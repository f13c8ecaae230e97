"""The fused step's hypervolume (dmo_nsga2_step with hv_ref set).  With three objectives on the deferred AUTO route the
device work of the volume runs on the truncation's lane beside the GP's variance contraction, over the population padded
with the reference point, and its reads follow the GP; every other route computes it after the GP.  Either way the volume
must be the bits of dmo_hypervolume_ranked on the population and ranks the step returns, on both M = 3 routes (sweep
below 4096 rank-0 rows inside the reference box, merge-sort tree above), when AUTO refines rows (the lane's work is
dropped and the volume computed again), on the float64 route and for 2, 4, 5 and 6 objectives.  Past eight objectives
the step fails as the ranked hypervolume does, and the context stays usable."""

import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _objectives(X, M, kind):
    if kind == "plane":  # every point of the plane sum(y) = M - 1 is non-dominated: fronts of thousands of rows
        Y = X[:, :M].copy()
        Y[:, M - 1] = (M - 1) - X[:, : M - 1].sum(axis=1)
        return Y
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)  # DTLZ2
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


class Run:
    """A resident population, a GP on its objectives and the buffers of dmo_nsga2_step.  kind "sphere": DTLZ2 targets
    and a population whose distance inputs are all 0.5, so that the parents lie on the unit sphere, a single front."""

    def __init__(self, L, d, N, pop, M, kind, seed, on_training=False):
        import dmosopt_b200 as b2

        rng = np.random.default_rng(seed)
        self.L, self.d, self.pop, self.M = L, d, pop, M
        xlb, xub = np.zeros(d), np.ones(d)
        Xtr = rng.random((N, d))
        sm = b2.GPR_Matern(Xtr, _objectives(Xtr, M, "dtlz2" if kind == "sphere" else kind), d, M, xlb, xub, optimizer=None)
        self.sm, self.gp = sm, sm._gp
        self.gp.predict(rng.random((64, d)), return_var=True, precision=L.GP_AUTO)  # calibration and tensor set-up
        x0 = Xtr[:pop].copy() if on_training else rng.random((pop, d))
        if kind == "sphere":
            x0[:, M - 1 :] = 0.5
        y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
        self.ref = y0.max(axis=0) + 0.1 * (y0.max(axis=0) - y0.min(axis=0))
        DA = L.DeviceArray
        self.x, self.y = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0)
        self.r = DA((pop,), np.int32).upload(L.rank_nd(y0).astype(np.int32))
        self.dic, self.dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
        self.dlb, self.dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
        self.nch = np.zeros(1, dtype=np.int64)
        self.stream = 10

    def step(self, precision, ref=None):
        L, d, M = self.L, self.d, self.M
        ref = self.ref if ref is None else ref
        hv = ctypes.c_double(-1.0)
        self.stream += 2
        L._check(L.load_library().dmo_nsga2_step(L.context(), self.gp._h, self.x.ptr, self.y.ptr, self.r.ptr, self.pop, d, M, 0.9, 0.1,
                                                 1.0 / d, self.dic.ptr, self.dim.ptr, self.dlb.ptr, self.dub.ptr, 777, self.stream, precision,
                                                 L.METRIC_NONE, 1, 1, ref.ctypes.data, self.nch.ctypes.data, ctypes.byref(hv)), "nsga2_step")
        return hv.value

    def ranked_hv(self):
        L = self.L
        h = ctypes.c_double(0.0)
        L._check(L.load_library().dmo_hypervolume_ranked(L.context(), self.y.ptr, self.pop, self.M, self.ref.ctypes.data, self.r.ptr,
                                                         ctypes.byref(h)), "hypervolume_ranked")
        return h.value

    def front(self):
        y, r = self.y.download(), self.r.download()
        return int(np.sum((r == 0) & np.all(y < self.ref, axis=1)))


# name: (d, N_train, pop, objectives, kind)
CASES = {
    "m2": (8, 512, 4096, 2, "plane"),
    "m3_sweep": (30, 1024, 8192, 3, "dtlz2"),
    "m3_tree": (30, 1024, 32768, 3, "sphere"),
    "m4": (8, 512, 2048, 4, "dtlz2"),
    "m5": (8, 512, 2048, 5, "dtlz2"),
    "m6": (8, 512, 1024, 6, "dtlz2"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_step_hypervolume_equals_ranked_hypervolume(L, case):
    d, N, pop, M, kind = CASES[case]
    run = Run(L, d, N, pop, M, kind, seed=31 + len(case))
    routes = set()
    for gen in range(3):
        L.profile_enable(True)
        hv = run.step(L.GP_AUTO)
        prof = L.profile_report()
        L.profile_enable(False)
        assert hv == run.ranked_hv() and hv > 0.0, (case, gen, hv)
        assert "step_hv" in prof, (case, gen, sorted(prof))
        if M == 3:
            # the lane builds the tree whenever the population reaches the threshold; the sweep runs after the GP, when
            # the rows the volume keeps stay below it
            assert run.gp.auto_info()["var_tensor"] and "hv3_tree" in prof, (case, gen, sorted(prof))
            n1 = run.front()
            routes.add("sweep" if "hv3" in prof else "tree")
            assert ("hv3" in prof) == (n1 < 4096), (case, gen, n1, sorted(prof))
    if case == "m3_sweep":
        assert routes == {"sweep"}, routes
    elif case == "m3_tree":
        assert "tree" in routes, (routes, run.front())


def test_step_hypervolume_when_auto_refines_rows(L):
    # the population starts on the training inputs: offspring that mutation barely moves have a variance near 0, which
    # AUTO recomputes in float64, so the truncation and the volume run again on the refined rows
    run = Run(L, 30, 4096, 4096, 3, "dtlz2", seed=2026, on_training=True)
    refined = []
    for gen in range(3):
        hv = run.step(L.GP_AUTO)
        refined.append(run.gp.auto_info()["last_refined"])
        assert hv == run.ranked_hv() and hv > 0.0, (gen, hv)
    assert run.gp.auto_info()["var_tensor"] and max(refined) > 0, refined


def test_step_hypervolume_on_the_float64_route(L):
    run = Run(L, 30, 1024, 8192, 3, "dtlz2", seed=404)
    for gen in range(2):
        L.profile_enable(True)
        hv = run.step(L.GP_FP64)
        prof = L.profile_report()
        L.profile_enable(False)
        assert hv == run.ranked_hv() and hv > 0.0, (gen, hv)
        # after the GP, on the rows it keeps: the sweep, and no tree over the whole population
        assert run.front() < 4096 and "hv3" in prof and "hv3_tree" not in prof, sorted(prof)


def test_step_past_eight_objectives_fails_like_the_ranked_hypervolume(L):
    run = Run(L, 12, 512, 1024, 10, "dtlz2", seed=99)
    with pytest.raises(L.DmoError) as step_err:
        run.step(L.GP_AUTO)
    with pytest.raises(L.DmoError) as ranked_err:
        run.ranked_hv()
    step_status, step_msg = str(step_err.value).split("failed ", 1)[1].split(": ", 1)
    ranked_status, ranked_msg = str(ranked_err.value).split("failed ", 1)[1].split(": ", 1)
    assert step_status == ranked_status and step_msg == ranked_msg, (str(step_err.value), str(ranked_err.value))
    # the context stays usable: the next step, without a reference point, succeeds
    L._check(L.load_library().dmo_nsga2_step(L.context(), run.gp._h, run.x.ptr, run.y.ptr, run.r.ptr, run.pop, run.d, run.M, 0.9, 0.1,
                                             1.0 / run.d, run.dic.ptr, run.dim.ptr, run.dlb.ptr, run.dub.ptr, 778, 90, L.GP_AUTO,
                                             L.METRIC_NONE, 1, 1, None, run.nch.ctypes.data, None), "nsga2_step")
    assert run.nch[0] > 0
