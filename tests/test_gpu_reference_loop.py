"""The real thing on hardware: the UNMODIFIED reference controller loop (dmosopt/MOASMO.py:196-470, MOASMO.epoch) driving
the GPU plugins by import path, the controller helpers routed to the GPU by install(), and the plain-C host of
include/dmosopt_b200.h executed on the GPU.

The tests that run the reference's own code take the dmosopt package that build() compiles into ``oracle/_ref``
(git-ignored; oracle/reference_build.py), ``$DMOSOPT_REF`` or ``baseline/_ref``, and skip without one; the install() test compares with stored reference results (tests/golden/helpers.npz).
"""

import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


def _zdt1(x):
    d = x.shape[1]
    g = 1.0 + 9.0 / (d - 1) * x[:, 1:].sum(axis=1)
    return np.column_stack((x[:, 0], g * (1.0 - np.sqrt(x[:, 0] / g))))


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("optimizer,kwargs", [("dmosopt_b200.NSGA2", {}), ("dmosopt_b200.AGEMOEA", {}), ("dmosopt_b200.SMPSO", {}), ("dmosopt_b200.CMAES", {})])
def test_unmodified_moasmo_epoch_drives_the_gpu_plugins(optimizer, kwargs):
    """MOASMO.epoch resolves optimizer_name / surrogate_method_name by import path (config.py:5-11), fits the surrogate
    (GPR_Matern, default precision = auto), runs the generation loop on the GPU and the resample step
    (MOEA.get_duplicates(best_x, x_0) + crowding, MOASMO.py:441-448)."""
    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    from dmosopt_b200 import _lib

    _lib.context()
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(11)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    Y = _zdt1(X)
    launches0 = _lib.launch_count()
    gen = MOASMO.epoch(
        6, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop,
        optimizer_name=optimizer, optimizer_kwargs=kwargs, surrogate_method_name="dmosopt_b200.GPR_Matern",
        surrogate_method_kwargs={"anisotropic": False, "optimizer": None}, local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    assert _lib.launch_count() > launches0  # the generations ran on the GPU library
    assert type(res["optimizer"]).__module__.startswith("dmosopt_b200")
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M)
    assert np.all(xr >= xlb) and np.all(xr <= xub)
    # the resampled points are predicted to improve on the training set: their predicted objectives are not dominated
    # by the bulk of the initial sample (ZDT1: f2 falls as the surrogate pushes g towards 1)
    assert np.median(yp[:, 1]) < np.median(Y[:, 1])
    # predictions stored by the epoch agree with the oracle restatement of the fitted model at the resampled points
    from oracle import gp as ogp

    sm = res["optimizer"].model.objective if hasattr(res["optimizer"], "model") else None
    if sm is not None and hasattr(sm, "smlist"):
        st = ogp.from_sklearn(sm.smlist, xlb, xub)
        mean_o, _ = ogp.predict(st, xr)
        ystd = np.array([o.y_std for o in st.objectives])
        assert np.max(np.abs(mean_o - yp) / np.maximum(np.abs(mean_o), ystd)) < 1e-5


@pytest.mark.skipif(_reference_path() is None, reason="reference package not shipped")
def test_reference_and_plugin_nsga2_agree_on_a_generation():
    """Same initial state and the same offspring: the reference's NSGA2.update_strategy (dda_ens + sortMO on the CPU)
    and the GPU plugin keep the same survivors, in the same order, with the same ranks."""
    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import NSGA2 as rNSGA2
        from dmosopt import model as rmodel
    finally:
        sys.path.remove(ref)
    import dmosopt_b200 as b2

    d, M, pop = 10, 3, 300
    rng = np.random.default_rng(3)
    bounds = np.column_stack((np.zeros(d), np.ones(d)))
    x0 = rng.random((pop, d))

    def f(x):
        return np.column_stack((x[:, 0] + x[:, 3:].sum(1) * 0.1, (1 - x[:, 0]) * (1 + x[:, 1]), x[:, 2] ** 2 + 0.5 * x[:, 1]))

    y0 = f(x0).astype(np.float32)
    ro = rNSGA2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=rmodel.Model(), distance_metric=None)
    ro.initialize_strategy(x0.astype(np.float32), y0.copy(), bounds, np.random.default_rng(1))
    bo = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=None, distance_metric=None)
    bo.initialize_strategy(x0.astype(np.float32), y0.copy(), bounds, np.random.default_rng(1))
    assert np.array_equal(ro.state.rank, bo.state.rank)
    for _ in range(3):
        x_gen, st = bo.generate()
        x_gen = np.array(x_gen)
        y_gen = f(x_gen)
        ro.state.population_parm = np.array(bo.state.population_parm, dtype=np.float32) if ro.state.population_parm.dtype == np.float32 else np.array(bo.state.population_parm)
        ro.update(x_gen, y_gen, {"crossover_indices": st["crossover_indices"], "mutation_indices": st["mutation_indices"]})
        bo.update(x_gen, y_gen, st)
        assert np.array_equal(np.asarray(ro.state.rank), np.asarray(bo.state.rank))
        assert np.array_equal(np.asarray(ro.state.population_obj), np.asarray(bo.state.population_obj))


def test_plain_c_host_runs_the_resident_step_on_the_gpu(tmp_path):
    """examples/nsga2_step.c: gcc -std=c99 against include/dmosopt_b200.h, linked with the in-tree library, executed."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    libdir = os.path.join(ROOT, "dmosopt_b200")
    exe = str(tmp_path / "nsga2_step")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "nsga2_step.c"),
                        "-L", libdir, "-ldmosopt_b200", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    run = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("generation")]
    assert len(lines) == 5
    hv = [float(ln.rsplit(" ", 1)[1]) for ln in lines]
    assert all(b >= a - 1e-12 for a, b in zip(hv, hv[1:])), hv  # elitist survival: the hypervolume never shrinks


_STUB_MODULES = {
    "MOEA": "def _absent(*a, **k):\n    raise AssertionError('not routed')\n\n"
            + "".join(f"{n} = _absent\n" for n in ("get_duplicates", "remove_duplicates", "sortMO", "orderMO", "remove_worst",
                                                    "crowding_distance_metric", "euclidean_distance_metric", "dda_ens")),
    "indicators": "def crowding_distance_metric(*a, **k):\n    raise AssertionError('not routed')\n",
    "dda": "def dda_ens(*a, **k):\n    raise AssertionError('not routed')\n",
    "hv": ("class AdaptiveHyperVolume:\n    dimension_threshold_exact = 6\n\n    def __init__(self, ref_point):\n"
           "        self.ref_point = ref_point\n        self.n_objectives = len(ref_point)\n\n"
           "    def compute_hypervolume(self, pareto_front, algorithm=None, verbose=False):\n        raise AssertionError('not routed')\n"),
}


def test_install_routes_controller_helpers_to_the_gpu_with_identical_results(golden, tmp_path):
    """dmosopt_b200.install(): the helpers the reference controller calls on its own modules -- MOEA.get_duplicates and
    MOEA.sortMO (MOASMO.get_best, MOASMO.py:581-639), MOEA.crowding_distance_metric (resample step, MOASMO.py:441-448)
    and the termination hypervolume (hv.py:123-189) -- are rebound to the GPU and give the reference's own results
    (tests/golden/helpers.npz).  The rebinding is exercised on a stand-in package with the reference's module layout."""
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib

    pkg = tmp_path / "refstub"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    for name, src in _STUB_MODULES.items():
        (pkg / f"{name}.py").write_text(src)
    g = golden("helpers")
    rng = np.random.default_rng(21)  # the inputs tests/golden/make_golden.py (gen_helpers) gave the reference
    n, d = 700, 9
    x = rng.random((n, d))
    y = np.column_stack((x[:, 0] + 0.1, (1.1 - x[:, 0]) * (1 + x[:, 1]), 0.2 + x[:, 2] ** 2 + x[:, 1]))
    y[50] = y[3]
    y[400] = y[3]
    x0 = rng.random((300, d))
    x0[:40] = x[100:140]
    ref_pt = y.max(axis=0) + 0.1
    sys.path.insert(0, str(tmp_path))
    try:
        import refstub.hv as rhv
        import refstub.MOEA as rMOEA

        launches0 = _lib.launch_count()
        patched = b2.install(package="refstub")
        try:
            assert any(name.endswith("get_duplicates") for name in patched)
            dup_x = rMOEA.get_duplicates(x, x0)
            dup_y = rMOEA.get_duplicates(y)
            xs, ys, rank, _, perm = rMOEA.sortMO(x[~dup_y], y[~dup_y], return_perm=True)
            cd = rMOEA.crowding_distance_metric(y[np.r_[0:50, 51:400, 401:n]])
            hv = rhv.AdaptiveHyperVolume(ref_pt).compute_hypervolume(y[:300])
        finally:
            b2.uninstall()
        assert _lib.launch_count() > launches0
        assert rMOEA.get_duplicates.__module__ == "refstub.MOEA"  # restored
    finally:
        sys.path.remove(str(tmp_path))
        for m in [m for m in sys.modules if m == "refstub" or m.startswith("refstub.")]:
            del sys.modules[m]
    assert np.array_equal(dup_x, g["dup_x"]) and dup_x.sum() == 40
    assert np.array_equal(dup_y, g["dup_y"])
    assert np.array_equal(np.asarray(rank), g["sort_rank"]) and np.array_equal(np.asarray(perm), g["sort_perm"])
    assert np.array_equal(xs, x[~dup_y][g["sort_perm"]]) and np.array_equal(ys, y[~dup_y][g["sort_perm"]])
    assert np.array_equal(cd, g["cd"])  # float64 bit-exact crowding (tie-free columns)
    assert abs(hv - float(g["hv"])) <= 1e-9 * abs(float(g["hv"]))
