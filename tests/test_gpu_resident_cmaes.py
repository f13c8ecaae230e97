"""The resident MO-CMA-ES surrogate epoch (dmosopt_b200.MOASMO.optimize on dmo_cmaes_step_record / dmo_cmaes_step_apply)
against the per-generation plugin loop, on the GPU.

1. MOASMO.optimize against MOASMO.optimize_per_generation from identically seeded generators: identical epoch results
   (dtypes included) and optimizer state (parents_x, parents_y, sigmas, A, Ainv, pc, psucc, rank, the next draw of
   ``local_random``), for every surrogate class, option and shape the route serves, and one more plugin generation
   after the epoch.
2. The two entry points against the plugin's generate -> predict -> update on crafted parent objectives: the
   hypervolume-improvement pick, a mid front with nothing chosen before it (its first k rows) and no mid front (k = 0);
   bad arguments refused before any launch.
3. The host traffic of a resident generation: the record, the codes and the parent indices down, the host draws and
   the host arithmetic up, no state copy, and no more waits than the plugin loop.
4. The reference's unmodified MOASMO.epoch with and without ``install(resident_epoch=True)``.
"""

import sys

import numpy as np
import pytest

from oracle import reference_build
from test_gpu_resident_posterior import CLASSES, DEEP, _dtlz2, surrogate

pytestmark = pytest.mark.gpu

REFERENCE = reference_build.reference_path()


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _make_surrogate(cls, d, M, N, precision):
    """(surrogate, xlb, xub, X, Y): the exact GPs fitted as given, the other classes from seeded hyper-parameters."""
    import dmosopt_b200 as b2

    if cls in ("GPR_Matern", "GPR_RBF"):
        rng = np.random.default_rng(5)
        xlb, xub = np.zeros(d), np.ones(d)
        X = rng.random((N, d))
        Y = _dtlz2(X, M)
        return getattr(b2, cls)(X, Y, d, M, xlb, xub, optimizer=None, precision=precision), xlb, xub, X, Y
    return surrogate(cls, d, M, N, precision)


class _StopAt:
    def __init__(self, n):
        self.n, self.seen = n, []

    def has_terminated(self, opt):
        self.seen.append((opt.n_gen, opt.n_eval, np.array(opt.x), np.array(opt.y)))
        return opt.n_gen > self.n


BASE = dict(cls="GPR_Matern", precision="fp64", d=7, M=3, N=256, pop=64, lam=1, gens=3, stop=None, initial=True)
CASES = {f"{c}-{p}": dict(cls=c, precision=p) for c in ("GPR_Matern", "GPR_RBF") + CLASSES for p in ("fp64", "tensor")}
CASES.update({
    "GPR_Matern-auto": dict(precision="auto"),
    "lambda2": dict(lam=2, pop=65, precision="auto"),
    "lambda2_even": dict(lam=2, pop=100, cls="SVGP_Matern", precision="tensor"),
    "odd_pop": dict(pop=101, cls="EGP_Matern", precision="fp64"),
    "no_initial": dict(initial=False, precision="auto"),
    "termination": dict(cls="MDGP_Matern", precision="tensor", stop=2, gens=10),
    # no generation runs: the state stays as initialize_strategy left it
    "terminate_at_once": dict(stop=0, gens=10),
    "zero_generations": dict(gens=0, cls="SVGP_Matern", precision="tensor"),
    "M2": dict(M=2, d=30, pop=200, N=512, precision="auto"),
    "M4": dict(M=4, pop=129, cls="CRV_Matern", precision="tensor"),
    "M12": dict(M=12, d=16, pop=96, precision="tensor"),  # most candidates non-dominated: the mid front's first k rows
    "M16": dict(M=16, d=20, pop=64, gens=2),
    "d40": dict(d=40, pop=200, precision="tensor"),  # the two-kernel tensor route
    # lambda * mu > 2^20 offspring: two candidate chunks of the predict
    "two_chunks": dict(pop=(1 << 20) + 2002, lam=2, d=5, M=2, gens=1, precision="tensor"),
    "c5_shape": dict(d=24, M=4, N=4096, pop=131072, gens=2, precision="auto"),
})


def _setup(c):
    import dmosopt_b200 as b2

    sm, xlb, xub, X, Y = _make_surrogate(c["cls"], c["d"], c["M"], c["N"], c["precision"])
    model = b2.Model(objective=sm)
    opt = b2.CMAES(popsize=c["pop"], nInput=c["d"], nOutput=c["M"], model=model, lambda_=c["lam"])
    return opt, model, sm, xlb, xub, X, Y


def _run(fn, c, seed=11, more=False):
    opt, model, sm, xlb, xub, X, Y = _setup(c)
    rng = np.random.default_rng(seed)
    stop = None if c["stop"] is None else _StopAt(c["stop"])
    initial = (X[:64], Y[:64]) if c["initial"] else None
    gen = fn(c["gens"], opt, model, c["d"], c["M"], xlb, xub, popsize=c["pop"], initial=initial, local_random=rng, termination=stop)
    with pytest.raises(StopIteration) as ex:
        next(gen)
    if more:  # one more plugin generation on whatever state the epoch left
        x_gen, state = opt.generate()
        opt.update(x_gen, sm.evaluate(x_gen), state)
    return ex.value.value, opt, rng, stop, sm


STATE = ("parents_x", "parents_y", "sigmas", "A", "Ainv", "pc", "psucc", "rank")


def _assert_state(sa, sb, msg=None):
    for f in STATE:
        u, v = np.asarray(getattr(sa, f)), np.asarray(getattr(sb, f))
        assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), (f, msg)


def _assert_same(a, b, results=True):
    res_a, opt_a, rng_a, stop_a, sm_a = a
    res_b, opt_b, rng_b, stop_b, sm_b = b
    if results:
        for f in ("best_x", "best_y", "gen_index", "x", "y"):
            u, v = getattr(res_a, f), getattr(res_b, f)
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), f
    _assert_state(opt_a.state, opt_b.state)
    assert rng_a.random() == rng_b.random()
    assert getattr(sm_a, "calls", None) == getattr(sm_b, "calls", None)
    if stop_a is not None:
        assert len(stop_a.seen) == len(stop_b.seen)
        for u, v in zip(stop_a.seen, stop_b.seen):
            assert u[:2] == v[:2] and u[2].dtype == v[2].dtype and np.array_equal(u[2], v[2]) and np.array_equal(u[3], v[3])


def _counting(L, monkeypatch, name="step_record"):
    calls = []
    f = getattr(L.CmaesResident, name)

    def counted(self, *args, **kwargs):
        calls.append(1)
        return f(self, *args, **kwargs)

    monkeypatch.setattr(L.CmaesResident, name, counted)
    return calls


# ------------------------------------------------------------------------------------ 1. epoch parity
@pytest.mark.parametrize("case", list(CASES))
def test_resident_epoch_equals_plugin_loop(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    calls = _counting(L, monkeypatch)
    res = _run(MOASMO.optimize, c)
    n_gens = c["gens"] if c["stop"] is None else c["stop"]
    assert len(calls) == n_gens, (case, len(calls))
    ref = _run(MOASMO.optimize_per_generation, c)
    assert len(calls) == n_gens
    _assert_same(res, ref)
    f32 = c["cls"] not in DEEP + ("GPR_Matern", "GPR_RBF")
    assert res[0].y.dtype == (np.float32 if f32 or n_gens == 0 else np.float64)  # the initial rows alone are float32
    assert res[1].state.parents_y.dtype == (np.float32 if f32 or n_gens == 0 else np.float64)
    if c["cls"] == "MDGP_Matern":
        assert res[4].calls == 1 + n_gens  # the initial evaluate, then one draw per generation


@pytest.mark.parametrize("case", ["GPR_Matern-auto", "MDGP_Matern-tensor", "lambda2", "SIV_Matern-fp64"])
def test_plugin_generation_after_the_resident_epoch(L, case):
    """The state the resident epoch leaves (the current half of its double buffer as the state's ResidentRows) carries a
    plugin generation exactly as the plugin loop's state does."""
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    _assert_same(_run(MOASMO.optimize, c, more=True), _run(MOASMO.optimize_per_generation, c, more=True), results=False)


# ------------------------------------------------------------------------------------ 2. the entry points
def _pair(cls, precision, d, M, pop, lam, parents_y, seed=3):
    """Two CMAES optimizers in the same state, on one surrogate, with crafted parent objectives."""
    import dmosopt_b200 as b2

    sm, xlb, xub, X, Y = _make_surrogate(cls, d, M, 256, precision)
    model = b2.Model(objective=sm)
    x = np.random.default_rng(seed).random((pop, d))
    y = sm.evaluate(x).astype(np.float32)  # once: a deep GP's next evaluate draws another key
    opts = []
    for _ in range(2):
        opt = b2.CMAES(popsize=pop, nInput=d, nOutput=M, model=model, lambda_=lam)
        opt.initialize_strategy(x, y, np.column_stack((xlb, xub)), np.random.default_rng(seed + 1))
        if parents_y is not None:
            opt.state.parents_y = parents_y.copy()
            opt.state.rank = np.zeros(pop, dtype=np.intp)
        opts.append(opt)
    return sm, model, opts


def _crafted(kind, pop, M, rng):
    if kind == "random":  # a cloud with several fronts of its own: some fronts fit whole, the mid front is picked by EHVI
        return 2.0 * rng.random((pop, M))
    if kind == "dominating_line":  # every parent dominates every offspring and none dominates another: k = 0
        t = np.arange(pop, dtype=np.float64)
        return np.column_stack([-1e3 - t] + [-1e3 + t] * (M - 1))
    # "first_k" (M = 2): the parents on an anti-diagonal that neither dominates nor is dominated by the offspring, so the
    # first front holds every parent and some offspring: more than pop rows, nothing chosen before the mid front
    t = rng.permutation(pop).astype(np.float64)
    return np.column_stack((t - 1e6, 1e6 - t))


ENTRY_CASES = [("GPR_Matern", "auto", 3, "random"), ("GPR_Matern", "fp64", 2, "dominating_line"), ("EGP_Matern", "tensor", 3, "random"),
               ("SVGP_Matern", "fp64", 8, "random"), ("MDGP_Matern", "tensor", 2, "first_k"), ("GPR_RBF", "tensor", 16, "random")]


@pytest.mark.parametrize("cls,precision,M,kind", ENTRY_CASES)
def test_entry_points_equal_the_plugin_generation(L, cls, precision, M, kind):
    from dmosopt_b200 import MOASMO

    d, pop, lam = max(6, M + 2), 97, 2  # DTLZ2 takes d >= M
    rng = np.random.default_rng(4)
    py = _crafted(kind, pop, M, rng)
    sm, model, (a, b) = _pair(cls, precision, d, M, pop, lam, py)
    step = MOASMO._CmaesStep(b, model, MOASMO._resident_posterior(sm))
    C = step.rows
    cuts = []
    for gen in range(3):
        draw = sm._draw_key() if cls == "MDGP_Matern" else (0, 0)
        x_gen, state = a.generate()
        if cls == "MDGP_Matern":
            sm.calls -= 1  # the same key again for the plugin's evaluate
        y_gen = sm.evaluate(x_gen)
        xr, yr = L.pinned_empty((C, d)), L.pinned_empty((C, M))
        step(xr, yr, None, draw)
        step.sync()
        # the front cut of this generation: (rows chosen whole, k)
        r = step.res.cand_rank.download()
        fronts = np.r_[0, np.cumsum(np.bincount(r, minlength=C + pop))]
        lo = int(fronts[np.flatnonzero(fronts <= pop)[-1]])
        cuts.append((lo, pop - lo))
        a.update(x_gen, y_gen, state)
        msg = (cls, precision, M, kind, gen)
        assert np.array_equal(xr, x_gen), msg
        assert np.array_equal(yr, np.asarray(y_gen, dtype=np.float64)), msg
        _assert_state(a.state, b.state, msg)
        assert a.local_random.random() == b.local_random.random(), msg
    lo, k = cuts[0]
    if kind == "dominating_line":
        assert k == 0, cuts
    elif kind == "first_k":
        assert lo == 0 and k == pop, cuts
    elif M <= 3:  # with more objectives most rows are non-dominated: any cut may come
        assert any(lo > 0 and k > 0 for lo, k in cuts), cuts


def test_record_refuses_bad_arguments_before_any_launch(L):
    from dmosopt_b200 import _lib

    d, M, pop, C = 5, 2, 16, 8
    gpr = _make_surrogate("GPR_Matern", d, M, 128, "fp64")[0]
    svgp = surrogate("SVGP_Matern", d, M, 128, "fp64")[0]
    wide = surrogate("EGP_Matern", d + 1, M, 128, "fp64")[0]
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    rng = np.random.default_rng(2)
    px, sg, A = L.resident_rows(rng.random((pop, d))), L.resident_rows(np.full((pop, d), 1e-3)), L.identity_rows(pop, d)
    py = DA((pop, M)).upload(rng.random((pop, M)))
    cx, cy, cr = DA((C, d)), DA((C + pop, M)), DA((C + pop,), np.int32)
    arz, js = rng.standard_normal((C, d)), rng.integers(0, pop // 2, C).astype(np.int64)
    xlb, xub = np.zeros(d), np.ones(d)
    xg, yg = L.pinned_empty((C, d)), L.pinned_empty((C, M))
    codes, pidx = L.pinned_empty((C + pop,), np.uint8), L.pinned_empty((C,), np.int64)

    def call(kind=_lib.POSTERIOR_GP, h=gpr._gp._h, var_route=0, prec=L.GP_FP64, stream=0, sc=d, parents=px.ptr, j=js, mu=pop // 2, n_off=C,
             cand=cy.ptr, x=xg, c=codes, M_=M):
        L.synchronize()
        l0 = L.launch_count()
        st = lib.dmo_cmaes_step_record(ctx, kind, h, 9, stream, var_route, prec, 0, 0, L._ptr(parents), sg.ptr, sc, A.ptr, py.ptr, pop, d, M_,
                                       arz.ctypes.data, L._ptr(j), n_off, mu, xlb.ctypes.data, xub.ctypes.data, cx.ptr, L._ptr(cand), cr.ptr,
                                       L._ptr(x), yg.ctypes.data, L._ptr(c), pidx.ctypes.data)
        return st, L.launch_count() - l0

    dev_js = DA((C,), np.int64).upload(js)
    bad_js = js.copy()
    bad_js[3] = pop // 2
    assert call(kind=3) == (2, 0)
    assert call(h=None) == (2, 0)
    assert call(var_route=1, prec=L.GP_AUTO) == (2, 0)
    assert call(kind=_lib.POSTERIOR_SVGP, h=svgp._h._h, var_route=0) == (2, 0)
    assert call(h=wide._gp._h, var_route=1) == (2, 0)
    assert call(sc=3) == (2, 0)
    assert call(parents=np.zeros((pop, d))) == (2, 0)
    assert call(cand=np.zeros((C + pop, M))) == (2, 0)
    assert call(j=dev_js) == (2, 0)
    assert call(j=bad_js) == (2, 0)
    assert call(j=js, mu=2) == (2, 0)  # js must lie below min(mu, pop)
    assert call(n_off=0) == (2, 0)
    assert call(x=None) == (2, 0)
    assert call(c=None) == (2, 0)
    assert call(M_=17) == (2, 0)
    st, launched = call()
    assert st == 0 and launched > 0
    L.synchronize()

    # the second call: indices out of range, device index arrays, outputs aliasing the state
    from dmosopt_b200.CMAES import _strategy_scalars

    opt = __import__("dmosopt_b200").CMAES(popsize=pop, nInput=d, nOutput=M)
    chosen = codes.astype(bool)
    h = _strategy_scalars(opt.opt_params, np.full(pop, 0.15), np.concatenate((pidx, np.arange(pop))), C, chosen, ~chosen)
    Ainv, pc = L.identity_rows(pop, d), L.resident_rows(np.zeros((pop, d)))
    outs = [L.resident_rows(np.zeros((pop, d))), L.resident_rows(np.zeros((pop, d))), L.identity_rows(pop, d), L.identity_rows(pop, d),
            L.resident_rows(np.zeros((pop, d))), DA((pop, M)), DA((pop,), np.int32)]
    i64 = lambda a: np.ascontiguousarray(a, dtype=np.int64)  # noqa: E731

    def apply(nc=i64(h.ch), ns=i64(h.src_idx), oc=i64(h.ch_off), out=None):
        L.synchronize()
        l0 = L.launch_count()
        op, sr, ss = i64(h.par), i64(h.seg_row), i64(h.seg_start)
        ps, of, ef = np.ascontiguousarray(h.off_psucc), np.ascontiguousarray(h.off_fac), np.ascontiguousarray(h.ev_fac)
        o = out or outs
        st = lib.dmo_cmaes_step_apply(ctx, px.ptr, sg.ptr, d, A.ptr, Ainv.ptr, pc.ptr, pop, d, M, cx.ptr, cy.ptr, cr.ptr, C, oc.shape[0],
                                      L._ptr(oc), op.ctypes.data, ps.ctypes.data, of.ctypes.data, sr.shape[0], sr.ctypes.data, ss.ctypes.data,
                                      ef.ctypes.data, L._ptr(nc), L._ptr(ns), xlb.ctypes.data, xub.ctypes.data, 0.2, 0.1, 0.44,
                                      *(a.ptr for a in o))
        return st, L.launch_count() - l0

    bad = i64(h.ch).copy()
    bad[0] = C + pop
    assert apply(nc=bad) == (2, 0)
    bad = i64(h.src_idx).copy()
    bad[-1] = pop
    assert apply(ns=bad) == (2, 0)
    assert apply(nc=DA((pop,), np.int64).upload(i64(h.ch))) == (2, 0)
    assert apply(out=[px] + outs[1:]) == (2, 0)
    if len(h.ch_off):
        bad = i64(h.ch_off).copy()
        bad[0] = C
        assert apply(oc=bad) == (2, 0)
    st, launched = apply()
    assert st == 0 and launched > 0
    L.synchronize()


# ------------------------------------------------------------------------------------ 3. host traffic
@pytest.mark.parametrize("case", ["GPR_Matern-auto", "SVGP_Matern-tensor"])
def test_resident_generation_traffic(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case], pop=8192, gens=3)
    pop, d, M = c["pop"], c["d"], c["M"]
    C = pop // 2
    per_gen = []
    f = MOASMO._CmaesStep.__call__

    def measured(self, *args, **kwargs):
        L.synchronize()
        b0 = L.transfer_bytes()
        out = f(self, *args, **kwargs)
        L.synchronize()
        b1 = L.transfer_bytes()
        per_gen.append((b1[0] - b0[0], b1[1] - b0[1]))
        return out

    monkeypatch.setattr(MOASMO._CmaesStep, "__call__", measured)
    L.synchronize()
    w0 = L.wait_count()
    res = _run(MOASMO.optimize, c)
    w_res = L.wait_count() - w0
    w0 = L.wait_count()
    ref = _run(MOASMO.optimize_per_generation, c)
    w_ref = L.wait_count() - w0
    _assert_same(res, ref)
    assert len(per_gen) == c["gens"]
    down = C * (d + M) * 8 + (C + pop) + C * 8  # the record, the codes, the parents of the offspring
    up = C * d * 8 + C * 8 + 2 * d * 8  # the normals, the parent draws, the bounds
    for h2d, d2h in per_gen:
        # no state row crosses the bus: the slack stays below one parameter row per parent
        assert down <= d2h < down + pop * d * 8 // 4, (h2d, d2h)
        # the host arithmetic: at most 4 values per offspring, 3 per parent event, 2 per new parent, the bounds again, and
        # the predict's own small uploads: no state row
        assert up <= h2d <= up + (4 * C + 3 * (C + pop) + 2 * pop + 1) * 8 + 2 * d * 8 + 65536, (h2d, d2h)
    assert w_res <= w_ref, (w_res, w_ref)


# ------------------------------------------------------------------------------------ 4. the reference's epoch
def _reference_epoch(MOASMO, seed):
    d, M, pop = 6, 2, 24
    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((40, d))
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.column_stack(((1.0 + g) * np.cos(0.5 * np.pi * X[:, 0]), (1.0 + g) * np.sin(0.5 * np.pi * X[:, 0])))
    gen = MOASMO.epoch(
        4, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop,
        optimizer_name="dmosopt_b200.CMAES", surrogate_method_name="dmosopt_b200.GPR_Matern",
        surrogate_method_kwargs={"anisotropic": False, "optimizer": None}, local_random=rng,
    )
    with pytest.raises(StopIteration) as ex:
        next(gen)
    return ex.value.args[0]


@pytest.mark.skipif(REFERENCE is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_unmodified_reference_epoch_same_with_resident_route(L, monkeypatch):
    import dmosopt_b200 as b2

    sys.path.insert(0, REFERENCE)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(REFERENCE)
    calls = _counting(L, monkeypatch)
    plain = _reference_epoch(MOASMO, 5)
    assert len(calls) == 0
    try:
        b2.install(resident_epoch=True)
        routed = _reference_epoch(MOASMO, 5)
    finally:
        b2.uninstall()
    assert len(calls) == 4
    assert sorted(plain) == sorted(routed)
    for k in plain:
        u, v = plain[k], routed[k]
        if isinstance(u, np.ndarray):
            assert u.dtype == v.dtype and np.array_equal(u, v), k
        elif k == "optimizer":
            assert type(u) is type(v)
        elif isinstance(u, (int, float, str, type(None))):
            assert u == v, k
