"""The resident SMPSO surrogate epoch (dmosopt_b200.MOASMO.optimize on dmo_smpso_step_record) against the per-generation
plugin loop, on the GPU.

1. MOASMO.optimize against MOASMO.optimize_per_generation from identically seeded generators: identical epoch results
   (dtypes included) and optimizer state (positions, objectives, velocities, ranks, success counter, operator
   parameters, Philox state, the next draw of ``local_random``), for every surrogate class, y-metric, option, swarm
   count and shape the route serves, and one more plugin generation after the epoch.
2. One dmo_smpso_step_record call against dmo_smpso_generate -> the public predict -> dmo_smpso_update on the same
   inputs, bit for bit; bad arguments refused before any launch.
3. The host traffic of a resident generation: the record and no state copy, no upload of the offspring's mean, and no
   more waits than the plugin loop.
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


BASE = dict(cls="GPR_Matern", precision="fp64", d=7, M=3, N=256, pop=64, S=5, gens=3, metric=None, adaptive=False, stop=None, initial=True)
CASES = {f"{c}-{p}": dict(cls=c, precision=p) for c in ("GPR_Matern", "GPR_RBF") + CLASSES for p in ("fp64", "tensor")}
CASES.update({
    "GPR_Matern-auto": dict(precision="auto"),
    "crowding": dict(metric="crowding", precision="auto"),
    "euclidean": dict(cls="SVGP_Matern", precision="tensor", metric="euclidean"),
    "adaptive_rates": dict(cls="EGP_Matern", precision="fp64", adaptive=True, gens=4),
    "termination": dict(cls="MDGP_Matern", precision="tensor", stop=2, gens=10, metric="crowding"),
    "no_initial": dict(initial=False, precision="auto"),
    # no generation runs: the state (ranks included) stays as initialize_strategy left it
    "terminate_at_once": dict(stop=0, gens=10, metric="crowding"),
    "zero_generations": dict(gens=0, cls="SVGP_Matern", precision="tensor"),
    "one_swarm": dict(S=1, pop=100),
    "two_swarms": dict(S=2, pop=101, cls="VGP_Matern", precision="tensor"),
    "pop2": dict(pop=2, metric="crowding"),  # no leader draws: the ind < 0 branch
    "pop3": dict(pop=3, metric="crowding", cls="MDSPP_Matern", precision="fp64"),
    "M2": dict(M=2, pop=333, precision="auto"),
    "M5": dict(M=5, pop=129, cls="CRV_Matern", precision="tensor"),
    "M9": dict(M=9, d=10, pop=96, precision="tensor", metric="euclidean"),
    "d40": dict(d=40, pop=200, precision="tensor"),  # the two-kernel tensor route
    # P = 4 pop > 2^20 rows: two candidate chunks of every predict route
    "two_chunks": dict(S=2, pop=(1 << 18) + 1001, gens=1, precision="tensor"),
    "two_chunks_svgp": dict(S=2, pop=(1 << 18) + 1001, gens=1, cls="SVGP_Matern", precision="tensor"),
    "c4_shape": dict(d=22, M=5, N=4096, pop=32768, S=5, gens=2, precision="auto"),
})


def _setup(c):
    import dmosopt_b200 as b2

    sm, xlb, xub, X, Y = _make_surrogate(c["cls"], c["d"], c["M"], c["N"], c["precision"])
    model = b2.Model(objective=sm)
    opt = b2.SMPSO(popsize=c["pop"], nInput=c["d"], nOutput=c["M"], model=model, distance_metric=c["metric"], swarm_size=c["S"],
                   adaptive_operator_rates=c["adaptive"])
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


def _assert_same(a, b, results=True):
    res_a, opt_a, rng_a, stop_a, sm_a = a
    res_b, opt_b, rng_b, stop_b, sm_b = b
    if results:
        for f in ("best_x", "best_y", "gen_index", "x", "y"):
            u, v = getattr(res_a, f), getattr(res_b, f)
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), f
    sa, sb = opt_a.state, opt_b.state
    for f in ("population_parm", "population_obj", "velocity"):
        u, v = getattr(sa, f), getattr(sb, f)
        assert u.dtype == v.dtype and np.array_equal(u, v), f
    assert len(sa.ranks) == len(sb.ranks)
    for u, v in zip(sa.ranks, sb.ranks):
        assert np.asarray(u).dtype == np.asarray(v).dtype and np.array_equal(u, v), "ranks"
    assert type(sa.successful_children) is type(sb.successful_children) and sa.successful_children == sb.successful_children
    pa, pb = opt_a.opt_params(), opt_b.opt_params()
    assert sorted(pa) == sorted(pb)
    for k in pa:
        if not callable(pa[k]):
            assert type(pa[k]) is type(pb[k]) and np.array_equal(np.asarray(pa[k]), np.asarray(pb[k])), k
    for f in ("_philox_seed", "_philox_stream"):  # drawn at the first generation: absent from both after none
        assert getattr(opt_a, f, None) == getattr(opt_b, f, None), f
    assert rng_a.random() == rng_b.random()
    assert getattr(sm_a, "calls", None) == getattr(sm_b, "calls", None)
    if stop_a is not None:
        assert len(stop_a.seen) == len(stop_b.seen)
        for u, v in zip(stop_a.seen, stop_b.seen):
            assert u[:2] == v[:2] and u[2].dtype == v[2].dtype and np.array_equal(u[2], v[2]) and np.array_equal(u[3], v[3])


# ------------------------------------------------------------------------------------ 1. epoch parity
@pytest.mark.parametrize("case", list(CASES))
def test_resident_epoch_equals_plugin_loop(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    calls = []
    step = L.SmpsoSwarms.step_record

    def counted(self, *args, **kwargs):
        calls.append(1)
        return step(self, *args, **kwargs)

    monkeypatch.setattr(L.SmpsoSwarms, "step_record", counted)
    res = _run(MOASMO.optimize, c)
    n_gens = c["gens"] if c["stop"] is None else c["stop"]
    assert len(calls) == n_gens, (case, len(calls))
    ref = _run(MOASMO.optimize_per_generation, c)
    assert len(calls) == n_gens
    _assert_same(res, ref)
    f32 = c["cls"] not in DEEP + ("GPR_Matern", "GPR_RBF")
    assert res[0].y.dtype == (np.float32 if f32 or n_gens == 0 else np.float64)  # the initial rows alone are float32
    if c["cls"] == "MDGP_Matern":
        assert res[4].calls == 1 + n_gens  # the initial evaluate, then one draw per generation


@pytest.mark.parametrize("case", ["GPR_Matern-auto", "MDGP_Matern-tensor", "two_swarms"])
def test_plugin_generation_after_the_resident_epoch(L, case):
    """The state the resident epoch leaves (host arrays and the device copy keyed to them) carries a plugin generation
    exactly as the plugin loop's state does."""
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    _assert_same(_run(MOASMO.optimize, c, more=True), _run(MOASMO.optimize_per_generation, c, more=True), results=False)


# ------------------------------------------------------------------------------------ 2. the entry point
ENTRY_CASES = [("GPR_Matern", "auto", 0), ("GPR_Matern", "fp64", 1), ("GPR_RBF", "tensor", 2), ("EGP_Matern", "tensor", 1),
               ("SVGP_Matern", "fp64", 2), ("MDGP_Matern", "tensor", 0), ("MDSPP_Matern", "fp64", 1)]


def _posterior(L, sm):
    from dmosopt_b200.MOASMO import _resident_posterior

    return _resident_posterior(sm)


@pytest.mark.parametrize("cls,precision,metric", ENTRY_CASES)
def test_step_equals_the_separate_entry_points(L, cls, precision, metric, monkeypatch):
    monkeypatch.setenv("DMOSOPT_B200_SMPSO_THREADS", "0")  # one dmo_smpso_update call for every swarm
    d, M, S, pop = 7, 3, 3, 257
    sm, xlb, xub, X, Y = _make_surrogate(cls, d, M, 256, precision)
    kind, h, prec, dtype, var_route = _posterior(L, sm)
    rng = np.random.default_rng(17)
    n = S * pop
    parm = rng.random((n, d)).astype(np.float32)
    obj = np.asarray(sm.evaluate(parm.astype(np.float64)), dtype=np.float32)
    vel = 0.1 * rng.standard_normal((n, d))
    a, b = L.SmpsoSwarms(parm, obj, vel, S, pop), L.SmpsoSwarms(parm, obj, vel, S, pop)
    ranks = L.DeviceArray((n,), np.int32)
    P = 2 * n
    xg, yg = L.pinned_empty((P, d)), L.pinned_empty((P, M))
    di = np.full(d, 20.0)
    for gen in range(2):
        sc = np.column_stack((0.1 + 0.4 * rng.random((S, 1)), 1.5 + rng.random((S, 1)), rng.random((S, 1)), 1.5 + rng.random((S, 1)),
                              rng.random((S, 1)), 0.5 + rng.random((S, 1)), rng.integers(0, pop, (S, 2)).astype(np.float64)))
        draw = (123, 7 + gen)
        a.step_record(kind, h, draw, var_route, di, xlb, xub, 1.0 / d, 31, 40 + gen, prec, dtype == np.float32, metric, sc, ranks, xg, yg)
        L.synchronize()
        x_gen = b.generate(di, xlb, xub, 1.0 / d, 31, 40 + gen)
        if kind == L.POSTERIOR_DGP:
            mean, _ = h.predict(x_gen, seed=draw[0], stream_id=draw[1], return_var=True, precision=prec)
        else:
            mean, _ = h.predict(x_gen, return_var=var_route, precision=prec)
        if dtype == np.float32:
            mean = mean.astype(np.float32).astype(np.float64)
        po, oo = np.empty((n, d), np.float32), np.empty((n, M), np.float32)
        r, _ = b.update(x_gen, mean, sc, xlb, xub, metric, po, oo)
        msg = (cls, precision, gen)
        assert np.array_equal(xg, x_gen) and np.array_equal(yg, mean), msg
        for u, v in ((a.parm, b.parm), (a.obj, b.obj), (a.vel, b.vel)):
            assert np.array_equal(u.download(), v.download()), msg
        assert np.array_equal(a.parm.download(), po.astype(np.float64)) and np.array_equal(a.obj.download(), oo.astype(np.float64)), msg
        assert np.array_equal(ranks.download(), r.reshape(-1)), msg


def test_step_refuses_bad_arguments_before_any_launch(L):
    from dmosopt_b200 import _lib

    d, M, S, pop = 6, 2, 2, 16
    n = S * pop
    gpr = _make_surrogate("GPR_Matern", d, M, 128, "fp64")[0]
    egp = surrogate("EGP_Matern", d, M, 128, "fp64")[0]
    svgp = surrogate("SVGP_Matern", d, M, 128, "fp64")[0]
    dgp = surrogate("MDGP_Matern", d, M, 128, "fp64")[0]
    wide = surrogate("EGP_Matern", d + 1, M, 128, "fp64")[0]
    tall = surrogate("EGP_Matern", d, M + 1, 128, "fp64")[0]
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    rng = np.random.default_rng(2)
    sw = L.SmpsoSwarms(rng.random((n, d)).astype(np.float32), rng.random((n, M)).astype(np.float32), rng.random((n, d)), S, pop)
    ranks = DA((n,), np.int32)
    host_parm = np.zeros((n, d))
    di, xlb, xub = np.full(d, 20.0), np.zeros(d), np.ones(d)
    good_sc = np.tile([0.3, 2.0, 0.5, 2.0, 0.5, 0.7, 1.0, 2.0], (S, 1))
    dev_sc = DA((S, 8)).upload(good_sc)
    xg, yg = L.pinned_empty((2 * n, d)), L.pinned_empty((2 * n, M))

    def call(kind=_lib.POSTERIOR_GP, h=gpr._gp._h, var_route=0, prec=L.GP_FP64, stream=0, parm=sw.parm.ptr, rk=ranks.ptr, sc=good_sc,
             x=xg, y=yg):
        L.synchronize()
        l0 = L.launch_count()
        scp = sc.ptr if isinstance(sc, L.DeviceArray) else sc.ctypes.data
        st = lib.dmo_smpso_step_record(ctx, kind, h, 9, stream, var_route, L._ptr(parm), sw.obj.ptr, sw.vel.ptr, S, pop, d, M, di.ctypes.data,
                                       xlb.ctypes.data, xub.ctypes.data, 1.0 / d, 5, 1, prec, 0, 1, scp, L._ptr(rk), L._ptr(x), L._ptr(y))
        return st, L.launch_count() - l0

    bad_leader = good_sc.copy()
    bad_leader[1, 7] = pop
    assert call(kind=3) == (2, 0)
    assert call(kind=-1) == (2, 0)
    assert call(h=None) == (2, 0)
    assert call(kind=_lib.POSTERIOR_GP, h=egp._gp._h, var_route=1, prec=L.GP_AUTO) == (2, 0)  # AUTO with flag 1
    assert call(kind=_lib.POSTERIOR_SVGP, h=svgp._h._h, var_route=0) == (2, 0)  # the mean-only predict is the exact GP's
    assert call(h=wide._gp._h, var_route=1) == (2, 0)
    assert call(h=tall._gp._h, var_route=1) == (2, 0)
    assert call(parm=host_parm) == (2, 0)
    assert call(rk=np.zeros(n, np.int32)) == (2, 0)
    assert call(sc=dev_sc) == (2, 0)
    assert call(x=None) == (2, 0)
    assert call(y=None) == (2, 0)
    assert call(sc=bad_leader) == (2, 0)
    assert call(kind=_lib.POSTERIOR_DGP, h=dgp._gp._h, var_route=1, stream=1 << 54) == (2, 0)
    st, launched = call(kind=_lib.POSTERIOR_DGP, h=dgp._gp._h, var_route=1, stream=(1 << 54) - 1)
    assert st == 0 and launched > 0
    st, launched = call(prec=L.GP_AUTO)
    assert st == 0 and launched > 0


# ------------------------------------------------------------------------------------ 3. host traffic
@pytest.mark.parametrize("case", ["GPR_Matern-auto", "SVGP_Matern-tensor"])
def test_resident_generation_traffic(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case], pop=4096, S=5, gens=3)
    S, pop, d, M = c["S"], c["pop"], c["d"], c["M"]
    P = 2 * S * pop
    per_gen = []
    step = L.SmpsoSwarms.step_record

    def measured(self, *args, **kwargs):
        L.synchronize()
        b0 = L.transfer_bytes()
        out = step(self, *args, **kwargs)
        L.synchronize()
        b1 = L.transfer_bytes()
        per_gen.append((b1[0] - b0[0], b1[1] - b0[1]))
        return out

    monkeypatch.setattr(L.SmpsoSwarms, "step_record", measured)
    L.synchronize()
    w0 = L.wait_count()
    res = _run(MOASMO.optimize, c)
    w_res = L.wait_count() - w0
    w0 = L.wait_count()
    ref = _run(MOASMO.optimize_per_generation, c)
    w_ref = L.wait_count() - w0
    _assert_same(res, ref)
    assert len(per_gen) == c["gens"]
    for h2d, d2h in per_gen:
        assert d2h - P * (d + M) * 8 < S * pop * d * 4, (h2d, d2h)
        assert h2d < S * pop * M * 8, (h2d, d2h)
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
        optimizer_name="dmosopt_b200.SMPSO", optimizer_kwargs={"swarm_size": 3}, surrogate_method_name="dmosopt_b200.GPR_Matern",
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
    calls = []
    step = L.SmpsoSwarms.step_record

    def counted(self, *args, **kwargs):
        calls.append(1)
        return step(self, *args, **kwargs)

    monkeypatch.setattr(L.SmpsoSwarms, "step_record", counted)
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
