"""The resident surrogate epoch with the EGP, variational and deep-GP surrogates (dmo_nsga2_step_record_posterior).

1. MOASMO.optimize on that entry point against the per-generation plugin loop (optimize_per_generation), for each of
   the eight classes in float64 and on the tensor path: identical epoch results (dtypes included), optimizer state,
   success counters, operator parameters, Philox state, next draw of ``local_random`` and MDGP's call counter.
2. One call against the separate entry points on the same Philox streams: tournament, variation, the public predict
   with a variance buffer, the float32 cast where evaluate makes it, parents under the children, remove_worst and the
   float32 rounding of the survivors.  Population, ranks, record and count bit for bit; the host waits are the composed
   calls' minus their four trailing waits and minus the predict's watchdog read-back where the step runs no
   contraction.  Bad arguments are refused with zero launches.
3. The mean the step uses against the public predict's mean with the variance requested, bit for bit, at a population
   whose offspring span two candidate chunks of every route.
"""

import numpy as np
import pytest

from test_deepgp_cpu import problem

pytestmark = pytest.mark.gpu

VARIATIONAL = ("SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern", "CRV_Matern")
DEEP = ("MDSPP_Matern", "MDGP_Matern")
CLASSES = ("EGP_Matern",) + VARIATIONAL + DEEP


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


def _constraints(X):
    return np.column_stack((0.7 - X[:, 0], X[:, 1] - 0.2 + 0.1 * X[:, 2]))


def _lower(rng, n, Z):
    q = np.tril(0.3 * rng.standard_normal((n, Z, Z)), -1)
    for i in range(n):
        q[i][np.diag_indices(Z)] = 0.2 + 0.5 * rng.random(Z)
    return q


def surrogate(name, d, M, N, precision, seed=5, iso=True):
    """One of the eight classes from given hyper-parameters (no training) on DTLZ2 data in the unit cube."""
    from dmosopt_b200 import model_gpflow as mf
    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((N, d))
    Y = _dtlz2(X, M)
    if name == "EGP_Matern":
        ls = np.sqrt(d) * (0.3 + 0.3 * rng.random((M, 1 if iso else d)))
        hp = dict(lengthscale=np.broadcast_to(ls, (M, d)).copy(), outputscale=0.5 + rng.random(M), noise=np.full(M, 1e-3),
                  weight=0.1 * rng.standard_normal((M, d)), bias=0.1 * rng.standard_normal(M))
        return mg.EGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision), xlb, xub, X, Y
    if name in VARIATIONAL:
        ls = np.sqrt(d) * (0.4 + 0.6 * rng.random((M, d)))
        var = 0.5 + rng.random(M)
        if name == "SIV_Matern":
            ls[:], var[:] = ls[0], var[0]
        hp = dict(lengthscales=ls, variance=var, likelihood_variance=1e-3)
        if name == "CRV_Matern":
            Zn = min(N, 160)
            hp.update(Z=X[rng.choice(N, Zn, replace=False)], q_mu=rng.standard_normal((M, Zn)), q_sqrt=_lower(rng, M, Zn),
                      W=rng.standard_normal((M, M)))
        cls = getattr(mf, name)
        return cls(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision, seed=seed, return_mean_variance=False), xlb, xub, X, Y
    hp, *_ = problem(rng, d, 3, M, 96, 64, J=3, quadrature=name == "MDSPP_Matern")
    return getattr(mg, name)(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision), xlb, xub, X, Y


# ------------------------------------------------------------------------------------ 1. epoch parity
class _StopAt:
    def __init__(self, n):
        self.n, self.seen = n, []

    def has_terminated(self, opt):
        self.seen.append((opt.n_gen, opt.n_eval, np.array(opt.x), np.array(opt.y)))
        return opt.n_gen > self.n


BASE = dict(d=7, M=3, N=256, pop=2048, gens=3, metric=None, feasibility=False, adaptive=False, stop=None)
CASES = {f"{c}-{p}": dict(cls=c, precision=p) for c in CLASSES for p in ("fp64", "tensor")}
CASES.update({
    "odd_pop": dict(cls="SVGP_Matern", precision="tensor", pop=3001),
    "crowding": dict(cls="EGP_Matern", precision="tensor", metric="crowding"),
    "euclidean": dict(cls="MDSPP_Matern", precision="fp64", metric="euclidean"),
    "feasibility": dict(cls="VGP_Matern", precision="fp64", feasibility=True),
    "adaptive_rates": dict(cls="MDGP_Matern", precision="tensor", adaptive=True, gens=4),
    "termination": dict(cls="CRV_Matern", precision="tensor", stop=2, gens=10),
    "bench_shape": dict(cls="EGP_Matern", precision="tensor", d=30, N=1024, pop=65536, gens=2),
})


def _run(fn, c, seed=11):
    import dmosopt_b200 as b2
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    sm, xlb, xub, X, Y = surrogate(c["cls"], c["d"], c["M"], c["N"], c["precision"])
    feas = LogisticFeasibilityModel(X, _constraints(X)) if c["feasibility"] else None
    model = b2.Model(objective=sm, feasibility=feas)
    opt = b2.NSGA2(popsize=c["pop"], nInput=c["d"], nOutput=c["M"], model=model, distance_metric=c["metric"],
                   adaptive_operator_rates=c["adaptive"])
    rng = np.random.default_rng(seed)
    stop = None if c["stop"] is None else _StopAt(c["stop"])
    gen = fn(c["gens"], opt, model, c["d"], c["M"], xlb, xub, popsize=c["pop"], initial=(X[:64], Y[:64]), local_random=rng, termination=stop)
    with pytest.raises(StopIteration) as ex:
        next(gen)
    return ex.value.value, opt, rng, stop, sm


def _assert_same(a, b):
    res_a, opt_a, rng_a, stop_a, sm_a = a
    res_b, opt_b, rng_b, stop_b, sm_b = b
    for f in ("best_x", "best_y", "gen_index", "x", "y"):
        u, v = getattr(res_a, f), getattr(res_b, f)
        assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), f
    sa, sb = opt_a.state, opt_b.state
    for f in ("population_parm", "population_obj", "rank"):
        u, v = np.asarray(getattr(sa, f)), np.asarray(getattr(sb, f))
        assert u.dtype == v.dtype and np.array_equal(u, v), f
    for f in ("successful_crossovers", "total_crossovers", "successful_mutations", "total_mutations"):
        u, v = getattr(sa, f), getattr(sb, f)
        assert type(u) is type(v) and u == v, (f, u, v)
    pa, pb = opt_a.opt_params(), opt_b.opt_params()
    assert sorted(pa) == sorted(pb)
    for k in pa:
        if not callable(pa[k]):
            assert type(pa[k]) is type(pb[k]) and np.array_equal(np.asarray(pa[k]), np.asarray(pb[k])), k
    assert opt_a._philox_seed == opt_b._philox_seed and opt_a._philox_stream == opt_b._philox_stream
    assert rng_a.random() == rng_b.random()
    assert getattr(sm_a, "calls", None) == getattr(sm_b, "calls", None)
    if stop_a is not None:
        assert len(stop_a.seen) == len(stop_b.seen)
        for u, v in zip(stop_a.seen, stop_b.seen):
            assert u[:2] == v[:2] and u[2].dtype == v[2].dtype and np.array_equal(u[2], v[2]) and np.array_equal(u[3], v[3])


@pytest.mark.parametrize("case", list(CASES))
def test_resident_epoch_equals_plugin_loop(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    calls = []
    post = L.nsga2_step_record_posterior

    def counted(*args, **kwargs):
        calls.append(kwargs.get("key"))
        return post(*args, **kwargs)

    def refuse(*args, **kwargs):
        raise AssertionError("nsga2_step_record reached by a posterior surrogate")

    monkeypatch.setattr(L, "nsga2_step_record_posterior", counted)
    monkeypatch.setattr(L, "nsga2_step_record", refuse)
    res = _run(MOASMO.optimize, c)
    n_gens = c["gens"] if c["stop"] is None else c["stop"]
    assert len(calls) == n_gens, (case, len(calls))
    assert all((k is not None) == c["feasibility"] for k in calls)
    ref = _run(MOASMO.optimize_per_generation, c)
    assert len(calls) == n_gens
    _assert_same(res, ref)
    f32 = c["cls"] not in DEEP
    assert res[0].y.dtype == (np.float32 if f32 else np.float64)
    if c["cls"] == "MDGP_Matern":
        assert res[4].calls == 1 + n_gens  # the initial evaluate, then one draw per generation


# ------------------------------------------------------------------------------------ 2. the entry point
KIND_CASES = [(c, p) for c in ("EGP_Matern", "SVGP_Matern", "CRV_Matern", "MDSPP_Matern", "MDGP_Matern") for p in ("fp64", "tensor")]


def _kind(L, sm):
    kind, h, prec, dtype = sm.resident_posterior()
    return kind, h, prec, dtype == np.float32


def _public_predict(L, lib, ctx, kind, h, X, P, mean, var, prec, draw):
    if kind == L.POSTERIOR_GP:
        return L._check(lib.dmo_gp_predict(ctx, h._h, X, P, mean, var, prec), "gp_predict")
    if kind == L.POSTERIOR_SVGP:
        return L._check(lib.dmo_svgp_predict(ctx, h._h, X, P, mean, var, prec), "svgp_predict")
    return L._check(lib.dmo_dgp_predict(ctx, h._h, X, P, draw[0], draw[1], None, mean, var, prec), "dgp_predict")


@pytest.mark.parametrize("cls,precision", KIND_CASES)
def test_step_equals_the_separate_entry_points(L, cls, precision):
    d, M, pop, metric = 7, 3, 2047, 1
    sm, xlb, xub, X, Y = surrogate(cls, d, M, 256, precision)
    kind, h, prec, f32 = _kind(L, sm)
    rng = np.random.default_rng(17)
    x0 = rng.random((pop, d))
    y0 = np.asarray(sm.evaluate(x0), dtype=np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
    sx, sy, sr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    cx, cy, cr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    poolsize = pop // 2
    if (pop & 1) and (poolsize & 1):
        poolsize += 1
    cap = pop + 1
    pool, perm, kind_d = DA((poolsize,), np.int64), DA((pop,), np.int64), DA((cap,), np.int32)
    Xs, Ys, var = DA((cap + pop, d)), DA((cap + pop, M)), DA((cap, M))
    xg, yg, cg = L.pinned_empty((cap, d)), L.pinned_empty((cap, M)), L.pinned_empty((4,), np.int64)
    nch_s, nch_c = np.zeros(1, dtype=np.int64), np.zeros(1, dtype=np.int64)
    seed, stream = 31, 40

    def waits_of(fn):
        w0 = L.wait_count()
        fn()
        return L.wait_count() - w0

    for gen in range(2):
        draw = (123, 7 + gen)
        w_step = waits_of(lambda: L._check(lib.dmo_nsga2_step_record_posterior(
            ctx, kind, h._h, draw[0], draw[1], None, sx.ptr, sy.ptr, sr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr, dlb.ptr, dub.ptr,
            seed, stream, prec, metric, int(f32), 1, L._ptr(xg), L._ptr(yg), L._ptr(cg), nch_s.ctypes.data), "nsga2_step_record_posterior"))
        L.synchronize()
        w = {}
        w["tournament"] = waits_of(lambda: L._check(lib.dmo_tournament(ctx, cr.ptr, None, pop, poolsize, seed, stream, pool.ptr, None), "tournament"))
        w["generate"] = waits_of(lambda: L._check(lib.dmo_nsga2_generate(ctx, cx.ptr, pop, d, pool.ptr, poolsize, pop, 0.9, 0.1, 1.0 / d, dic.ptr,
                                                                          dim.ptr, dlb.ptr, dub.ptr, seed, stream + 1, Xs.ptr, kind_d.ptr,
                                                                          nch_c.ctypes.data, None), "generate"))
        P = int(nch_c[0])
        w["predict"] = waits_of(lambda: _public_predict(L, lib, ctx, kind, h, Xs.ptr, P, Ys.ptr, var.ptr, prec, draw))
        if f32:
            L.round_f32(Ys.ptr, P * M)
        L.memcpy(Xs.offset(P * d), cx.ptr, pop * d * 8)
        L.memcpy(Ys.offset(P * M), cy.ptr, pop * M * 8)
        w["truncate"] = waits_of(lambda: L._check(lib.dmo_remove_worst(ctx, Xs.ptr, Ys.ptr, P + pop, d, M, metric, None, 0, pop, cx.ptr, cy.ptr,
                                                                       cr.ptr, perm.ptr), "remove_worst"))
        L.round_f32(cy.ptr, pop * M)
        msg = (cls, precision, gen)
        assert int(nch_s[0]) == P, msg
        for a, b in zip((sx, sy, sr), (cx, cy, cr)):
            assert np.array_equal(a.download(), b.download()), msg
        xs, ys, k, pm = Xs.download()[:P], Ys.download()[:P], kind_d.download()[:P], perm.download()
        assert np.array_equal(xg[:P], xs) and np.array_equal(yg[:P], ys), msg
        if f32:
            assert np.array_equal(yg[:P], yg[:P].astype(np.float32)), msg
        kept = k[pm[pm < P]]
        assert cg.tolist() == [np.count_nonzero(k < 2), np.count_nonzero(k == 2), np.count_nonzero(kept < 2), np.count_nonzero(kept == 2)], msg
        # separate: tournament 1, generate 2 (count + trailing), predict 1 + the tensor watchdog's read-back, truncation
        # its own + 1.  The step keeps the count, the truncation's own and the watchdog only where a contraction runs (the
        # deep GP's hidden layer)
        tensor = precision == "tensor"
        assert w["tournament"] == 1 and w["generate"] == 2 and w["predict"] == (2 if tensor else 1), (msg, w)
        skipped = 1 if tensor and kind != L.POSTERIOR_DGP else 0
        assert w_step == sum(w.values()) - 4 - skipped, (msg, w_step, w)
        stream += 2


def test_step_refuses_bad_arguments_before_any_launch(L):
    from dmosopt_b200 import _lib

    d, M, pop = 6, 2, 64
    egp = surrogate("EGP_Matern", d, M, 128, "fp64")[0]
    dgp = surrogate("MDGP_Matern", d, M, 128, "fp64")[0]
    egp_wide = surrogate("EGP_Matern", d + 1, M, 128, "fp64")[0]
    egp_tall = surrogate("EGP_Matern", d, M + 1, 128, "fp64")[0]
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    rng = np.random.default_rng(2)
    px, py, pr = DA((pop, d)).upload(rng.random((pop, d))), DA((pop, M)).upload(rng.random((pop, M))), DA((pop,), np.int32).upload(np.zeros(pop, np.int32))
    dic, dim, xlb, xub = np.full(d, 1.0), np.full(d, 20.0), np.zeros(d), np.ones(d)
    xg, yg, cg = L.pinned_empty((pop + 1, d)), L.pinned_empty((pop + 1, M)), L.pinned_empty((4,), np.int64)
    nch = np.zeros(1, dtype=np.int64)

    def feas(width):
        J = 1
        return L.FeasModel(np.ones(J, dtype=np.int32), np.zeros((J, width)), np.eye(width)[None, : width - 1, :] * np.ones((J, 1, 1)),
                           np.zeros((J, width - 1)), np.ones((J, width - 1)), np.ones((J, width - 1)), np.zeros(J))

    good_key, bad_key = feas(d), feas(d + 1)

    def call(kind=_lib.POSTERIOR_GP, h=egp._gp._h, key=None, n=pop, x=xg, y=yg, c=cg, prec=L.GP_FP64, stream=0):
        L.synchronize()
        l0 = L.launch_count()
        st = lib.dmo_nsga2_step_record_posterior(ctx, kind, h, 9, stream, None if key is None else key._h, px.ptr, py.ptr, pr.ptr, n, d, M,
                                                 0.9, 0.1, 1.0 / d, dic.ctypes.data, dim.ctypes.data, xlb.ctypes.data, xub.ctypes.data, 5, 1,
                                                 prec, 0, 1, 1, L._ptr(x), L._ptr(y), L._ptr(c), nch.ctypes.data)
        return st, L.launch_count() - l0

    assert call(h=None) == (2, 0)
    assert call(kind=3) == (2, 0)
    assert call(kind=-1) == (2, 0)
    assert call(h=egp_wide._gp._h) == (2, 0)
    assert call(h=egp_tall._gp._h) == (2, 0)
    assert call(key=bad_key) == (2, 0)
    assert call(x=None) == (2, 0)
    assert call(y=None) == (2, 0)
    assert call(c=None) == (2, 0)
    assert call(n=1) == (2, 0)
    assert call(prec=L.GP_AUTO) == (2, 0)
    assert call(kind=_lib.POSTERIOR_DGP, h=dgp._gp._h, stream=1 << 54) == (2, 0)
    st, launched = call(kind=_lib.POSTERIOR_DGP, h=dgp._gp._h, stream=(1 << 54) - 1, key=good_key)
    assert st == 0 and launched > 0
    st, launched = call(key=good_key)
    assert st == 0 and launched > 0


# ------------------------------------------------------------------------------------ 3. the step's mean bits
MEAN_CASES = [("EGP_Matern", True), ("EGP_Matern", False), ("SVGP_Matern", True), ("CRV_Matern", True), ("MDSPP_Matern", True),
              ("MDGP_Matern", True)]


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
@pytest.mark.parametrize("cls,iso", MEAN_CASES)
def test_step_mean_is_the_predict_mean_with_variance(L, cls, iso, precision):
    # every predict chunks its candidates at 2^20 rows at most: offspring past that span two chunks on every route.
    # EGP isotropic runs the fused producer without its K* stores on the tensor path, anisotropic with three covariances
    # the two-kernel route without its contraction
    d, M = 7, 3
    pop = (1 << 20) + 1001
    sm, xlb, xub, X, Y = surrogate(cls, d, M, 256, precision, iso=iso)
    kind, h, prec, _ = _kind(L, sm)
    rng = np.random.default_rng(3)
    x0 = rng.random((pop, d))
    DA = L.DeviceArray
    px, py = DA((pop, d)).upload(x0), DA((pop, M)).upload(rng.random((pop, M)))
    pr = DA((pop,), np.int32).upload(np.zeros(pop, np.int32))
    xg, yg, cg = L.pinned_empty((pop + 1, d)), L.pinned_empty((pop + 1, M)), L.pinned_empty((4,), np.int64)
    draw = (77, 3)
    P = L.nsga2_step_record_posterior(kind, h, draw, px, py, pr, 0.9, 0.1, 1.0 / d, 1.0, 20.0, xlb, xub, 5, 2, prec, L.METRIC_NONE, False, False,
                                      xg, yg, cg)
    L.synchronize()
    assert P > (1 << 20)
    if kind == L.POSTERIOR_DGP:
        mean, var = h.predict(xg[:P], seed=draw[0], stream_id=draw[1], return_var=True, precision=prec)
    else:
        mean, var = h.predict(xg[:P], return_var=True, precision=prec)
    assert var is not None and np.all(np.isfinite(mean))
    assert np.array_equal(yg[:P], mean), (cls, precision, int(np.count_nonzero(yg[:P] != mean)))
