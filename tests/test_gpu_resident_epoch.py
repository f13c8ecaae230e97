"""The resident surrogate epoch (dmosopt_b200.MOASMO.optimize on dmo_nsga2_step_record) against the per-generation
plugin loop, on the GPU.

The plugin loop is the same ``optimize`` with the route disabled (``optimize_per_generation``), given an identically
seeded ``local_random``: the epoch results, the optimizer state after the epoch and the next draw of ``local_random`` must
be identical.  dmo_nsga2_step_record itself must equal dmo_nsga2_step (mean only, no hypervolume) bit for bit, record what
the separate entry points produce on the same Philox streams, wait on the host exactly as often as dmo_nsga2_step, and
refuse bad arguments before it launches anything.  Epochs the resident step does not cover must never reach it."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


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


class _StopAt:
    """Stops before generation n + 1; keeps what it was shown."""

    def __init__(self, n):
        self.n, self.seen = n, []

    def has_terminated(self, opt):
        self.seen.append((opt.n_gen, opt.n_eval, np.array(opt.x), np.array(opt.y), opt.c))
        return opt.n_gen > self.n


# name: dict(d, M, N, pop, gens, surrogate, precision, metric, initial, on_training, feasibility, adaptive, stop)
BASE = dict(d=7, M=3, N=512, pop=3001, gens=3, surrogate="GPR_Matern", precision="auto", metric=None, initial=True,
            on_training=False, feasibility=False, adaptive=False, stop=None)
CASES = {
    "odd_pop": {},
    "bench_shape": dict(d=30, N=1024, pop=65536, gens=2),
    "many_objectives": dict(M=9, pop=2048, d=10),
    "crowding": dict(metric="crowding"),
    "euclidean": dict(metric="euclidean"),
    "fp64": dict(precision="fp64", pop=2048),
    "tensor": dict(precision="tensor", pop=2048),
    # the population starts on the training inputs: offspring that mutation barely moves sit next to them
    "auto_on_training": dict(d=30, N=4096, pop=4096, on_training=True, initial=False),
    "rbf": dict(surrogate="GPR_RBF", pop=2048),
    "feasibility": dict(feasibility=True, pop=2048),
    "adaptive_rates": dict(adaptive=True, gens=4, pop=2048),
    "termination": dict(stop=2, gens=10, pop=2048),
    "no_initial": dict(initial=False, pop=2048),
}


def _setup(c, seed=7):
    import dmosopt_b200 as b2
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(seed)
    d, M = c["d"], c["M"]
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((c["N"], d))
    Y = _dtlz2(X, M)
    sm = getattr(b2, c["surrogate"])(X, Y, d, M, xlb, xub, optimizer=None, precision=c["precision"])
    feas = LogisticFeasibilityModel(X, _constraints(X)) if c["feasibility"] else None
    model = b2.Model(objective=sm, feasibility=feas)
    kw = {}
    if c["on_training"]:
        kw["initial_sampling_method"] = lambda local_random, n, nInput, lb, ub: X[:n].copy()
    opt = b2.NSGA2(popsize=c["pop"], nInput=d, nOutput=M, model=model, distance_metric=c["metric"], adaptive_operator_rates=c["adaptive"], **kw)
    initial = (X[:64], Y[:64]) if c["initial"] else None
    return opt, model, xlb, xub, initial


def _run(fn, c, seed=11):
    opt, model, xlb, xub, initial = _setup(c)
    rng = np.random.default_rng(seed)
    stop = None if c["stop"] is None else _StopAt(c["stop"])
    gen = fn(c["gens"], opt, model, opt.nInput, opt.nOutput, xlb, xub, popsize=opt.popsize, initial=initial, local_random=rng,
             termination=stop)
    with pytest.raises(StopIteration) as ex:
        next(gen)
    return ex.value.value, opt, rng, stop


def _assert_same(a, b):
    res_a, opt_a, rng_a, stop_a = a
    res_b, opt_b, rng_b, stop_b = b
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
        if callable(pa[k]):
            continue
        assert type(pa[k]) is type(pb[k]) and np.array_equal(np.asarray(pa[k]), np.asarray(pb[k])), k
    assert opt_a._philox_seed == opt_b._philox_seed and opt_a._philox_stream == opt_b._philox_stream
    assert rng_a.random() == rng_b.random()
    if stop_a is not None:
        assert len(stop_a.seen) == len(stop_b.seen)
        for u, v in zip(stop_a.seen, stop_b.seen):
            assert u[0] == v[0] and u[1] == v[1] and u[4] is None and v[4] is None
            assert u[2].dtype == v[2].dtype and np.array_equal(u[2], v[2]) and u[3].dtype == v[3].dtype and np.array_equal(u[3], v[3])


@pytest.mark.parametrize("case", list(CASES))
def test_resident_epoch_equals_plugin_loop(L, case, monkeypatch):
    from dmosopt_b200 import MOASMO

    c = dict(BASE, **CASES[case])
    calls = []
    record = L.nsga2_step_record

    def counted(*args, **kwargs):
        calls.append(kwargs.get("key"))
        return record(*args, **kwargs)

    monkeypatch.setattr(L, "nsga2_step_record", counted)
    res = _run(MOASMO.optimize, c)
    n_gens = c["gens"] if c["stop"] is None else c["stop"]
    assert len(calls) == n_gens, (case, len(calls))
    assert all((k is not None) == c["feasibility"] for k in calls)
    monkeypatch.setattr(L, "nsga2_step_record", record)
    ref = _run(MOASMO.optimize_per_generation, c)
    assert len(calls) == n_gens
    _assert_same(res, ref)
    assert res[0].gen_index.max() == n_gens


def _device_case(L, d, M, N, pop, seed):
    import dmosopt_b200 as b2

    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    sm = b2.GPR_Matern(Xtr, _dtlz2(Xtr, M), d, M, xlb, xub, optimizer=None)
    x0 = rng.random((pop, d))
    y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    return sm, xlb, xub, x0, y0, r0


@pytest.mark.parametrize("pop,d,N,metric", [(8193, 30, 1024, 0), (4096, 12, 512, 1), (2047, 7, 256, 2)])
def test_record_equals_step_and_the_separate_entry_points(L, pop, d, N, metric):
    M = 3
    sm, xlb, xub, x0, y0, r0 = _device_case(L, d, M, N, pop, seed=pop)
    gp = sm._gp
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
    pops = {k: (DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)) for k in ("step", "rec", "comp")}
    poolsize = pop // 2
    if (pop & 1) and (poolsize & 1):
        poolsize += 1
    cap = pop + 1
    pool, perm, kind = DA((poolsize,), np.int64), DA((pop,), np.int64), DA((cap,), np.int32)
    Xs, Ys = DA((cap + pop, d)), DA((cap + pop, M))
    nch_s, nch_r, nch_c = (np.zeros(1, dtype=np.int64) for _ in range(3))
    seed, stream = 99, 20
    prec = L.GP_AUTO

    def waits_of(fn):
        w0 = L.wait_count()
        fn()
        return L.wait_count() - w0

    # where the record goes: page-locked host memory, device memory, pageable host memory (one wait per output)
    dests = [
        ("pinned", L.pinned_empty((cap, d)), L.pinned_empty((cap, M)), L.pinned_empty((4,), np.int64), 0),
        ("device", DA((cap, d)), DA((cap, M)), DA((4,), np.int64), 0),
        ("pageable", np.empty((cap, d)), np.empty((cap, M)), np.empty(4, dtype=np.int64), 3),
    ]
    for gen, (where, xg, yg, cg, extra) in enumerate(dests):
        sx, sy, sr = pops["step"]
        w_step = waits_of(lambda: L._check(lib.dmo_nsga2_step(ctx, gp._h, sx.ptr, sy.ptr, sr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr,
                                                              dlb.ptr, dub.ptr, seed, stream, prec, metric, 0, 1, None, nch_s.ctypes.data, None),
                                           "nsga2_step"))
        rx, ry, rr = pops["rec"]
        w_rec = waits_of(lambda: L._check(lib.dmo_nsga2_step_record(ctx, gp._h, None, rx.ptr, ry.ptr, rr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr,
                                                                    dim.ptr, dlb.ptr, dub.ptr, seed, stream, prec, metric, 1, L._ptr(xg),
                                                                    L._ptr(yg), L._ptr(cg), nch_r.ctypes.data), "nsga2_step_record"))
        L.synchronize()
        msg = (pop, where, gen)
        assert w_rec == w_step + extra, (msg, w_rec, w_step)
        P = int(nch_r[0])
        assert int(nch_s[0]) == P, msg
        for a, b in zip(pops["step"], pops["rec"]):
            assert np.array_equal(a.download(), b.download()), msg

        # the same generation from the separate entry points
        cx, cy, cr = pops["comp"]
        L._check(lib.dmo_tournament(ctx, cr.ptr, None, pop, poolsize, seed, stream, pool.ptr, None), "tournament")
        L._check(lib.dmo_nsga2_generate(ctx, cx.ptr, pop, d, pool.ptr, poolsize, pop, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr, dlb.ptr, dub.ptr, seed,
                                        stream + 1, Xs.ptr, kind.ptr, nch_c.ctypes.data, None), "generate")
        assert int(nch_c[0]) == P, msg
        L._check(lib.dmo_gp_predict(ctx, gp._h, Xs.ptr, P, Ys.ptr, None, prec), "gp_predict")
        L.memcpy(Xs.offset(P * d), cx.ptr, pop * d * 8)
        L.memcpy(Ys.offset(P * M), cy.ptr, pop * M * 8)
        L._check(lib.dmo_remove_worst(ctx, Xs.ptr, Ys.ptr, P + pop, d, M, metric, None, 0, pop, cx.ptr, cy.ptr, cr.ptr, perm.ptr), "remove_worst")
        L.round_f32(cy.ptr, pop * M)
        for a, b in zip(pops["comp"], pops["rec"]):
            assert np.array_equal(a.download(), b.download()), msg

        xs, ys, k, pm = Xs.download()[:P], Ys.download()[:P], kind.download()[:P], perm.download()
        got = [np.asarray(a.download() if isinstance(a, DA) else a) for a in (xg, yg, cg)]
        assert np.array_equal(got[0][:P], xs) and np.array_equal(got[1][:P], ys), msg
        kept = k[pm[pm < P]]
        want = [np.count_nonzero(k < 2), np.count_nonzero(k == 2), np.count_nonzero(kept < 2), np.count_nonzero(kept == 2)]
        assert got[2].tolist() == want, (msg, got[2], want)
        assert want[0] + want[1] == P and want[2] + want[3] > 0
        stream += 2


def _feas_model(L, d):
    J = 1
    return L.FeasModel(np.ones(J, dtype=np.int32), np.zeros((J, d)), np.eye(d)[None, : d - 1, :] * np.ones((J, 1, 1)), np.zeros((J, d - 1)),
                       np.ones((J, d - 1)), np.ones((J, d - 1)), np.zeros(J))


def test_record_refuses_bad_arguments_before_any_launch(L):
    d, M, pop = 6, 2, 64
    sm, xlb, xub, x0, y0, r0 = _device_case(L, d, M, 128, pop, seed=1)
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    px, py, pr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    dic, dim = np.full(d, 1.0), np.full(d, 20.0)
    xg, yg, cg = L.pinned_empty((pop + 1, d)), L.pinned_empty((pop + 1, M)), L.pinned_empty((4,), np.int64)
    nch = np.zeros(1, dtype=np.int64)
    good_key, bad_key = _feas_model(L, d), _feas_model(L, d + 1)

    def call(key=None, n=pop, x=xg, y=yg, c=cg):
        L.synchronize()
        l0 = L.launch_count()
        st = lib.dmo_nsga2_step_record(ctx, sm._gp._h, None if key is None else key._h, px.ptr, py.ptr, pr.ptr, n, d, M, 0.9, 0.1, 1.0 / d,
                                       dic.ctypes.data, dim.ctypes.data, xlb.ctypes.data, xub.ctypes.data, 5, 1, L.GP_FP64, 0, 1,
                                       L._ptr(x), L._ptr(y), L._ptr(c), nch.ctypes.data)
        return st, L.launch_count() - l0

    assert call(key=bad_key) == (2, 0)
    assert call(x=None) == (2, 0)
    assert call(y=None) == (2, 0)
    assert call(c=None) == (2, 0)
    assert call(n=1) == (2, 0)
    st, launched = call(key=good_key)  # the same call with a key of the right width runs
    assert st == 0 and launched > 0


def _fallback_setups():
    import dmosopt_b200 as b2
    from dmosopt_b200.model_gpytorch import MEGP_Matern
    from dmosopt_b200.parallel import ShardedSurrogate

    d, M, pop = 6, 2, 512
    rng = np.random.default_rng(3)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((256, d))
    Y = _dtlz2(X, M)

    def gpr(**kw):
        return b2.GPR_Matern(X, Y, d, M, xlb, xub, optimizer=None, **kw)

    def megp():
        hp = dict(lengthscale=np.full(d, 0.8), covar_factor=np.ones((M, 1)), var=np.full(M, 0.5), task_noises=np.full(M, 1e-3), noise=1e-3,
                  weights=np.zeros((M, d)), biases=np.zeros(M))
        return MEGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp)

    def nsga2(model, **kw):
        return b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=model, **kw)

    def agemoea(model, **kw):
        return b2.AGEMOEA(popsize=pop, nInput=d, nOutput=M, model=model, **kw)

    # name: (surrogate factory, optimizer factory, optimize_mean_variance)
    return xlb, xub, (X[:32], Y[:32]), {
        "agemoea": (gpr, agemoea, {}, False),
        "megp": (megp, nsga2, {}, False),
        "mean_variance": (lambda: gpr(return_mean_variance=True), nsga2, {"optimize_mean_variance": True}, True),
        "adaptive_population_size": (gpr, nsga2, {"adaptive_population_size": True}, False),
        "callable_metric": (gpr, nsga2, {"distance_metric": lambda y: y[:, 0]}, False),
        "sharded": (lambda: ShardedSurrogate(gpr()), nsga2, {}, False),
    }


@pytest.mark.parametrize("case", ["agemoea", "megp", "mean_variance", "adaptive_population_size", "callable_metric", "sharded"])
def test_ineligible_epochs_run_the_plugin_loop(L, case, monkeypatch):
    import dmosopt_b200 as b2
    from dmosopt_b200 import MOASMO

    def refuse(*args, **kwargs):
        raise AssertionError("nsga2_step_record reached by an ineligible epoch")

    monkeypatch.setattr(L, "nsga2_step_record", refuse)
    out = []
    for fn in (MOASMO.optimize, MOASMO.optimize_per_generation):
        xlb, xub, initial, setups = _fallback_setups()
        make_sm, make_opt, kw, mv = setups[case]
        model = b2.Model(objective=make_sm(), return_mean_variance=mv)
        opt = make_opt(model, **kw)
        assert not MOASMO.resident_eligible(opt, model, mv)
        rng = np.random.default_rng(21)
        # with mean-variance objectives the initial rows would need their variances too: the epoch starts without them
        gen = fn(3, opt, model, opt.nInput, opt.nOutput, xlb, xub, popsize=opt.popsize, initial=None if mv else initial, local_random=rng,
                 optimize_mean_variance=mv)
        with pytest.raises(StopIteration) as ex:
            next(gen)
        out.append((ex.value.value, rng.random()))
    (a, ra), (b, rb) = out
    assert ra == rb
    for f in ("best_x", "best_y", "gen_index", "x", "y"):
        u, v = getattr(a, f), getattr(b, f)
        assert u.dtype == v.dtype and np.array_equal(u, v), (case, f)
