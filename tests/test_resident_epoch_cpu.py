"""Host logic of the resident surrogate epoch (dmosopt_b200.MOASMO.optimize) without a GPU.

The ``_lib`` calls are the oracle-backed test seam (fake_backend), and ``nsga2_step_record`` is composed here from the
seam's tournament, variation, GP posterior and truncation, in the order dmo_nsga2_step_record runs them.  Checked:
which epochs are eligible, the generator protocol, that the resident epoch leaves the same results and optimizer state
as the per-generation loop, and that ``install(resident_epoch=True)`` / ``uninstall()`` patch and restore the
reference's ``MOASMO.optimize`` while a plain ``install()`` leaves it alone.
"""

import sys

import numpy as np
import pytest

import fake_backend
from oracle import reference_build

REFERENCE = reference_build.reference_path()


class _DeviceArray:
    """A NumPy stand-in for _lib.DeviceArray."""

    def __init__(self, shape, dtype=np.float64):
        self.a = np.zeros(shape, dtype=dtype)
        self.shape, self.dtype = self.a.shape, self.a.dtype
        self.ptr = self

    def upload(self, a):
        self.a[...] = a
        return self

    def download(self):
        return self.a.copy()


def _step_record(gp, pop_x, pop_y, rank, crossover_prob, mutation_prob, mutation_rate, di_crossover, di_mutation, xlb, xub, seed,
                 stream_id, precision, metric, round_to_f32, x_gen, y_gen, counts, key=None):
    assert key is None
    pop = pop_x.shape[0]
    pool = fake_backend.tournament(rank.a, int(round(pop / 2.0)), seed, stream_id)
    xg, kind = fake_backend.nsga2_generate(pop_x.a, pool, pop, crossover_prob, mutation_prob, mutation_rate, di_crossover, di_mutation,
                                           xlb, xub, seed, stream_id + 1)
    P = xg.shape[0]
    yg, _ = gp.predict(xg, return_var=False, precision=precision)
    Xo, Yo, r, perm = fake_backend.remove_worst(np.vstack((xg, pop_x.a)), np.vstack((yg, pop_y.a)), pop, metric)
    pop_x.a[:] = Xo
    pop_y.a[:] = Yo.astype(np.float32) if round_to_f32 else Yo
    rank.a[:] = r
    x_gen[:P], y_gen[:P] = xg, yg
    kept = kind[perm[perm < P]]
    counts[:] = [np.count_nonzero(kind < 2), np.count_nonzero(kind == 2), np.count_nonzero(kept < 2), np.count_nonzero(kept == 2)]
    return P


@pytest.fixture
def fake(monkeypatch):
    from dmosopt_b200 import _lib

    fake_backend.install(monkeypatch)
    calls = []

    def record(*args, **kwargs):
        calls.append(1)
        return _step_record(*args, **kwargs)

    monkeypatch.setattr(_lib, "nsga2_step_record", record)
    monkeypatch.setattr(_lib, "DeviceArray", _DeviceArray)
    monkeypatch.setattr(_lib, "pinned_empty", lambda shape, dtype=np.float64: np.empty(shape, dtype=dtype))
    monkeypatch.setattr(_lib, "synchronize", lambda: None)
    monkeypatch.setattr(_lib, "mirror_register", lambda host, dev: None)  # host arrays only: no device mirrors
    return calls


def _dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


def _setup(d=5, M=2, pop=24, N=40, seed=3, metric=None, **opt_kwargs):
    import dmosopt_b200 as b2

    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((N, d))
    sm = b2.GPR_Matern(X, _dtlz2(X, M), d, M, xlb, xub, optimizer=None)
    model = b2.Model(objective=sm)
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=model, distance_metric=metric, **opt_kwargs)
    return opt, model, xlb, xub, (X[:8], _dtlz2(X[:8], M))


class _StopAt:
    def __init__(self, n):
        self.n, self.seen = n, []

    def has_terminated(self, opt):
        self.seen.append((opt.n_gen, opt.n_eval, opt.x.copy(), opt.y.copy()))
        return opt.n_gen > self.n


def _run(route, gens=3, seed=11, initial=True, termination=None, **setup):
    from dmosopt_b200 import MOASMO

    opt, model, xlb, xub, init = _setup(**setup)
    rng = np.random.default_rng(seed)
    fn = MOASMO.optimize if route == "resident" else MOASMO.optimize_per_generation
    gen = fn(gens, opt, model, opt.nInput, opt.nOutput, xlb, xub, popsize=opt.popsize, initial=init if initial else None,
             local_random=rng, termination=termination)
    with pytest.raises(StopIteration) as ex:
        next(gen)
    return ex.value.value, opt, rng


def _assert_same(a, b):
    res_a, opt_a, rng_a = a
    res_b, opt_b, rng_b = b
    for f in ("best_x", "best_y", "gen_index", "x", "y"):
        u, v = getattr(res_a, f), getattr(res_b, f)
        assert u.dtype == v.dtype and np.array_equal(u, v), f
    sa, sb = opt_a.state, opt_b.state
    for f in ("population_parm", "population_obj", "rank"):
        u, v = getattr(sa, f), getattr(sb, f)
        assert u.dtype == v.dtype and np.array_equal(u, v), f
    for f in ("successful_crossovers", "total_crossovers", "successful_mutations", "total_mutations"):
        u, v = getattr(sa, f), getattr(sb, f)
        assert type(u) is type(v) and u == v, (f, u, v)
    pa, pb = opt_a.opt_params(), opt_b.opt_params()
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert type(pa[k]) is type(pb[k]) and np.array_equal(np.asarray(pa[k]), np.asarray(pb[k])), k
    assert opt_a._philox_stream == opt_b._philox_stream and opt_a._philox_seed == opt_b._philox_seed
    assert rng_a.random() == rng_b.random()


@pytest.mark.parametrize("metric", [None, "crowding", "euclidean"])
def test_resident_epoch_equals_per_generation_loop(fake, metric):
    res = _run("resident", metric=metric)
    assert len(fake) == 3
    _assert_same(res, _run("per_generation", metric=metric))


def test_resident_epoch_odd_population_without_initial(fake):
    res = _run("resident", pop=23, initial=False, gens=4)
    assert len(fake) == 4
    _assert_same(res, _run("per_generation", pop=23, initial=False, gens=4))


def test_resident_epoch_adaptive_operator_rates(fake):
    kw = dict(gens=5, adaptive_operator_rates=True)
    res = _run("resident", **kw)
    assert len(fake) == 5
    _assert_same(res, _run("per_generation", **kw))


def test_resident_epoch_termination_stops_at_the_same_generation(fake):
    t_res, t_ref = _StopAt(2), _StopAt(2)
    res = _run("resident", gens=10, termination=t_res)
    assert len(fake) == 2
    _assert_same(res, _run("per_generation", gens=10, termination=t_ref))
    assert len(t_res.seen) == len(t_ref.seen) == 3
    for u, v in zip(t_res.seen, t_ref.seen):
        assert u[0] == v[0] and u[1] == v[1] and np.array_equal(u[2], v[2]) and np.array_equal(u[3], v[3])


def test_eligibility():
    import dmosopt_b200 as b2
    from dmosopt_b200.MOASMO import resident_eligible

    class _FakeGP:
        pass

    class _Surrogate(b2.GPR_Matern):
        pass

    def gp(cls=b2.GPR_Matern, mean_variance=False):
        sm = cls.__new__(cls)
        sm._gp, sm.return_mean_variance = _FakeGP(), mean_variance
        return sm

    def nsga2(model, **kw):
        return b2.NSGA2(popsize=10, nInput=3, nOutput=2, model=model, **kw)

    m = b2.Model(objective=gp())
    assert resident_eligible(nsga2(m, distance_metric=None), m)
    assert resident_eligible(nsga2(m, distance_metric="crowding"), m)
    assert resident_eligible(nsga2(m, distance_metric="euclidean"), m)
    assert resident_eligible(nsga2(m, adaptive_operator_rates=True), m)
    m_rbf = b2.Model(objective=gp(b2.GPR_RBF))
    assert resident_eligible(nsga2(m_rbf), m_rbf)

    assert not resident_eligible(nsga2(m), m, optimize_mean_variance=True)
    assert not resident_eligible(nsga2(m, adaptive_population_size=True), m)
    assert not resident_eligible(nsga2(m, distance_metric=lambda y: y[:, 0]), m)
    assert not resident_eligible(b2.AGEMOEA(popsize=10, nInput=3, nOutput=2, model=m), m)
    for sm in (gp(mean_variance=True), gp(_Surrogate), None):
        mm = b2.Model(objective=sm)
        assert not resident_eligible(nsga2(mm), mm)
    # a host x-metric (not the GPU feasibility model's rank)
    opt = nsga2(m)
    opt.x_distance_metrics = [lambda x: x[:, 0]]
    assert not resident_eligible(opt, m)


def test_generator_protocol_without_surrogate_still_yields(fake):
    """With model.objective None the epoch yields x and takes y back (MOASMO.py:57-58, 107-108)."""
    from dmosopt_b200 import MOASMO

    opt, model, xlb, xub, _ = _setup()
    sm = model.objective
    model.objective = None
    gen = MOASMO.optimize(2, opt, model, opt.nInput, opt.nOutput, xlb, xub, popsize=opt.popsize, local_random=np.random.default_rng(1))
    x = next(gen)
    n = 0
    try:
        while True:
            x = gen.send(sm.evaluate(x))
            n += 1
    except StopIteration as ex:
        res = ex.value
    assert n == 2 and len(fake) == 0
    assert res.gen_index.max() == 2 and res.x.shape[0] == res.y.shape[0]


def test_install_patches_and_restores_optimize_only_when_asked():
    if REFERENCE is None:
        pytest.skip("reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
    import dmosopt_b200 as b2

    sys.path.insert(0, REFERENCE)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(REFERENCE)
    original = MOASMO.optimize
    try:
        names = b2.install()
        assert MOASMO.optimize is original and not any(n.endswith(".optimize") for n in names)
        names = b2.install(resident_epoch=True)
        assert MOASMO.optimize is not original and "dmosopt.MOASMO.optimize" in names
        b2.uninstall()
        assert MOASMO.optimize is original
        b2.install(resident_epoch=True)
        assert MOASMO.optimize is not original
    finally:
        b2.uninstall()
    assert MOASMO.optimize is original


def _reference_epoch(MOASMO, seed):
    d, M, pop = 6, 2, 24
    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((40, d))
    Y = _dtlz2(X, M)
    gen = MOASMO.epoch(
        4, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop,
        optimizer_name="dmosopt_b200.NSGA2", surrogate_method_name="dmosopt_b200.GPR_Matern",
        surrogate_method_kwargs={"anisotropic": False, "optimizer": None}, local_random=rng,
    )
    with pytest.raises(StopIteration) as ex:
        next(gen)
    return ex.value.args[0]


@pytest.mark.skipif(REFERENCE is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_unmodified_reference_epoch_same_with_resident_route(fake):
    import dmosopt_b200 as b2

    sys.path.insert(0, REFERENCE)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(REFERENCE)
    plain = _reference_epoch(MOASMO, 5)
    assert len(fake) == 0
    try:
        b2.install(resident_epoch=True)
        routed = _reference_epoch(MOASMO, 5)
    finally:
        b2.uninstall()
    assert len(fake) == 4
    assert sorted(plain) == sorted(routed)
    for k in plain:
        u, v = plain[k], routed[k]
        if isinstance(u, np.ndarray):
            assert u.dtype == v.dtype and np.array_equal(u, v), k
        elif k == "optimizer":
            assert type(u) is type(v)
        elif isinstance(u, (int, float, str, type(None))):
            assert u == v, k
