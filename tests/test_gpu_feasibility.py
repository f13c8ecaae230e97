"""Logistic feasibility model on the GPU (csrc/feasibility.cu, dmosopt_b200/feasibility.py): the reference's recorded
predictions, the batched L1-logistic grid search against oracle/feasibility.py, the edges of the shape envelope, the
resident NSGA-II update with the feasibility key, and the unmodified reference's MOASMO.epoch."""

import numpy as np
import pytest

from oracle import feasibility as of

pytestmark = pytest.mark.gpu

DATASETS = ("tnk", "d30", "single")


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def golden_hyper(g, name):
    hp = []
    for j in range(g[f"{name}_C"].shape[1]):
        p = f"{name}_{j}_"
        k = int(g[p + "k"])
        hp.append(None if k == 0 else (k, float(g[p + "C"]), g[p + "pca_mean"], g[p + "components"], g[p + "scaler_mean"],
                                       g[p + "scaler_scale"], g[p + "coef"], float(g[p + "intercept"])))
    return hp


def tnk(X):
    c0 = -(np.square(X[:, 0]) + np.square(X[:, 1]) - 1.0 - 0.1 * np.cos(16.0 * np.arctan(X[:, 0] / X[:, 1])))
    c1 = 2 * (np.square(X[:, 0] - 0.5) + np.square(X[:, 1] - 0.5)) - 1
    return np.column_stack((c0, c1))


def noisy(rng, N, d):
    """d inputs, two constraints with 10 % label noise and unbalanced classes (no intercept-only optimum sits at t = 0)."""
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    a = X @ rng.standard_normal(d)
    b = X[:, 0] - X[:, -1]
    C = np.column_stack((a - np.quantile(a, 0.35), b - np.quantile(b, 0.6)))
    flip = rng.random(C.shape) < 0.1
    return X, np.where(flip, -C, C)


# ------------------------------------------------------------------------------------------ the reference's predictions
@pytest.mark.parametrize("name", DATASETS)
def test_golden_hyperparameters_give_the_reference_predictions(L, golden, name):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    g = golden("feasibility")
    m = LogisticFeasibilityModel(None, None, hyperparameters=golden_hyper(g, name))
    Q = g[f"{name}_query"]
    e_p = np.max(np.abs(m.predict_proba(Q)[:, :, 1] - g[f"{name}_proba"]))
    e_r = np.max(np.abs(m.rank(Q) - g[f"{name}_rank"]))
    print(f"{name}: max |proba - reference| {e_p:.3e}, max |rank - reference| {e_r:.3e}")
    assert e_p <= 1e-11 and e_r <= 1e-11
    pred = m.predict(Q)
    assert pred.shape == (Q.shape[0], g[f"{name}_C"].shape[1])
    assert np.array_equal(pred, (g[f"{name}_proba"].T > 0.5).astype(pred.dtype))


# ------------------------------------------------------------------------------------------ the fit against the oracle
def _fit_cases():
    rng = np.random.default_rng(3)
    X = rng.uniform(0.0, np.pi, (200, 2))
    yield "tnk", X, tnk(X)
    yield "d6", *noisy(np.random.default_rng(4), 253, 6)


@pytest.mark.parametrize("case", ["tnk", "d6"])
def test_fit_matches_the_oracle(L, case):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    X, C = dict((n, (x, c)) for n, x, c in _fit_cases())[case]
    m = LogisticFeasibilityModel(X, C)
    d = X.shape[1]
    ref = []
    for j in range(C.shape[1]):
        c = (C[:, j] > 0).astype(int)
        hp, detail, _ = of.grid_search(X, c, problems=True)
        ref.append(hp)
        info = m.fit_info["per_constraint"][j]
        bad = (info["iters"] >= 0) & ~info["converged"]
        assert not bad.any(), (np.argwhere(bad), info["kkt"][bad], info["iters"][bad])
        for (f, ci, k), (w, b, F, cor) in detail.items():
            Fg = info["objective"][f, ci, k - 1]
            assert Fg <= F * (1 + 1e-9), (j, f, ci, k, Fg, F)
            cg = info["coef"][f, ci, k - 1]
            wo = np.append(w, b)
            wg = np.append(cg[:k], cg[d - 1])
            assert np.max(np.abs(wg - wo)) <= 1e-6 * np.max(np.abs(wo)), (j, f, ci, k)
            if cor is not None:
                tr = of.test_folds(c) != f
                Z = of.dataset(X, tr)[4]
                assert np.min(np.abs(Z[~tr, :k] @ w + b)) > 1e-6, "a held-out row sits on the boundary"
                assert info["correct"][f, ci, k - 1] == cor
        assert m.hyperparameters[j][:2] == hp[:2]
    Q = np.random.default_rng(5).random((1000, d)) * (np.pi if case == "tnk" else np.linspace(1.0, 3.0, d))
    assert np.max(np.abs(m.rank(Q) - of.rank(ref, Q))) <= 1e-6


def test_fit_repeats_and_hyperparameters_round_trip(L):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    X, C = noisy(np.random.default_rng(6), 300, 8)
    a, b = LogisticFeasibilityModel(X, C), LogisticFeasibilityModel(X, C)
    for j in (0, 1):
        for key in ("objective", "coef", "kkt", "iters", "correct"):
            assert np.array_equal(a.fit_info["per_constraint"][j][key], b.fit_info["per_constraint"][j][key], equal_nan=True)
        for u, v in zip(a.hyperparameters[j], b.hyperparameters[j]):
            assert np.array_equal(u, v)
    r = LogisticFeasibilityModel(None, None, hyperparameters=a.hyperparameters)
    Q = np.random.default_rng(7).random((5000, 8))
    assert np.array_equal(r.rank(Q), a.rank(Q))
    assert np.array_equal(r.predict_proba(Q), a.predict_proba(Q))


def test_sklearn_fit_is_read_out_and_predicted_on_the_gpu(L):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    X, C = noisy(np.random.default_rng(8), 150, 4)
    m = LogisticFeasibilityModel(X, C, fit="sklearn")
    Q = np.random.default_rng(9).random((300, 4))
    assert np.max(np.abs(m.rank(Q) - of.rank(m.hyperparameters, Q))) <= 1e-12


# ------------------------------------------------------------------------------------------ edges
def test_single_class_and_single_member_minority(L):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(10)
    X = rng.random((121, 5))  # N not a multiple of 5
    c1 = -np.ones(121)
    c1[40] = 1.0
    C = np.column_stack((-np.ones(121), c1, X[:, 1] - 0.3))
    m = LogisticFeasibilityModel(X, C)
    assert m.hyperparameters[0] is None
    assert m.hyperparameters[1][:2] == (1, float(of.C_GRID[0]))  # every fold mean is NaN: the first grid point
    assert m.hyperparameters[2][:2] == of.grid_search(X, (C[:, 2] > 0).astype(int))[:2]
    Q = rng.random((50, 5))
    P = m.predict_proba(Q)[:, :, 1]
    assert np.all(P[0] == 1.0)
    assert np.max(np.abs(P - of.proba(of.fit(X, C), Q))) <= 1e-6


def test_d2_duplicates_and_constant_column(L):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(11)
    X = rng.random((80, 2))
    X = np.vstack((X, X[:20]))  # duplicate rows
    C = (X[:, :1] + 0.3 * X[:, 1:] - 0.55)
    m = LogisticFeasibilityModel(X, C)
    assert m.hyperparameters[0][0] == 1
    assert m.hyperparameters[0][:2] == of.grid_search(X, (C[:, 0] > 0).astype(int))[:2]
    Xc = np.column_stack((X, np.full(len(X), 0.25)))  # a constant column: its direction is the last component
    mc = LogisticFeasibilityModel(Xc, C)
    hp = of.grid_search(Xc, (C[:, 0] > 0).astype(int))
    assert mc.hyperparameters[0][:2] == hp[:2]
    Q = np.column_stack((rng.random((200, 2)), np.full(200, 0.25)))
    assert np.max(np.abs(mc.rank(Q) - of.rank([hp], Q))) <= 1e-6


@pytest.mark.parametrize("J,d", [(1, 3), (32, 90)])
def test_constraint_and_dimension_limits(L, J, d):
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(J + d)
    N = 400
    X = rng.random((N, d))
    C = X[:, :J] + 0.2 * X[:, 1:J + 1] - 0.6
    m = LogisticFeasibilityModel(X, C)
    assert len(m.hyperparameters) == J
    left = sum(m.fit_info["per_constraint"][j]["not_converged"] for j in range(J))
    print(f"J {J} d {d}: {left} problems short of the KKT tolerance")
    if d <= 10:
        assert left == 0
    Q = rng.random((2000, d))
    r = m.rank(Q)
    assert r.shape == (2000,) and np.all((r >= 0) & (r <= 1))
    assert np.max(np.abs(r - of.rank(m.hyperparameters, Q))) <= 1e-10


def test_shapes_past_the_limits_are_refused(L):
    from dmosopt_b200 import _lib
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(12)
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((50, 91)), rng.standard_normal((50, 1)))
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((50, 4)), rng.standard_normal((50, 33)))
    d, J = 91, 1
    with pytest.raises(_lib.DmoError, match="d=91"):
        _lib.feas_fit(rng.random((10, d)), np.ones((J, 10)), np.zeros((J, 10)), np.zeros((6 * J, d)), np.zeros((6 * J, d - 1, d)), [1.0])
    with pytest.raises(_lib.DmoError, match="N=4"):
        _lib.feas_fit(rng.random((4, 3)), np.ones((1, 4)), np.zeros((1, 4)), np.zeros((6, 3)), np.zeros((6, 2, 3)), [1.0])
    m = LogisticFeasibilityModel(*noisy(rng, 60, 3))
    with pytest.raises(ValueError):
        m.rank(rng.random((5, 4)))


# ------------------------------------------------------------------------------------------ resident NSGA-II update
def test_nsga2_update_with_the_device_key_equals_the_host_path(L):
    import types

    import dmosopt_b200 as b2
    from dmosopt_b200.MOEA import remove_worst
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(13)
    d, M, pop = 6, 2, 256
    X, C = noisy(rng, 300, d)
    fm = LogisticFeasibilityModel(X, C)
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=types.SimpleNamespace(objective=None, feasibility=fm), distance_metric=None)
    assert opt.x_distance_metrics == [fm.rank]

    def f(x):
        return np.column_stack((x[:, 0], 1 - np.sqrt(np.abs(x[:, 0])) + x[:, 1:].sum(axis=1)))

    x0 = rng.random((pop, d)) * np.linspace(1.0, 3.0, d)
    bounds = np.column_stack((np.zeros(d), np.linspace(1.0, 3.0, d)))
    opt.initialize_strategy(x0, f(x0), bounds, rng)
    x_gen, state = opt.generate()
    y_gen = f(np.asarray(x_gen))
    parm, obj = np.array(opt.state.population_parm), opt.state.population_obj.copy()
    xs, ys, rank, perm = remove_worst(np.vstack((x_gen, parm)), np.vstack((y_gen, obj)), pop, x_distance_metrics=[fm.rank],
                                      y_distance_metrics=None, return_perm=True)
    xd, yd, rd, pd = L.remove_worst_pair(x_gen, y_gen, parm, obj, pop, key=fm.device_model)
    assert np.array_equal(pd, perm) and np.array_equal(rd, rank) and np.array_equal(xd, xs) and np.array_equal(yd, ys)
    h0, _ = L.transfer_bytes()
    opt.update(x_gen, y_gen, state)
    h1, _ = L.transfer_bytes()
    assert h1 - h0 <= 2 * pop * M * 8, "x rows were uploaded for the feasibility key"
    assert np.array_equal(opt.state.population_parm, xs)
    assert np.array_equal(opt.state.population_obj, ys.astype(opt.state.population_obj.dtype))
    assert np.array_equal(opt.state.rank, rank)


# ------------------------------------------------------------------------------------------ through the unmodified reference
def _reference():
    from oracle import reference_build

    return reference_build.reference_path()


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_reference_epoch_with_the_gpu_feasibility_model(L, monkeypatch):
    import sys

    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    nsga2_mod = sys.modules["dmosopt_b200.NSGA2"]  # the package re-exports the class under the module's name

    ref = _reference()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    keys = []
    orig = nsga2_mod._device_feasibility_key

    def spy(metrics):
        k = orig(metrics)
        keys.append((metrics, k))
        return k

    monkeypatch.setattr(nsga2_mod, "_device_feasibility_key", spy)
    rng = np.random.default_rng(14)
    d, pop = 2, 64
    xlb, xub = np.zeros(d), np.full(d, np.pi)
    X = rng.uniform(0.0, np.pi, (120, d))
    gen = MOASMO.epoch(
        3, ["x0", "x1"], ["y1", "y2"], xlb, xub, 0.25, X, X.copy(), tnk(X), pop=pop, optimizer_name="dmosopt_b200.NSGA2",
        optimizer_kwargs={}, surrogate_method_name="dmosopt_b200.GPR_Matern", surrogate_method_kwargs={"optimizer": None},
        feasibility_method_name="logreg", surrogate_custom_training="dmosopt_b200.feasibility.train_with_feasibility",
        local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    assert keys, "the optimizer never updated with a feasibility metric"
    for metrics, k in keys:
        assert len(metrics) == 1 and isinstance(metrics[0].__self__, LogisticFeasibilityModel) and k is not None
    xr = res["x_resample"]
    assert xr.shape[1] == d and len(xr) > 0
