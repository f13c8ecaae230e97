"""The logistic feasibility model's restatement (oracle/feasibility.py) against the reference's fixture and against
scikit-learn; the host-side pieces of dmosopt_b200.feasibility (folds, PCA, limits) without a GPU."""

import warnings

import numpy as np
import pytest

from oracle import feasibility as of

DATASETS = ("tnk", "d30", "single")


def golden_hyper(g, name):
    hp = []
    J = g[f"{name}_C"].shape[1]
    for j in range(J):
        p = f"{name}_{j}_"
        k = int(g[p + "k"])
        if k == 0:
            hp.append(None)
            continue
        hp.append((k, float(g[p + "C"]), g[p + "pca_mean"], g[p + "components"], g[p + "scaler_mean"], g[p + "scaler_scale"],
                   g[p + "coef"], float(g[p + "intercept"])))
    return hp


@pytest.mark.parametrize("name", DATASETS)
def test_oracle_rebuilds_the_reference_predictions(golden, name):
    g = golden("feasibility")
    hp = golden_hyper(g, name)
    Q = g[f"{name}_query"]
    assert np.max(np.abs(of.proba(hp, Q) - g[f"{name}_proba"])) <= 1e-12
    assert np.max(np.abs(of.rank(hp, Q) - g[f"{name}_rank"])) <= 1e-12


def test_golden_single_class_constraint_has_probability_one(golden):
    g = golden("feasibility")
    assert int(g["d30_1_k"]) == 0
    assert np.all(g["d30_proba"][1] == 1.0)


@pytest.mark.parametrize("seed,n,pos", [(0, 50, 0.4), (1, 103, 0.1), (2, 37, 0.5), (3, 120, 1 / 120)])
def test_folds_equal_stratified_kfold(seed, n, pos):
    from sklearn.model_selection import StratifiedKFold

    from dmosopt_b200.feasibility import stratified_test_folds

    rng = np.random.default_rng(seed)
    c = (rng.random(n) < pos).astype(int)
    c[rng.integers(n)] = 1
    c[rng.integers(n)] = 0
    folds = of.test_folds(c)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        splits = list(StratifiedKFold(5).split(np.zeros((n, 1)), c))
    for f, (tr, te) in enumerate(splits):
        assert np.array_equal(np.flatnonzero(folds == f), te)
        assert np.array_equal(np.flatnonzero(folds != f), tr)
    assert np.array_equal(stratified_test_folds(c), folds)


@pytest.mark.parametrize("n,d", [(200, 2), (300, 6), (400, 30)])
def test_pca_equals_covariance_eigh(n, d):
    from sklearn.decomposition import PCA

    from dmosopt_b200.feasibility import pca_components

    rng = np.random.default_rng(n + d)
    X = rng.standard_normal((n, d)) @ rng.standard_normal((d, d)) + rng.standard_normal(d)
    p = PCA(svd_solver="covariance_eigh").fit(X)
    m, V = of.pca(X)
    assert np.max(np.abs(m - p.mean_)) <= 1e-12
    assert np.max(np.abs(V - p.components_)) <= 1e-12
    m2, V2 = pca_components(X)
    assert np.max(np.abs(m2 - p.mean_)) <= 1e-12 and np.max(np.abs(V2 - p.components_)) <= 1e-12


# saga stops at once when w stays 0 (its stopping rule watches the coefficients), so C is kept where w moves
@pytest.mark.parametrize("C", [0.3, 1.0, 20.0])
def test_l1_optimum_matches_tight_saga(C):
    from sklearn.linear_model import LogisticRegression

    rng = np.random.default_rng(int(C * 100))
    Z = rng.standard_normal((60, 3))
    y = (Z @ [1.0, -0.5, 0.0] + 0.8 * rng.standard_normal(60) > 0.2).astype(int)
    w, b, F = of.l1_logistic(Z, y, C)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        lr = LogisticRegression(penalty="l1", solver="saga", C=C, tol=1e-12, max_iter=100000).fit(Z, y)
    Fs = of.objective(Z, y, C, lr.coef_[0], lr.intercept_[0])
    assert F <= Fs * (1 + 1e-9) and abs(F - Fs) <= 1e-9 * abs(Fs)


def test_grid_choice_equals_gridsearchcv():
    from sklearn.decomposition import PCA
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import GridSearchCV
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    rng = np.random.default_rng(5)
    X = rng.standard_normal((80, 3)) * [3.0, 1.0, 0.3]
    c = (X[:, 0] + 0.3 * rng.standard_normal(80) > 0.5).astype(int)
    hp, _, means = of.grid_search(X, c, problems=True)
    ppl = make_pipeline(PCA(svd_solver="covariance_eigh"), StandardScaler(),
                        LogisticRegression(penalty="l1", solver="saga", tol=1e-12, max_iter=100000))
    grid = {"pca__n_components": range(1, 3), "logisticregression__C": of.C_GRID}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gs = GridSearchCV(ppl, grid, n_jobs=1).fit(X, c)
    # at C = 1e-4 w stays 0 and saga stops before its intercept converges (see above): compare the rows with C >= 1
    assert np.allclose(gs.cv_results_["mean_test_score"][4:], means.ravel()[4:], atol=1e-12)
    assert (hp[0], hp[1]) == (gs.best_params_["pca__n_components"], gs.best_params_["logisticregression__C"])


def test_single_member_minority_picks_the_first_grid_point():
    rng = np.random.default_rng(9)
    X = rng.random((40, 3))
    c = np.zeros(40, dtype=int)
    c[11] = 1
    hp, _, means = of.grid_search(X, c, problems=True)
    assert np.all(np.isnan(means)) and (hp[0], hp[1]) == (1, of.C_GRID[0])


def test_d1_raises():
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    X = np.linspace(0, 1, 20)[:, None]
    C = (X - 0.5).reshape(-1, 1)
    with pytest.raises(ValueError):
        of.fit(X, C)
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(X, C)


def test_limits_are_refused_on_the_host():
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(0)
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((50, 91)), rng.standard_normal((50, 1)))
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((50, 3)), rng.standard_normal((50, 33)))
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((65537, 2)), rng.standard_normal((65537, 1)))
    with pytest.raises(ValueError):
        LogisticFeasibilityModel(rng.random((50, 3)), rng.standard_normal((50, 1)), fit="saga")


def test_all_single_class_constraints_need_no_classifier():
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    rng = np.random.default_rng(1)
    X = rng.random((30, 4))
    m = LogisticFeasibilityModel(X, -np.ones((30, 2)))
    assert m.hyperparameters == [None, None]
    Q = rng.random((7, 4))
    assert np.array_equal(m.rank(Q), np.ones(7))
    assert np.array_equal(m.predict(Q), np.ones((7, 2), dtype=np.int64))
    assert np.array_equal(m.predict_proba(Q)[:, :, 1], np.ones((2, 7)))
