"""MEGP_Matern training on the GPU (row A19): dmo_mtgp_lml_grad against the dense torch autograd oracle
(oracle/megp_train.py, no block decomposition), megp_fit's Adam loop against torch.optim.Adam on that oracle, the fitted
surrogate against the hyper-parameters path and the dense posterior, and the unmodified reference controller training
the plugin without gpytorch."""

import sys

import numpy as np
import pytest

from oracle import megp, megp_train

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _zdt1(x):
    d = x.shape[1]
    g = 1.0 + 9.0 / (d - 1) * x[:, 1:].sum(axis=1)
    return np.column_stack((x[:, 0], g * (1.0 - np.sqrt(x[:, 0] / g))))


def _data(rng, N, d, M):
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, (t + 2) % d] + 0.2 * t * X[:, -1] ** 2 for t in range(M)])
    yn, _, _ = megp.normalise_y(Y)
    return X, yn


def _hyper(rng, d, M, tiny=False):
    F = rng.standard_normal((M, 1))
    var = 0.1 + 0.5 * rng.random(M)
    if tiny:  # one task with a ~1e-8 covariance factor and var: a tiny lambda_j
        F[-1, 0], var[-1] = 1e-8, 1e-8
    return dict(length_scale=np.exp(rng.uniform(np.log(0.05), np.log(5.0), d)), B=F @ F.T + np.diag(var),
                D=np.geomspace(2e-3, 2e-2, M), weight=0.3 * rng.standard_normal((M, d)), bias=0.2 * rng.standard_normal(M))


def _check_against_oracle(L, X, yn, hp):
    lml, g = L.mtgp_lml_grad(X, yn, *hp.values())
    ref, rg = megp_train.lml_and_grad_torch(X, yn, *hp.values())
    assert abs(lml - ref) <= 1e-10 * abs(ref), (lml, ref)
    for k in rg:
        err, scale = np.abs(g[k] - rg[k]).max(), np.abs(rg[k]).max()
        assert err <= 1e-8 * scale, (k, err, scale)
    return lml, g


@pytest.mark.parametrize("N", [150, 333])
@pytest.mark.parametrize("d", [2, 12, 40])
@pytest.mark.parametrize("M", [1, 2, 3, 5])
def test_lml_grad_vs_autograd_oracle(L, M, d, N):
    rng = np.random.default_rng(1000 * M + 10 * d + N)
    X, yn = _data(rng, N, d, M)
    _check_against_oracle(L, X, yn, _hyper(rng, d, M))


def test_lml_grad_with_a_tiny_task_eigenvalue(L):
    rng = np.random.default_rng(77)
    X, yn = _data(rng, 333, 12, 3)
    _check_against_oracle(L, X, yn, _hyper(rng, 12, 3, tiny=True))


def test_lml_grad_is_bit_identical_to_create_and_deterministic(L):
    rng = np.random.default_rng(5)
    N, d, M = 333, 7, 3
    X, yn = _data(rng, N, d, M)
    hp = _hyper(rng, d, M)
    a = L.mtgp_lml_grad(X, yn, *hp.values())
    b = L.mtgp_lml_grad(X, yn, *hp.values())
    assert a[0] == b[0] and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])
    h = L.MTGPHandle(X, yn, hp["length_scale"], hp["B"], hp["D"], hp["weight"], hp["bias"], np.zeros(M), np.ones(M), np.zeros(d), np.ones(d))
    assert h.lml == a[0]


def test_adam_trajectory_matches_torch(L):
    from dmosopt_b200.model_gpytorch import megp_fit, megp_initial_raw

    rng = np.random.default_rng(8)
    N, d, M = 200, 8, 3
    X, yn = _data(rng, N, d, M)
    raw0 = megp_initial_raw(d, M, seed=3)
    _, info = megp_fit(X, yn, n_iter=300, initial_raw=raw0)
    raw_ref, loss_ref, _ = megp_train.train_adam_torch(X, yn, raw0, n_iter=300)
    assert info["iterations"] == 300 and len(loss_ref) == 300
    assert np.all(np.abs(info["loss"] - loss_ref) <= 1e-9 * np.abs(loss_ref))
    for k in raw_ref:
        assert np.abs(info["raw"][k] - raw_ref[k]).max() <= 1e-7, k


def test_default_fit_stops_like_the_oracle_trainer(L):
    from dmosopt_b200.model_gpytorch import megp_fit, megp_initial_raw, megp_natural

    rng = np.random.default_rng(9)
    N, d, M = 200, 6, 2
    X = rng.random((N, d))
    yn, _, _ = megp.normalise_y(_zdt1(X))
    hp, info = megp_fit(X, yn, seed=0)
    _, loss_ref, reason_ref = megp_train.train_adam_torch(X, yn, megp_initial_raw(d, M, seed=0))

    def criteria(reason):  # the tests that held, without their formatted values
        return [r.split(" (")[0] for r in reason.split("; ")]

    assert info["iterations"] == len(loss_ref) and criteria(info["stop_reason"]) == criteria(reason_ref), (info["stop_reason"], reason_ref)
    assert info["iterations"] < 5000
    lml0, _ = L.mtgp_lml_grad(X, yn, *megp_natural(megp_initial_raw(d, M, seed=0)))
    B = megp.task_covariance(hp["covar_factor"], hp["var"])
    lml1, _ = L.mtgp_lml_grad(X, yn, hp["lengthscale"], B, hp["task_noises"] + hp["noise"], hp["weights"], hp["biases"])
    assert lml1 > lml0
    hpb, _ = megp_fit(X, yn, lengthscale_bounds=(0.3, 2.0), n_iter=1200)
    assert np.all(hpb["lengthscale"] >= 0.3) and np.all(hpb["lengthscale"] <= 2.0)


def test_fitted_surrogate_is_the_hyperparameter_path(L):
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    rng = np.random.default_rng(10)
    N, d, M = 180, 5, 3
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    X = xlb + rng.random((N, d)) * (xub - xlb)
    Y = np.column_stack([np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] for t in range(M)]) * (1.0 + np.arange(M))
    Xs = xlb + rng.random((250, d)) * (xub - xlb)
    sm = MEGP_Matern(X, Y, d, M, xlb, xub, fit="gpu", n_iter=300, seed=2)
    assert sm.fit_info["iterations"] == 300 and len(sm.fit_info["loss"]) == 300
    hp = sm.hyperparameters
    B = megp.task_covariance(hp["covar_factor"], hp["var"])
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], B, hp["task_noises"] + hp["noise"], hp["weights"], hp["biases"])
    assert abs(sm.log_marginal_likelihood_value - st.lml) <= 1e-9 * abs(st.lml)
    em, ev = megp.predict(st, Xs)
    prior = (np.diag(st.B) + st.D) * st.y_std**2
    for precision, tol in (("fp64", 2e-6), ("tensor", 1e-5)):
        a = MEGP_Matern(X, Y, d, M, xlb, xub, fit="gpu", n_iter=300, seed=2, precision=precision).predict(Xs)
        b = MEGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision).predict(Xs)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.all(np.abs(a[0] - em).max(axis=0) <= tol * np.abs(em).max(axis=0))
        assert np.all(np.abs(a[1] - ev).max(axis=0) <= tol * prior)


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("optimizer", ["dmosopt_b200.CMAES", "dmosopt_b200.AGEMOEA"])
def test_unmodified_moasmo_epoch_trains_megp_on_the_gpu(L, optimizer):
    """The reference examples' configuration (surrogate_method_name "megp" with CMAES / AGEMOEA) with no surrogate
    keywords: without gpytorch the plugin trains on the GPU."""
    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(12)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    Y = _zdt1(X)
    gen = MOASMO.epoch(
        4, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name=optimizer,
        optimizer_kwargs={}, surrogate_method_name="dmosopt_b200.model_gpytorch.MEGP_Matern", surrogate_method_kwargs={},
        local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    sm = MEGP_Matern(X, Y, d, M, xlb, xub)
    assert sm.fit_info is not None and sm.fit_info["iterations"] >= 51
    mean, _ = sm.predict(xr)
    assert np.allclose(yp, mean, rtol=1e-4, atol=1e-4 * np.abs(mean).max())
