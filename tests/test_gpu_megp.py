"""MEGP_Matern on the GPU (row A19, parity unpinned: gpytorch is absent, so the hyper-parameters are given, not trained).

The multitask posterior through dmo_mtgp_create / dmo_mtgp_predict against the dense float64 restatement in
oracle/megp.py, which builds the (N M) x (N M) covariance explicitly and does not use the block decomposition of the
GPU path; the one-task model against EGP_Matern; and the unmodified reference controller driving the plugin.
"""

import functools
import sys

import numpy as np
import pytest

from oracle import megp

pytestmark = pytest.mark.gpu

N_TRAIN, N_CAND = 520, 300  # neither a multiple of 256: padded training rows and candidate rows are exercised


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _hyperparameters(rng, d, M):
    return dict(lengthscale=0.6 + 0.8 * rng.random(d), covar_factor=rng.standard_normal((M, 1)), var=0.2 + 0.5 * rng.random(M),
                task_noises=np.geomspace(1e-3, 8e-3, M), noise=1e-3, weights=0.2 * rng.standard_normal((M, d)),
                biases=0.1 * rng.standard_normal(M))


@functools.lru_cache(maxsize=None)
def _case(M, d):
    """Training data, hyper-parameters, candidates and the dense oracle's answers for one shape (computed once)."""
    rng = np.random.default_rng(100 * M + d)
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    X = xlb + rng.random((N_TRAIN, d)) * (xub - xlb)
    Y = np.column_stack([np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] + 0.1 * t * X[:, -1] ** 2 for t in range(M)])
    Y = Y * (1.0 + np.arange(M)) + np.arange(M)
    hp = _hyperparameters(rng, d, M)
    B = megp.task_covariance(hp["covar_factor"], hp["var"])
    D = hp["task_noises"] + hp["noise"]
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], B, D, hp["weights"], hp["biases"])
    Xs = xlb + rng.random((N_CAND, d)) * (xub - xlb)
    Xs[:20] = X[:20] + 1e-3 * rng.standard_normal((20, d))  # next to training points: small posterior variance
    mean, var = megp.predict(st, Xs)
    return X, Y, xlb, xub, hp, st, Xs, mean, var


@pytest.mark.parametrize("d", [2, 12, 40])
@pytest.mark.parametrize("M", [1, 2, 3, 5])
def test_megp_vs_dense_oracle(L, M, d):
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    X, Y, xlb, xub, hp, st, Xs, em, ev = _case(M, d)
    prior = (np.diag(st.B) + st.D) * st.y_std**2
    scale = np.abs(em).max(axis=0)
    for precision, tol in (("fp64", 2e-6), ("tensor", 1e-5)):  # float32 outputs bound the fp64 path
        sm = MEGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision)
        mean, var = sm.predict(Xs)
        assert mean.dtype == np.float32 and var.dtype == np.float32
        assert mean.shape == (N_CAND, M) and var.shape == (N_CAND, M)
        assert np.all(np.abs(mean - em).max(axis=0) <= tol * scale), (precision, np.abs(mean - em).max(axis=0) / scale)
        assert np.all(np.abs(var - ev).max(axis=0) <= tol * prior), (precision, np.abs(var - ev).max(axis=0) / prior)
        assert np.array_equal(sm.evaluate(Xs), mean)


@pytest.mark.parametrize("M,d", [(1, 12), (3, 2), (5, 40)])
def test_megp_log_marginal_likelihood_vs_dense_oracle(L, M, d):
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    X, Y, xlb, xub, hp, st, *_ = _case(M, d)
    sm = MEGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp)
    assert abs(sm.log_marginal_likelihood_value - st.lml) <= 1e-9 * abs(st.lml)


def test_megp_with_one_task_is_egp(L):
    """M = 1: the multitask model is EGP with output scale B_11 and noise D_1.  The two normalise the targets with
    float32 resp. float64 statistics, so they agree to float32 rounding of those."""
    from dmosopt_b200.model_gpytorch import EGP_Matern, MEGP_Matern

    X, Y, xlb, xub, hp, st, Xs, *_ = _case(1, 12)
    m1, v1 = MEGP_Matern(X, Y, 12, 1, xlb, xub, hyperparameters=hp).predict(Xs)
    ehp = dict(lengthscale=hp["lengthscale"][None, :], outputscale=[st.B[0, 0]], noise=[st.D[0]], weight=hp["weights"], bias=hp["biases"])
    m2, v2 = EGP_Matern(X, Y, 12, 1, xlb, xub, hyperparameters=ehp).predict(Xs)
    prior = (st.B[0, 0] + st.D[0]) * st.y_std[0] ** 2
    assert np.abs(m1 - m2).max() <= 1e-6 * np.abs(m2).max()
    assert np.abs(v1 - v2).max() <= 1e-6 * prior


def test_megp_argument_checks(L):
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    X, Y, xlb, xub, hp, *_ = _case(2, 2)
    h = MEGP_Matern(X, Y, 2, 2, xlb, xub, hyperparameters=hp)._gp
    with pytest.raises(L.DmoError):  # no AUTO calibration for the multitask model
        h.predict(X[:4], precision=L.GP_AUTO)
    bad = dict(hp, task_noises=[-1.0, 1e-3], noise=0.0)
    with pytest.raises(L.DmoError):  # D must be positive
        MEGP_Matern(X, Y, 2, 2, xlb, xub, hyperparameters=bad)
    for precision in (L.GP_FP64, L.GP_TENSOR):  # mean-only predicts give the same mean
        mean, var = h.predict(X[:7], return_var=False, precision=precision)
        assert var is None and np.array_equal(mean, h.predict(X[:7], precision=precision)[0])


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


def _zdt1(x):
    d = x.shape[1]
    g = 1.0 + 9.0 / (d - 1) * x[:, 1:].sum(axis=1)
    return np.column_stack((x[:, 0], g * (1.0 - np.sqrt(x[:, 0] / g))))


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("optimizer", ["dmosopt_b200.CMAES", "dmosopt_b200.AGEMOEA"])
def test_unmodified_moasmo_epoch_drives_megp(L, optimizer):
    """The reference examples' pairings (examples/example_dmosopt_zdt1.py: cmaes + megp; zdt2 / zdt3: age + megp):
    MOASMO.epoch resolves the surrogate by import path, fits it (fixed hyper-parameters), runs the generations and the
    resample step."""
    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(11)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    Y = _zdt1(X)
    hp = dict(lengthscale=np.full(d, 0.7), covar_factor=[[0.8], [-0.3]], var=[0.4, 0.6], task_noises=[1e-3, 2e-3], noise=1e-4,
              weights=np.zeros((M, d)), biases=np.zeros(M))
    launches0 = L.launch_count()
    gen = MOASMO.epoch(
        6, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name=optimizer,
        optimizer_kwargs={}, surrogate_method_name="dmosopt_b200.model_gpytorch.MEGP_Matern",
        surrogate_method_kwargs={"hyperparameters": hp}, local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    assert L.launch_count() > launches0
    assert type(res["optimizer"]).__module__.startswith("dmosopt_b200")
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
    assert np.all(xr >= xlb) and np.all(xr <= xub)
    # the stored predictions are the plugin's posterior mean at the resampled points
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    mean, _ = MEGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp).predict(xr)
    assert np.allclose(yp, mean, rtol=1e-4, atol=1e-4 * np.abs(mean).max())
