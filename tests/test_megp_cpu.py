"""MEGP_Matern (row A19, multitask exact GP) without a GPU: the dense oracle against the single-task oracle and scipy, the
block decomposition the GPU path uses restated in NumPy against the dense oracle, and the read-out of a trained gpytorch
model on a stand-in built from torch tensors (gpytorch itself is not installed)."""

from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import egp, megp


def _problem(rng, N, d, M, noise=(2e-3, 5e-3, 1e-2, 3e-3, 8e-3)):
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    X = xlb + rng.random((N, d)) * (xub - xlb)
    cols = [np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] ** 2 for t in range(M)]
    Y = np.column_stack(cols) * np.arange(1, M + 1) + 3.0
    F = rng.standard_normal((M, 1))
    B = megp.task_covariance(F, 0.1 + rng.random(M))
    D = np.asarray(noise[:M], dtype=np.float64)
    hp = dict(lengthscale=0.5 + rng.random(d), B=B, D=D, weight=0.2 * rng.standard_normal((M, d)), bias=0.1 * rng.standard_normal(M))
    return X, Y, xlb, xub, hp


def test_dense_oracle_with_one_task_is_the_single_task_oracle():
    rng = np.random.default_rng(0)
    X, Y, xlb, xub, hp = _problem(rng, 80, 4, 1)
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["B"], hp["D"], hp["weight"], hp["bias"])
    e = egp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"][None, :], [hp["B"][0, 0]], hp["D"], hp["weight"], hp["bias"])
    Xs = xlb + rng.random((50, 4)) * (xub - xlb)
    m1, v1 = megp.predict(st, Xs)
    m2, v2 = egp.predict(e, Xs)
    assert m1.dtype == np.float32 and v1.dtype == np.float32
    # the multitask model normalises the targets with float32 statistics (and + 1e-12): float32-level differences only
    assert np.abs(m1 - m2).max() <= 1e-6 * np.abs(m2).max()
    assert np.abs(v1 - v2).max() <= 1e-6 * (hp["B"][0, 0] + hp["D"][0]) * e.objectives[0].y_std ** 2


@pytest.mark.parametrize("M", [2, 3])
def test_dense_oracle_log_marginal_likelihood_is_the_gaussian_logpdf(M):
    from scipy.stats import multivariate_normal

    rng = np.random.default_rng(1)
    X, Y, xlb, xub, hp = _problem(rng, 40, 3, M)
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["B"], hp["D"], hp["weight"], hp["bias"])
    C = megp.dense_covariance(megp.kernel_matrix(st.X_train, st.X_train, st.lengthscale, megp.MATERN52), st.B, st.D)
    yn, _, _ = megp.normalise_y(Y)
    r = (yn - (st.X_train @ st.weight.T + st.bias)).reshape(-1)
    ref = multivariate_normal.logpdf(r, mean=np.zeros(len(r)), cov=C)
    assert abs(st.lml - ref) <= 1e-10 * abs(ref)


@pytest.mark.parametrize("M", [1, 2, 3, 5])
def test_block_decomposition_matches_the_dense_posterior(M):
    """The algebra of csrc/gp_multitask.cu in float64 NumPy: D^-1/2 B D^-1/2 = Q diag(lam) Q', one GP per block with
    kernel lam_j K + I on the rotated residuals, mixed back with c_tj = lam_j Q_tj sqrt(D_t)."""
    from scipy.linalg import cho_solve, cholesky, solve_triangular

    rng = np.random.default_rng(2 + M)
    d = 3
    X, Y, xlb, xub, hp = _problem(rng, 60, d, M)
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["B"], hp["D"], hp["weight"], hp["bias"])
    Xs = xlb + rng.random((40, d)) * (xub - xlb)
    m_dense, v_dense = megp.predict(st, Xs)

    N = st.X_train.shape[0]
    sq = np.sqrt(st.D)
    lam, Q = np.linalg.eigh(st.B / np.outer(sq, sq))
    yn, _, _ = megp.normalise_y(Y)
    res = (yn - (st.X_train @ st.weight.T + st.bias)) / sq  # (N, M)
    rhat = res @ Q  # (N, M): column j is the rotated residual of block j
    K = megp.kernel_matrix(st.X_train, st.X_train, st.lengthscale, megp.MATERN52)
    xn = (Xs - st.xlb) / st.xrng
    Ks = megp.kernel_matrix(xn, st.X_train, st.lengthscale, megp.MATERN52)
    c = lam[None, :] * Q * sq[:, None]  # c[t, j]
    km, vn, lml = np.empty((len(Xs), M)), np.empty((len(Xs), M)), 0.0
    for j in range(M):
        Lj = cholesky(lam[j] * K + np.eye(N), lower=True)
        aj = cho_solve((Lj, True), rhat[:, j])
        km[:, j] = Ks @ aj
        V = solve_triangular(Lj, Ks.T, lower=True)
        vn[:, j] = np.einsum("ij,ij->j", V, V)
        lml += -0.5 * rhat[:, j] @ aj - np.sum(np.log(np.diag(Lj))) - 0.5 * N * np.log(2 * np.pi)
    lml -= 0.5 * N * np.sum(np.log(st.D))
    mean = xn @ st.weight.T + st.bias + km @ c.T
    var = np.maximum(0.0, np.diag(st.B) + st.D - vn @ (c * c).T)
    mean = (st.y_std * mean + st.y_mean).astype(np.float32)
    var = (st.y_std**2 * var).astype(np.float32)
    assert np.abs(mean - m_dense).max() <= 1e-6 * np.abs(m_dense).max()
    assert np.all(np.abs(var - v_dense).max(axis=0) <= 1e-6 * (np.diag(st.B) + st.D) * st.y_std**2)
    assert abs(lml - st.lml) <= 1e-9 * abs(st.lml)


def _stub_model(rng, N, d, M, wrapped):
    torch = pytest.importorskip("torch")
    covar = NS(data_covar_module=NS(lengthscale=torch.tensor(0.5 + rng.random((1, d)), dtype=torch.float32)),
               task_covar_module=NS(covar_factor=torch.tensor(rng.standard_normal((M, 1)), dtype=torch.float32),
                                    var=torch.tensor(0.1 + rng.random(M), dtype=torch.float32)))
    means = [NS(weights=torch.tensor(rng.standard_normal((d, 1)), dtype=torch.float32), bias=torch.tensor([0.1 * t], dtype=torch.float32))
             for t in range(M)]
    return NS(covar_module=NS(module=covar) if wrapped else covar,
              likelihood=NS(task_noises=torch.tensor(1e-3 * (1 + np.arange(M)), dtype=torch.float32), noise=torch.tensor([2e-4]),
                            has_task_noise=True, has_global_noise=True),
              mean_module=NS(base_means=means),
              train_inputs=(torch.tensor(rng.random((N, d)), dtype=torch.float32),),
              train_targets=torch.tensor(rng.standard_normal((N, M)), dtype=torch.float32))


@pytest.mark.parametrize("wrapped", [False, True])
def test_hyperparameter_readout_of_a_trained_model(wrapped):
    """megp_hyperparameters reads gpytorch's attribute names (MultitaskKernel.data_covar_module / task_covar_module,
    MultitaskGaussianLikelihood.task_noises / noise, MultitaskMean.base_means[t].weights / bias) through an optional
    MultiDeviceKernel wrapper, and takes the training tensors from the model."""
    from dmosopt_b200.model_gpytorch import megp_hyperparameters

    rng = np.random.default_rng(5)
    N, d, M = 30, 4, 3
    model = _stub_model(rng, N, d, M, wrapped)
    xn, yn, hp = megp_hyperparameters(model)
    cm = model.covar_module.module if wrapped else model.covar_module
    assert xn.shape == (N, d) and yn.shape == (N, M) and xn.dtype == np.float64
    assert np.array_equal(xn, model.train_inputs[0].numpy().astype(np.float64))
    assert np.array_equal(yn, model.train_targets.numpy().astype(np.float64))
    assert np.array_equal(hp["lengthscale"], cm.data_covar_module.lengthscale.numpy().reshape(-1).astype(np.float64))
    assert hp["covar_factor"].shape == (M, 1) and hp["var"].shape == (M,)
    assert np.array_equal(hp["task_noises"], model.likelihood.task_noises.numpy().astype(np.float64))
    assert hp["noise"] == pytest.approx(2e-4, rel=1e-6)
    assert hp["weights"].shape == (M, d) and np.array_equal(hp["weights"][1], model.mean_module.base_means[1].weights.numpy().reshape(-1).astype(np.float64))
    assert np.allclose(hp["biases"], [0.0, 0.1, 0.2])
    B = megp.task_covariance(hp["covar_factor"], hp["var"])
    assert np.allclose(B, B.T) and np.all(np.linalg.eigvalsh(B) > 0)


def test_precision_auto_is_refused():
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    with pytest.raises(ValueError):
        MEGP_Matern(np.zeros((4, 2)), np.zeros((4, 2)), 2, 2, np.zeros(2), np.ones(2), precision="auto", hyperparameters={})


def test_plugin_target_normalisation_matches_the_oracle():
    from dmosopt_b200.model_gpytorch import normalise_targets

    rng = np.random.default_rng(6)
    Y = rng.standard_normal((50, 3)) * [1.0, 10.0, 0.1] + [0.0, 5.0, -2.0]
    Y[:, 2] = 4.0  # a constant column: std 0 -> 1
    a, b = normalise_targets(Y), megp.normalise_y(Y)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
