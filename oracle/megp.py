"""Oracle: multitask exact-GP posterior (MEGP_Matern, row A19 of SURVEY.md section 8a).

Test infrastructure only (see oracle/__init__.py).

PARITY UNPINNED.  The reference path is ``MEGP_Matern.predict`` (``dmosopt/model_gpytorch.py:1872-1919``): one
``gpytorch.models.ExactGP`` (``GPyTorchMultitaskExactGPModelMatern``, ``:510-571``) with ``MultitaskMean(LinearMean)``,
``MultitaskKernel(MaternKernel(nu=2.5, ard_num_dims=d), rank=1)`` and ``MultitaskGaussianLikelihood``; ``predict``
evaluates ``likelihood(model(x))``.  The arithmetic lives in gpytorch 1.13 + linear-operator 0.5.3 (``uv.lock:520-522,
837-839``), which are neither installed in this image nor vendored in the reference, and the reference holds no test or
golden vector for this path.  What follows restates the textbook exact posterior of that model densely, in float64,
without the block decomposition the GPU path uses (csrc/gp_multitask.cu), so that it checks that decomposition:

  x_n  = (x - xlb) / xrng,  xrng = xub - xlb (1 where the range is ~0)          model_gpytorch.py:1662-1664, 1679-1682
  y_n  = (y - mean(y)) / (std(y) + 1e-12), mean / std float32 (std 0 -> 1)      model_gpytorch.py:1686-1703
  m_t(x) = w_t . x_n + b_t                                                       MultitaskMean(LinearMean)
  k(x, x') = (1 + sqrt5 r + 5 r^2 / 3) exp(-sqrt5 r),  r = ||(x - x') / l||      MaternKernel(nu=2.5, ARD), shared by the tasks
  B    = F F' + diag(v)                                                          IndexKernel(rank=1): covar_factor, var
  D_t  = task_noises[t] + noise                                                  MultitaskGaussianLikelihood (rank 0)
  C    = K (x) B + I_N (x) diag(D)   (rows ordered point-major, task-minor)       MultitaskKernel + likelihood
  mean_t(x_*) = m_t(x_*) + (k_* (x) B[t])' C^-1 (y_n - m(X))
  var_t(x_*)  = B_tt + D_t - (k_* (x) B[t])' C^-1 (k_* (x) B[t])               (exact: fast_pred_var=False)
  log p(y_n)  = -r' C^-1 r / 2 - log|C| / 2 - N M log(2 pi) / 2
  out  = std * mean + mean(y),  std^2 * var  (float32 arrays)                    model_gpytorch.py:1915-1916
"""

from dataclasses import dataclass

import numpy as np
from scipy.linalg import cho_solve, cholesky, solve_triangular

from .gp import MATERN52, kernel_matrix

LOG_2PI = np.log(2.0 * np.pi)


@dataclass
class MEGPState:
    X_train: np.ndarray  # (N,d) normalised inputs
    xlb: np.ndarray
    xrng: np.ndarray
    lengthscale: np.ndarray  # (d,)
    B: np.ndarray  # (M,M) task covariance
    D: np.ndarray  # (M,) noise per task
    weight: np.ndarray  # (M,d)
    bias: np.ndarray  # (M,)
    y_mean: np.ndarray  # (M,)
    y_std: np.ndarray  # (M,)
    L: np.ndarray  # (NM,NM) lower Cholesky factor of C
    alpha: np.ndarray  # (NM,) C^-1 (y_n - m(X)), point-major
    lml: float


def normalise_y(yin):
    """model_gpytorch.py:1686-1703."""
    yin = np.asarray(yin, dtype=np.float64)
    mean = np.asarray(yin.mean(axis=0), dtype=np.float32)
    std = np.asarray(yin.std(axis=0), dtype=np.float32)
    std = np.where(std == 0.0, np.float32(1.0), std)
    return (yin - mean.astype(np.float64)) / (std.astype(np.float64) + 1e-12), mean.astype(np.float64), std.astype(np.float64)


def task_covariance(covar_factor, var):
    """IndexKernel.covar_matrix: F F' + diag(v)."""
    v = np.ravel(np.asarray(var, dtype=np.float64))
    F = np.asarray(covar_factor, dtype=np.float64).reshape(len(v), -1)
    return F @ F.T + np.diag(v)


def dense_covariance(K, B, D):
    """C = K (x) B + I_N (x) diag(D), rows point-major (index n * M + t)."""
    N = K.shape[0]
    return np.kron(K, B) + np.kron(np.eye(N), np.diag(D))


def fit_fixed(xin, yin, xlb, xub, lengthscale, B, D, weight, bias):
    """Posterior state for given hyper-parameters (training itself is out of scope)."""
    xin = np.asarray(xin, dtype=np.float64)
    yin = np.asarray(yin, dtype=np.float64)
    if yin.ndim == 1:
        yin = yin.reshape(-1, 1)
    xlb = np.asarray(xlb, dtype=np.float64)
    xub = np.asarray(xub, dtype=np.float64)
    xrng = np.where(np.isclose(xub - xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - xlb)
    xn = (xin - xlb) / xrng
    yn, ymean, ystd = normalise_y(yin)
    N, d = xn.shape
    M = yn.shape[1]
    ls = np.broadcast_to(np.asarray(lengthscale, dtype=np.float64).reshape(-1), (d,)).copy()
    B = np.asarray(B, dtype=np.float64).reshape(M, M)
    D = np.asarray(D, dtype=np.float64).reshape(M)
    w = np.asarray(weight, dtype=np.float64).reshape(M, d)
    b = np.asarray(bias, dtype=np.float64).reshape(M)
    C = dense_covariance(kernel_matrix(xn, xn, ls, MATERN52), B, D)
    r = (yn - (xn @ w.T + b)).reshape(-1)
    L = cholesky(C, lower=True)
    alpha = cho_solve((L, True), r)
    lml = -0.5 * float(r @ alpha) - float(np.sum(np.log(np.diag(L)))) - 0.5 * N * M * LOG_2PI
    return MEGPState(xn, xlb, xrng, ls, B, D, w, b, ymean, ystd, L, alpha, lml)


def predict(st: MEGPState, xin):
    """(mean, variance), each (P, M) float32 as the reference returns them."""
    xin = np.asarray(xin, dtype=np.float64)
    if xin.ndim == 1:
        xin = xin.reshape(1, -1)
    xn = (xin - st.xlb) / st.xrng
    P, M = xn.shape[0], st.B.shape[0]
    Ks = kernel_matrix(xn, st.X_train, st.lengthscale, MATERN52)  # (P, N)
    mean = np.empty((P, M))
    var = np.empty((P, M))
    for t in range(M):
        Kt = np.kron(Ks, st.B[t][None, :])  # (P, N M): cross covariance of task t at x_* with every (point, task)
        mu = xn @ st.weight[t] + st.bias[t] + Kt @ st.alpha
        V = solve_triangular(st.L, Kt.T, lower=True)
        v = np.maximum(0.0, st.B[t, t] + st.D[t] - np.einsum("ij,ij->j", V, V))
        mean[:, t] = st.y_std[t] * mu + st.y_mean[t]
        var[:, t] = st.y_std[t] ** 2 * v
    return mean.astype(np.float32), var.astype(np.float32)
