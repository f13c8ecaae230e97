"""Oracle: the GPflow variational posteriors behind dmosopt's SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern and
CRV_Matern predict (dmosopt/model.py:290-318, 509-537, 730-757, 953-981, 1143-1172).

Test infrastructure only (see oracle/__init__.py).

Parity is UNPINNED: the reference pins GPflow 2.9.2 (``uv.lock:497-498``), which is neither installed nor vendored here.
This module restates the whitened posterior predict_f (latent f, no likelihood noise) densely in float64:

  per latent l:  Kzz = s k(Z, Z) + jitter I (jitter 1e-2, model.py:17),  Lz = chol(Kzz),  A = Lz^-1 s k(Z, x*)
                 mean_l = A' q_mu_l,   var_l = s - colsum(A o A) + colsum((q_sqrt_l' A) o (q_sqrt_l' A))
  outputs:       mean = g_mean W',  var = g_var (W o W)'   (W = I except LinearCoregionalization)
  dmosopt:       mean * y_std + y_mean cast to float32;  var * y_std**2, float32 for SVGP / VGP (y_std float64), float64
                 for CRV / SIV / SPV (y_std float32, squared in float32)

and the optimal whitened q for a Gaussian likelihood (Titsias 2009): B = I + A A' / sigma^2 with A = Lz^-1 K(Z, X)
(SVGP) or A = Lz' (VGP, whose f(X) = Lz v sees the jitter), q_mu = B^-1 A y / sigma^2, S = B^-1.  No QR, no operator planes: the q_sqrt term is the dense product above.
"""

import numpy as np
from scipy.linalg import cholesky, solve_triangular
from scipy.spatial.distance import cdist

JITTER = 1e-2


def matern52(A, B, variance, lengthscales):
    r = cdist(A / lengthscales, B / lengthscales)
    K = np.sqrt(5.0) * r
    return variance * (1.0 + K + K * K / 3.0) * np.exp(-K)


def latent_predict(xn, Z, variance, lengthscales, q_mu, q_sqrt, jitter=JITTER):
    """One latent GP: mean (P,), var (P,) of f at normalised inputs xn (P,d)."""
    Lz = cholesky(matern52(Z, Z, variance, lengthscales) + jitter * np.eye(Z.shape[0]), lower=True)
    A = solve_triangular(Lz, matern52(Z, xn, variance, lengthscales), lower=True)
    LTA = q_sqrt.T @ A
    return A.T @ q_mu, (variance - np.sum(A * A, axis=0)) + np.sum(LTA * LTA, axis=0)


def predict(kind, xin, xlb, xrng, Z, variance, lengthscales, q_mu, q_sqrt, y_mean, y_std, W=None, jitter=JITTER):
    """dmosopt's predict of class ``kind`` ("svgp", "vgp", "siv", "spv", "crv"): (mean, var) with the reference's dtypes.
    Z (L,Z,d), variance (L,), lengthscales (L,d), q_mu (L,Z), q_sqrt (L,Z,Z); y_mean float32, y_std float64 for svgp / vgp
    and float32 otherwise."""
    xn = (np.asarray(xin, dtype=np.float64) - xlb) / xrng
    L = len(variance)
    g = [latent_predict(xn, Z[l], variance[l], lengthscales[l], q_mu[l], q_sqrt[l], jitter) for l in range(L)]
    gm = np.stack([m for m, _ in g], axis=1)
    gv = np.stack([v for _, v in g], axis=1)
    W = np.eye(L) if W is None else np.asarray(W, dtype=np.float64)
    mean, var = gm @ W.T, gv @ (W * W).T
    y_mean = np.asarray(y_mean, dtype=np.float32)
    if kind in ("svgp", "vgp"):
        ys = np.asarray(y_std, dtype=np.float64)
        return (ys * mean + y_mean.astype(np.float64)).astype(np.float32), (var * ys ** 2).astype(np.float32)
    ys = np.asarray(y_std, dtype=np.float32)
    return (ys.astype(np.float64) * mean + y_mean.astype(np.float64)).astype(np.float32), var * (ys ** 2).astype(np.float64)


def optimal_q(xn, y, Z, variance, lengthscales, noise, jitter=JITTER, inducing_is_data=False):
    """Titsias optimum in whitened coordinates for one latent: q_mu (Z,), S = q_sqrt q_sqrt' (Z,Z).  SVGP: the data term
    is f(X) = K(X, Z) Lz^-T v, A = Lz^-1 K(Z, X).  inducing_is_data (GPflow's VGP, Z = X): f(X) = Lz v, A = Lz'."""
    Lz = cholesky(matern52(Z, Z, variance, lengthscales) + jitter * np.eye(Z.shape[0]), lower=True)
    A = Lz.T if inducing_is_data else solve_triangular(Lz, matern52(Z, xn, variance, lengthscales), lower=True)
    B = np.eye(Z.shape[0]) + A @ A.T / noise
    return np.linalg.solve(B, A @ y / noise), np.linalg.inv(B)
