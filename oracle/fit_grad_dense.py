"""Oracle: the exact log marginal likelihood and its hyper-parameter gradient in closed form, densely in float64.

Test infrastructure only (see oracle/__init__.py).

The torch autograd oracles (oracle/egp_train.py, oracle/megp_train.py) build an N x N x d difference tensor and keep
the whole graph; that does not fit the training sizes the fits run at (N 2048 - 4096).  This module computes the same
quantities from the textbook identities, one input coordinate at a time, in O(N^2) memory:

  d lml / d theta = 1/2 sum_ij W_ij dK_ij / d theta,   W = alpha alpha' - K^-1,  alpha = K^-1 (y - m(X))
  Matern-5/2:  k(r) = (1 + r + r^2 / 3) e^-r,  r = sqrt5 ||(x - x') / l||
               dk / dl_k = 5/3 (1 + r) e^-r (x_k - x'_k)^2 / l_k^3      (finite, and 0, at r = 0)
  linear mean m(x) = w . x + b:  d lml / d w = X' alpha,  d lml / d b = sum alpha

EGP (dmo_gp_lml_grad): one GP per objective, K = s k + noise I.  MEGP (dmo_mtgp_lml_grad): C = K (x) B + I (x) diag(D)
(rows point-major, task-minor) with alpha (N, M) = C^-1 r reshaped, and W = alpha alpha' - C^-1 contracted with B over
the task indices for the length scales (A B A' - sum_st C^-1[(i s), (j t)] B_st), with K for B's entries and on the
diagonal for D.  B's entries are independent parameters, as in the autograd oracle.  tests/test_shape_limits_cpu.py
checks this module against the autograd oracles.
"""

import numpy as np
from scipy.linalg import cho_factor, cho_solve

from .megp import LOG_2PI


def _unit_matern(X, ls):
    """(k, g) with k = Matern52(X / ls) and g = 5/3 (1 + r) e^-r (dk / dl_k = g (x_k - x'_k)^2 / l_k^3); r^2 is summed one
    coordinate at a time (no Gram-form cancellation)."""
    N, d = X.shape
    r2 = np.zeros((N, N))
    for k in range(d):
        dk = (X[:, k, None] - X[None, :, k]) / ls[k]
        r2 += dk * dk
    r = np.sqrt(5.0 * r2)
    e = np.exp(-r)
    return (1.0 + r + r * r / 3.0) * e, (5.0 / 3.0) * (1.0 + r) * e


def _length_scale_grad(X, ls, WG):
    """1/2 sum_ij WG_ij (x_ik - x_jk)^2 / l_k^3 for every k: WG already holds W o g (and any scale factor)."""
    d = X.shape[1]
    out = np.empty(d)
    for k in range(d):
        dk = X[:, k, None] - X[None, :, k]
        out[k] = 0.5 * np.sum(WG * dk * dk) / ls[k] ** 3
    return out


def egp_lml_and_grad(xn, yn, lengthscale, outputscale, noise, weight, bias):
    """(lml (M,), grads) with the keys and shapes of dmosopt_b200._lib.gp_lml_grad (and of egp_train.lml_and_grad_torch)."""
    X = np.asarray(xn, dtype=np.float64)
    N, d = X.shape
    Y = np.asarray(yn, dtype=np.float64).reshape(N, -1)
    M = Y.shape[1]
    ls_all = np.asarray(lengthscale, dtype=np.float64).reshape(M, d)
    s_all, nz_all = np.asarray(outputscale, dtype=np.float64).reshape(M), np.asarray(noise, dtype=np.float64).reshape(M)
    w_all, b_all = np.asarray(weight, dtype=np.float64).reshape(M, d), np.asarray(bias, dtype=np.float64).reshape(M)
    lml = np.empty(M)
    g = {"length_scale": np.empty((M, d)), "outputscale": np.empty(M), "noise": np.empty(M), "weight": np.empty((M, d)),
         "bias": np.empty(M)}
    for m in range(M):
        k, gk = _unit_matern(X, ls_all[m])
        K = s_all[m] * k
        K[np.diag_indices(N)] += nz_all[m]
        cf = cho_factor(K, lower=True)
        res = Y[:, m] - (X @ w_all[m] + b_all[m])
        alpha = cho_solve(cf, res)
        W = np.outer(alpha, alpha) - cho_solve(cf, np.eye(N))
        lml[m] = -0.5 * res @ alpha - np.sum(np.log(np.diag(cf[0]))) - 0.5 * N * LOG_2PI
        g["outputscale"][m] = 0.5 * np.sum(W * k)
        g["noise"][m] = 0.5 * np.trace(W)
        g["length_scale"][m] = _length_scale_grad(X, ls_all[m], s_all[m] * W * gk)
        g["weight"][m] = X.T @ alpha
        g["bias"][m] = alpha.sum()
    return lml, g


def megp_lml_and_grad(xn, yn, lengthscale, B, D, weight, bias):
    """(lml, grads) with the keys and shapes of dmosopt_b200._lib.mtgp_lml_grad (and of megp_train.lml_and_grad_torch)."""
    X = np.asarray(xn, dtype=np.float64)
    N, d = X.shape
    Y = np.asarray(yn, dtype=np.float64).reshape(N, -1)
    M = Y.shape[1]
    ls = np.broadcast_to(np.asarray(lengthscale, dtype=np.float64).reshape(-1), (d,))
    Bm, Dv = np.asarray(B, dtype=np.float64).reshape(M, M), np.asarray(D, dtype=np.float64).reshape(M)
    w, b = np.asarray(weight, dtype=np.float64).reshape(M, d), np.asarray(bias, dtype=np.float64).reshape(M)
    k, gk = _unit_matern(X, ls)
    C = np.kron(k, Bm) + np.kron(np.eye(N), np.diag(Dv))
    cf = cho_factor(C, lower=True)
    res = (Y - (X @ w.T + b)).reshape(-1)
    alpha = cho_solve(cf, res)
    lml = -0.5 * res @ alpha - np.sum(np.log(np.diag(cf[0]))) - 0.5 * N * M * LOG_2PI
    C = None
    Ci = cho_solve(cf, np.eye(N * M)).reshape(N, M, N, M)  # C^-1[(i s), (j t)]
    cf = None
    A = alpha.reshape(N, M)
    # W4[i, s, j, t] = A_is A_jt - C^-1[(i s), (j t)], contracted without forming W4
    WB = A @ Bm @ A.T - np.einsum("isjt,st->ij", Ci, Bm, optimize=True)
    g = {"length_scale": _length_scale_grad(X, ls, WB * gk),
         "B": 0.5 * (np.einsum("is,ij,jt->st", A, k, A, optimize=True) - np.einsum("isjt,ij->st", Ci, k, optimize=True)),
         "D": 0.5 * (np.einsum("is,is->s", A, A) - np.einsum("isis->s", Ci)),
         "weight": A.T @ X, "bias": A.sum(0)}
    return float(lml), g
