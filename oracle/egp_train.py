"""Oracle: training of the independent exact GPs (EGP_Matern, row A19 of SURVEY.md section 8a).

Test infrastructure only (see oracle/__init__.py).

PARITY UNPINNED (gpytorch is absent; see oracle/egp.py).  Each objective's exact log marginal likelihood with torch
float64 autograd on the dense N x N covariance K = s Matern52(X / l) + noise I (so it checks the hand-derived gradient of
csrc/gp_multitask_fit.cu's dmo_gp_lml_grad), and the Adam loop of EGP_Matern's training for one objective
(dmosopt/model_gpytorch.py:2023-2126) with torch.optim.Adam on gpytorch 1.13's parameterisation (DESIGN.md section 4.4;
not checked against gpytorch).
"""

import numpy as np

from .megp import LOG_2PI


def _lml_torch(X, y, ls, s, noise, w, b):
    """log p(y) of one objective: X (N,d), y (N,), ls (d,), s and noise scalars, w (d,), b scalar (torch tensors)."""
    import torch

    N = X.shape[0]
    xs = X / ls
    diff = xs[:, None, :] - xs[None, :, :]
    r2 = (diff * diff).sum(-1)
    eye = torch.eye(N, dtype=torch.bool)
    r = torch.sqrt(torch.where(eye, torch.ones_like(r2), r2)) * np.sqrt(5.0)
    r = torch.where(eye, torch.zeros_like(r), r)  # no sqrt'(0) on the diagonal
    K = s * (1.0 + r + r * r / 3.0) * torch.exp(-r) + noise * torch.eye(N, dtype=X.dtype)
    res = (y - (X @ w + b)).reshape(-1, 1)
    L = torch.linalg.cholesky(K)
    alpha = torch.cholesky_solve(res, L)
    return -0.5 * (res * alpha).sum() - torch.log(torch.diagonal(L)).sum() - 0.5 * N * LOG_2PI


def lml_and_grad_torch(xn, yn, lengthscale, outputscale, noise, weight, bias):
    """(lml (M,), grads) for normalised inputs xn (N,d) and targets yn (N,M), one independent GP per column: grads holds
    d lml_m / d length_scale (M,d), outputscale (M,), noise (M,), weight (M,d), bias (M,) -- the keys of
    dmosopt_b200._lib.gp_lml_grad."""
    import torch

    X = torch.tensor(np.asarray(xn, dtype=np.float64))
    Y = np.asarray(yn, dtype=np.float64).reshape(X.shape[0], -1)
    N, d = X.shape
    M = Y.shape[1]
    shapes = {"length_scale": (M, d), "outputscale": (M,), "noise": (M,), "weight": (M, d), "bias": (M,)}
    vals = dict(zip(shapes, (lengthscale, outputscale, noise, weight, bias)))
    lml = np.empty(M)
    g = {k: np.empty(s) for k, s in shapes.items()}
    for m in range(M):
        p = {k: torch.tensor(np.asarray(v, dtype=np.float64).reshape(shapes[k])[m], requires_grad=True) for k, v in vals.items()}
        f = _lml_torch(X, torch.tensor(Y[:, m]), p["length_scale"], p["outputscale"], p["noise"], p["weight"], p["bias"])
        f.backward()
        lml[m] = float(f.detach())
        for k in shapes:
            g[k][m] = p[k].grad.numpy()
    return lml, g


def natural_torch(p, lengthscale_bounds=None):
    """gpytorch's transforms on one objective's torch raw parameters (rows of one, the layout of
    dmosopt_b200.model_gpytorch.egp_initial_raw(d, 1)): (length_scale (d,), outputscale, noise, weight (d,), bias)."""
    import torch
    from torch.nn.functional import softplus

    if lengthscale_bounds is None:
        ls = softplus(p["raw_lengthscale"][0])
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        ls = lo + (hi - lo) * torch.sigmoid(p["raw_lengthscale"][0])
    return ls, softplus(p["raw_outputscale"][0]), 1e-4 + softplus(p["raw_noise"][0]), p["weights"][0], p["bias"][0]


def train_adam_torch(xn, y, raw0, lengthscale_bounds=None, lr=0.01, n_iter=5000, min_loss_pct_change=0.1):
    """EGP_Matern's training loop for one objective on the dense torch model from the raw parameters raw0 (rows of one):
    torch.optim.Adam on loss = -lml / N, the loss of iteration it recorded before its step, the exact-GP early-stopping
    rule asked from iteration 50 on.  y (N,) normalised targets.  Returns (raw, losses, stop_reason)."""
    import torch

    from dmosopt_b200.model_gpytorch import EarlyStopping

    X = torch.tensor(np.asarray(xn, dtype=np.float64))
    yt = torch.tensor(np.asarray(y, dtype=np.float64).reshape(-1))
    N = X.shape[0]
    p = {k: torch.tensor(np.array(v, dtype=np.float64), requires_grad=True) for k, v in raw0.items()}
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    stopper = EarlyStopping(threshold_pct=min_loss_pct_change)
    losses, reason = [], "n_iter"
    for it in range(n_iter):
        opt.zero_grad()
        loss = -_lml_torch(X, yt, *natural_torch(p, lengthscale_bounds)) / N
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if it >= stopper.warmup_iterations:
            stop, why = stopper.should_stop(it, np.array(losses))
            if stop:
                reason = why
                break
    return {k: v.detach().numpy().copy() for k, v in p.items()}, np.asarray(losses), reason
