"""Oracle: training of the multitask exact GP (MEGP_Matern, row A19 of SURVEY.md section 8a).

Test infrastructure only (see oracle/__init__.py).

PARITY UNPINNED (gpytorch is absent; see oracle/megp.py).  The exact log marginal likelihood and its gradient with torch
float64 autograd on the dense (N M) x (N M) covariance (no block decomposition, so it checks both the decomposition of
csrc/gp_multitask.cu and the hand-derived gradient of csrc/gp_multitask_fit.cu), and the Adam loop of MEGP_Matern's
training (dmosopt/model_gpytorch.py:1722-1829) with torch.optim.Adam on gpytorch 1.13's parameterisation (DESIGN.md
section 4.4; not checked against gpytorch).
"""

import numpy as np

from .megp import LOG_2PI


def _lml_torch(X, Y, ls, B, D, w, b):
    import torch

    N, M = Y.shape
    xs = X / ls
    diff = xs[:, None, :] - xs[None, :, :]
    r2 = (diff * diff).sum(-1)
    eye = torch.eye(N, dtype=torch.bool)
    r = torch.sqrt(torch.where(eye, torch.ones_like(r2), r2)) * np.sqrt(5.0)
    r = torch.where(eye, torch.zeros_like(r), r)  # no sqrt'(0) on the diagonal
    K = (1.0 + r + r * r / 3.0) * torch.exp(-r)
    C = torch.kron(K, B) + torch.kron(torch.eye(N, dtype=X.dtype), torch.diag(D))
    res = (Y - (X @ w.T + b)).reshape(-1, 1)
    L = torch.linalg.cholesky(C)
    alpha = torch.cholesky_solve(res, L)
    return -0.5 * (res * alpha).sum() - torch.log(torch.diagonal(L)).sum() - 0.5 * N * M * LOG_2PI


def lml_and_grad_torch(xn, yn, lengthscale, B, D, weight, bias):
    """(lml, grads) for normalised inputs xn (N,d) and targets yn (N,M): grads holds d lml / d length_scale (d,),
    B (M,M, entries independent), D (M,), weight (M,d), bias (M,) -- the keys of dmosopt_b200._lib.mtgp_lml_grad."""
    import torch

    X = torch.tensor(np.asarray(xn, dtype=np.float64))
    Y = torch.tensor(np.asarray(yn, dtype=np.float64).reshape(X.shape[0], -1))
    N, d = X.shape
    M = Y.shape[1]
    p = {k: torch.tensor(np.asarray(v, dtype=np.float64).reshape(s), requires_grad=True)
         for k, v, s in (("length_scale", np.broadcast_to(np.ravel(lengthscale), (d,)), (d,)), ("B", B, (M, M)), ("D", D, (M,)),
                         ("weight", weight, (M, d)), ("bias", bias, (M,)))}
    lml = _lml_torch(X, Y, p["length_scale"], p["B"], p["D"], p["weight"], p["bias"])
    lml.backward()
    return float(lml.detach()), {k: v.grad.numpy().copy() for k, v in p.items()}


def natural_torch(p, lengthscale_bounds=None):
    """gpytorch's transforms on torch raw parameters: (length_scale, B, D, weight, bias)."""
    import torch
    from torch.nn.functional import softplus

    if lengthscale_bounds is None:
        ls = softplus(p["raw_lengthscale"])
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        ls = lo + (hi - lo) * torch.sigmoid(p["raw_lengthscale"])
    F = p["covar_factor"]
    B = F @ F.T + torch.diag(softplus(p["raw_var"]))
    D = (1e-4 + softplus(p["raw_task_noises"])) + (1e-4 + softplus(p["raw_noise"]))[0]
    return ls, B, D, p["weights"], p["biases"]


def train_adam_torch(xn, yn, raw0, lengthscale_bounds=None, lr=0.01, n_iter=5000, min_loss_pct_change=0.1):
    """MEGP_Matern's training loop on the dense torch model from the raw parameters raw0 (dict of arrays, the keys of
    dmosopt_b200.model_gpytorch.megp_initial_raw): torch.optim.Adam on loss = -lml / (N M), the loss of iteration it
    recorded before its step, the exact-GP early-stopping rule asked from iteration 50 on.  Returns (raw, losses,
    stop_reason)."""
    import torch

    from dmosopt_b200.model_gpytorch import EarlyStopping

    X = torch.tensor(np.asarray(xn, dtype=np.float64))
    Y = torch.tensor(np.asarray(yn, dtype=np.float64).reshape(X.shape[0], -1))
    N, M = Y.shape
    p = {k: torch.tensor(np.array(v, dtype=np.float64), requires_grad=True) for k, v in raw0.items()}
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    stopper = EarlyStopping(threshold_pct=min_loss_pct_change)
    losses, reason = [], "n_iter"
    for it in range(n_iter):
        opt.zero_grad()
        loss = -_lml_torch(X, Y, *natural_torch(p, lengthscale_bounds)) / (N * M)
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if it >= stopper.warmup_iterations:
            stop, why = stopper.should_stop(it, np.array(losses))
            if stop:
                reason = why
                break
    return {k: v.detach().numpy().copy() for k, v in p.items()}, np.asarray(losses), reason
