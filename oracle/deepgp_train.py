"""Oracle: training of the two-layer deep GPs behind dmosopt's MDSPP_Matern and MDGP_Matern (dmosopt/model_gpytorch.py
:185-247, 359-416 the models, :991-1269 / :1308-1585 the loops), gpytorch's DSPP and DeepGP.

Test infrastructure only (see oracle/__init__.py).

Parity is UNPINNED: the reference pins gpytorch 1.13 (``uv.lock``), which is neither installed nor vendored here.  Each
step of its loss is restated below, one comment per step, densely in torch float64, with gradients by autograd.  The
loop uses torch.optim.Adam and torch.optim.lr_scheduler.ReduceLROnPlateau themselves.

raw: the raw parameters by name (dmosopt_b200.model_gpytorch.DEEPGP_RAW_KEYS): hidden_inducing_points (Z1,d),
hidden_raw_lengthscale (H,), hidden_raw_outputscale (H,), hidden_variational_mean (H,Z1), hidden_chol_variational_covar
(H,Z1,Z1), mean_weights (d,), mean_bias (1,), last_inducing_points (T,Z2,H), last_raw_lengthscale (T,),
last_raw_outputscale (T,), last_variational_mean (T,Z2), last_chol_variational_covar (T,Z2,Z2), mean_constant (1,),
raw_task_noises (T,), raw_noise (1,), quad_sites (J,H) (MDSPP).
"""

import math

import numpy as np
import torch

JITTER = 1e-4  # settings.variational_cholesky_jitter for float32 models
MIN_VARIANCE = 1e-6  # settings.min_variance for float32
NOISE_LOWER = 1e-4  # GreaterThan(1e-4) on the task noises and the global noise


def _t(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float64))


def _lengthscale(x, bounds):
    # Positive(): softplus; Interval(lo, hi): lo + (hi - lo) sigmoid
    if bounds is None:
        return torch.nn.functional.softplus(x)
    lo, hi = float(bounds[0]), float(bounds[1])
    return lo + (hi - lo) * torch.sigmoid(x)


def _matern(a, b, s, ls):
    # ScaleKernel(MaternKernel(nu=2.5)): s (1 + sqrt5 r + 5 r^2 / 3) exp(-sqrt5 r), r = ||a - b|| / ell; the distance is
    # clamped at 1e-30 before the square root, as gpytorch's covar_dist does
    d2 = (((a[:, None, :] - b[None, :, :]) / ls) ** 2).sum(-1)
    q = torch.sqrt(torch.clamp_min(5.0 * d2, 1e-30))
    return s * ((1.0 + q + q * q / 3.0) * torch.exp(-q))


def _unit(x, Z, s, ls, mu, chol, jitter):
    """One whitened VariationalStrategy unit at the rows x: (a' mu, diag variance, KL)."""
    # Kzz = s k(Z, Z) + jitter I = Lz Lz' (no psd_safe_cholesky retry)
    Lz = torch.linalg.cholesky(_matern(Z, Z, s, ls) + jitter * torch.eye(Z.shape[0], dtype=torch.float64))
    # a = Lz^-1 s k(Z, x)
    a = torch.linalg.solve_triangular(Lz, _matern(Z, x, s, ls), upper=False)
    # CholeskyVariationalDistribution: Lq = tril(chol_variational_covar)
    Lq = torch.tril(chol)
    # predictive variance diag: s + jitter - a'a + ||Lq' a||^2 (jitter added to k(x, x))
    v = (s + jitter) - (a * a).sum(0) + ((Lq.T @ a) ** 2).sum(0)
    # KL(N(mu, Lq Lq') || N(0, I)) = (||Lq||_F^2 + mu'mu - Z - sum log Lq_ii^2) / 2
    kl = 0.5 * ((Lq * Lq).sum() + mu @ mu - Z.shape[0] - torch.log(torch.diagonal(Lq) ** 2).sum())
    return a.T @ mu, v, kl


def loss(raw, xb, yb, N, eps=None, lengthscale_bounds=None, jitter=JITTER, min_variance=MIN_VARIANCE):
    """-DeepApproximateMLL(VariationalELBO(likelihood, model, num_data=N)) of one minibatch (xb (B,d), yb (B,T)) as a
    torch scalar; raw holds torch tensors (leaves for autograd).  eps (J,B,H): the MDGP draws; None: quad_sites."""
    xb, yb = _t(xb), _t(yb)
    B = xb.shape[0]
    H = raw["hidden_raw_outputscale"].shape[0]
    T = raw["last_raw_outputscale"].shape[0]
    kl = 0.0
    # hidden layer: H units over x, one inducing matrix shared by all, isotropic length scale per unit, one LinearMean
    pm = xb @ raw["mean_weights"] + raw["mean_bias"][0]
    m1, v1 = [], []
    for h in range(H):
        s = torch.nn.functional.softplus(raw["hidden_raw_outputscale"][h])
        ls = _lengthscale(raw["hidden_raw_lengthscale"][h], lengthscale_bounds)
        m, v, k = _unit(xb, raw["hidden_inducing_points"], s, ls, raw["hidden_variational_mean"][h],
                        raw["hidden_chol_variational_covar"][h], jitter)
        m1.append(pm + m)
        v1.append(v)
        kl = kl + k
    m1, v1 = torch.stack(m1, 1), torch.stack(v1, 1)
    # MultitaskMultivariateNormal.variance clamps at min_variance (the clamp blocks the gradient); sd1 = sqrt
    sd1 = torch.sqrt(torch.clamp_min(v1, min_variance))
    # layer-2 inputs u_j = m1 + e_j o sd1: DSPP's quad_sites (J,H) or DeepGP's rsample draws
    e = raw["quad_sites"][:, None, :].expand(-1, B, H) if eps is None else _t(eps)
    J = e.shape[0]
    u = (m1[None] + e * sd1[None]).reshape(J * B, H)
    # MultitaskGaussianLikelihood: sigma2_t = task_noise_t + noise, both 1e-4 + softplus
    s2 = (NOISE_LOWER + torch.nn.functional.softplus(raw["raw_task_noises"])) + (NOISE_LOWER + torch.nn.functional.softplus(raw["raw_noise"][0]))
    c = raw["mean_constant"][0]
    y = yb.repeat(J, 1)
    ell = 0.0
    for t in range(T):
        # last layer: per-task inducing points and isotropic length scale, ConstantMean c shared by the tasks
        s = torch.nn.functional.softplus(raw["last_raw_outputscale"][t])
        ls = _lengthscale(raw["last_raw_lengthscale"][t], lengthscale_bounds)
        m, v, k = _unit(u, raw["last_inducing_points"][t], s, ls, raw["last_variational_mean"][t], raw["last_chol_variational_covar"][t],
                        jitter)
        kl = kl + k
        # expected log likelihood with the latent variance clamped first: -1/2 [((y - m)^2 + v) / s2 + log s2 + log 2 pi]
        vc = torch.clamp_min(v, min_variance)
        ell = ell + (-0.5 * (((y[:, t] - (c + m)) ** 2 + vc) / s2[t] + torch.log(s2[t]) + math.log(2.0 * math.pi))).sum()
    # DeepApproximateMLL: the mean over the J sites of the ELL summed over tasks and divided by the batch size; the KL of
    # every unit over num_data
    return -(ell / (J * B)) + kl / N


def loss_grad(raw_np, xb, yb, N, eps=None, lengthscale_bounds=None, jitter=JITTER, min_variance=MIN_VARIANCE):
    """(loss float, {name: gradient array}) at the NumPy raw parameters."""
    raw = {k: _t(v).clone().requires_grad_(True) for k, v in raw_np.items()}
    L = loss(raw, xb, yb, N, eps, lengthscale_bounds, jitter, min_variance)
    L.backward()
    return float(L.detach()), {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(v.shape)) for k, v in raw.items()}


def fit_loop(raw_np, xn, yn, perms, batch_size, lr, eps_fn=None, lengthscale_bounds=None, jitter=JITTER, min_variance=MIN_VARIANCE):
    """The reference's loop over the given epoch permutations: a torch.optim.Adam step per batch, the epoch loss the
    unweighted mean of its batch losses, ReduceLROnPlateau(mode="min", patience=3, threshold=0.01) stepped on it.
    eps_fn(step, batch) -> (J,B,H) draws for MDGP (None: quadrature).  Returns (epoch losses, lr of each epoch, raw)."""
    raw = {k: _t(v).clone().requires_grad_(True) for k, v in raw_np.items()}
    # parameters that get no gradient (DSPP's hidden quad_sites, raw_quad_weights) never move: not listed
    opt = torch.optim.Adam(list(raw.values()), lr=lr)
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, mode="min", patience=3, threshold=0.01)
    xn, yn = np.asarray(xn, dtype=np.float64), np.asarray(yn, dtype=np.float64)
    N = xn.shape[0]
    losses, lrs, step = [], [], 0
    for perm in perms:
        lrs.append(opt.param_groups[0]["lr"])
        batch_losses = []
        for b0 in range(0, N, batch_size):
            idx = np.asarray(perm[b0 : b0 + batch_size])
            opt.zero_grad()
            L = loss(raw, xn[idx], yn[idx], N, None if eps_fn is None else eps_fn(step, idx), lengthscale_bounds, jitter, min_variance)
            L.backward()
            batch_losses.append(float(L.detach()))
            opt.step()
            step += 1
        losses.append(float(np.mean(batch_losses)))
        sched.step(losses[-1])
    return np.asarray(losses), lrs, {k: v.detach().numpy().copy() for k, v in raw.items()}
