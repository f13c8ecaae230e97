"""Oracle: training of the GPflow variational surrogates behind dmosopt's SVGP_Matern, VGP_Matern, SIV_Matern,
SPV_Matern and CRV_Matern (dmosopt/model.py:98-1179).

Test infrastructure only (see oracle/__init__.py).

Parity is UNPINNED: the reference pins gpflow 2.9.2 / tensorflow 2.14 (``uv.lock``), neither installed nor vendored here.
This module restates, densely in torch float64:

  * the minibatch ELBO of one GPflow model with L whitened latents (q_l = N(m_l, S_l)), outputs f = W g:
        ELBO = (N / B) sum_b sum_m E_q log N(y_bm | f_bm, sigma2_m) - sum_l KL(q_l || N(0, I))
    SVGP forms: A = Lz^-1 K(Z, X_b), mu = A' m, v = s - colsum(A o A) + colsum(A o S A);  VGP: A = Lz' over the batch
    columns, v = colsum(A o S A); Lz = chol(s k(Z, Z) + jitter I).  Hyper-parameter gradients come from autograd.
  * the natural-gradient step, derived by autograd alone: the loss -ELBO as a function of the expectation parameters
    eta1 = m, eta2 = S + m m' of each latent, and theta <- theta - gamma grad_eta(loss) on the natural parameters
    theta1 = S^-1 m, theta2 = -S^-1 / 2.  No closed form of the update is used.
  * the training loop on a given batch stream, with keras' Adam and the reference's transforms.
"""

import numpy as np
import torch

JITTER = 1e-2
LOG_2PI = float(np.log(2.0 * np.pi))


def _t(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float64))


def matern52(A, B, variance, lengthscales):
    """variance Matern52(A / l, B / l) with a gradient that stays finite at zero distance."""
    D = (A / lengthscales)[:, None, :] - (B / lengthscales)[None, :, :]
    r2 = (D * D).sum(-1)
    pos = r2 > 0
    r = torch.where(pos, torch.sqrt(torch.where(pos, r2, torch.ones_like(r2))), torch.zeros_like(r2)) * np.sqrt(5.0)
    return variance * (1.0 + r + r * r / 3.0) * torch.exp(-r)


def latent_moments(X, Z, batch, s, ls, m, S, vgp, jitter=JITTER):
    """mu (B,), v (B,) of one latent at the batch rows of X (VGP: Z is X)."""
    Kzz = matern52(Z, Z, s, ls) + jitter * torch.eye(Z.shape[0], dtype=torch.float64)
    Lz = torch.linalg.cholesky(Kzz)
    if vgp:
        A = Lz.T[:, batch]
        return A.T @ m, ((S @ A) * A).sum(0)
    A = torch.linalg.solve_triangular(Lz, matern52(Z, X[batch], s, ls), upper=False)
    return A.T @ m, s - (A * A).sum(0) + ((S @ A) * A).sum(0)


def kl_white(m, S):
    return 0.5 * (torch.trace(S) + m @ m - m.shape[0] - torch.logdet(S))


def elbo_parts(X, Y, Z, batch, s, ls, noise, W, ms, Ss, vgp, jitter=JITTER):
    """(ell (M,), kl (L,)) as torch tensors.  X (N,d), Y (N,M), Z (Z,d) (VGP: X), batch (B,) indices, s (L,), ls (L,d),
    noise (M,), W (M,L), ms / Ss lists of the latents' m (Z,) and S (Z,Z)."""
    N, B = X.shape[0], len(batch)
    L = len(ms)
    mom = [latent_moments(X, Z, batch, s[l], ls[l], ms[l], Ss[l], vgp, jitter) for l in range(L)]
    mu = torch.stack([a for a, _ in mom])  # (L,B)
    v = torch.stack([b for _, b in mom])
    mf, vf = W @ mu, (W * W) @ v  # (M,B)
    y = Y[batch].T
    ell = (-0.5 * (LOG_2PI + torch.log(noise))[:, None] - ((y - mf) ** 2 + vf) / (2.0 * noise[:, None])).sum(1) * (N / B)
    kl = torch.stack([kl_white(ms[l], Ss[l]) for l in range(L)])
    return ell, kl


def elbo_and_grad(X, Y, Z, batch, variance, lengthscales, noise, W, q_mu, q_sqrt, vgp, jitter=JITTER):
    """numpy (ell (M,), kl (L,), grads) with d ELBO / d variance (L,), length_scale (L,d), noise (M,), W (M,L) at the
    given q (q_mu (L,Z), q_sqrt (L,Z,Z))."""
    X, Y = _t(X), _t(Y).reshape(X.shape[0], -1)
    Zt = X if vgp else _t(Z)
    s = _t(variance).clone().requires_grad_(True)
    ls = _t(lengthscales).clone().requires_grad_(True)
    nz = _t(noise).clone().requires_grad_(True)
    L = s.shape[0]
    Wt = (torch.eye(L, dtype=torch.float64) if W is None else _t(W)).clone().requires_grad_(True)
    ms = [_t(q_mu[l]) for l in range(L)]
    Ss = [_t(q_sqrt[l]) @ _t(q_sqrt[l]).T for l in range(L)]
    ell, kl = elbo_parts(X, Y, Zt, torch.as_tensor(np.asarray(batch)), s, ls, nz, Wt, ms, Ss, vgp, jitter)
    (ell.sum() - kl.sum()).backward()
    g = {"variance": s.grad.numpy(), "length_scale": ls.grad.numpy(), "noise": nz.grad.numpy(), "W": Wt.grad.numpy()}
    return ell.detach().numpy(), kl.detach().numpy(), g


def natgrad_step(X, Y, Z, batch, variance, lengthscales, noise, W, q_mu, q_sqrt, gamma, vgp, jitter=JITTER):
    """One natural-gradient step: (q_mu (L,Z), q_sqrt (L,Z,Z) lower triangular) after it."""
    X, Y = _t(X), _t(Y).reshape(X.shape[0], -1)
    Zt = X if vgp else _t(Z)
    s, ls, nz = _t(variance), _t(lengthscales), _t(noise)
    L = s.shape[0]
    Wt = torch.eye(L, dtype=torch.float64) if W is None else _t(W)
    m0 = [_t(q_mu[l]) for l in range(L)]
    S0 = [_t(q_sqrt[l]) @ _t(q_sqrt[l]).T for l in range(L)]
    eta1 = [m.clone().requires_grad_(True) for m in m0]
    eta2 = [(S + torch.outer(m, m)).clone().requires_grad_(True) for m, S in zip(m0, S0)]
    ms = eta1
    Ss = [e2 - torch.outer(e1, e1) for e1, e2 in zip(eta1, eta2)]
    ell, kl = elbo_parts(X, Y, Zt, torch.as_tensor(np.asarray(batch)), s, ls, nz, Wt, ms, Ss, vgp, jitter)
    loss = -(ell.sum() - kl.sum())
    g = torch.autograd.grad(loss, eta1 + eta2)
    q_mu_new, q_sqrt_new = [], []
    for l in range(L):
        P = torch.linalg.inv(S0[l])
        th1 = P @ m0[l] - gamma * g[l]
        th2 = -0.5 * P - gamma * 0.5 * (g[L + l] + g[L + l].T)
        S = torch.linalg.inv(-2.0 * th2)
        S = 0.5 * (S + S.T)
        q_mu_new.append((S @ th1).numpy())
        q_sqrt_new.append(torch.linalg.cholesky(S).numpy())
    return np.stack(q_mu_new), np.stack(q_sqrt_new)


def _softplus(x):
    return np.logaddexp(0.0, x)


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def train(kind, X, Y, Z, batches, n_iter, *, gamma, adam_lr=0.01, lengthscale_bounds=(1e-6, 100.0), likelihood_sigma=1e-4, W0=None,
          jitter=JITTER):
    """The reference's loop for ONE GPflow model on a given batch stream ``batches`` (an iterator of index arrays, drawn
    in the order natural-gradient batch, Adam batch, then every 10th iteration the logging batch; VGP: full data and
    the ELBO logged every iteration).  kind "svgp" / "vgp" (one latent), "siv", "spv", "crv" (M latents).  Returns the
    ELBO log and the final (variance, lengthscales, noise, W, q_mu, q_sqrt).  Adam is restated from keras 2.14."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64).reshape(X.shape[0], -1)
    N, d = X.shape
    M = Y.shape[1]
    L = M
    vgp = kind == "vgp"
    Zn = X.shape[0] if vgp else np.asarray(Z).shape[0]
    K = 1 if kind == "siv" else L
    lo, hi = lengthscale_bounds
    raw = {"ls": np.full((K, d), np.log((1.0 - lo) / (hi - 1.0))), "s": np.full(K, np.log(np.expm1(1.0))),
           "nz": np.array([np.log(np.expm1(likelihood_sigma - 1e-6))])}
    if kind == "crv":
        raw["W"] = np.array(W0, dtype=np.float64)
    adam_m = {k: np.zeros_like(v) for k, v in raw.items()}
    adam_v = {k: np.zeros_like(v) for k, v in raw.items()}
    q_mu, q_sqrt = np.zeros((L, Zn)), np.stack([np.eye(Zn)] * L)

    def natural():
        ls = np.broadcast_to(lo + (hi - lo) * _sigmoid(raw["ls"]), (L, d)).copy()
        s = np.broadcast_to(_softplus(raw["s"]), (L,)).copy()
        return s, ls, np.full(M, 1e-6 + _softplus(raw["nz"][0])), raw.get("W")

    full = np.arange(N)
    log = []
    for it in range(n_iter):
        s, ls, nz, W = natural()
        q_mu, q_sqrt = natgrad_step(X, Y, Z, full if vgp else next(batches), s, ls, nz, W, q_mu, q_sqrt, gamma, vgp, jitter)
        _, _, g = elbo_and_grad(X, Y, Z, full if vgp else next(batches), s, ls, nz, W, q_mu, q_sqrt, vgp, jitter)
        gl = g["length_scale"] if K == L else g["length_scale"].sum(0, keepdims=True)
        gs = g["variance"] if K == L else g["variance"].sum(keepdims=True)
        sg = _sigmoid(raw["ls"])
        grads = {"ls": -gl * (hi - lo) * sg * (1.0 - sg), "s": -gs * _sigmoid(raw["s"]), "nz": -np.array([g["noise"].sum()]) * _sigmoid(raw["nz"])}
        if "W" in raw:
            grads["W"] = -g["W"]
        t = it + 1
        alpha = adam_lr * np.sqrt(1.0 - 0.999**t) / (1.0 - 0.9**t)
        for k, gk in grads.items():
            adam_m[k] = adam_m[k] + (gk - adam_m[k]) * 0.1
            adam_v[k] = adam_v[k] + (gk * gk - adam_v[k]) * 0.001
            raw[k] = raw[k] - alpha * adam_m[k] / (np.sqrt(adam_v[k]) + 1e-7)
        if vgp or it % 10 == 0:
            s, ls, nz, W = natural()
            ell, kl, _ = elbo_and_grad(X, Y, Z, full if vgp else next(batches), s, ls, nz, W, q_mu, q_sqrt, vgp, jitter)
            log.append(float(ell.sum() - kl.sum()))
    s, ls, nz, W = natural()
    return np.asarray(log), (s, ls, nz, W, q_mu, q_sqrt)
