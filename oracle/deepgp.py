"""Oracle: the two-layer deep GP predict behind dmosopt's MDSPP_Matern and MDGP_Matern (dmosopt/model_gpytorch.py
:991-1306, 1308-1620), gpytorch's DSPP and DeepGP with two whitened variational layers.

Test infrastructure only (see oracle/__init__.py).  gpytorch is not installed here, so each step below is restated from
its source as we know it, one comment per step, for a reviewer who has it to check.  Float64 throughout.

hp (the ``hyperparameters=`` dict of dmosopt_b200.model_gpytorch.MDSPP_Matern / MDGP_Matern):
  hidden_inducing_points (H,Z1,d), hidden_outputscale (H,), hidden_lengthscale (H,d), hidden_variational_mean (H,Z1),
  hidden_chol_variational_covar (H,Z1,Z1), mean_weights (d,), mean_bias; last_inducing_points (T,Z2,H), last_outputscale
  (T,), last_lengthscale (T,H), last_variational_mean (T,Z2), last_chol_variational_covar (T,Z2,Z2), mean_constant;
  task_noises (T,), noise; quad_sites (J,H) (MDSPP only).
"""

import numpy as np

from oracle.variational import latent_predict

JITTER = 1e-4  # settings.variational_cholesky_jitter for float32 models
MIN_VARIANCE = 1e-6  # settings.min_variance for float32


def layer(xn, Z, s, ls, q_mu, chol, prior_mean, jitter=JITTER):
    """One whitened VariationalStrategy unit at xn (P,d): (mean (P,), var (P,)).
    VariationalStrategy.forward (whitened): Lz = chol(K(Z,Z) + jitter I), mean = mu(x) + k(x,Z) Lz^-T q_mu,
    var = k(x,x) + jitter - ||Lz^-1 k||^2 + ||L_q' Lz^-1 k||^2 (the jitter is added to k(x,x) as well, the difference from
    gpflow's posterior); CholeskyVariationalDistribution masks chol_variational_covar to its lower triangle."""
    m, v = latent_predict(xn, Z, s, ls, q_mu, np.tril(chol), jitter)
    return m + prior_mean, v + jitter


def hidden(xn, hp, jitter=JITTER, min_variance=MIN_VARIANCE):
    """Hidden layer: (mean1 (P,H), sd1 (P,H)).
    LinearMean(input_dims): one w, b for every unit (not batched); ScaleKernel(MaternKernel(nu=2.5)) with batch shape H;
    MultivariateNormal.variance clamps at settings.min_variance before the square root."""
    pm = xn @ np.asarray(hp["mean_weights"], dtype=np.float64).reshape(-1) + float(hp["mean_bias"])
    H = len(hp["hidden_outputscale"])
    out = [layer(xn, hp["hidden_inducing_points"][h], hp["hidden_outputscale"][h], hp["hidden_lengthscale"][h],
                 hp["hidden_variational_mean"][h], hp["hidden_chol_variational_covar"][h], pm, jitter) for h in range(H)]
    m1 = np.stack([m for m, _ in out], axis=1)
    v1 = np.maximum(np.stack([v for _, v in out], axis=1), min_variance)
    return m1, np.sqrt(v1)


def predict(xin, xlb, xrng, hp, y_mean, y_std, eps=None, jitter=JITTER, min_variance=MIN_VARIANCE):
    """(mean (P,T), var (P,T)) of MDSPP (eps None: hp["quad_sites"]) or MDGP (eps (J,P,H): the draws).
    DSPPLayer: u_j = mu + xi_j o sigma with the layer's quad_sites (J,H), the same for every candidate; DeepGPLayer:
    Normal(mu, sigma).rsample() over num_likelihood_samples; either way u_j is formed once and expanded over the tasks.
    Last layer: ConstantMean (one c for every task), per-task inducing points and kernels.  MultitaskGaussianLikelihood
    adds task_noises[t] + noise; .variance clamps each site's variance at min_variance.  The model's predict returns
    batch_preds.mean.mean(0) and .variance.mean(0): an unweighted average over the sites (DSPP's quadrature weights are
    not used and there is no between-site spread term); dmosopt then un-normalises with y_std and y_mean."""
    xn = (np.asarray(xin, dtype=np.float64) - np.asarray(xlb, dtype=np.float64)) / np.asarray(xrng, dtype=np.float64)
    m1, sd1 = hidden(xn, hp, jitter, min_variance)
    if eps is None:
        sites = np.asarray(hp["quad_sites"], dtype=np.float64)
        eps = np.broadcast_to(sites[:, None, :], (sites.shape[0],) + m1.shape)
    J = eps.shape[0]
    T = len(hp["last_outputscale"])
    c = float(hp["mean_constant"])
    noise = np.asarray(hp["task_noises"], dtype=np.float64) + float(hp["noise"])
    ms, vs = np.zeros((xn.shape[0], T)), np.zeros((xn.shape[0], T))
    for j in range(J):
        u = m1 + eps[j] * sd1
        for t in range(T):
            m, v = layer(u, hp["last_inducing_points"][t], hp["last_outputscale"][t], hp["last_lengthscale"][t],
                         hp["last_variational_mean"][t], hp["last_chol_variational_covar"][t], c, jitter)
            ms[:, t] += m
            vs[:, t] += np.maximum(v + noise[t], min_variance)
    ys = np.asarray(y_std, dtype=np.float64)
    return ys * (ms / J) + np.asarray(y_mean, dtype=np.float64), ys * ys * (vs / J)
