"""gpytorch surrogates on the GPU path: the exact GPs ``EGP_Matern`` and ``MEGP_Matern`` (row A19), and the deep GPs
``MDSPP_Matern`` and ``MDGP_Matern`` (their posterior and training; see the end of this module).

Drop-ins for ``dmosopt.model_gpytorch.EGP_Matern`` (dmosopt/model_gpytorch.py:1927-2235) and
``dmosopt.model_gpytorch.MEGP_Matern`` (:1623-1926), selected in dmosopt by
``surrogate_method_name="dmosopt_b200.model_gpytorch.EGP_Matern"`` (or ``.MEGP_Matern``).  Both train either through
the reference class itself, which needs gpytorch (``fit="reference"``: after training, the hyper-parameters and the
model's own normalised training tensors are read out), or on the GPU without gpytorch (``fit="gpu"``: the reference's
Adam loop and early stopping around the exact log marginal likelihood and its gradient, ``egp_fit`` with
``dmo_gp_lml_grad`` and ``megp_fit`` with ``dmo_mtgp_lml_grad``).  The posterior is then factorised once in float64,
and every ``predict`` / ``evaluate`` runs on the GPU.

* ``EGP_Matern``: M independent GPs (ARD length scales, output scale, noise, linear-mean weights / bias per objective);
  ``dmo_gp_create`` / ``dmo_gp_set_linear_mean`` / ``dmo_gp_predict``.
* ``MEGP_Matern``: one multitask GP over all objectives, covariance K_x (x) B + I (x) D (shared ARD Matern-5/2 K_x,
  rank-1 IndexKernel B, task + global noise D, linear mean per task); ``dmo_mtgp_create`` / ``dmo_mtgp_predict``.  The
  (N*M) x (N*M) system splits exactly into M single-output blocks that share one K_* (csrc/gp_multitask.cu).

The predictive variance is the exact one (gpytorch's ``fast_pred_var=False``); ``fast_pred_var=True`` (LOVE) is a
low-rank approximation of it.  gpytorch is not available here, so training through the reference classes is
untested; the read-out of a trained model is tested on a stand-in with gpytorch's attribute names, and the
posterior arithmetic against oracle/egp.py and oracle/megp.py through the ``hyperparameters=`` constructor path
(tests/test_gpu_parity.py::test_egp_linear_mean_*, tests/test_gpu_megp.py).
"""

import numpy as np

from . import _lib


def _matern52_ard(xn, ls):
    """s-free Matern-5/2 Gram matrix of the normalised training inputs (float64, host, once per epoch)."""
    xs = xn / ls
    sq = np.sum(xs * xs, axis=1)
    d2 = np.maximum(sq[:, None] + sq[None, :] - 2.0 * (xs @ xs.T), 0.0)
    r = np.sqrt(d2) * np.sqrt(5.0)
    return (1.0 + r + r * r / 3.0) * np.exp(-r)


class EGP_Matern:
    """M independent exact GPs; the reference constructor signature (model_gpytorch.py:1928-1950) plus ``precision``
    ("fp64", the default, or "tensor"), ``hyperparameters`` (dict with lengthscale (M,d), outputscale (M,), noise
    (M,), weight (M,d), bias (M,)): when given, training is skipped, and ``fit``: "gpu" trains with egp_fit (Adam on the
    exact log marginal likelihood of every objective, on the GPU), "reference" through the reference class (needs
    gpytorch; every keyword is forwarded); None uses the reference class where it can train and "gpu" otherwise.  The
    GPU fit has no noise prior (``gp_likelihood_sigma``) and no batched-model mode (``batch_size``); it ignores
    ``preconditioner_size``, ``fast_pred_var`` and ``use_cuda`` (the likelihood is exact, the variance always the exact
    one).  After a fit ``hyperparameters`` and ``fit_info`` (one dict per objective) hold the result."""

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, seed=None, gp_lengthscale_bounds=None, gp_likelihood_sigma=None,
                 preconditioner_size=100, adam_lr=0.01, fast_pred_var=True, n_iter=5000, min_loss_pct_change=0.1,
                 return_mean_variance=False, batch_size=None, use_cuda=False, nan="remove", top_k=None, logger=None,
                 precision="fp64", hyperparameters=None, fit=None, **kwargs):
        if fit not in (None, "gpu", "reference"):
            raise ValueError(f"EGP_Matern: fit must be 'gpu', 'reference' or None (got {fit!r})")
        # the exact-GP predict (dmo_gp_create) is narrower than the training: refuse before any training starts
        if nInput > _lib.GP_PREDICT_MAX_D:
            raise ValueError(f"EGP_Matern: the GPU predict takes at most {_lib.GP_PREDICT_MAX_D} input dimensions (got nInput={nInput})")
        if nOutput > _lib.GP_PREDICT_MAX_M:
            raise ValueError(f"EGP_Matern: the GPU predict takes at most {_lib.GP_PREDICT_MAX_M} objectives (got nOutput={nOutput})")
        self.nInput, self.nOutput = nInput, nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        xub = np.asarray(xub, dtype=np.float64)
        self.xrng = np.where(np.isclose(xub - self.xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - self.xlb)  # model_gpytorch.py:1965-1967
        self.return_mean_variance = return_mean_variance
        self.logger = logger
        self.precision = _lib.GP_TENSOR if precision in ("tensor", _lib.GP_TENSOR) else _lib.GP_FP64
        self.stats = {}
        self.fit_info = None
        if hyperparameters is None and fit is None:
            fit = "reference" if _reference_can_train() else "gpu"
        if hyperparameters is None and fit == "gpu":
            if gp_likelihood_sigma is not None:
                raise ValueError("EGP_Matern: the GPU fit has no noise prior (gp_likelihood_sigma); use fit='reference'")
            if batch_size is not None:
                raise ValueError("EGP_Matern: the GPU fit trains one exact GP per objective (batch_size=None); use fit='reference'")
        if hyperparameters is None and fit == "reference":
            ref_kwargs = dict(seed=seed, gp_lengthscale_bounds=gp_lengthscale_bounds, gp_likelihood_sigma=gp_likelihood_sigma,
                              preconditioner_size=preconditioner_size, adam_lr=adam_lr, fast_pred_var=fast_pred_var, n_iter=n_iter,
                              min_loss_pct_change=min_loss_pct_change, batch_size=batch_size, use_cuda=use_cuda, nan=nan,
                              top_k=top_k, **kwargs)
            xn, yn, ymean, ystd, hyperparameters = self._fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, logger, ref_kwargs)
        else:
            xin = np.asarray(xin, dtype=np.float64)
            yin = np.asarray(yin, dtype=np.float64)
            if yin.ndim == 1:
                yin = yin.reshape(-1, 1)
            if hyperparameters is None:
                xin, yin = filter_and_top_k(xin, yin, nan, top_k)  # model_gpytorch.py:1974-1977
            xn = (xin - self.xlb) / self.xrng
            ymean = yin.mean(axis=0)
            ystd = yin.std(axis=0)
            ystd = np.where(ystd == 0.0, 1.0, ystd)  # handle_zeros_in_scale, model_gpytorch.py:1995-2001
            yn = (yin - ymean) / ystd
            if hyperparameters is None:
                hyperparameters, self.fit_info = egp_fit(xn, yn, lengthscale_bounds=gp_lengthscale_bounds, adam_lr=adam_lr, n_iter=n_iter,
                                                         min_loss_pct_change=min_loss_pct_change, seed=seed, logger=logger)
        self.hyperparameters = hyperparameters
        self._upload(xn, yn, ymean, ystd, hyperparameters)

    @staticmethod
    def _fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, logger, kwargs):
        """Train with the reference class (unchanged) and read the fitted state out of its gpytorch models."""
        try:
            from dmosopt.model_gpytorch import EGP_Matern as RefEGP
        except Exception as e:  # dmosopt or gpytorch missing
            raise RuntimeError("dmosopt_b200.model_gpytorch.EGP_Matern trains through dmosopt.model_gpytorch.EGP_Matern, "
                               "which requires dmosopt and the GPyTorch library; pass hyperparameters= to skip training") from e
        ref = RefEGP(xin, yin, nInput, nOutput, xlb, xub, logger=logger, **kwargs)
        hp = {"lengthscale": [], "outputscale": [], "noise": [], "weight": [], "bias": []}
        yn_cols = []
        for m in ref.smlist:
            cm = getattr(m.covar_module, "module", m.covar_module)  # MultiDeviceKernel wraps the ScaleKernel
            hp["lengthscale"].append(cm.base_kernel.lengthscale.detach().cpu().numpy().reshape(-1))
            hp["outputscale"].append(float(cm.outputscale.detach().cpu()))
            hp["noise"].append(float(m.likelihood.noise.detach().cpu().reshape(-1)[0]))
            hp["weight"].append(m.mean_module.weights.detach().cpu().numpy().reshape(-1))
            hp["bias"].append(float(m.mean_module.bias.detach().cpu().reshape(-1)[0]))
            yn_cols.append(m.train_targets.detach().cpu().numpy().reshape(-1).astype(np.float64))
        xn = ref.smlist[0].train_inputs[0].detach().cpu().numpy().astype(np.float64)
        return xn, np.column_stack(yn_cols), np.asarray(ref.y_train_mean, dtype=np.float64), np.asarray(ref.y_train_std, dtype=np.float64), hp

    def _upload(self, xn, yn, ymean, ystd, hp):
        """Posterior state of every objective -> HBM, once per epoch."""
        from scipy.linalg import cho_solve, cholesky

        M, d = self.nOutput, self.nInput
        ls = np.asarray(hp["lengthscale"], dtype=np.float64).reshape(M, d)
        s = np.asarray(hp["outputscale"], dtype=np.float64).reshape(M)
        nz = np.asarray(hp["noise"], dtype=np.float64).reshape(M)
        w = np.asarray(hp["weight"], dtype=np.float64).reshape(M, d)
        b = np.asarray(hp["bias"], dtype=np.float64).reshape(M)
        alphas, factors = [], []
        for m in range(M):
            K = s[m] * _matern52_ard(xn, ls[m])
            K[np.diag_indices_from(K)] += nz[m]
            Lm = cholesky(K, lower=True)
            alphas.append(cho_solve((Lm, True), yn[:, m] - (xn @ w[m] + b[m])))
            factors.append(Lm)
        self._gp = _lib.GPHandle(
            X_train=xn, alpha=np.stack(alphas), factor=np.stack(factors), constant=s, length_scale=list(ls), noise=nz,
            y_mean=np.asarray(ymean, dtype=np.float64).reshape(M), y_std=np.asarray(ystd, dtype=np.float64).reshape(M),
            xlb=self.xlb, xub=self.xlb + self.xrng, kernel=_lib.KERNEL_MATERN52, factor_is_inverse=False,
        )
        self._gp.set_linear_mean(w, b)

    def predict(self, xin):
        """model_gpytorch.py:2188-2228: (mean (P, M), variance (P, M)) as float32 arrays."""
        xin = np.asarray(xin, dtype=np.float64)
        if xin.ndim == 1:
            xin = xin.reshape((1, self.nInput))
        mean, var = self._gp.predict(xin, return_var=True, precision=self.precision)
        return mean.astype(np.float32), var.astype(np.float32)

    def evaluate(self, x):
        """model_gpytorch.py:2230-2235."""
        mean, var = self.predict(x)
        return (mean, var) if self.return_mean_variance else mean

    def resident_posterior(self):
        """(kind, handle, precision, mean dtype) of the posterior MOASMO's resident epoch steps on: ``evaluate`` returns
        this handle's mean with the variance requested, as float32."""
        return _lib.POSTERIOR_GP, getattr(self, "_gp", None), self.precision, np.float32


# ----------------------------------------------------------------------------------------------------------- MEGP
def filter_samples(y, x, nan="remove"):
    """MOEA.filter_samples (dmosopt/MOEA.py:445-467) for the ``nan=`` modes: "remove" drops rows with a NaN objective,
    "max" replaces NaNs by max(1e3 * column max, 1e5), a number replaces them by that number."""
    y = np.array(y, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    if nan == "max":
        m = np.max(np.nan_to_num(y), axis=0)
        for c in range(y.shape[1]):
            y[:, c] = np.nan_to_num(y[:, c], nan=max(1e3 * m[c], 1e5))
        return y, x
    if nan == "remove":
        keep = ~np.any(np.isnan(y), axis=1)
        return y[keep], x[keep]
    return np.nan_to_num(y, nan=nan), x


def filter_and_top_k(xin, yin, nan, top_k):
    """The reference surrogates' sample selection before normalisation: filter_samples for a non-None ``nan``, then for
    an integer ``top_k`` below the sample count the first ``top_k`` samples of a non-dominated sort (MOEA.top_k_MO)."""
    if nan is not None:
        yin, xin = filter_samples(yin, xin, nan=nan)
    if isinstance(top_k, int) and xin.shape[0] > top_k:
        from .MOEA import sortMO

        xs, ys, *_ = sortMO(xin, yin)
        xin, yin = xs[:top_k], ys[:top_k]
    return xin, yin


def normalise_targets(yin):
    """model_gpytorch.py:1686-1703: float32 per-task mean and standard deviation (a zero deviation becomes 1), then
    (y - mean) / (std + 1e-12)."""
    yin = np.asarray(yin, dtype=np.float64)
    ymean = np.asarray([np.mean(yin[:, i]) for i in range(yin.shape[1])], dtype=np.float32)
    ystd = np.asarray([np.std(yin[:, i]) for i in range(yin.shape[1])], dtype=np.float32)
    ystd[ystd == 0.0] = 1.0
    yn = (yin - ymean.astype(np.float64)) / (ystd.astype(np.float64) + 1e-12)
    return yn, ymean.astype(np.float64), ystd.astype(np.float64)


def megp_hyperparameters(gp_model):
    """Read a trained ``GPyTorchMultitaskExactGPModelMatern`` (dmosopt/model_gpytorch.py:510-571) out into
    (xn (N,d), yn (N,M), hyperparameters): its own normalised training tensors and the ``hyperparameters=`` dict of
    ``MEGP_Matern`` -- ARD length scales of the shared Matern kernel, the IndexKernel's covar_factor (M, rank) and var (M,),
    the likelihood's task_noises (M,) and global noise, and the LinearMean weights (M,d) / biases (M,) of every task."""

    def arr(t):
        return t.detach().cpu().numpy().astype(np.float64)

    cm = getattr(gp_model.covar_module, "module", gp_model.covar_module)  # MultiDeviceKernel wraps the MultitaskKernel
    task = cm.task_covar_module
    lik = gp_model.likelihood
    M = int(task.covar_factor.shape[-2])
    weights, biases = [], []
    for m in gp_model.mean_module.base_means:
        if hasattr(m, "weights"):
            weights.append(arr(m.weights).reshape(-1))
            biases.append(float(arr(m.bias).reshape(-1)[0]))
        else:  # ConstantMean (linear_mean=False)
            weights.append(None)
            biases.append(float(arr(m.constant).reshape(-1)[0]))
    xn = arr(gp_model.train_inputs[0])
    N, d = xn.shape
    hp = {
        "lengthscale": arr(cm.data_covar_module.lengthscale).reshape(-1),
        "covar_factor": arr(task.covar_factor).reshape(M, -1),
        "var": arr(task.var).reshape(M),
        "task_noises": arr(lik.task_noises).reshape(M) if getattr(lik, "has_task_noise", True) else np.zeros(M),
        "noise": float(arr(lik.noise).reshape(-1)[0]) if getattr(lik, "has_global_noise", True) else 0.0,
        "weights": np.stack([np.zeros(d) if w is None else w for w in weights]),
        "biases": np.asarray(biases, dtype=np.float64),
    }
    return xn, arr(gp_model.train_targets).reshape(N, M), hp


class EarlyStopping:
    """The early-stopping rule of the reference's exact-GP training: ``AdaptiveEarlyStopping`` with
    ``EarlyStoppingConfig.for_model_type(EXACT_GP)`` (dmosopt/model_gpytorch.py:588-812), restated.

    Four tests on the loss history, over a window of the last 200 losses: the mean percentage change between successive
    losses is below ``threshold_pct`` (needs 201 losses); the largest absolute change is below 1e-3; the change from the
    window's first to its last loss is below 1e-2 relative (not tested when the first is below 1e-3 in magnitude); the
    means of the first and second half of the window differ by less than 2e-2 relative to the window mean (+ 1e-3)
    (needs 400 losses).  From iteration 1000 on, when at least two tests hold at ``patience`` = 2 successive calls the
    rule stops, with the reasons of the tests that hold; a call with fewer than two resets the count."""

    def __init__(self, threshold_pct=0.1, min_iterations=1000, window_size=200, patience=2, warmup_iterations=50,
                 relative_tolerance=1e-2, absolute_tolerance=1e-3):
        self.threshold_pct, self.min_iterations, self.window = threshold_pct, min_iterations, window_size
        self.patience, self.warmup_iterations = patience, warmup_iterations
        self.rtol, self.atol = relative_tolerance, absolute_tolerance
        self.count = 0

    def _tests(self, h):
        w, atol = self.window, self.atol
        out = []
        if len(h) >= w + 1:
            win = h[-w:]
            pct = np.mean(np.abs(np.diff(win) / np.maximum(np.abs(win[:-1]), atol)) * 100)
            out.append(f"Mean % change ({pct:.4f}%) < threshold" if pct < self.threshold_pct else "")
        if len(h) >= w:
            win = h[-w:]
            big = np.max(np.abs(np.diff(win)))
            out.append(f"Max absolute change ({big:.2e}) converged" if big < atol else "")
            if abs(win[0]) >= atol:
                rel = abs((win[-1] - win[0]) / win[0])
                out.append(f"Relative change ({rel:.2e}) converged" if rel < self.rtol else "")
        if len(h) >= 2 * w:
            mid = len(h) - w
            diff = abs(np.mean(h[mid : mid + w // 2]) - np.mean(h[-w // 2 :]))
            rel = diff / (abs(np.mean(h[-w:])) + atol)
            out.append(f"Loss plateau detected (relative difference: {rel:.2e})" if rel < 2 * self.rtol else "")
        return [r for r in out if r]

    def should_stop(self, iteration, loss_history):
        """(stop, reason) after the loss of ``iteration`` was appended to ``loss_history``."""
        reasons = self._tests(np.asarray(loss_history))
        if iteration < self.min_iterations:
            return False, ""
        if len(reasons) >= 2:
            self.count += 1
            if self.count >= self.patience:
                return True, "; ".join(reasons)
        else:
            self.count = 0
        return False, ""


# gpytorch 1.13's parameterisation of the MEGP model (see DESIGN.md section 4.4), in NumPy float64
_NOISE_LOWER = 1e-4  # GreaterThan(1e-4) on the task noises and the global noise


def _softplus(x):
    x = np.asarray(x, dtype=np.float64)
    return np.where(x > 20.0, x, np.log1p(np.exp(np.minimum(x, 20.0))))  # torch.nn.functional.softplus, threshold 20


def _softplus_grad(x):
    x = np.asarray(x, dtype=np.float64)
    z = np.exp(np.minimum(x, 20.0))
    return np.where(x > 20.0, 1.0, z / (z + 1.0))


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, dtype=np.float64)))


def megp_initial_raw(d, M, seed=None):
    """Initial raw parameters: raw_lengthscale 0, covar_factor and raw_var N(0, 1), raw_task_noises and raw_noise 0,
    one N(0, 1) draw of the LinearMean weights / bias shared by every task.  Draws from np.random.default_rng(seed),
    seed None meaning 0, in the order covar_factor, raw_var, weights, bias."""
    rng = np.random.default_rng(0 if seed is None else seed)
    F = rng.standard_normal((M, 1))
    raw_var = rng.standard_normal(M)
    w = rng.standard_normal(d)
    b = rng.standard_normal()
    return {"raw_lengthscale": np.zeros(d), "covar_factor": F, "raw_var": raw_var, "raw_task_noises": np.zeros(M),
            "raw_noise": np.zeros(1), "weights": np.tile(w, (M, 1)), "biases": np.full(M, b)}


def megp_natural(raw, lengthscale_bounds=None):
    """raw parameters -> (length_scale (d,), B (M,M), D (M,), weight (M,d), bias (M,))."""
    if lengthscale_bounds is None:
        ls = _softplus(raw["raw_lengthscale"])
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        ls = lo + (hi - lo) * _sigmoid(raw["raw_lengthscale"])
    F = raw["covar_factor"]
    B = F @ F.T + np.diag(_softplus(raw["raw_var"]))
    D = (_NOISE_LOWER + _softplus(raw["raw_task_noises"])) + (_NOISE_LOWER + _softplus(raw["raw_noise"]))[0]
    return ls, B, D, raw["weights"], raw["biases"]


def megp_raw_grad(raw, g, lengthscale_bounds=None):
    """Chain rule: gradients with respect to (length_scale, B with independent entries, D, weight, bias) -> gradients
    with respect to the raw parameters."""
    x = raw["raw_lengthscale"]
    if lengthscale_bounds is None:
        gl = g["length_scale"] * _softplus_grad(x)
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        s = _sigmoid(x)
        gl = g["length_scale"] * ((hi - lo) * (s * (1.0 - s)))
    gB = g["B"]
    return {"raw_lengthscale": gl, "covar_factor": (gB + gB.T) @ raw["covar_factor"],
            "raw_var": np.diag(gB) * _softplus_grad(raw["raw_var"]), "raw_task_noises": g["D"] * _softplus_grad(raw["raw_task_noises"]),
            "raw_noise": np.array([np.sum(g["D"])]) * _softplus_grad(raw["raw_noise"]), "weights": g["weight"], "biases": g["bias"]}


def _fma(a, b, c):
    """a * b + c with one rounding (as torch's CPU kernels compute lerp / addcmul): the product split exactly
    (Dekker), the sum exactly (Knuth's two-sum), the two error terms added before the final rounding."""
    p = a * b
    t = 134217729.0 * a  # 2^27 + 1
    ah = t - (t - a)
    t = 134217729.0 * b
    bh = t - (t - b)
    al, bl = a - ah, b - bh
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    s = p + c
    z = s - p
    return s + (((p - (s - z)) + (c - z)) + e)


class Adam:
    """torch.optim.Adam with its defaults (betas 0.9 / 0.999, eps 1e-8, no weight decay) on a dict of float64 arrays,
    in torch's order of operations and roundings: m <- fma(1 - b1, g - m, m) (lerp); v <- fma((1 - b2) g, g, v b2)
    (addcmul); denom = sqrt(v) / sqrt(1 - b2^t) + eps; p <- p + (-(lr / (1 - b1^t)) m) / denom (addcdiv)."""

    def __init__(self, lr=0.01, betas=(0.9, 0.999), eps=1e-8):
        self.lr, self.b1, self.b2, self.eps = lr, betas[0], betas[1], eps
        self.t, self.m, self.v = 0, {}, {}

    def step(self, params, grads):
        self.t += 1
        bc1 = 1.0 - self.b1**self.t
        bc2_sqrt = (1.0 - self.b2**self.t) ** 0.5
        step_size = self.lr / bc1
        for k, g in grads.items():
            m = self.m.get(k, np.zeros_like(g))
            v = self.v.get(k, np.zeros_like(g))
            m = _fma(np.full_like(g, 1.0 - self.b1), g - m, m)
            v = _fma((1.0 - self.b2) * g, g, v * self.b2)
            self.m[k], self.v[k] = m, v
            params[k] = params[k] + ((-step_size) * m) / (np.sqrt(v) / bc2_sqrt + self.eps)


def megp_fit(xn, yn, *, lengthscale_bounds=None, adam_lr=0.01, n_iter=5000, min_loss_pct_change=0.1, seed=None, logger=None,
             initial_raw=None):
    """Train the MEGP model on the GPU: the reference's Adam loop (dmosopt/model_gpytorch.py:1722-1829) on the exact
    log marginal likelihood and its gradient (dmo_mtgp_lml_grad).  xn (N,d) normalised inputs, yn (N,M) normalised
    targets.  Loss = -lml / (N M) (gpytorch's ExactMarginalLogLikelihood); the loss logged at iteration it is the one
    before that iteration's step.  Returns (hyperparameters, info): the ``hyperparameters=`` dict of MEGP_Matern at the
    final parameters, and info with ``loss`` (array), ``iterations``, ``stop_reason`` and ``raw`` (final raw parameters).
    ``initial_raw`` replaces the seeded initial draws (megp_initial_raw)."""
    xn = np.ascontiguousarray(xn, dtype=np.float64)
    yn = np.ascontiguousarray(yn, dtype=np.float64).reshape(xn.shape[0], -1)
    N, d = xn.shape
    M = yn.shape[1]
    raw = megp_initial_raw(d, M, seed) if initial_raw is None else {k: np.array(v, dtype=np.float64) for k, v in initial_raw.items()}
    adam = Adam(lr=adam_lr)
    stopper = EarlyStopping(threshold_pct=min_loss_pct_change)
    losses, reason = [], "n_iter"
    for it in range(n_iter):
        ls, B, D, w, b = megp_natural(raw, lengthscale_bounds)
        lml, g = _lib.mtgp_lml_grad(xn, yn, ls, B, D, w, b)
        loss = -lml / (N * M)
        graw = megp_raw_grad(raw, g, lengthscale_bounds)
        adam.step(raw, {k: v * (-1.0 / (N * M)) for k, v in graw.items()})
        losses.append(loss)
        if it % 100 == 0 and logger is not None:
            noise = _NOISE_LOWER + float(_softplus(raw["raw_noise"])[0])
            logger.info(f"MEGP_Matern: iter {it}/{n_iter} - Loss: {loss:.3f}  noise: {noise:.3f}")
        if it >= stopper.warmup_iterations:
            stop, why = stopper.should_stop(it, np.array(losses))
            if stop:
                if logger is not None:
                    logger.info(f"MEGP_Matern: early stop at iteration {it + 1}: {why}")
                reason = why
                break
    ls, B, D, w, b = megp_natural(raw, lengthscale_bounds)
    hp = {"lengthscale": ls, "covar_factor": raw["covar_factor"].copy(), "var": _softplus(raw["raw_var"]),
          "task_noises": _NOISE_LOWER + _softplus(raw["raw_task_noises"]), "noise": _NOISE_LOWER + float(_softplus(raw["raw_noise"])[0]),
          "weights": w.copy(), "biases": b.copy()}
    return hp, {"loss": np.asarray(losses), "iterations": len(losses), "stop_reason": reason, "raw": raw}


# gpytorch 1.13's parameterisation of GPyTorchExactGPModelMatern (dmosopt/model_gpytorch.py:455-508; DESIGN.md section 4.4),
# one row per objective: raw_lengthscale (M,d), raw_outputscale (M,), raw_noise (M,), weights (M,d), bias (M,)
EGP_MAX_BATCH = 8  # objectives per dmo_gp_lml_grad call


def egp_initial_raw(d, M, seed=None):
    """Initial raw parameters: raw_lengthscale, raw_outputscale and raw_noise 0; the LinearMean weights and bias N(0, 1),
    drawn from np.random.default_rng(seed), seed None meaning 0, objective by objective: weights (d), then bias."""
    rng = np.random.default_rng(0 if seed is None else seed)
    w, b = np.empty((M, d)), np.empty(M)
    for m in range(M):
        w[m] = rng.standard_normal(d)
        b[m] = rng.standard_normal()
    return {"raw_lengthscale": np.zeros((M, d)), "raw_outputscale": np.zeros(M), "raw_noise": np.zeros(M), "weights": w, "bias": b}


def egp_natural(raw, lengthscale_bounds=None):
    """raw parameters -> (length_scale (M,d), outputscale (M,), noise (M,), weight (M,d), bias (M,))."""
    if lengthscale_bounds is None:
        ls = _softplus(raw["raw_lengthscale"])
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        ls = lo + (hi - lo) * _sigmoid(raw["raw_lengthscale"])
    return ls, _softplus(raw["raw_outputscale"]), _NOISE_LOWER + _softplus(raw["raw_noise"]), raw["weights"], raw["bias"]


def egp_raw_grad(raw, g, lengthscale_bounds=None):
    """Chain rule: gradients with respect to (length_scale, outputscale, noise, weight, bias), the keys of
    _lib.gp_lml_grad -> gradients with respect to the raw parameters."""
    x = raw["raw_lengthscale"]
    if lengthscale_bounds is None:
        gl = g["length_scale"] * _softplus_grad(x)
    else:
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        s = _sigmoid(x)
        gl = g["length_scale"] * ((hi - lo) * (s * (1.0 - s)))
    return {"raw_lengthscale": gl, "raw_outputscale": g["outputscale"] * _softplus_grad(raw["raw_outputscale"]),
            "raw_noise": g["noise"] * _softplus_grad(raw["raw_noise"]), "weights": g["weight"], "bias": g["bias"]}


def egp_fit(xn, yn, *, lengthscale_bounds=None, adam_lr=0.01, n_iter=5000, min_loss_pct_change=0.1, seed=None, logger=None,
            initial_raw=None):
    """Train the EGP model on the GPU: per objective the reference's Adam loop (dmosopt/model_gpytorch.py:2023-2126) on
    the exact log marginal likelihood and its gradient (dmo_gp_lml_grad).  xn (N,d) normalised inputs, yn (N,M)
    normalised targets.  Per objective: loss = -lml_m / N, the loss logged at iteration it is the one before that
    iteration's step, its own Adam and early-stopping rule.  The objectives advance in lockstep, one dmo_gp_lml_grad call
    per iteration and group of at most EGP_MAX_BATCH objectives still training; an objective that stops leaves the batch.
    Every objective's arithmetic is its own (the call is deterministic per objective, the host steps work on per-objective
    arrays), so its trajectory is bit-identical to training it alone.  Returns (hyperparameters, info): the
    ``hyperparameters=`` dict of EGP_Matern at the final parameters, and one dict per objective with ``loss`` (array),
    ``iterations``, ``stop_reason`` and ``raw`` (its final raw parameters, rows of one).  ``initial_raw`` (the layout of
    egp_initial_raw) replaces the seeded initial draws."""
    xn = np.ascontiguousarray(xn, dtype=np.float64)
    yn = np.ascontiguousarray(yn, dtype=np.float64).reshape(xn.shape[0], -1)
    N, d = xn.shape
    M = yn.shape[1]
    raw0 = egp_initial_raw(d, M, seed) if initial_raw is None else initial_raw
    raws = [{k: np.array(np.asarray(v, dtype=np.float64)[m : m + 1]) for k, v in raw0.items()} for m in range(M)]
    adams = [Adam(lr=adam_lr) for _ in range(M)]
    stoppers = [EarlyStopping(threshold_pct=min_loss_pct_change) for _ in range(M)]
    losses = [[] for _ in range(M)]
    reasons = ["n_iter"] * M
    active = list(range(M))
    for it in range(n_iter):
        if not active:
            break
        stopped = []
        for g0 in range(0, len(active), EGP_MAX_BATCH):
            group = active[g0 : g0 + EGP_MAX_BATCH]
            nat = [egp_natural(raws[m], lengthscale_bounds) for m in group]
            lml, g = _lib.gp_lml_grad(xn, yn[:, group], *(np.concatenate([p[i] for p in nat]) for i in range(5)))
            for j, m in enumerate(group):
                loss = -lml[j] / N
                graw = egp_raw_grad(raws[m], {k: v[j : j + 1] for k, v in g.items()}, lengthscale_bounds)
                adams[m].step(raws[m], {k: v * (-1.0 / N) for k, v in graw.items()})
                losses[m].append(loss)
                if it % 100 == 0 and logger is not None:
                    noise = _NOISE_LOWER + float(_softplus(raws[m]["raw_noise"])[0])
                    logger.info(f"EGP_Matern: iter {it}/{n_iter} - Loss: {loss:.3f}  noise: {noise:.3f}")
                if it >= stoppers[m].warmup_iterations:
                    stop, why = stoppers[m].should_stop(it, np.array(losses[m]))
                    if stop:
                        if logger is not None:
                            logger.info(f"EGP_Matern: early stop at iteration {it + 1}: {why}")
                        reasons[m] = why
                        stopped.append(m)
        active = [m for m in active if m not in stopped]
    nat = [egp_natural(r, lengthscale_bounds) for r in raws]
    hp = {k: np.concatenate([p[i] for p in nat]) for i, k in enumerate(("lengthscale", "outputscale", "noise", "weight", "bias"))}
    info = [{"loss": np.asarray(losses[m]), "iterations": len(losses[m]), "stop_reason": reasons[m], "raw": raws[m]} for m in range(M)]
    return hp, info


def _reference_can_train():
    """True when dmosopt.model_gpytorch imports with gpytorch available."""
    try:
        import dmosopt.model_gpytorch as ref
    except Exception:
        return False
    return bool(getattr(ref, "_has_gpytorch", False))


class MEGP_Matern:
    """Multitask exact-GP surrogate; the reference constructor signature (model_gpytorch.py:1624-1647) plus
    ``precision`` ("fp64", the default, or "tensor"; there is no "auto" calibration for this model),
    ``hyperparameters`` (dict with lengthscale (d,), covar_factor (M, rank), var (M,), task_noises (M,), noise, weights
    (M,d), biases (M,)): when given, training is skipped, and ``fit``: "gpu" trains with megp_fit (Adam on the exact
    log marginal likelihood, on the GPU), "reference" through the reference class (needs gpytorch); None uses the
    reference class where it can train and "gpu" otherwise.  After a fit ``hyperparameters`` and ``fit_info`` hold the
    result.  ``log_marginal_likelihood_value`` is the exact log marginal likelihood of the normalised targets under the
    model."""

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, seed=None, gp_lengthscale_bounds=None, gp_likelihood_sigma=None,
                 batch_size=None, preconditioner_size=100, adam_lr=0.01, fast_pred_var=False, n_iter=5000,
                 min_loss_pct_change=0.1, return_mean_variance=False, use_cuda=False, nan="remove", top_k=None, logger=None,
                 precision="fp64", hyperparameters=None, fit=None, **kwargs):
        codes = {"fp64": _lib.GP_FP64, "tensor": _lib.GP_TENSOR, _lib.GP_FP64: _lib.GP_FP64, _lib.GP_TENSOR: _lib.GP_TENSOR}
        if precision not in codes:
            raise ValueError(f"MEGP_Matern: precision must be 'fp64' or 'tensor' (got {precision!r})")
        if fit not in (None, "gpu", "reference"):
            raise ValueError(f"MEGP_Matern: fit must be 'gpu', 'reference' or None (got {fit!r})")
        self.precision = codes[precision]
        if self.precision == _lib.GP_TENSOR and nInput > _lib.GP_PREDICT_MAX_D:  # refused before any training starts
            raise ValueError(f"MEGP_Matern: the tensor-core predict takes at most {_lib.GP_PREDICT_MAX_D} input dimensions "
                             f"(got nInput={nInput}); use precision='fp64'")
        self.nInput, self.nOutput = nInput, nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        xub = np.asarray(xub, dtype=np.float64)
        self.xrng = np.where(np.isclose(xub - self.xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - self.xlb)  # model_gpytorch.py:1662-1664
        self.return_mean_variance = return_mean_variance
        self.logger = logger
        self.fit_info = None
        if hyperparameters is None and fit is None:
            fit = "reference" if _reference_can_train() else "gpu"
        if hyperparameters is None and fit == "gpu" and gp_likelihood_sigma is not None:
            raise ValueError("MEGP_Matern: the GPU fit has no noise prior (gp_likelihood_sigma); use fit='reference'")
        if hyperparameters is None and fit == "reference":
            ref_kwargs = dict(seed=seed, gp_lengthscale_bounds=gp_lengthscale_bounds, gp_likelihood_sigma=gp_likelihood_sigma,
                              batch_size=batch_size, preconditioner_size=preconditioner_size, adam_lr=adam_lr,
                              fast_pred_var=fast_pred_var, n_iter=n_iter, min_loss_pct_change=min_loss_pct_change,
                              use_cuda=use_cuda, nan=nan, top_k=top_k, **kwargs)
            xn, yn, ymean, ystd, hyperparameters = self._fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, logger, ref_kwargs)
        else:
            yin = np.asarray(yin, dtype=np.float64).reshape(len(yin), -1)
            xin = np.asarray(xin, dtype=np.float64)
            xin, yin = filter_and_top_k(xin, yin, nan, top_k)  # model_gpytorch.py:1668-1671
            xn = (xin - self.xlb) / self.xrng
            yn, ymean, ystd = normalise_targets(yin)
            if hyperparameters is None:
                if logger is not None:
                    logger.info("MEGP_Matern: optimizing regressor...")
                hyperparameters, self.fit_info = megp_fit(xn, yn, lengthscale_bounds=gp_lengthscale_bounds, adam_lr=adam_lr,
                                                          n_iter=n_iter, min_loss_pct_change=min_loss_pct_change, seed=seed,
                                                          logger=logger)
        self.hyperparameters = hyperparameters
        self._upload(xn, yn, ymean, ystd, hyperparameters)

    @staticmethod
    def _fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, logger, kwargs):
        """Train with the reference class (unchanged) and read the fitted state out of its gpytorch model."""
        try:
            from dmosopt.model_gpytorch import MEGP_Matern as RefMEGP
        except Exception as e:  # dmosopt or gpytorch missing
            raise RuntimeError("dmosopt_b200.model_gpytorch.MEGP_Matern trains through dmosopt.model_gpytorch.MEGP_Matern, "
                               "which requires dmosopt and the GPyTorch library; pass hyperparameters= to skip training") from e
        ref = RefMEGP(xin, yin, nInput, nOutput, np.asarray(xlb), np.asarray(xub), logger=logger, **kwargs)
        xn, yn, hp = megp_hyperparameters(ref.sm)
        return xn, yn, np.asarray(ref.y_train_mean, dtype=np.float64), np.asarray(ref.y_train_std, dtype=np.float64), hp

    def _upload(self, xn, yn, ymean, ystd, hp):
        """Multitask posterior -> HBM, once per epoch."""
        M, d = self.nOutput, self.nInput
        F = np.asarray(hp["covar_factor"], dtype=np.float64).reshape(M, -1)
        B = F @ F.T + np.diag(np.asarray(hp["var"], dtype=np.float64).reshape(M))  # IndexKernel covar_matrix
        B = 0.5 * (B + B.T)
        D = np.asarray(hp["task_noises"], dtype=np.float64).reshape(M) + float(np.ravel(hp["noise"])[0])
        ls = np.broadcast_to(np.asarray(hp["lengthscale"], dtype=np.float64).reshape(-1), (d,))
        self._gp = _lib.MTGPHandle(xn, np.asarray(yn, dtype=np.float64).reshape(-1, M), ls, B, D,
                                   np.asarray(hp["weights"], dtype=np.float64).reshape(M, d), np.asarray(hp["biases"], dtype=np.float64).reshape(M),
                                   ymean, ystd, self.xlb, self.xlb + self.xrng)
        self.log_marginal_likelihood_value = self._gp.lml

    def predict(self, xin):
        """model_gpytorch.py:1872-1919: (mean (P, M), variance (P, M)) of likelihood(model(x)) as float32 arrays."""
        xin = np.asarray(xin, dtype=np.float64)
        if xin.ndim == 1:
            xin = xin.reshape((1, self.nInput))
        mean, var = self._gp.predict(xin, return_var=True, precision=self.precision)
        return mean.astype(np.float32), var.astype(np.float32)

    def evaluate(self, x):
        """model_gpytorch.py:1921-1926."""
        mean, var = self.predict(x)
        return (mean, var) if self.return_mean_variance else mean


# ------------------------------------------------------------------------------------------------------ deep GPs
DEEPGP_JITTER = 1e-4  # gpytorch's settings.variational_cholesky_jitter for the float32 models the reference trains
DEEPGP_MIN_VARIANCE = 1e-6  # gpytorch's settings.min_variance for float32
MDGP_DEFAULT_SEED = 0x5EED_D6B  # the Philox key of MDGP_Matern's draws when seed is None

_DEEPGP_KEYS = {
    # key: (shape in terms of H, T, Z1, Z2, J, d; None for a scalar)
    "hidden_inducing_points": ("H", "Z1", "d"), "hidden_outputscale": ("H",), "hidden_lengthscale": ("H", "d"),
    "hidden_variational_mean": ("H", "Z1"), "hidden_chol_variational_covar": ("H", "Z1", "Z1"), "mean_weights": ("d",),
    "mean_bias": None, "last_inducing_points": ("T", "Z2", "H"), "last_outputscale": ("T",), "last_lengthscale": ("T", "H"),
    "last_variational_mean": ("T", "Z2"), "last_chol_variational_covar": ("T", "Z2", "Z2"), "mean_constant": None,
    "task_noises": ("T",), "noise": None,
}


def deepgp_hyperparameters(model, nInput, nOutput, quadrature):
    """Read a trained ``GPyTorchMultitaskDSPPMatern`` / ``GPyTorchMultitaskDeepGPMatern`` (dmosopt/model_gpytorch.py
    :185-277, 359-453) out into the ``hyperparameters=`` dict of MDSPP_Matern / MDGP_Matern, by gpytorch's attribute
    names.  Inducing points shared by the hidden units are expanded to one plane per unit, a single length scale per unit
    to all input dimensions, and chol_variational_covar is masked to its lower triangle (as
    CholeskyVariationalDistribution does).  Refuses any strategy but a whitened VariationalStrategy and any distribution
    but a CholeskyVariationalDistribution."""

    def arr(t):
        return np.asarray(t.detach().cpu().numpy(), dtype=np.float64)

    def unit(layer, name, n_units, in_dims):
        vs = layer.variational_strategy
        if type(vs).__name__ != "VariationalStrategy":
            raise ValueError(f"{name}: a whitened VariationalStrategy is required (got {type(vs).__name__})")
        dist = vs._variational_distribution
        if type(dist).__name__ != "CholeskyVariationalDistribution":
            raise ValueError(f"{name}: a CholeskyVariationalDistribution is required (got {type(dist).__name__})")
        Z = arr(vs.inducing_points)
        Z = np.broadcast_to(Z.reshape((-1,) + Z.shape[-2:]), (n_units,) + Z.shape[-2:]).copy()
        cm = getattr(layer.covar_module, "module", layer.covar_module)  # MultiDeviceKernel wraps the ScaleKernel
        ls = arr(cm.base_kernel.lengthscale).reshape(n_units, -1)
        return {"inducing_points": Z, "outputscale": arr(cm.outputscale).reshape(n_units),
                "lengthscale": np.broadcast_to(ls, (n_units, in_dims)).copy(),
                "variational_mean": arr(dist.variational_mean).reshape(n_units, Z.shape[1]),
                "chol_variational_covar": np.tril(arr(dist.chol_variational_covar).reshape(n_units, Z.shape[1], Z.shape[1]))}

    H = int(model.hidden_layer.output_dims)
    hid = unit(model.hidden_layer, "hidden_layer", H, nInput)
    last = unit(model.last_layer, "last_layer", nOutput, H)
    hp = {f"hidden_{k}": v for k, v in hid.items()}
    hp.update({f"last_{k}": v for k, v in last.items()})
    mm = model.hidden_layer.mean_module
    hp["mean_weights"] = arr(mm.weights).reshape(nInput)
    hp["mean_bias"] = float(arr(mm.bias).reshape(-1)[0])
    hp["mean_constant"] = float(arr(model.last_layer.mean_module.constant).reshape(-1)[0])
    lik = model.likelihood
    hp["task_noises"] = arr(lik.task_noises).reshape(nOutput) if getattr(lik, "has_task_noise", True) else np.zeros(nOutput)
    hp["noise"] = float(arr(lik.noise).reshape(-1)[0]) if getattr(lik, "has_global_noise", True) else 0.0
    if quadrature:
        hp["quad_sites"] = arr(model.last_layer.quad_sites).reshape(-1, H)  # J from the parameter's shape
    return hp


def deepgp_check_hyperparameters(hp, nInput, nOutput, quadrature, who):
    """float64 copies of the ``hyperparameters=`` arrays, their shapes checked; a ValueError names the first problem."""
    if not isinstance(hp, dict):
        raise ValueError(f"{who}: hyperparameters must be a dict (got {type(hp).__name__})")
    keys = dict(_DEEPGP_KEYS, **({"quad_sites": ("J", "H")} if quadrature else {}))
    missing = [k for k in keys if k not in hp]
    if missing:
        raise ValueError(f"{who}: hyperparameters is missing {', '.join(missing)}")
    out = {k: np.asarray(hp[k], dtype=np.float64) for k in keys}
    def lead(k, axis):  # axis 0 or -1 of array k; -1 for a scalar
        return out[k].shape[axis] if out[k].ndim >= 1 else -1

    dims = {"d": nInput, "T": nOutput, "H": lead("hidden_outputscale", 0), "Z1": lead("hidden_variational_mean", -1),
            "Z2": lead("last_variational_mean", -1), "J": lead("quad_sites", 0) if quadrature else -1}
    for k, shape in keys.items():
        want = () if shape is None else tuple(dims[s] for s in shape)
        if out[k].shape != want:
            raise ValueError(f"{who}: hyperparameters[{k!r}] must have shape {want}, got {out[k].shape}")
        if not np.all(np.isfinite(out[k])):
            raise ValueError(f"{who}: hyperparameters[{k!r}] must be finite")
    return out


# ---- deep GP training on the GPU (fit="gpu-seeded")
DEEPGP_FIT_MAX_Z = 128  # inducing points per layer of dmo_dgp_fit (one CTA holds K(Z, Z) in shared memory)
DEEPGP_FIT_MAX_HT = 8  # hidden units and tasks
DEEPGP_FIT_MAX_D = 90  # input dimensions
DSPP_NUM_QUAD_SITES = 3  # gpytorch DSPPLayer's default num_quad_sites

# raw parameters of the deep GP, in the order of the flat vector of dmo_dgp_fit (include/dmosopt_b200.h): key -> shape
DEEPGP_RAW_KEYS = ("hidden_inducing_points", "hidden_raw_lengthscale", "hidden_raw_outputscale", "hidden_variational_mean",
                   "hidden_chol_variational_covar", "mean_weights", "mean_bias", "last_inducing_points", "last_raw_lengthscale",
                   "last_raw_outputscale", "last_variational_mean", "last_chol_variational_covar", "mean_constant", "raw_task_noises",
                   "raw_noise", "quad_sites")


def deepgp_raw_shapes(d, T, H, Z1, Z2, quadrature):
    """{key: shape} of the raw parameters, in flat-vector order."""
    shapes = {"hidden_inducing_points": (Z1, d), "hidden_raw_lengthscale": (H,), "hidden_raw_outputscale": (H,),
              "hidden_variational_mean": (H, Z1), "hidden_chol_variational_covar": (H, Z1, Z1), "mean_weights": (d,), "mean_bias": (1,),
              "last_inducing_points": (T, Z2, H), "last_raw_lengthscale": (T,), "last_raw_outputscale": (T,),
              "last_variational_mean": (T, Z2), "last_chol_variational_covar": (T, Z2, Z2), "mean_constant": (1,),
              "raw_task_noises": (T,), "raw_noise": (1,)}
    if quadrature:
        shapes["quad_sites"] = (DSPP_NUM_QUAD_SITES, H)
    return shapes


def deepgp_flatten(raw):
    """raw dict -> the flat float64 vector of dmo_dgp_fit."""
    return np.concatenate([np.asarray(raw[k], dtype=np.float64).reshape(-1) for k in DEEPGP_RAW_KEYS if k in raw])


def deepgp_unflatten(flat, shapes):
    """The flat vector -> raw dict with the given {key: shape}."""
    out, o = {}, 0
    for k, shp in shapes.items():
        n = int(np.prod(shp))
        out[k] = np.asarray(flat[o : o + n], dtype=np.float64).reshape(shp).copy()
        o += n
    return out


def deepgp_initial_raw(xn, T, *, quadrature, num_hidden_dims=3, num_inducing_points=128, rng=None):
    """Initial raw parameters of the reference's DSPP / DeepGP model (dmosopt/model_gpytorch.py:185-247, 359-416) at the
    normalised inputs xn (N,d).  Z = min(num_inducing_points, N) in both layers.  Raw length scales, output scales and
    noises 0; chol_variational_covar I; mean constant 0.  Draws from ``rng`` (np.random.Generator) in this order: the
    hidden inducing points, kmeans2(xn, xn[permutation(N)[:Z]], minit="matrix"); the LinearMean weights (d) and bias;
    the hidden variational means (H,Z) then the last-layer ones (T,Z), both 1e-3 N(0,1); the last-layer inducing points
    (T,Z,H) N(0,1); the quadrature sites (3,H) N(0,1) (quadrature only)."""
    from scipy.cluster.vq import kmeans2

    xn = np.asarray(xn, dtype=np.float64)
    N, d = xn.shape
    H = int(num_hidden_dims)
    Z = min(int(num_inducing_points), N)
    perm = rng.permutation(N)
    Z1 = kmeans2(xn, xn[perm[:Z]].copy(), minit="matrix")[0]
    w = rng.standard_normal(d)
    b = rng.standard_normal(1)
    mu1 = 1e-3 * rng.standard_normal((H, Z))
    mu2 = 1e-3 * rng.standard_normal((T, Z))
    Z2 = rng.standard_normal((T, Z, H))
    raw = {"hidden_inducing_points": Z1, "hidden_raw_lengthscale": np.zeros(H), "hidden_raw_outputscale": np.zeros(H),
           "hidden_variational_mean": mu1, "hidden_chol_variational_covar": np.tile(np.eye(Z), (H, 1, 1)), "mean_weights": w,
           "mean_bias": b, "last_inducing_points": Z2, "last_raw_lengthscale": np.zeros(T), "last_raw_outputscale": np.zeros(T),
           "last_variational_mean": mu2, "last_chol_variational_covar": np.tile(np.eye(Z), (T, 1, 1)), "mean_constant": np.zeros(1),
           "raw_task_noises": np.zeros(T), "raw_noise": np.zeros(1)}
    if quadrature:
        raw["quad_sites"] = rng.standard_normal((DSPP_NUM_QUAD_SITES, H))
    return raw


def deepgp_natural(raw, lengthscale_bounds=None):
    """raw parameters -> the ``hyperparameters=`` dict of MDSPP_Matern / MDGP_Matern: the shared hidden inducing points
    expanded to one plane per unit, each isotropic length scale broadcast over its unit's input dimensions, chol masked to
    its lower triangle, the transforms applied."""

    def ls(x):
        if lengthscale_bounds is None:
            return _softplus(x)
        lo, hi = float(lengthscale_bounds[0]), float(lengthscale_bounds[1])
        return lo + (hi - lo) * _sigmoid(x)

    Z1 = np.asarray(raw["hidden_inducing_points"], dtype=np.float64)
    H = raw["hidden_raw_outputscale"].shape[0]
    d = Z1.shape[1]
    hp = {"hidden_inducing_points": np.broadcast_to(Z1, (H,) + Z1.shape).copy(), "hidden_outputscale": _softplus(raw["hidden_raw_outputscale"]),
          "hidden_lengthscale": np.repeat(ls(raw["hidden_raw_lengthscale"])[:, None], d, axis=1),
          "hidden_variational_mean": raw["hidden_variational_mean"].copy(),
          "hidden_chol_variational_covar": np.tril(raw["hidden_chol_variational_covar"]), "mean_weights": raw["mean_weights"].copy(),
          "mean_bias": float(raw["mean_bias"][0]), "last_inducing_points": raw["last_inducing_points"].copy(),
          "last_outputscale": _softplus(raw["last_raw_outputscale"]), "last_lengthscale": np.repeat(ls(raw["last_raw_lengthscale"])[:, None], H, axis=1),
          "last_variational_mean": raw["last_variational_mean"].copy(), "last_chol_variational_covar": np.tril(raw["last_chol_variational_covar"]),
          "mean_constant": float(raw["mean_constant"][0]), "task_noises": _NOISE_LOWER + _softplus(raw["raw_task_noises"]),
          "noise": _NOISE_LOWER + float(_softplus(raw["raw_noise"])[0])}
    if "quad_sites" in raw:
        hp["quad_sites"] = raw["quad_sites"].copy()
    return hp


class ReduceLROnPlateau:
    """torch.optim.lr_scheduler.ReduceLROnPlateau(mode="min", patience=3, threshold=0.01) with torch's other defaults
    (factor 0.1, threshold_mode "rel", cooldown 0, min_lr 0, eps 1e-8), restated: a loss below best (1 - threshold) is an
    improvement and resets the count of bad epochs; when the count exceeds patience the lr becomes max(lr factor,
    min_lr) if that lowers it by more than eps, and the count restarts."""

    def __init__(self, lr, factor=0.1, patience=3, threshold=0.01, min_lr=0.0, eps=1e-8):
        self.lr, self.factor, self.patience, self.threshold, self.min_lr, self.eps = float(lr), factor, patience, threshold, min_lr, eps
        self.best = float("inf")
        self.num_bad_epochs = 0

    def step(self, metric):
        """The lr after the epoch loss ``metric``."""
        current = float(metric)
        if current < self.best * (1.0 - self.threshold):
            self.best = current
            self.num_bad_epochs = 0
        else:
            self.num_bad_epochs += 1
        if self.num_bad_epochs > self.patience:
            new_lr = max(self.lr * self.factor, self.min_lr)
            if self.lr - new_lr > self.eps:
                self.lr = new_lr
            self.num_bad_epochs = 0
        return self.lr


def deepgp_stopper(quadrature, min_loss_pct_change):
    """The reference's AdaptiveEarlyStopping for the deep GPs: DEEP_STOCHASTIC (MDSPP, from epoch 2000) or DEEP_GP (MDGP,
    from 1500); window 500, patience 3, warmup 200, threshold_pct = min_loss_pct_change."""
    return EarlyStopping(threshold_pct=min_loss_pct_change, min_iterations=2000 if quadrature else 1500, window_size=500, patience=3,
                         warmup_iterations=200)


def deepgp_fit(xn, yn, *, quadrature, num_hidden_dims=3, num_inducing_points=128, lengthscale_bounds=None, adam_lr=0.1, n_iter=2000,
               min_loss_pct_change=1.0, batch_size=None, seed=None, logger=None, initial_raw=None):
    """Train MDSPP_Matern (quadrature) or MDGP_Matern on the GPU: the reference's loop (dmosopt/model_gpytorch.py:1179-1216,
    1495-1532) on the minibatch loss and gradient of dmo_dgp_fit.  xn (N,d) normalised inputs, yn (N,T) normalised targets.

    Per epoch: a fresh permutation of the rows, batches of batch_size (default 10 for MDSPP, 50 for MDGP; the last may be
    partial), one Adam step each, all on the device; the epoch loss is the unweighted mean of the batch losses and steps
    ReduceLROnPlateau; every 100 epochs the reference's log line; from epoch 200 the early-stopping rule, which -- as in
    the reference, whose ``break`` sits inside ``if logger is not None`` -- stops the loop only when a logger is given.
    MDGP draws J = batch_size samples per row (num_likelihood_samples during the reference's training) from Philox4x32-10
    keyed by the seed and the step counter.  Randomness: np.random.default_rng(seed) (seed None meaning 0) makes the
    initial draws (deepgp_initial_raw, made even when ``initial_raw`` replaces them) and then one permutation per epoch.

    Returns (hyperparameters, info): the ``hyperparameters=`` dict at the final parameters, and info with ``loss`` (epoch
    losses), ``lr`` (the lr of each epoch), ``iterations``, ``stop_reason`` and ``raw`` (final raw parameters)."""
    xn = np.ascontiguousarray(xn, dtype=np.float64)
    yn = np.ascontiguousarray(yn, dtype=np.float64).reshape(xn.shape[0], -1)
    N, d = xn.shape
    T = yn.shape[1]
    H = int(num_hidden_dims)
    B = int(batch_size if batch_size is not None else (10 if quadrature else 50))
    B = min(B, N)
    name = "MDSPP_Matern" if quadrature else "MDGP_Matern"
    seed_v = 0 if seed is None else int(seed)
    rng = np.random.default_rng(seed_v)
    raw = deepgp_initial_raw(xn, T, quadrature=quadrature, num_hidden_dims=H, num_inducing_points=num_inducing_points, rng=rng)
    if initial_raw is not None:
        raw = {k: np.array(v, dtype=np.float64) for k, v in initial_raw.items()}
    Z1 = raw["hidden_variational_mean"].shape[1]
    Z2 = raw["last_variational_mean"].shape[1]
    shapes = deepgp_raw_shapes(d, T, H, Z1, Z2, quadrature)
    J = DSPP_NUM_QUAD_SITES if quadrature else B
    state = _lib.DGPFitState(xn, yn, H, Z1, Z2, J, quadrature, B, lengthscale_bounds=lengthscale_bounds, jitter=DEEPGP_JITTER,
                             min_variance=DEEPGP_MIN_VARIANCE)
    state.set_params(deepgp_flatten(raw))
    sched = ReduceLROnPlateau(adam_lr)
    stopper = deepgp_stopper(quadrature, min_loss_pct_change)
    losses, lrs, reason, step = [], [], "n_iter", 0
    nb = -(-N // B)
    for it in range(n_iter):
        lr = sched.lr
        batch_losses = state.epoch(rng.permutation(N), B, lr, seed=seed_v, step0=step)
        step += nb
        mean_loss = float(np.mean(batch_losses))
        losses.append(mean_loss)
        lrs.append(lr)
        sched.step(mean_loss)
        if it % 100 == 0 and logger is not None:
            noise = _NOISE_LOWER + float(_softplus(state.get_params()[-(1 + (J * H if quadrature else 0))]))
            sep = "  " if quadrature else "  noise:  "
            logger.info(f"{name}: iter {it}/{n_iter} - Loss: {mean_loss:.3f}{sep}{noise:.3f}")
        if it >= stopper.warmup_iterations:
            stop, why = stopper.should_stop(it, np.array(losses))
            if stop and logger is not None:
                logger.info(f"{name}: early stop at iteration {it + 1}: {why}")
                reason = why
                break
    raw = deepgp_unflatten(state.get_params(), shapes)
    state.close()
    hp = deepgp_natural(raw, lengthscale_bounds)
    return hp, {"loss": np.asarray(losses), "lr": np.asarray(lrs), "iterations": len(losses), "stop_reason": reason, "raw": raw}


class _DeepGP:
    """Shared construction and predict of MDSPP_Matern and MDGP_Matern (see their docstrings)."""

    NAME = ""
    QUADRATURE = False

    def _setup(self, xin, yin, nInput, nOutput, xlb, xub, fit, precision, hyperparameters, jitter, return_mean_variance, nan, top_k,
               logger, ref_kwargs):
        codes = {"fp64": _lib.GP_FP64, "tensor": _lib.GP_TENSOR, _lib.GP_FP64: _lib.GP_FP64, _lib.GP_TENSOR: _lib.GP_TENSOR}
        who = self.NAME
        if precision not in codes:
            raise ValueError(f"{who}: precision must be 'fp64' or 'tensor' (got {precision!r})")
        if fit not in (None, "gpu", "gpu-seeded", "reference"):
            raise ValueError(f"{who}: fit must be 'reference', 'gpu-seeded', 'gpu' or None (got {fit!r})")
        if fit == "gpu":
            raise ValueError(f"{who}: training on the GPU with torch's own random streams is not built yet; fit='gpu-seeded' "
                             "trains on the GPU with seeded streams (or use fit='reference', or pass hyperparameters=)")
        self.precision = codes[precision]
        if self.precision == _lib.GP_TENSOR and nInput > _lib.GP_PREDICT_MAX_D:
            raise ValueError(f"{who}: the tensor-core predict takes at most {_lib.GP_PREDICT_MAX_D} input dimensions "
                             f"(got nInput={nInput}); use precision='fp64'")
        self.nInput, self.nOutput = nInput, nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        xub = np.asarray(xub, dtype=np.float64)
        self.xrng = np.where(np.isclose(xub - self.xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - self.xlb)  # model_gpytorch.py:1034-1036
        self.return_mean_variance = return_mean_variance
        self.logger = logger
        self.fit_info = None
        if hyperparameters is None and fit == "gpu-seeded":
            self._check_gpu_fit(nInput, nOutput, len(xin), ref_kwargs)
        if hyperparameters is not None or fit == "gpu-seeded":
            yin = np.asarray(yin, dtype=np.float64).reshape(len(yin), -1)
            xin, yin = filter_and_top_k(np.asarray(xin, dtype=np.float64), yin, nan, top_k)
            # float64 statistics (the reference's are float32); handle_zeros_in_scale
            ymean = yin.mean(axis=0)
            ystd = yin.std(axis=0)
            ystd = np.where(ystd < 10 * np.finfo(np.float64).eps, 1.0, ystd)
            if hyperparameters is None:
                if logger is not None:
                    logger.info(f"{who}: optimizing regressor...")
                xn = (xin - self.xlb) / self.xrng
                hyperparameters, self.fit_info = deepgp_fit(
                    xn, (yin - ymean) / ystd, quadrature=self.QUADRATURE, num_hidden_dims=ref_kwargs["num_hidden_dims"],
                    num_inducing_points=ref_kwargs["num_inducing_points"], lengthscale_bounds=ref_kwargs["gp_lengthscale_bounds"],
                    adam_lr=ref_kwargs["adam_lr"], n_iter=ref_kwargs["n_iter"], min_loss_pct_change=ref_kwargs["min_loss_pct_change"],
                    batch_size=ref_kwargs["batch_size"], seed=ref_kwargs["seed"], logger=logger)
            hp = deepgp_check_hyperparameters(hyperparameters, nInput, nOutput, self.QUADRATURE, who)
        else:
            try:
                import dmosopt.model_gpytorch as ref
            except Exception as e:
                raise RuntimeError(f"dmosopt_b200.model_gpytorch.{who} trains through dmosopt.model_gpytorch.{who}, which requires "
                                   "dmosopt and the GPyTorch library; pass hyperparameters= to skip training") from e
            if not getattr(ref, "_has_gpytorch", False):
                raise RuntimeError(f"dmosopt_b200.model_gpytorch.{who} trains through dmosopt.model_gpytorch.{who}, which requires "
                                   "the GPyTorch library; pass hyperparameters= to skip training")
            model = getattr(ref, who)(xin, yin, nInput, nOutput, np.asarray(xlb), np.asarray(xub), logger=logger, nan=nan, top_k=top_k,
                                      **ref_kwargs)
            hp = deepgp_hyperparameters(model.sm, nInput, nOutput, self.QUADRATURE)
            ymean = np.asarray(model.y_train_mean, dtype=np.float64)
            ystd = np.asarray(model.y_train_std, dtype=np.float64)
        self.hyperparameters = hp
        self.y_train_mean, self.y_train_std = ymean, ystd
        self._gp = _lib.DGPHandle(
            hp["hidden_inducing_points"], hp["hidden_outputscale"], hp["hidden_lengthscale"], hp["hidden_variational_mean"],
            np.tril(hp["hidden_chol_variational_covar"]), hp["mean_weights"], float(hp["mean_bias"]), hp["last_inducing_points"],
            hp["last_outputscale"], hp["last_lengthscale"], hp["last_variational_mean"], np.tril(hp["last_chol_variational_covar"]),
            float(hp["mean_constant"]), hp["task_noises"] + float(hp["noise"]), ymean, ystd, self.xlb, self.xrng,
            quad_sites=hp.get("quad_sites"), n_sites=self._n_sites(), jitter=jitter, min_variance=DEEPGP_MIN_VARIANCE)

    def _check_gpu_fit(self, nInput, nOutput, N, kw):
        """Refuse, before any training starts, what dmo_dgp_fit does not train."""
        who = self.NAME
        if kw.get("gp_likelihood_sigma") is not None:
            raise ValueError(f"{who}: the GPU fit has no noise prior (gp_likelihood_sigma); use fit='reference'")
        H = int(kw["num_hidden_dims"])
        if not 1 <= H <= DEEPGP_FIT_MAX_HT or not 1 <= nOutput <= DEEPGP_FIT_MAX_HT:
            raise ValueError(f"{who}: the GPU fit takes 1 to {DEEPGP_FIT_MAX_HT} hidden units and objectives (got num_hidden_dims={H}, "
                             f"nOutput={nOutput}); use fit='reference'")
        if nInput > DEEPGP_FIT_MAX_D:
            raise ValueError(f"{who}: the GPU fit takes at most {DEEPGP_FIT_MAX_D} input dimensions (got nInput={nInput}); "
                             "use fit='reference'")
        if min(int(kw["num_inducing_points"]), N) > DEEPGP_FIT_MAX_Z:  # the reference clips Z at N
            raise ValueError(f"{who}: the GPU fit takes at most {DEEPGP_FIT_MAX_Z} inducing points per layer (got "
                             f"num_inducing_points={kw['num_inducing_points']}); use fit='reference'")

    def _n_sites(self):
        return None

    def _draw_key(self):
        return 0, 0

    def predict(self, xin):
        """(mean (P, T), variance (P, T)) as float64 arrays (the reference returns float32)."""
        xin = np.asarray(xin, dtype=np.float64)
        if xin.ndim == 1:
            xin = xin.reshape((1, self.nInput))
        seed, stream_id = self._draw_key()
        return self._gp.predict(xin, seed=seed, stream_id=stream_id, return_var=True, precision=self.precision)

    def evaluate(self, x):
        mean, var = self.predict(x)
        return (mean, var) if self.return_mean_variance else mean

    def resident_posterior(self):
        """(kind, handle, precision, mean dtype) of the posterior MOASMO's resident epoch steps on: ``evaluate`` returns
        this handle's mean with the variance requested, as float64.  Each step takes its draw key from ``_draw_key``, as
        each predict does."""
        return _lib.POSTERIOR_DGP, getattr(self, "_gp", None), self.precision, np.float64


class MDSPP_Matern(_DeepGP):
    """Deep sigma-point process surrogate: the reference constructor signature (model_gpytorch.py:991-1019) plus
    ``precision`` ("fp64", the default, or "tensor": the hidden layer's variance through the split-fp16 contraction, d <=
    64), ``hyperparameters`` (dict, see oracle/deepgp.py and ``deepgp_check_hyperparameters``; training is skipped and the
    y statistics are computed in float64), ``jitter`` (gpytorch's variational_cholesky_jitter, 1e-4 for float32 models)
    and ``fit`` ("reference" or None: train through the reference class, which needs gpytorch; "gpu-seeded": train on the
    GPU with deepgp_fit, seeded streams in place of torch's; "gpu", replaying torch's streams, is refused).  After a
    GPU fit ``fit_info`` holds the epoch losses, the lr history, the epoch count, the stop reason and the raw parameters.

    predict is deterministic: the hidden layer's mean and standard deviation are combined with the learned quadrature
    sites ``last_layer.quad_sites`` (J of them, J from the parameter's shape, not ``Q``), the last layer is evaluated at
    each site, and the result is the reference's ``batch_preds.mean.mean(0)`` / ``.variance.mean(0)``: an unweighted
    average over the sites (the learned quadrature weights are not used, and there is no between-site spread term).
    ``fast_pred_var``, ``preconditioner_size`` and ``use_cuda`` are ignored; the reference's ``batch_size`` only affects
    its training."""

    NAME = "MDSPP_Matern"
    QUADRATURE = True

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, num_hidden_dims=3, Q=8, num_inducing_points=128, seed=None,
                 gp_lengthscale_bounds=None, gp_likelihood_sigma=None, linear_mean=True, preconditioner_size=100, adam_lr=0.1,
                 fast_pred_var=False, n_iter=2000, min_loss_pct_change=1.0, batch_size=10, return_mean_variance=False, use_cuda=False,
                 nan="remove", top_k=None, logger=None, precision="fp64", hyperparameters=None, jitter=DEEPGP_JITTER, fit=None,
                 **kwargs):
        ref_kwargs = dict(num_hidden_dims=num_hidden_dims, Q=Q, num_inducing_points=num_inducing_points, seed=seed,
                          gp_lengthscale_bounds=gp_lengthscale_bounds, gp_likelihood_sigma=gp_likelihood_sigma, linear_mean=linear_mean,
                          preconditioner_size=preconditioner_size, adam_lr=adam_lr, fast_pred_var=fast_pred_var, n_iter=n_iter,
                          min_loss_pct_change=min_loss_pct_change, batch_size=batch_size, use_cuda=use_cuda, **kwargs)
        self._setup(xin, yin, nInput, nOutput, xlb, xub, fit, precision, hyperparameters, jitter, return_mean_variance, nan, top_k,
                    logger, ref_kwargs)


class MDGP_Matern(_DeepGP):
    """Doubly stochastic deep GP surrogate: the reference constructor signature (model_gpytorch.py:1308-1335) plus
    ``precision``, ``hyperparameters``, ``jitter`` and ``fit`` as MDSPP_Matern, and ``num_samples`` (10: gpytorch's
    default num_likelihood_samples, which the reference sets only during training).

    predict is a Monte Carlo average over ``num_samples`` draws of the hidden layer's output per candidate, as the
    reference's: mean and variance are the unweighted averages over the draws.  The draws come from Philox4x32-10 keyed
    by ``seed`` (None: MDGP_DEFAULT_SEED) with the call index as stream, so every predict draws afresh and the sequence of
    predicts is reproducible from (seed, call index).  torch's random stream is not reproduced."""

    NAME = "MDGP_Matern"
    QUADRATURE = False

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, num_hidden_dims=3, num_inducing_points=128, seed=None,
                 gp_lengthscale_bounds=None, gp_likelihood_sigma=None, linear_mean=True, preconditioner_size=100, adam_lr=0.1,
                 fast_pred_var=False, n_iter=2000, min_loss_pct_change=1.0, batch_size=50, return_mean_variance=False, use_cuda=False,
                 nan="remove", top_k=None, logger=None, precision="fp64", hyperparameters=None, jitter=DEEPGP_JITTER, fit=None,
                 num_samples=10, **kwargs):
        self.num_samples = int(num_samples)
        self.seed = MDGP_DEFAULT_SEED if seed is None else int(seed)
        self.calls = 0
        ref_kwargs = dict(num_hidden_dims=num_hidden_dims, num_inducing_points=num_inducing_points, seed=seed,
                          gp_lengthscale_bounds=gp_lengthscale_bounds, gp_likelihood_sigma=gp_likelihood_sigma, linear_mean=linear_mean,
                          preconditioner_size=preconditioner_size, adam_lr=adam_lr, fast_pred_var=fast_pred_var, n_iter=n_iter,
                          min_loss_pct_change=min_loss_pct_change, batch_size=batch_size, use_cuda=use_cuda, **kwargs)
        self._setup(xin, yin, nInput, nOutput, xlb, xub, fit, precision, hyperparameters, jitter, return_mean_variance, nan, top_k,
                    logger, ref_kwargs)

    def _n_sites(self):
        return self.num_samples

    def _draw_key(self):
        self.calls += 1
        return self.seed, self.calls - 1
