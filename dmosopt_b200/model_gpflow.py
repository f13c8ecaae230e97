"""The GPflow variational surrogates of dmosopt/model.py (SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern, CRV_Matern) with
their posterior on the GPU (dmo_svgp_create / dmo_svgp_predict).

Every class keeps the reference's constructor keywords and adds:

- ``precision``: "fp64" (default) or "tensor" (split-fp16 wgmma variance contraction, ~1e-5 of the prior);
- ``hyperparameters``: a dict with GPflow's names -- ``lengthscales`` (L,d) (SIV: (1,d), one shared kernel),
  ``variance`` (L,), ``likelihood_variance`` (scalar or (L,)), and optionally ``Z`` ((Z,d) shared or (L,Z,d)), ``q_mu``
  (L,Z), ``q_sqrt`` (L,Z,Z) lower triangular and ``W`` (M,L, CRV only).  Without ``Z`` the inducing points follow the
  reference's rule with ``np.random.default_rng(seed)`` instead of the global generator (a documented deviation); without
  ``q_mu`` / ``q_sqrt`` q is set to its optimum for the Gaussian likelihood (dmo_svgp_optimal_q).  CRV requires q and W.
  This trains nothing: the kernel hyper-parameters are taken as given.
- ``fit``: "gpu" trains on the GPU (svgp_fit: natural-gradient steps on q, keras' Adam on the hyper-parameters, the
  reference's stopping rule; the reference's training keywords apply) and keeps ``hyperparameters`` and ``fit_info``;
  "reference" trains through the reference class (needs gpflow and tensorflow) and reads its ``posterior()`` objects out
  by gpflow 2.9.2's attribute names; None means "reference" when gpflow imports.

The variance is that of the latent f (GPflow's predict_f: no likelihood noise).  ``predict``'s ``batch_size`` split of
the reference is row-independent and is not repeated.
"""

import numpy as np

from . import _lib
from .model_gpytorch import filter_and_top_k

JITTER = 1e-2  # the reference sets gpflow's default jitter to 10e-3 at import (dmosopt/model.py:17)


def _gpflow_available():
    try:
        import gpflow  # noqa: F401
    except Exception:
        return False
    return True


def _np(x):
    return np.asarray(x.numpy() if hasattr(x, "numpy") else x, dtype=np.float64)


def _matern_params(k):
    if type(k).__name__ != "Matern52":
        raise ValueError(f"expected a gpflow Matern52 kernel, got {type(k).__name__}")
    return float(_np(k.variance)), np.atleast_1d(_np(k.lengthscales))


def read_gpflow_posterior(post, d):
    """State of one gpflow 2.9.2 posterior object (``gp_model.posterior()``): a dict with Z (L,Z,d), variance (L,),
    lengthscales (L,d), q_mu (L,Z), q_sqrt (L,Z,Z) and W (M,L) or None.  A posterior with whiten=False or a non-zero mean
    function is refused, so that it can never be mis-predicted."""
    white = getattr(post, "whiten", getattr(post, "white", None))
    if white is not True:
        raise ValueError("only whitened variational posteriors (whiten=True) are supported")
    mf = getattr(post, "mean_function", None)
    if mf is not None and type(mf).__name__ != "Zero":
        raise ValueError(f"only a zero mean function is supported, got {type(mf).__name__}")
    qd = getattr(post, "q_dist", None)
    q_mu = _np(qd.q_mu if qd is not None else post.q_mu)
    q_sqrt = _np(qd.q_sqrt if qd is not None else post.q_sqrt)
    Zn = q_mu.shape[0]
    L = q_mu.shape[1] if q_mu.ndim == 2 else 1
    q_mu = q_mu.reshape(Zn, L).T.copy()
    if q_sqrt.ndim == 2:  # q_diag: (Z, L) standard deviations
        q_sqrt = np.stack([np.diag(q_sqrt[:, l]) for l in range(L)])
    q_sqrt = q_sqrt.reshape(L, Zn, Zn)
    iv = post.X_data
    if hasattr(iv, "inducing_variable_list"):
        Zs = [_np(v.Z) for v in iv.inducing_variable_list]
    elif hasattr(iv, "inducing_variable"):
        Zs = [_np(iv.inducing_variable.Z)] * L
    elif hasattr(iv, "Z"):
        Zs = [_np(iv.Z)] * L
    else:  # VGP: the posterior's X_data are the training inputs
        Zs = [_np(iv)] * L
    kern = post.kernel
    W = None
    if hasattr(kern, "W"):  # LinearCoregionalization
        W = _np(kern.W)
        kernels = list(kern.kernels)
    elif hasattr(kern, "kernels"):  # SeparateIndependent
        kernels = list(kern.kernels)
    elif hasattr(kern, "kernel"):  # SharedIndependent
        kernels = [kern.kernel] * L
    else:
        kernels = [kern] * L
    if len(kernels) != L or len(Zs) != L:
        raise ValueError(f"posterior with {L} latent GPs has {len(kernels)} kernels and {len(Zs)} inducing sets")
    var, ls = zip(*[_matern_params(k) for k in kernels])
    ls = np.stack([np.broadcast_to(v, (d,)) for v in ls]).astype(np.float64)
    return dict(Z=np.stack([z.reshape(Zn, d) for z in Zs]), variance=np.asarray(var, dtype=np.float64), lengthscales=ls,
                q_mu=q_mu, q_sqrt=q_sqrt, W=W)


def choose_inducing(xn, inducing_fraction, min_inducing, rng):
    """The reference's inducing-point rule (dmosopt/model.py:862-869): every point when round(fraction N) < min_inducing,
    else that many distinct rows drawn without replacement."""
    N = xn.shape[0]
    m = int(round(inducing_fraction * N))
    if m < min_inducing:
        return xn.copy()
    return xn[rng.choice(N, size=m, replace=False), :].copy()


# ---- training on the GPU (fit="gpu") ---------------------------------------------------------------------------------
# The reference's parameterisation (DESIGN.md section 4.4, restated from gpflow 2.9.2, not checked against it): length
# scales lo + (hi - lo) sigmoid(raw) (bounded_parameter), kernel variance softplus(raw), likelihood variance
# 1e-6 + softplus(raw); W (CRV) untransformed.  Z, q_mu and q_sqrt are not trained by Adam.
LIKELIHOOD_LOWER = 1e-6
TRAIN_DEFAULTS = {"svgp": dict(batch_size=50, natgrad_gamma=0.1, n_iter=30000), "vgp": dict(batch_size=None, natgrad_gamma=1.0, n_iter=3000)}


def _softplus(x):
    return np.logaddexp(0.0, x)


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _inv_softplus(y):
    y = np.asarray(y, dtype=np.float64)
    return y + np.log(-np.expm1(-y))


class KerasAdam:
    """keras 2.14's Adam (beta 0.9 / 0.999, epsilon 1e-7) on a dict of float64 arrays: m <- m + (g - m)(1 - b1),
    v <- v + (g^2 - v)(1 - b2), p <- p - lr sqrt(1 - b2^t) / (1 - b1^t) m / (sqrt(v) + eps)."""

    def __init__(self, lr=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
        self.lr, self.b1, self.b2, self.eps = lr, beta_1, beta_2, epsilon
        self.t, self.m, self.v = 0, {}, {}

    def step(self, params, grads):
        self.t += 1
        alpha = self.lr * np.sqrt(1.0 - self.b2**self.t) / (1.0 - self.b1**self.t)
        for k, g in grads.items():
            m = self.m.get(k, np.zeros_like(g))
            v = self.v.get(k, np.zeros_like(g))
            m = m + (g - m) * (1.0 - self.b1)
            v = v + (g * g - v) * (1.0 - self.b2)
            self.m[k], self.v[k] = m, v
            params[k] = params[k] - alpha * m / (np.sqrt(v) + self.eps)


def mean_elbo_pct_change(elbo_log):
    """The reference's stopping statistic: mean percent change of the ELBO log over its last 100 differences."""
    elbo_change = np.convolve(elbo_log, np.array([1, -1]), "same")[1:]
    return float(np.mean((elbo_change / np.abs(elbo_log[1:]) * 100)[-100:]))


class MinibatchStream:
    """Consecutive B-slices of a stream of independent permutations of range(N) drawn from np.random.default_rng(seed)
    (the reference shuffles a repeated tf.data set; a documented deviation)."""

    def __init__(self, N, B, seed):
        self.N, self.B = int(N), int(B)
        self.rng = np.random.default_rng(seed)
        self.buf = np.empty(0, dtype=np.int64)

    def next(self):
        while self.buf.shape[0] < self.B:
            self.buf = np.concatenate([self.buf, self.rng.permutation(self.N).astype(np.int64)])
        b, self.buf = self.buf[: self.B], self.buf[self.B :]
        return b


class _FitModel:
    """One GPflow model in training: its state on the GPU, raw parameters, Adam, batch stream and ELBO log.  outs: the
    columns of Y it models; K: distinct kernels (1: SIV's shared kernel, else one per latent)."""

    def __init__(self, xn, yn, Z, outs, L, K, vgp, opts, seed, W0):
        self.outs, self.L, self.K, self.vgp = outs, L, K, vgp
        self.N, d = xn.shape
        self.state = _lib.SVGPFitState(xn, yn[:, outs], Z, L, jitter=JITTER, inducing_is_data=vgp)
        lo, hi = opts["lengthscale_bounds"]
        self.lo, self.hi = float(lo), float(hi)
        self.raw = {"lengthscale": np.full((K, d), np.log((1.0 - self.lo) / (self.hi - 1.0))),
                    "variance": np.full(K, _inv_softplus(1.0)),
                    "noise": np.array([_inv_softplus(opts["likelihood_sigma"] - LIKELIHOOD_LOWER)])}
        if W0 is not None:
            self.raw["W"] = np.array(W0, dtype=np.float64)
        self.adam = KerasAdam(lr=opts["adam_lr"])
        B = self.N if vgp or opts["batch_size"] is None else min(int(opts["batch_size"]), self.N)
        self.stream = None if vgp else MinibatchStream(self.N, B, seed)
        self.elbo_log, self.iterations, self.stop_reason = [], 0, "n_iter"

    def natural(self):
        M = len(self.outs)
        ls = np.broadcast_to(self.lo + (self.hi - self.lo) * _sigmoid(self.raw["lengthscale"]), (self.L, self.raw["lengthscale"].shape[1]))
        s = np.broadcast_to(_softplus(self.raw["variance"]), (self.L,))
        noise = np.full(M, LIKELIHOOD_LOWER + _softplus(self.raw["noise"][0]))
        return np.ascontiguousarray(s), np.ascontiguousarray(ls), noise, self.raw.get("W")

    def batch(self):
        return np.arange(self.N, dtype=np.int64) if self.stream is None else self.stream.next()

    def elbo(self, batch):
        ell, kl, _ = self.state.elbo_grad(batch, *self.natural(), grad=False)
        return float(np.sum(ell) - np.sum(kl))

    def step(self, gamma):
        """Natural-gradient step on one batch, then an Adam step on the next at the new q."""
        self.state.natgrad(self.batch(), *self.natural(), gamma=gamma)
        s, ls, noise, W = self.natural()
        _, _, g = self.state.elbo_grad(self.batch(), s, ls, noise, W)
        raw = self.raw
        gl = g["length_scale"] if self.K == self.L else g["length_scale"].sum(axis=0, keepdims=True)
        gs = g["variance"] if self.K == self.L else g["variance"].sum(keepdims=True)
        sg = _sigmoid(raw["lengthscale"])
        # loss = -ELBO: gradients with respect to the raw parameters, negated
        grads = {"lengthscale": -gl * ((self.hi - self.lo) * (sg * (1.0 - sg))),
                 "variance": -gs * _sigmoid(raw["variance"]),
                 "noise": -np.array([np.sum(g["noise"])]) * _sigmoid(raw["noise"])}
        if "W" in raw:
            grads["W"] = -g["W"]
        self.adam.step(raw, grads)


def svgp_fit(kind, xn, yn, Z=None, *, lengthscale_bounds=(1e-6, 100.0), likelihood_sigma=1e-4, natgrad_gamma=None, adam_lr=0.01,
             n_iter=None, min_elbo_pct_change=0.1, batch_size=-1, seed=None, logger=None, W0=None, name=None):
    """Train a variational surrogate on the GPU with the reference's loop (dmosopt/model.py:98-1179): per iteration a
    natural-gradient step on q (batch b1), an Adam step on the hyper-parameters at the new q (batch b2) and, every 10th
    iteration, the ELBO on batch b3 appended to the log (VGP: full data, the ELBO after every iteration); the stopping
    rule from iteration 2000 (VGP: 200).  kind: "svgp" / "vgp" (one model per output, trained in lockstep; a model
    that stops leaves the loop), "siv" (one model, one shared kernel), "spv" (one model, a kernel per output) or "crv"
    (like spv, plus W (M,M) trained by Adam, initial W0).  xn (N,d), yn (N,M) normalised; Z (Z,d) shared, or
    (M,Z,d) one set per output for svgp; None for vgp.  natgrad_gamma / n_iter / batch_size default to the reference's
    per class.  Returns (hyperparameters, info): the ``hyperparameters=`` dict of the class (with Z, q_mu, q_sqrt and W),
    and info with ``elbo`` (one log per model), ``iterations`` and ``stop_reason`` (one per model)."""
    xn = np.ascontiguousarray(xn, dtype=np.float64)
    yn = np.ascontiguousarray(yn, dtype=np.float64).reshape(xn.shape[0], -1)
    N, d = xn.shape
    M = yn.shape[1]
    vgp = kind == "vgp"
    dflt = TRAIN_DEFAULTS["vgp" if vgp else "svgp"]
    gamma = dflt["natgrad_gamma"] if natgrad_gamma is None else float(natgrad_gamma)
    n_iter = dflt["n_iter"] if n_iter is None else int(n_iter)
    batch_size = dflt["batch_size"] if batch_size == -1 else batch_size
    name = name or {"svgp": "SVGP_Matern", "vgp": "VGP_Matern", "siv": "SIV_Matern", "spv": "SPV_Matern", "crv": "CRV_Matern"}[kind]
    opts = dict(lengthscale_bounds=lengthscale_bounds, likelihood_sigma=float(likelihood_sigma), adam_lr=adam_lr, batch_size=batch_size)
    base = 0 if seed is None else int(seed)
    if kind in ("svgp", "vgp"):
        Zs = [None] * M if vgp else list(np.broadcast_to(np.asarray(Z, dtype=np.float64), (M,) + np.shape(Z)[-2:]))
        models = [_FitModel(xn, yn, Zs[i], [i], 1, 1, vgp, opts, [base, i], None) for i in range(M)]
    else:
        Zs = np.asarray(Z, dtype=np.float64).reshape(-1, d)
        models = [_FitModel(xn, yn, Zs, list(range(M)), M, 1 if kind == "siv" else M, False, opts, [base, 0],
                            W0 if kind == "crv" else None)]
    log_every, warmup, report = (1, 200, 100) if vgp else (10, 2000, 1000)
    active = list(models)
    for it in range(n_iter):
        if not active:
            break
        for mdl in list(active):
            mdl.step(gamma)
            mdl.iterations = it + 1
            if it % log_every == 0:
                mdl.elbo_log.append(mdl.elbo(mdl.batch()))
            if it % report == 0 and logger is not None:
                logger.info(f"{name}: iteration {it} likelihood: {mdl.elbo_log[-1]:.04f}")
            if it >= warmup:
                pct = mean_elbo_pct_change(np.asarray(mdl.elbo_log))
                if it % 1000 == 0 and logger is not None:
                    logger.info(f"{name}: iteration {it} mean elbo pct change: {pct:.04f}")
                if pct < min_elbo_pct_change:
                    if logger is not None:
                        logger.info(f"{name}: likelihood change at iteration {it + 1} is less than {min_elbo_pct_change} percent")
                    mdl.stop_reason = "elbo_pct_change"
                    active.remove(mdl)
    nat = [m.natural() for m in models]
    qs = [m.state.q() for m in models]
    hp = {"lengthscales": np.concatenate([n[1] for n in nat]), "variance": np.concatenate([n[0] for n in nat]),
          "likelihood_variance": np.concatenate([n[2] for n in nat]), "q_mu": np.concatenate([q[0] for q in qs]),
          "q_sqrt": np.concatenate([q[1] for q in qs])}
    if not vgp:
        hp["Z"] = np.stack(Zs) if kind == "svgp" else np.broadcast_to(Zs, (M,) + Zs.shape).copy()
    if kind == "crv":
        hp["W"] = models[0].raw["W"].copy()
    info = {"elbo": [np.asarray(m.elbo_log) for m in models], "iterations": [m.iterations for m in models],
            "stop_reason": [m.stop_reason for m in models]}
    return hp, info


class _VariationalGP:
    """Shared body of the five classes: data selection and normalisation as the reference's, then the posterior state
    (from the reference fit or from ``hyperparameters``) uploaded to one dmo_svgp."""

    name = None
    std_dtype = np.float32  # dtype of y_train_std
    f32_var = False  # variance cast to float32 (SVGP, VGP), else float64
    per_output_inducing = False  # SVGP: its own Z per output
    all_points = False  # VGP: Z = the training inputs

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, seed=None, batch_size=None, inducing_fraction=0.2, min_inducing=100,
                 return_mean_variance=False, num_latent_gps=None, nan="remove", top_k=None, logger=None, precision="fp64",
                 hyperparameters=None, fit=None, **kwargs):
        self.nInput, self.nOutput = nInput, nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        xub = np.asarray(xub, dtype=np.float64)
        self.xub = xub
        self.xrng = np.where(np.isclose(xub - self.xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - self.xlb)
        self.batch_size = batch_size
        self.logger = logger
        self.return_mean_variance = return_mean_variance
        self.precision = _lib.GP_TENSOR if precision in ("tensor", _lib.GP_TENSOR) else _lib.GP_FP64
        self.stats = {}
        self.fit_info = None
        if self.precision == _lib.GP_TENSOR and nInput > _lib.GP_PREDICT_MAX_D:  # refused before any training starts
            raise ValueError(f"{self.name}: the tensor-core predict takes at most {_lib.GP_PREDICT_MAX_D} input dimensions "
                             f"(got nInput={nInput}); use precision='fp64'")
        if hyperparameters is not None and fit is not None:
            raise ValueError(f"{self.name}: fit={fit!r} and hyperparameters= conflict; pass one of them")
        if fit not in (None, "reference", "gpu"):
            raise ValueError(f"{self.name}: fit must be 'gpu', 'reference' or None (got {fit!r})")
        if self.name == "CRV_Matern" and fit == "gpu" and num_latent_gps not in (None, nOutput):
            raise ValueError(f"CRV_Matern: the GPU fit builds one kernel per output and an (M, M) W; num_latent_gps must be "
                             f"None or nOutput={nOutput} (got {num_latent_gps})")
        if hyperparameters is None and fit != "gpu":
            if fit is None:
                if not _gpflow_available():
                    raise RuntimeError(f"{self.name}: training needs gpflow and tensorflow, which are not importable; pass "
                                       "hyperparameters= (lengthscales, variance, likelihood_variance) to predict without them, "
                                       "or fit='gpu' to train on the GPU")
                fit = "reference"
            if batch_size is not None:  # else the reference class's own default (50 for the SVGP forms, None for VGP)
                kwargs["batch_size"] = batch_size
            ref = self._fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, seed=seed, inducing_fraction=inducing_fraction,
                                           min_inducing=min_inducing, num_latent_gps=num_latent_gps, nan=nan, top_k=top_k,
                                           logger=logger, **kwargs)
            import gpflow

            posts = getattr(ref, "smlist", None) or [ref.sm]
            states = [read_gpflow_posterior(p, nInput) for p in posts]
            st = {k: np.concatenate([s[k] for s in states]) for k in ("Z", "variance", "lengthscales", "q_mu", "q_sqrt")}
            st["W"] = states[0]["W"]
            self.y_train_mean = np.asarray(ref.y_train_mean, dtype=np.float32)
            self.y_train_std = np.asarray(ref.y_train_std, dtype=self.std_dtype)
            self._upload(st, float(gpflow.config.default_jitter()))
            return
        xin = np.asarray(xin, dtype=np.float64)
        yin = np.asarray(yin, dtype=np.float64)
        if yin.ndim == 1:
            yin = yin.reshape(-1, 1)
        xin, yin = filter_and_top_k(xin, yin, nan, top_k)
        xn = (xin - self.xlb) / self.xrng
        N = xn.shape[0]
        self.y_train_mean = np.asarray([np.mean(yin[:, i]) for i in range(nOutput)], dtype=np.float32)
        std = [np.std(yin[:, i], axis=0) for i in range(nOutput)]
        self.y_train_std = np.asarray([s if s != 0.0 else 1.0 for s in std], dtype=self.std_dtype)  # handle_zeros_in_scale
        yn = np.column_stack([(yin[:, i] - self.y_train_mean[i]) / self.y_train_std[i] for i in range(nOutput)])
        if fit == "gpu":
            hyperparameters = self._fit_on_gpu(xn, yn, nOutput, seed, inducing_fraction, min_inducing, batch_size, logger, kwargs)
        hp = hyperparameters
        L = nOutput if self.name != "CRV_Matern" else int(num_latent_gps or nOutput)
        ls = np.asarray(hp["lengthscales"], dtype=np.float64).reshape(-1, nInput)
        var = np.asarray(hp["variance"], dtype=np.float64).reshape(-1)
        ls = np.broadcast_to(ls, (L, nInput)).copy()
        var = np.broadcast_to(var, (L,)).copy()
        noise = np.broadcast_to(np.asarray(hp["likelihood_variance"], dtype=np.float64).reshape(-1), (L,)).copy()
        if self.all_points:
            if "Z" in hp:
                raise ValueError("VGP_Matern: the inducing points are the training inputs; hyperparameters take no Z")
            Z = np.broadcast_to(xn, (L,) + xn.shape).copy()
        elif "Z" in hp:
            Z = np.asarray(hp["Z"], dtype=np.float64)
            Z = np.broadcast_to(Z, (L,) + Z.shape[-2:]).copy()
        else:
            rng = np.random.default_rng(seed)
            if self.per_output_inducing:
                Z = np.stack([choose_inducing(xn, inducing_fraction, min_inducing, rng) for _ in range(L)])
            else:
                z0 = choose_inducing(xn, inducing_fraction, min_inducing, rng)
                Z = np.broadcast_to(z0, (L,) + z0.shape).copy()
        W = hp.get("W")
        if "q_mu" in hp and "q_sqrt" in hp:
            q_mu = np.asarray(hp["q_mu"], dtype=np.float64).reshape(L, -1)
            q_sqrt = np.asarray(hp["q_sqrt"], dtype=np.float64).reshape(L, Z.shape[1], Z.shape[1])
        else:
            if self.name == "CRV_Matern":
                raise ValueError("CRV_Matern: hyperparameters need q_mu, q_sqrt and W (its latents are coupled through W)")
            q_mu, q_sqrt = _lib.svgp_optimal_q(xn, yn.T, Z, var, ls, noise, jitter=JITTER, inducing_is_data=self.all_points)
        if self.name == "CRV_Matern" and W is None:
            raise ValueError("CRV_Matern: hyperparameters need W (M, L)")
        self.hyperparameters = dict(hp, Z=Z, q_mu=q_mu, q_sqrt=q_sqrt)
        if fit == "gpu" and self.all_points:
            del self.hyperparameters["Z"]  # the training inputs: hyperparameters= takes no Z for VGP
        self._upload(dict(Z=Z, variance=var, lengthscales=ls, q_mu=q_mu, q_sqrt=q_sqrt, W=W), JITTER)

    def _fit_on_gpu(self, xn, yn, nOutput, seed, inducing_fraction, min_inducing, batch_size, logger, kw):
        """svgp_fit on the normalised data, with the inducing points of the hyperparameters= path (the same seeded
        draws) and, for CRV, W ~ N(0, 1) drawn next from the same generator; fit_info keeps the training record."""
        kind = {"SVGP_Matern": "svgp", "VGP_Matern": "vgp", "SIV_Matern": "siv", "SPV_Matern": "spv", "CRV_Matern": "crv"}[self.name]
        rng = np.random.default_rng(seed)
        Z = None
        if self.per_output_inducing:
            Z = np.stack([choose_inducing(xn, inducing_fraction, min_inducing, rng) for _ in range(nOutput)])
        elif not self.all_points:
            Z = choose_inducing(xn, inducing_fraction, min_inducing, rng)
        W0 = rng.standard_normal((nOutput, nOutput)) if kind == "crv" else None
        opts = {k: kw[k] for k in ("natgrad_gamma", "adam_lr", "n_iter", "min_elbo_pct_change") if kw.get(k) is not None}
        if kw.get("gp_lengthscale_bounds") is not None:
            opts["lengthscale_bounds"] = kw["gp_lengthscale_bounds"]
        if kw.get("gp_likelihood_sigma") is not None:
            opts["likelihood_sigma"] = kw["gp_likelihood_sigma"]
        if batch_size is not None:
            opts["batch_size"] = batch_size
        hp, self.fit_info = svgp_fit(kind, xn, yn, Z, seed=seed, logger=logger, W0=W0, name=self.name, **opts)
        return hp

    def _fit_with_reference(self, xin, yin, nInput, nOutput, xlb, xub, **kw):
        """Train with the reference class (unchanged)."""
        import dmosopt.model as ref_model

        return getattr(ref_model, self.name)(xin, yin, nInput, nOutput, xlb, xub, return_mean_variance=self.return_mean_variance, **kw)

    def _upload(self, st, jitter):
        ys64 = self.y_train_std.astype(np.float64)
        vscale = (self.y_train_std ** 2).astype(np.float64)  # float32 squares for CRV / SIV / SPV, as the reference's
        self._h = _lib.SVGPHandle(st["Z"], st["variance"], st["lengthscales"], st["q_mu"], st["q_sqrt"], self.y_train_mean.astype(np.float64),
                                  ys64, self.xlb, self.xrng, W=st["W"], jitter=jitter, y_var_scale=vscale)

    def predict(self, xin, batch_size=None):
        x = np.asarray(xin, dtype=np.float64)
        if x.ndim == 1:
            x = x.reshape(1, self.nInput)
        mean, var = self._h.predict(x, return_var=True, precision=self.precision)
        return mean.astype(np.float32), var.astype(np.float32 if self.f32_var else np.float64)

    def evaluate(self, x):
        mean, var = self.predict(x)
        if self.return_mean_variance:
            return mean, var
        return mean

    def resident_posterior(self):
        """(kind, handle, precision, mean dtype) of the posterior MOASMO's resident epoch steps on: ``evaluate`` returns
        this handle's mean with the variance requested, as float32."""
        return _lib.POSTERIOR_SVGP, getattr(self, "_h", None), self.precision, np.float32


class SVGP_Matern(_VariationalGP):
    """dmosopt/model.py:769-988: one SVGP per output, each with its own inducing points."""

    name = "SVGP_Matern"
    std_dtype = np.float64
    f32_var = True
    per_output_inducing = True

    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, return_mean_variance=True, **kwargs):
        super().__init__(xin, yin, nInput, nOutput, xlb, xub, return_mean_variance=return_mean_variance, **kwargs)


class VGP_Matern(_VariationalGP):
    """dmosopt/model.py:991-1179: one VGP per output over all training points."""

    name = "VGP_Matern"
    std_dtype = np.float64
    f32_var = True
    all_points = True


class SIV_Matern(_VariationalGP):
    """dmosopt/model.py:328-544: one SVGP, shared inducing points and one shared kernel (SharedIndependent)."""

    name = "SIV_Matern"


class SPV_Matern(_VariationalGP):
    """dmosopt/model.py:547-766: one SVGP, copies of one set of inducing points and one kernel per output."""

    name = "SPV_Matern"


class CRV_Matern(_VariationalGP):
    """dmosopt/model.py:98-325: one SVGP with L latent GPs mixed into the outputs by W (LinearCoregionalization)."""

    name = "CRV_Matern"
