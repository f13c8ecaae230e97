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
- ``fit``: "reference" trains through the reference class (needs gpflow and tensorflow) and reads its ``posterior()``
  objects out by gpflow 2.9.2's attribute names; None means "reference" when gpflow imports.

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
        if hyperparameters is not None and fit is not None:
            raise ValueError(f"{self.name}: fit={fit!r} and hyperparameters= conflict; pass one of them")
        if hyperparameters is None:
            if fit is None:
                if not _gpflow_available():
                    raise RuntimeError(f"{self.name}: training needs gpflow and tensorflow, which are not importable; pass "
                                       "hyperparameters= (lengthscales, variance, likelihood_variance) to predict without them")
                fit = "reference"
            if fit != "reference":
                raise ValueError(f"{self.name}: fit must be 'reference' or None (got {fit!r})")
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
        self._upload(dict(Z=Z, variance=var, lengthscales=ls, q_mu=q_mu, q_sqrt=q_sqrt, W=W), JITTER)

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
