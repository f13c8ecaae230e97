"""Exact-GP surrogates on the GPU path: drop-ins for ``dmosopt.model.GPR_Matern`` / ``GPR_RBF``.

Reference: dmosopt/model.py:1182-1275 (GPR_Matern) and :1278-1364 (GPR_RBF); selected in dmosopt by
``surrogate_method_name="dmosopt_b200.GPR_Matern"`` (dmosopt/MOASMO.py:516-530).  The constructor
signature, ``predict`` / ``evaluate`` and the ``return_mean_variance`` switch are the reference's.

Scope (SURVEY.md section 8a row A18 / section 2 row 12): the per-generation call -- ``predict`` -- runs on the GPU
(dmo_gp_predict).  The once-per-epoch fit (section 8f row N1) runs on the GPU as well (``fit="gpu"``, the default): for
given hyper-parameters the kernel matrix, its Cholesky factor, alpha and the log marginal likelihood come from
dmo_gp_fit (csrc/gp_fit.cu); with ``optimizer="sceua"`` the reference's SCE-UA search (dmosopt/model.py:1419-1753, used
when dmosopt is importable; a bounded derivative-free SciPy search otherwise) drives that evaluation instead of
scikit-learn's host Cholesky; ``optimizer=None`` keeps the initial theta (the BASELINE.md configuration).
``fit="sklearn"`` is the previous behaviour: scikit-learn's ``GaussianProcessRegressor.fit`` on the host.  Either way the
result is a list of scikit-learn regressors (``smlist``, as the reference keeps) whose posterior state is uploaded once.
"""

import numpy as np

from . import _lib


def _filter_nan_rows(y, x):
    mask = ~np.any(np.isnan(y), axis=1)
    return y[mask], x[mask]


def _host_optimizer(optimizer, seed, logger):
    """sklearn ``optimizer=`` argument for the requested method (fit-time only)."""
    if optimizer is None:
        return None
    try:  # the reference's optimisers, when dmosopt itself is installed next to this package
        from functools import partial

        from dmosopt.model import dlib_optimizer, sceua_optimizer

        if optimizer == "dlib":
            return partial(dlib_optimizer, logger)
        return partial(sceua_optimizer, seed, logger)
    except Exception:
        if logger is not None:
            logger.warning("dmosopt_b200: dmosopt.model optimisers unavailable, fitting with scikit-learn's L-BFGS-B")
        return "fmin_l_bfgs_b"


class _GPRBase:
    _kernel_code = _lib.KERNEL_MATERN52
    _default_noise = 1e-6
    _name = "GPR_Matern"

    def __init__(
        self,
        xin,
        yin,
        nInput,
        nOutput,
        xlb,
        xub,
        optimizer="sceua",
        seed=None,
        length_scale_bounds=(1e-3, 100.0),
        constant_kernel_bounds=(1e-4, 1e3),
        noise_level_bounds=(1e-9, 1e-2),
        anisotropic=False,
        return_mean_variance=False,
        nan="remove",
        top_k=None,
        logger=None,
        precision="auto",
        fit="gpu",
        **kwargs,
    ):
        from sklearn.gaussian_process import GaussianProcessRegressor
        from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

        self.nInput = nInput
        self.nOutput = nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        self.xub = np.asarray(xub, dtype=np.float64)
        self.xrg = self.xub - self.xlb
        self.logger = logger
        self.return_mean_variance = return_mean_variance
        # "auto" (default): the tensor-core path wherever a per-model calibration against the float64 path holds the
        # 1e-5 bar, float64 for the rest (csrc/gp.cu, DMO_GP_AUTO); "tensor" / "fp64" force one arithmetic
        codes = {"auto": _lib.GP_AUTO, "tensor": _lib.GP_TENSOR, "fp64": _lib.GP_FP64,
                 _lib.GP_AUTO: _lib.GP_AUTO, _lib.GP_TENSOR: _lib.GP_TENSOR, _lib.GP_FP64: _lib.GP_FP64}
        if precision not in codes:
            raise ValueError(f"{self._name}: precision must be 'auto', 'tensor' or 'fp64' (got {precision!r})")
        self.precision = codes[precision]
        self.stats = {}

        xin = np.asarray(xin, dtype=np.float64)
        yin = np.asarray(yin, dtype=np.float64)
        if yin.ndim == 1:
            yin = yin.reshape(-1, 1)
        if nan is not None and self._name == "GPR_Matern":  # model.py:1209-1210
            yin, xin = _filter_nan_rows(yin, xin)
        if isinstance(top_k, int) and xin.shape[0] > top_k:  # model.py:1212, MOEA.top_k_MO
            from .MOEA import sortMO

            xs, ys, *_ = sortMO(xin, yin)
            xin, yin = xs[:top_k], ys[:top_k]

        x = (xin - self.xlb) / self.xrg  # model.py:1217-1218
        y = np.nan_to_num(np.copy(yin))
        length_scale = np.asarray([0.5] * nInput) if anisotropic else 0.5
        if self._kernel_code == _lib.KERNEL_MATERN52:
            stationary = Matern(length_scale=length_scale, length_scale_bounds=length_scale_bounds, nu=2.5)
        else:
            stationary = RBF(length_scale=length_scale, length_scale_bounds=length_scale_bounds)
        kernel = ConstantKernel(1, constant_kernel_bounds) * stationary + WhiteKernel(
            noise_level=self._default_noise, noise_level_bounds=noise_level_bounds
        )
        if fit not in ("gpu", "sklearn"):
            raise ValueError(f"{self._name}: fit must be 'gpu' or 'sklearn' (got {fit!r})")
        optf = _host_optimizer(optimizer, seed, logger)
        if fit == "gpu":
            self.smlist = self._fit_on_gpu(kernel, optf, x, y, logger)
        else:
            smlist = []
            for i in range(nOutput):
                if logger is not None:
                    logger.info(f"{self._name}: creating regressor for output {i + 1} of {nOutput}...")
                gpr = GaussianProcessRegressor(kernel=kernel, optimizer=optf, normalize_y=True)
                gpr.fit(x, y[:, i])
                smlist.append(gpr)
            self.smlist = smlist
        self._upload()

    def _fit_on_gpu(self, kernel, optf, x, y, logger):
        """GaussianProcessRegressor.fit restated around dmo_gp_fit (sklearn/gaussian_process/_gpr.py:fit): targets are
        normalised per output, theta = log(constant, length scale(s), noise) is either kept or searched by the optimiser
        with -log marginal likelihood evaluated on the GPU, and the final Cholesky factor / alpha of every output come from
        one batched call.  Returns scikit-learn regressors carrying that state (their own predict works on it)."""
        from sklearn.gaussian_process import GaussianProcessRegressor

        M, d = self.nOutput, self.nInput
        y_mean = np.mean(y, axis=0)
        y_std = np.std(y, axis=0)
        y_std = np.where(y_std < 10 * np.finfo(np.float64).eps, 1.0, y_std)  # sklearn _handle_zeros_in_scale
        yn = ((y - y_mean) / y_std).T.copy()  # (M, N)
        jitter = 1e-10  # GaussianProcessRegressor(alpha=1e-10)

        def unpack(theta):
            v = np.exp(np.asarray(theta, dtype=np.float64))
            return v[0], v[1:-1], v[-1]  # constant, length scale(s), noise

        thetas = []
        for i in range(M):
            theta = np.array(kernel.theta, dtype=np.float64)
            if optf is not None:
                if logger is not None:
                    logger.info(f"{self._name}: optimising the hyper-parameters of output {i + 1} of {M} (likelihood on the GPU)...")

                def obj_func(th, eval_gradient=False, _i=i):
                    c, ls, nz = unpack(th)
                    try:
                        _, _, lml = _lib.gp_fit(x, yn[_i : _i + 1], [c], [np.broadcast_to(ls, (d,))], [nz], kernel=self._kernel_code, jitter=jitter,
                                                want_L=False, want_alpha=False)
                        val = -float(lml[0])
                    except _lib.DmoError:  # not positive definite at this theta: what sklearn maps to -inf likelihood
                        val = np.inf
                    return val, None

                if callable(optf):
                    theta, _ = optf(obj_func, theta, kernel.bounds)
                else:  # "fmin_l_bfgs_b" has no gradient here: bounded derivative-free search instead
                    from scipy.optimize import minimize

                    res = minimize(lambda th: obj_func(th)[0], theta, method="Powell", bounds=kernel.bounds, options={"xtol": 1e-3, "ftol": 1e-6})
                    theta = res.x
            thetas.append(np.asarray(theta, dtype=np.float64))
        cs, lss, nzs = zip(*[unpack(t) for t in thetas])
        L, alpha, lml = _lib.gp_fit(x, yn, list(cs), [np.broadcast_to(ls, (d,)) for ls in lss], list(nzs), kernel=self._kernel_code, jitter=jitter)
        smlist = []
        for i in range(M):
            gpr = GaussianProcessRegressor(kernel=kernel, optimizer=None, normalize_y=True)
            gpr.kernel_ = kernel.clone_with_theta(thetas[i])
            gpr.X_train_, gpr.y_train_ = x, yn[i]
            gpr._y_train_mean, gpr._y_train_std = y_mean[i], y_std[i]
            gpr.alpha_, gpr.L_ = alpha[i], L[i]
            gpr.log_marginal_likelihood_value_ = float(lml[i])
            gpr.n_features_in_ = d
            gpr._rng = None
            smlist.append(gpr)
        return smlist

    def _upload(self):
        """Posterior state of every objective -> HBM (dmo_gp_create), once per epoch."""
        sm = self.smlist
        d = self.nInput
        self._gp = _lib.GPHandle(
            X_train=np.asarray(sm[0].X_train_, dtype=np.float64),
            alpha=np.stack([np.ravel(g.alpha_) for g in sm]),
            factor=np.stack([np.asarray(g.L_, dtype=np.float64) for g in sm]),  # L^-1 is formed on the GPU
            constant=[g.kernel_.k1.k1.constant_value for g in sm],
            length_scale=[np.broadcast_to(np.asarray(g.kernel_.k1.k2.length_scale, dtype=np.float64), (d,)) for g in sm],
            noise=[g.kernel_.k2.noise_level for g in sm],
            y_mean=[np.ravel(g._y_train_mean)[0] for g in sm],
            y_std=[np.ravel(g._y_train_std)[0] for g in sm],
            xlb=self.xlb,
            xub=self.xub,
            kernel=self._kernel_code,
            factor_is_inverse=False,
        )

    def predict(self, xin):
        """model.py:1254-1268: (mean (P, M), variance (P, M))."""
        xin = np.asarray(xin, dtype=np.float64)
        if xin.ndim == 1:
            xin = xin.reshape((1, self.nInput))
        return self._gp.predict(xin, return_var=True, precision=self.precision)

    def evaluate(self, x):
        """model.py:1270-1275."""
        if self.return_mean_variance:
            return self.predict(x)
        x = np.asarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x.reshape((1, self.nInput))
        mean, _ = self._gp.predict(x, return_var=False, precision=self.precision)
        return mean


class GPR_Matern(_GPRBase):
    _kernel_code = _lib.KERNEL_MATERN52
    _default_noise = 1e-6
    _name = "GPR_Matern"


class GPR_RBF(_GPRBase):
    _kernel_code = _lib.KERNEL_RBF
    _default_noise = 1e-5
    _name = "GPR_RBF"


class Model:
    """dmosopt.model.Model (dmosopt/model.py:70-95): container handed to the optimizers."""

    def __init__(self, return_mean_variance=False, objective=None, feasibility=None, sensitivity=None, **kwargs):
        self.objective = objective
        self.feasibility = feasibility
        self.sensitivity = sensitivity
        self.stats = {}
        self.return_mean_variance = return_mean_variance

    def get_stats(self):
        for part in (self.objective, self.feasibility, self.sensitivity):
            if part is not None:
                self.stats.update(getattr(part, "stats", {}))
        return self.stats.copy()
