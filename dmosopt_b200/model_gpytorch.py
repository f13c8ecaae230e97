"""gpytorch exact-GP surrogate on the GPU path: ``EGP_Matern`` (row A19).

Drop-in for ``dmosopt.model_gpytorch.EGP_Matern`` (dmosopt/model_gpytorch.py:1927-2235), selected in dmosopt by
``surrogate_method_name="dmosopt_b200.model_gpytorch.EGP_Matern"``.  As with the scikit-learn surrogates, *fitting*
stays with the host library -- here the reference class itself, which needs gpytorch -- and only the posterior is
taken over: after training, the hyper-parameters (ARD length scales, output scale, noise, linear-mean weights / bias)
and the model's own normalised training tensors are read out, K + sigma^2 I is factorised once in float64, and every
``predict`` / ``evaluate`` runs on the GPU through ``dmo_gp_create`` / ``dmo_gp_set_linear_mean`` / ``dmo_gp_predict``.

The predictive variance is the exact one (gpytorch's ``fast_pred_var=False``); the reference's default
``fast_pred_var=True`` (LOVE) is a low-rank approximation of it.  gpytorch is not part of this image, so the
extraction from a trained gpytorch model is untested here; the posterior arithmetic is tested against oracle/egp.py
through the ``hyperparameters=`` constructor path (tests/test_gpu_parity.py::test_egp_linear_mean_*).

``MEGP_Matern`` (multitask Kronecker model, model_gpytorch.py:1872-1919) couples the objectives in one (N*M) x (N*M)
system and is not covered.
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
    def __init__(self, xin, yin, nInput, nOutput, xlb, xub, return_mean_variance=False, logger=None, precision="fp64",
                 hyperparameters=None, **kwargs):
        self.nInput, self.nOutput = nInput, nOutput
        self.xlb = np.asarray(xlb, dtype=np.float64)
        xub = np.asarray(xub, dtype=np.float64)
        self.xrng = np.where(np.isclose(xub - self.xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - self.xlb)  # model_gpytorch.py:1965-1967
        self.return_mean_variance = return_mean_variance
        self.logger = logger
        self.precision = _lib.GP_TENSOR if precision in ("tensor", _lib.GP_TENSOR) else _lib.GP_FP64
        self.stats = {}
        if hyperparameters is None:
            xn, yn, ymean, ystd, hyperparameters = self._fit_with_reference(xin, yin, nInput, nOutput, xlb, xub, logger, kwargs)
        else:
            xin = np.asarray(xin, dtype=np.float64)
            yin = np.asarray(yin, dtype=np.float64)
            if yin.ndim == 1:
                yin = yin.reshape(-1, 1)
            xn = (xin - self.xlb) / self.xrng
            ymean = yin.mean(axis=0)
            ystd = yin.std(axis=0)
            ystd = np.where(ystd == 0.0, 1.0, ystd)  # handle_zeros_in_scale, model_gpytorch.py:1995-2001
            yn = (yin - ymean) / ystd
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
