"""Sensitivity analysis without SALib: drop-ins for dmosopt's ``default_sa_methods`` (``dmosopt/sa.py``).

    sensitivity_method_name="dmosopt_b200.sa.SA_DGSM"     # or "dmosopt_b200.sa.SA_FAST"

``MOASMO.analyze_sensitivity`` resolves the name with ``import_object_by_path``, constructs the class with
``(xlb, xub, param_names, objective_names)`` and calls ``analyze(model)``; the result becomes the per-dimension
``di_mutation`` / ``di_crossover`` of the optimizer.  Both classes keep the reference's constructor, ``sample`` and
``analyze`` and follow SALib 1.5's definitions (restated in ``oracle/sa.py``; SALib itself is not needed):

* ``SA_DGSM``: derivative-based global sensitivity measures on the forward-difference design around unscrambled Sobol
  base points (1024 skipped, delta 0.01 of the range).  ``analyze`` returns ``{"S1": {output: dgsm (d,)}}``;
  ``statistics`` also gives vi, vi_std and the bootstrap confidence (100 replicates, 95 %).
* ``SA_FAST``: extended FAST with interference factor 4 (``num_samples`` > 64).  ``analyze`` returns
  ``{"S1": ..., "ST": ...}``.

The designs are built on the GPU into page-locked host arrays that keep a device copy, so the surrogates of this
package predict them without uploading them; any other model's ``evaluate`` sees an ordinary read-only NumPy array.
``analyze`` asks nothing of the model but ``evaluate(X)``; a ``(mean, variance)`` pair is reduced to its mean.  The DGSM
statistics run on the GPU; the eFAST spectra (d M transforms of length N) stay in ``numpy.fft``.

The random draws (eFAST phases, DGSM bootstrap indices) come from ``numpy.random.default_rng(seed)``; ``seed`` is an
extra keyword (an int, a Generator or None).
"""

import math
import warnings

import numpy as np

from . import _lib


class _SensitivityMethod:
    def __init__(self, lo_bounds, hi_bounds, param_names, output_names, logger=None, seed=None):
        self.xlb = np.asarray(lo_bounds, dtype=np.float64).reshape(-1)
        self.xub = np.asarray(hi_bounds, dtype=np.float64).reshape(-1)
        if self.xlb.shape != (len(param_names),) or self.xub.shape != (len(param_names),):
            raise ValueError(f"{type(self).__name__}: {len(param_names)} parameter names but bounds of {self.xlb.shape[0]} and {self.xub.shape[0]} entries")
        self.problem = {"num_vars": len(param_names), "names": list(param_names), "bounds": list(zip(self.xlb, self.xub))}
        self.output_names = list(output_names)
        self.logger = logger
        self.rng = seed if isinstance(seed, np.random.Generator) else np.random.default_rng(seed)

    def _evaluate(self, model, X):
        Y = model.evaluate(X)
        if isinstance(Y, tuple):  # return_mean_variance
            Y = Y[0]
        Y = np.asarray(Y, dtype=np.float64)
        if Y.ndim == 1:
            Y = Y[:, None]
        if Y.shape != (X.shape[0], len(self.output_names)):
            raise ValueError(f"{type(self).__name__}: model.evaluate returned shape {Y.shape} for {X.shape[0]} rows and "
                             f"{len(self.output_names)} outputs")
        return Y


class SA_DGSM(_SensitivityMethod):
    """DGSM (SALib 1.5 ``finite_diff.sample`` + ``dgsm.analyze``) with the design and the statistics on the GPU."""

    skip = 1024
    delta = 0.01
    num_resamples = 100
    conf_level = 0.95

    def base_points(self, num_samples):
        from scipy.stats import qmc

        s = qmc.Sobol(self.problem["num_vars"], scramble=False)
        s.fast_forward(self.skip)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # scipy warns when N is not a power of two
            return s.random(int(num_samples))

    def sample(self, num_samples=10000):
        """(N (d+1), d) read-only design: each base point followed by its d forward-difference neighbours."""
        return _lib.sa_dgsm_design(self.base_points(num_samples), self.xlb, self.xub, self.delta)

    def statistics(self, X, Y):
        """{vi, vi_std, dgsm, conf}, each (M, d), of the design X and its outputs Y (N (d+1), M); draws the bootstrap
        indices (num_resamples, N) from ``self.rng``."""
        N = X.shape[0] // (X.shape[1] + 1)
        idx = self.rng.integers(0, N, size=(self.num_resamples, N), dtype=np.int32)
        return _lib.sa_dgsm_stats(X, Y, self.xlb, self.xub, idx, self.conf_level)

    def analyze(self, model, num_samples=10000):
        X = self.sample(num_samples)
        try:
            st = self.statistics(X, self._evaluate(model, X))
        finally:
            _lib.mirror_drop(X)  # release the design's device copy now rather than when X is collected
        return {"S1": dict(zip(self.output_names, st["dgsm"]))}


class SA_FAST(_SensitivityMethod):
    """eFAST (SALib 1.5 ``fast_sampler.sample`` + ``fast.analyze``, M = 4) with the design on the GPU."""

    M = 4

    def frequencies(self, N):
        """(d,) frequencies: omega_0 for the parameter of a block, then the complementary set in order."""
        d, M = self.problem["num_vars"], self.M
        if N <= 4 * M**2:
            raise ValueError(f"SA_FAST: the sample size must exceed 4 M^2 = {4 * M * M} (got num_samples={N})")
        omega = np.zeros(d)
        omega[0] = math.floor((N - 1) / (2 * M))
        m = math.floor(omega[0] / (2 * M))
        if m >= d - 1:
            omega[1:] = np.floor(np.linspace(1, m, d - 1))
        else:
            omega[1:] = np.arange(d - 1) % m + 1
        return omega

    def sample(self, num_samples=10000):
        """(N d, d) read-only design; one random phase per block, drawn from ``self.rng``."""
        N = int(num_samples)
        omega = self.frequencies(N)
        phi = 2 * math.pi * self.rng.random(self.problem["num_vars"])
        return _lib.sa_fast_design(N, omega, phi, self.xlb, self.xub)

    def indices(self, Y, N):
        """(S1, ST), each (M_out, d), from the outputs Y (N d, M_out) of the design."""
        d, M = self.problem["num_vars"], self.M
        omega0 = math.floor((N - 1) / (2 * M))
        f = np.fft.rfft(Y.reshape(d, N, -1), axis=1)
        Sp = (np.abs(f[:, 1 : math.ceil(N / 2)]) / N) ** 2  # (d, ceil(N/2) - 1, M_out)
        V = 2 * Sp.sum(axis=1)
        D1 = 2 * Sp[:, np.arange(1, M + 1) * omega0 - 1].sum(axis=1)
        Dt = 2 * Sp[:, : math.floor(omega0 / 2)].sum(axis=1)
        return (D1 / V).T, (1 - Dt / V).T

    def analyze(self, model, num_samples=10000):
        X = self.sample(num_samples)
        try:
            Y = self._evaluate(model, X)
        finally:
            _lib.mirror_drop(X)
        S1, ST = self.indices(Y, int(num_samples))
        return {"S1": dict(zip(self.output_names, S1)), "ST": dict(zip(self.output_names, ST))}
