"""NumPy restatement of the two sensitivity-analysis methods dmosopt registers (``dmosopt/config.py`` default_sa_methods):
DGSM (derivative-based global sensitivity measures on a forward-difference Sobol design) and eFAST (extended Fourier
amplitude sensitivity test), as SALib 1.5 defines them.  SALib is neither installed nor vendored, so parity with it is
unpinned; the definitions below are the ones ``dmosopt_b200/sa.py`` and ``csrc/sa.cu`` follow.

Every random draw (the eFAST phases, the DGSM bootstrap indices) is an argument, so a device result can be replayed.
"""

import math

import numpy as np

DGSM_SKIP = 1024  # Sobol points skipped before the base points
DGSM_DELTA = 0.01  # forward-difference step in the unit cube
FAST_M = 4  # eFAST interference factor

# Cody-Waite split of pi/2 (fdlibm's pio2_1, pio2_2, pio2_2t): P1 and P2 carry 33 significant bits each, so n * P1 and
# n * P2 are exact for n < 2^20; P3 is the remainder rounded to a double
_PIO2_1 = 1.57079632673412561417e00
_PIO2_2 = 6.07710050630396597660e-11
_PIO2_3 = 2.02226624879595063154e-21
_TWO_OVER_PI = 6.36619772367581382433e-01
_PIO2 = math.pi / 2
_INV_PI = 1 / math.pi


def dgsm_base(N, d):
    """(N, d) base points: unscrambled Sobol after skipping DGSM_SKIP points."""
    import warnings

    from scipy.stats import qmc

    s = qmc.Sobol(d, scramble=False)
    s.fast_forward(DGSM_SKIP)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # "balance properties" warning for N not a power of two
        return s.random(N)


def dgsm_design(B, lb, ub, delta=DGSM_DELTA):
    """(N (d+1), d): row i(d+1) is B_i, row i(d+1)+1+j is B_i + delta e_j, every row scaled to lb + u (ub - lb)."""
    B = np.asarray(B, dtype=np.float64)
    N, d = B.shape
    lb, ub = np.asarray(lb, dtype=np.float64), np.asarray(ub, dtype=np.float64)
    U = np.repeat(B, d + 1, axis=0).reshape(N, d + 1, d)
    j = np.arange(d)
    U[:, 1 + j, j] += delta
    return (U * (ub - lb) + lb).reshape(N * (d + 1), d)


def dgsm_stats(X, Y, lb, ub, idx, conf_level=0.95):
    """vi, vi_std, dgsm, conf, each (M, d), from the design X (N (d+1), d), its outputs Y (N (d+1), M) and the bootstrap
    base indices idx (R, N): conf = z_{(1+c)/2} * std(ddof=1) of dgsm over the R resampled base sets."""
    from scipy.stats import norm

    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    d = X.shape[1]
    N = X.shape[0] // (d + 1)
    M = Y.shape[1]
    rng_ = np.asarray(ub, dtype=np.float64) - np.asarray(lb, dtype=np.float64)
    Xr = X.reshape(N, d + 1, d)
    Yr = Y.reshape(N, d + 1, M)
    z = norm.ppf(0.5 + conf_level / 2)
    out = {k: np.empty((M, d)) for k in ("vi", "vi_std", "dgsm", "conf")}
    for j in range(d):
        dx = Xr[:, 1 + j, j] - Xr[:, 0, j]
        for m in range(M):
            yb = Yr[:, 0, m]
            q2 = ((Yr[:, 1 + j, m] - yb) / dx) ** 2
            vi = np.mean(q2)
            out["vi"][m, j], out["vi_std"][m, j] = vi, np.std(q2)
            out["dgsm"][m, j] = vi * rng_[j] ** 2 / (np.var(yb) * np.pi**2)
            s = np.mean(q2[idx], axis=1) * rng_[j] ** 2 / (np.var(yb[idx], axis=1) * np.pi**2)  # one replicate per row of idx
            out["conf"][m, j] = z * s.std(ddof=1)
    return out


def fast_frequencies(N, d, M=FAST_M):
    """(d,) eFAST frequencies: omega_0 for the parameter of interest, then the complementary set."""
    if N <= 4 * M**2:
        raise ValueError(f"eFAST needs N > 4 M^2 = {4 * M * M} samples (got N={N})")
    omega = np.zeros(d)
    omega[0] = math.floor((N - 1) / (2 * M))
    m = math.floor(omega[0] / (2 * M))
    if m >= d - 1:
        omega[1:] = np.floor(np.linspace(1, m, d - 1))
    else:
        omega[1:] = np.arange(d - 1) % m + 1
    return omega


def triangle(theta):
    """arcsin(sin(theta)) for 0 <= theta < 2^20 pi/2, by exact reduction to n pi/2 + r: r, pi/2 - |r|, -r, |r| - pi/2
    for n = 0, 1, 2, 3 mod 4.  The composition arcsin(sin(.)) evaluated as written is ill-conditioned next to the peaks
    (a last-bit error in sin near +-1 moves arcsin by up to ~1e-8); this form is accurate to about an ulp everywhere."""
    theta = np.asarray(theta, dtype=np.float64)
    n = np.rint(theta * _TWO_OVER_PI)
    r = ((theta - n * _PIO2_1) - n * _PIO2_2) - n * _PIO2_3
    q = n.astype(np.int64) & 3
    a = np.abs(r)
    return np.select([q == 0, q == 1, q == 2], [r, _PIO2 - a, -r], a - _PIO2)


def fast_design(N, omega, phi, lb, ub):
    """(N d, d) eFAST design: block i gives parameter i omega_0 and the others omega_1.. in order; column j of block i
    is 0.5 + arcsin(sin(omega_j s_k + phi_i)) / pi, s_k = 2 pi k / N, scaled to lb + x (ub - lb)."""
    omega = np.asarray(omega, dtype=np.float64)
    d = omega.shape[0]
    lb, ub = np.asarray(lb, dtype=np.float64), np.asarray(ub, dtype=np.float64)
    s = (2 * math.pi / N) * np.arange(N)
    X = np.empty((N * d, d))
    for i in range(d):
        w = np.empty(d)
        w[i] = omega[0]
        w[np.arange(d) != i] = omega[1:]
        x = 0.5 + _INV_PI * triangle(w[None, :] * s[:, None] + phi[i])
        X[i * N : (i + 1) * N] = x * (ub - lb) + lb
    return X


def fast_indices(Y, N, d, M=FAST_M):
    """(S1, ST), each (M_out, d), of the eFAST design's outputs Y (N d, M_out)."""
    Y = np.asarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    omega0 = math.floor((N - 1) / (2 * M))
    S1 = np.empty((Y.shape[1], d))
    ST = np.empty((Y.shape[1], d))
    for m in range(Y.shape[1]):
        for i in range(d):
            f = np.fft.fft(Y[i * N : (i + 1) * N, m])
            Sp = np.power(np.absolute(f[np.arange(1, math.ceil(N / 2))]) / N, 2)
            V = 2 * np.sum(Sp)
            D1 = 2 * np.sum(Sp[np.arange(1, M + 1) * int(omega0) - 1])
            Dt = 2 * np.sum(Sp[np.arange(math.floor(omega0 / 2))])
            S1[m, i], ST[m, i] = D1 / V, 1 - Dt / V
    return S1, ST
