"""Oracle: WFG1 and the many-objective MaF problems, vectorised over rows (test infrastructure only, see oracle/__init__.py).

Restates dmosopt/benchmarks/moo_benchmarks.py wfg1 :286-332, maf1 :384-419, maf2 :422-457 and maf4 :460-497 next to
the DTLZ / WFG4 / ZDT restatements of oracle/benchmarks.py; pinned to the reference by tests/golden/benchmarks.npz (rows
evaluated one at a time by the reference itself).
"""

import numpy as np

from .benchmarks import _g_sphere, _product_form


def wfg1(X, M=3):
    """Raises ValueError, as the reference does, where a maximum window is empty ((M - 2) (d - M + 1) >= d)."""
    X = np.atleast_2d(X)
    d = X.shape[1]
    k = M - 1
    ll = d - k
    y = X / (2 * np.arange(1, d + 1))
    t2 = y.copy()
    with np.errstate(invalid="ignore"):  # y < 0 (y ** 0.02) and infinite y (cos, sin) give nan in the reference as well
        t2[:, k:] = 0.35 + 0.65 * y[:, k:] ** 0.02
        xv = np.empty((X.shape[0], M))
        for i in range(M - 1):
            xv[:, i] = np.max(t2[:, i * ll : (i + 1) * ll], axis=1)
        xv[:, -1] = np.mean(t2[:, -ll:], axis=1)
        f = _product_form(xv, M, 1.0, lambda v: 1 - np.cos(v * np.pi / 2), lambda v: 1 - np.sin(v * np.pi / 2))
    return f * (1 + np.arange(1, M + 1))


def maf1(X, M=5):
    X = np.atleast_2d(X)
    xm = X[:, -(X.shape[1] - M + 1) :] - 0.5
    g = np.sum(xm**2 - np.cos(20 * np.pi * xm), axis=1)
    return _product_form(X, M, 1 + g, lambda v: v, lambda v: 1 - v)


def maf2(X, M=5):
    X = np.atleast_2d(X)
    return _product_form(X, M, 1 + _g_sphere(X, M), lambda v: np.cos(v * np.pi / 2), lambda v: np.sin(v * np.pi / 2))


def maf4(X, M=5):
    # the reference multiplies by the Python int 10 ** (2 i); float() of it is the correctly rounded double
    return maf2(X, M) * np.array([float(10 ** (2 * i)) for i in range(M)])
