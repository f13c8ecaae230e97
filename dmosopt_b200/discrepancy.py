"""Uniformity scores of a design (dmosopt/discrepancy.py): the L2 discrepancies on the GPU, the other two in NumPy.

Same names and return values as the reference: ``MD2`` (modified), ``CD2`` (centred), ``SD2`` (symmetric) and ``WD2``
(wrap-around) L2 discrepancies [Hickernell 1998], ``MinDist``, ``corrscore`` and ``all``.

Each discrepancy is sqrt(D1 + c2 D2 + c3 D3), where D2 sums a product over the s coordinates of each row and D3 sums a
product over the s coordinates of every ordered pair of rows (n^2 s terms).  The GPU (``dmo_l2_discrepancy_terms``)
sums D2 and D3 in a fixed blocked order, so results repeat bit for bit, but the order is not the reference's.  The
terms cancel heavily at large s (D^2 is a small difference of numbers near (4/3)^s or (13/12)^s), so the agreement is
stated on D^2: |D^2 - D^2_ref| <= ``d2_bound(...)``, derived as in ``sampling.screen_margin``.

Two behaviours of the reference are kept as they are:

* ``MinDist`` takes its minimum over j >= i, which includes the zero distance of every row to itself, so it returns
  0.0 for every design with a finite row (1e32 for an empty one);
* ``corrscore`` is the sum of squared upper-triangle entries of ``np.corrcoef(X)``, which correlates the rows, not the
  columns.
"""

import math

import numpy as np

from . import _lib

_U = 2.0**-53


def _terms(X, metric):
    X = np.asarray(X, dtype=np.float64)
    n, s = X.shape
    D2, D3 = _lib.l2_discrepancy_terms(X, metric)
    return n, s, D2, D3


def d2_bound(n, s, *magnitudes):
    """Bound on |D^2 - D^2_ref| given the magnitudes of the three terms of D^2: each side is within
    (n^2 + 7 s + 4) u (|D1| + |c2 D2| + |c3 D3|) of the exact value (sequential sums of n^2 positive products of s
    factors, each factor a few roundings); doubled for the two sides, with 1.01 for second-order terms."""
    return 2.02 * (float(n) * n + 7.0 * s + 4.0) * _U * sum(abs(m) for m in magnitudes)


def MD2(X):
    """Modified L2-discrepancy."""
    n, s, D2, D3 = _terms(X, "MD2")
    return math.sqrt((4.0 / 3.0) ** s + D2 * (-(2 ** (1 - s)) / float(n)) + D3 / (n**2))


def CD2(X):
    """Centred L2-discrepancy."""
    n, s, D2, D3 = _terms(X, "CD2")
    return math.sqrt((13.0 / 12.0) ** s + D2 * (-2.0 / n) + D3 / (n**2))


def SD2(X):
    """Symmetric L2-discrepancy."""
    n, s, D2, D3 = _terms(X, "SD2")
    return math.sqrt((4.0 / 3.0) ** s + D2 * (-2.0 / n) + D3 * ((2**s) / float(n**2)))


def WD2(X):
    """Wrap-around L2-discrepancy."""
    n, s, _, D3 = _terms(X, "WD2")
    return math.sqrt(-((4.0 / 3.0) ** s) + D3 / (n**2))


def MinDist(X):
    """Minimum of the distances |X_i - X_j| over j >= i, starting from 1e32 (see the module docstring: 0.0 whenever a
    row is finite, since j = i is included)."""
    X = np.asarray(X)
    best = 1.0e32
    for i in range(X.shape[0]):
        d = np.sqrt(np.sum((X[i] - X[i:]) ** 2, axis=1))
        d = d[~np.isnan(d)]
        if d.size:
            best = min(best, float(d.min()))
    return best


def corrscore(X):
    """Sum of squared correlations above the diagonal of ``np.corrcoef(X)`` (between rows, as the reference has it)."""
    return np.sum(np.triu(np.corrcoef(X), 1) ** 2)


def all(X):
    """Every score, printed and returned as a dict keyed by name."""
    r = {"MD2": MD2(X), "CD2": CD2(X), "SD2": SD2(X), "WD2": WD2(X), "MinDist": MinDist(X), "corrscore": corrscore(X)}
    for k, v in r.items():
        print(f"The result of {k} is: {v}")
    return r
