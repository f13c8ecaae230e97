"""NumPy restatement of the good-lattice-point search and the L2 discrepancies (dmosopt/GLP.py, discrepancy.py).

The discrepancies here keep the reference's operation order, vectorised over rows or row pairs: per-element factors
rounded one operation at a time, products taken over the coordinates in order from 1.0, and sums taken sequentially
(``np.cumsum``) over rows, or over row pairs in row-major order.  Scalar ``a ** 2`` terms go through NumPy float64
scalars as in the reference (the C library's pow, which is not always a * a).  So ``cd2`` equals the reference's CD2
bit for bit, at sizes the reference's Python loops cannot finish.
"""

import itertools
import math

import numpy as np


def _sq_scalar(A):
    """Elementwise a ** 2 evaluated on NumPy float64 scalars."""
    A = np.asarray(A, dtype=np.float64)
    return np.array([np.float64(a) ** 2 for a in A.ravel()]).reshape(A.shape)


def euler(n):
    """The reference's float totient: n prod (1 - 1/p) over distinct primes, truncated."""
    primes, m, f = [], n, 2
    while f < m:
        while m % f == 0:
            primes.append(f)
            m //= f
        f += 1
    if m > 1:
        primes.append(m)
    phi = n * (1 - 1.0 / primes[0])
    for a, b in zip(primes, primes[1:]):
        if b != a:
            phi *= 1 - 1.0 / b
    return int(phi)


def candidates(n, s):
    """(lattice, rows, H (C, s)) in the reference's order; powers with Python integers, as the reference forms them."""
    m = euler(n)
    plusone = m / n < 0.9
    N = n + 1 if plusone else n
    units = [i for i in range(N) if math.gcd(i, N) == 1]
    if m < 20 and s < 4:
        mm = euler(N) if plusone else m
        H = [[units[c] for c in comb] for comb in itertools.combinations(range(mm), s)]
    else:
        H = []
        for a in units:
            if a < 2:
                continue
            pw = sorted((a**t) % N for t in range(1, s))
            if pw[0] != 1 and all(pw[i] != pw[i - 1] for i in range(1, len(pw))):
                H.append([(a**t) % N for t in range(s)])
    return N, N - 1 if plusone else N, np.array(H, dtype=np.int64).reshape(-1, s)


def design(h, N, rows):
    u = np.mod(np.arange(1, rows + 1)[:, None] * np.asarray(h, dtype=np.int64)[None, :], N).astype(np.float64)
    u[u == 0] = N
    return (u - 0.5) / rows


def _pair_sum(X, factor):
    """Sequential row-major sum over (k, j) of prod_i factor(X[k, i], X[j, i])."""
    n, s = X.shape
    P = np.ones((n, n))
    for i in range(s):
        P = P * factor(X[:, i][:, None], X[:, i][None, :])
    return np.cumsum(P.ravel())[-1]


def _row_sum(F):
    """Sequential sum over rows of prod_i F[k, i]."""
    p = np.ones(F.shape[0])
    for i in range(F.shape[1]):
        p = p * F[:, i]
    return np.cumsum(p)[-1]


def cd2_terms(X):
    X = np.asarray(X, dtype=np.float64)
    A = np.abs(X - 0.5)
    D2 = _row_sum(1 + 0.5 * A - 0.5 * _sq_scalar(A))
    D3 = _pair_sum(X, lambda x, y: 1 + 0.5 * np.abs(x - 0.5) + 0.5 * np.abs(y - 0.5) - 0.5 * np.abs(x - y))
    return D2, D3


def cd2(X):
    n, s = np.shape(X)
    D2, D3 = cd2_terms(X)
    return math.sqrt((13.0 / 12.0) ** s + D2 * (-2.0 / n) + D3 / (n**2))


def md2(X):
    X = np.asarray(X, dtype=np.float64)
    n, s = X.shape
    D2 = _row_sum(3 - _sq_scalar(X))
    D3 = _pair_sum(X, lambda x, y: 2 - np.maximum(x, y))
    return math.sqrt((4.0 / 3.0) ** s + D2 * (-(2 ** (1 - s)) / float(n)) + D3 / (n**2))


def sd2(X):
    X = np.asarray(X, dtype=np.float64)
    n, s = X.shape
    D2 = _row_sum(1 + 2 * X - 2 * _sq_scalar(X))
    D3 = _pair_sum(X, lambda x, y: 1 - np.abs(x - y))
    return math.sqrt((4.0 / 3.0) ** s + D2 * (-2.0 / n) + D3 * ((2**s) / float(n**2)))


def wd2(X):
    X = np.asarray(X, dtype=np.float64)
    n, s = X.shape
    D3 = _pair_sum(X, lambda x, y: 3.0 / 2.0 - np.abs(x - y) * (1 - np.abs(x - y)))
    return math.sqrt(-((4.0 / 3.0) ** s) + D3 / (n**2))


def select(H, N, rows):
    """Index of the first candidate with the smallest CD2 (the reference's ``if d < D`` from D = 1e32), and the CD2s."""
    d = np.array([cd2(design(h, N, rows)) for h in H])
    best, D = None, 1e32
    for i, v in enumerate(d):
        if v < D:
            best, D = i, v
    return best, d


def glp(n, s, rng):
    """The reference's GLP.sample: the discarded (N, s) uniform draw, then the selected lattice design."""
    N, rows, H = candidates(n, s)
    X = rng.uniform(0, 1, size=[N, s])
    if H.shape[0]:
        best, _ = select(H, N, rows)
        X = design(H[best], N, rows)
    return X
