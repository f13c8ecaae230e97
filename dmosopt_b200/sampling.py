"""Good-lattice-point initial designs with the generator search on the GPU: a drop-in for dmosopt's ``glp``.

    dmosopt_params["initial_method"] = "dmosopt_b200.sampling.glp"

``MOASMO.xinit`` resolves the name with ``import_object_by_path`` and calls ``glp(n, s, local_random, maxiter)``.
``glp``, ``GoodLatticePointsDesign`` and ``GoodLatticePointsDesignDecorrelation`` keep the signatures of
``dmosopt/sampling.py`` and return the reference's design bit for bit for the same generator state, leaving the
generator in the same state afterwards.

The search (dmosopt/GLP.py):

* the lattice: with m = phi(n) evaluated as the reference does (a float product over the prime factors, truncated),
  m / n < 0.9 selects the lattice of n + 1 points with its last point dropped ("plusone"), otherwise the lattice of n;
* the candidates: when m < 20 and s < 4, every s-combination of the first m' units of the lattice (m' = phi of the
  lattice size, recomputed in the plusone case); otherwise the power vectors (1, a, ..., a^(s-1)) mod n' of the units
  2 <= a < n' whose powers a^1 .. a^(s-1) are distinct and differ from 1.  Enumerated on the host in exact integers;
* both searches draw ``local_random.uniform(0, 1, size=[n', s])`` (n' = lattice size) and discard it; it is the result
  when no candidate exists (then the design has n' rows);
* each candidate's design x_ki = (u - 0.5) / rows, u = ((k + 1) h_i mod n') with 0 replaced by n', is scored by its
  centred L2 discrepancy, and the first candidate with the smallest score wins.

The scores are screened on the GPU for all candidates at once (``_lib.glp_cd2_terms``).  Those sums run in a different
order from the reference's, so the candidates within a rigorous rounding margin of the smallest screened score are
rescored in the reference's own operation order (``_exact_cd2``) and the selection is made on those values; the pick
is the reference's.

``maxiter > 0`` adds the ranked Gram-Schmidt decorrelation of ``dmosopt/sampling.py``, in NumPy with the same
operations in the same order: it is a chain of s^2 dependent rank steps with nothing to parallelise.

Refused with ``ValueError`` where the reference fails: n < 2 (its Euler function indexes an empty factor list), s < 1,
and s = 1 on the power-vector branch (it indexes an empty power list).
"""

import itertools
import math
import operator

import numpy as np

from . import _lib

_U = 2.0**-53  # unit roundoff of float64
_PAIRS_CHUNK = 1 << 24  # pair products per exact-pass call (128 MB)


def _prime_factors(n):
    """Distinct prime factors of n >= 2, ascending."""
    p, f = [], 2
    while f * f <= n:
        if n % f == 0:
            p.append(f)
            while n % f == 0:
                n //= f
        f += 1
    if n > 1:
        p.append(n)
    return p


def euler_phi(n):
    """phi(n) as the reference evaluates it: n (1 - 1/p) over the distinct primes p in float64, truncated to int (this
    can fall one short of the exact totient, and the branch choice and the column count follow the float value)."""
    if n < 2:
        raise ValueError(f"glp: n={n} has no prime factor; the good-lattice-point design needs n >= 2")
    p = _prime_factors(n)
    fai = n * (1 - 1.0 / p[0])
    for q in p[1:]:
        fai *= 1 - 1.0 / q
    return int(fai)


def _units(n, start):
    return np.array([i for i in range(start, n) if math.gcd(i, n) == 1], dtype=np.int64)


def power_vectors(lattice, s):
    """(C, s) int64: (1, a, ..., a^(s-1)) mod lattice for each unit 2 <= a < lattice, in increasing a, whose powers
    a^1 .. a^(s-1) mod lattice are pairwise distinct and all differ from 1."""
    if s < 2:
        raise ValueError(f"glp: s={s} on the power-vector branch; the reference needs s >= 2 there (it indexes the empty list of powers a^1 .. a^(s-1))")
    a = _units(lattice, 2)
    P = np.empty((a.shape[0], s), dtype=np.int64)
    P[:, 0] = 1 % lattice
    for t in range(1, s):
        P[:, t] = P[:, t - 1] * a % lattice  # < lattice^2 < 2^62
    S = np.sort(P[:, 1:], axis=1)
    bad = (S[:, 0] == 1) | np.any(S[:, 1:] == S[:, :-1], axis=1)
    return np.ascontiguousarray(P[~bad])


def column_vectors(lattice, s, m):
    """(C, s) int64: the units of the lattice at every s-combination (itertools order) of the column indices 0 .. m-1."""
    h = _units(lattice, 0)
    combos = np.array(list(itertools.combinations(range(m), s)), dtype=np.int64).reshape(-1, s)
    return np.ascontiguousarray(h[combos])


def candidates(n, s):
    """(lattice, rows, H): the lattice size, the design's row count and the (C, s) candidate multipliers, in the
    reference's candidate order."""
    n, s = operator.index(n), operator.index(s)
    if s < 1:
        raise ValueError(f"glp: s={s}; a design needs at least one dimension")
    m = euler_phi(n)
    plusone = float(m) / n < 0.9
    lattice = n + 1 if plusone else n
    if m < 20 and s < 4:
        H = column_vectors(lattice, s, euler_phi(lattice) if plusone else m)
    else:
        H = power_vectors(lattice, s)
    return lattice, lattice - 1 if plusone else lattice, H


def lattice_design(h, lattice, rows):
    """(rows, s) design of the multipliers h: x_ki = (u - 0.5) / rows, u = (k + 1) h_i mod lattice, 0 -> lattice."""
    u = np.outer(np.arange(1, rows + 1, dtype=np.int64), np.asarray(h, dtype=np.int64)) % lattice
    u[u == 0] = lattice
    return (u.astype(np.float64) - 0.5) / rows


def screen_margin(D1, t2, t3, rows, s):
    """Half-width within which a screened CD2^2 and the reference's may differ, per candidate.

    Both evaluate D^2 = D1 - t2 + t3 with t2 = 2 D2 / n and t3 = D3 / n^2 from the same coordinates.  Every pair factor
    (1 + a_k/2 + a_j/2 - |x_k - x_j|/2 >= 1, since |x_k - x_j| <= a_k + a_j) and every row factor (in [7/8, 1]) carries
    at most 4 roundings of at most 1.5 u each relative to it, and a product of s factors adds s more: a product is
    within 7 s u of exact.  A sequential sum of N positive terms is within (N - 1) u of exact (the reference sums n^2
    pair products and n row products this way; the GPU's blocked sums are better), and forming D^2 adds 3 roundings of
    at most u M with M = D1 + t2 + t3.  So each side lies within gamma M of the exact D^2, gamma = (n^2 + 7 s + 4) u
    to first order; the bound below doubles it for the two sides and takes a factor 1.01 for the second-order terms."""
    gamma = (float(rows) * rows + 7.0 * s + 4.0) * _U
    return 2.02 * gamma * (D1 + t2 + t3)


def _cd2_row_table(lattice, rows):
    """CD2's row factor 1 + 0.5 a - 0.5 a**2, a = |x - 0.5|, for x of u = 1 .. lattice, with NumPy float64 scalar
    operations as the reference evaluates it (a scalar ``a ** 2`` goes through the C library's pow, which is not always
    a * a)."""
    xv = (np.arange(1, lattice + 1, dtype=np.float64) - 0.5) / rows
    T = np.empty(lattice + 1)
    for u in range(1, lattice + 1):
        a = abs(xv[u - 1] - 0.5)
        T[u] = 1 + 0.5 * a - 0.5 * a**2
    return T


def _exact_cd2(H, lattice, rows, s):
    """CD2 of each lattice in H (L, s) in the reference's operation order: D2 from the row table, multiplied along
    each row and summed down the rows sequentially; D3 from the GPU's pair products (dmo_glp_cd2_pairs) summed
    sequentially in row-major order; D1 and the square root in Python floats."""
    T = _cd2_row_table(lattice, rows)
    D1 = (13.0 / 12.0) ** s
    per = max(1, _PAIRS_CHUNK // (rows * rows))
    out = []
    for l0 in range(0, H.shape[0], per):
        Hc = H[l0 : l0 + per]
        P = _lib.glp_cd2_pairs(Hc, lattice, rows)
        D3 = np.cumsum(P, axis=1)[:, -1]
        for h, d3 in zip(Hc, D3):
            u = np.outer(np.arange(1, rows + 1, dtype=np.int64), h) % lattice
            u[u == 0] = lattice
            dd2 = np.ones(rows)
            for i in range(s):
                dd2 = dd2 * T[u[:, i]]
            D2 = np.cumsum(dd2)[-1]
            out.append(math.sqrt(D1 + D2 * (-2.0 / rows) + d3 / (rows**2)))
    return np.array(out)


def select(H, lattice, rows):
    """Index in H of the reference's pick (first candidate with the smallest CD2), and the shortlist that was rescored
    exactly.  Screening on the GPU, then the exact pass over every candidate within the margin of the smallest
    screened D^2."""
    s = H.shape[1]
    d2, d3 = _lib.glp_cd2_terms(H, lattice, rows)
    D1 = (13.0 / 12.0) ** s
    t2, t3 = 2.0 * d2 / rows, d3 / (float(rows) * rows)
    sq = D1 - t2 + t3
    margin = screen_margin(D1, t2, t3, rows, s)
    short = np.flatnonzero(sq <= sq.min() + 2.0 * margin.max())
    d = _exact_cd2(H[short], lattice, rows, s)
    best, D = None, 1e32
    for i, v in zip(short, d):
        if v < D:
            best, D = int(i), v
    return best, short


def GoodLatticePointsDesign(n, s, local_random):
    """Good-lattice-point design of n points in s dimensions (dmosopt ``GLP.sample``); see the module docstring."""
    lattice, rows, H = candidates(n, s)
    X = local_random.uniform(0, 1, size=[lattice, operator.index(s)])
    if H.shape[0] > 0:
        best, _ = select(H, lattice, rows)
        X = lattice_design(H[best], lattice, rows)
    return X


def _rank(z):
    r = np.empty(z.shape[0])
    r[z.argsort()] = np.arange(z.shape[0])
    return r


def _detrend(x, y):
    xm = x - x.mean()
    ym = y - y.mean()
    b = (xm * ym).sum() / (xm**2.0).sum()
    return y - b * xm


def decorrelate(x, n, s):
    """One ranked Gram-Schmidt iteration in place: forward over column pairs (j, k < j), then backward (j descending,
    k from s-1 down to j+1); column k becomes the centred ranks / n of its residual against column j."""
    for j in range(1, s):
        for k in range(j):
            x[:, k] = (_rank(_detrend(x[:, j], x[:, k])) + 0.5) / n
    for j in range(s - 2, -1, -1):
        for k in range(s - 1, j, -1):
            x[:, k] = (_rank(_detrend(x[:, j], x[:, k])) + 0.5) / n
    return x


def GoodLatticePointsDesignDecorrelation(n, s, local_random, maxiter=5):
    """GoodLatticePointsDesign followed by ``maxiter`` ranked Gram-Schmidt iterations."""
    x = GoodLatticePointsDesign(n, s, local_random)
    for _ in range(maxiter):
        x = decorrelate(x, n, s)
    return x


def glp(n, s, local_random, maxiter=0):
    """Short name of GoodLatticePointsDesign (``maxiter`` > 0: with decorrelation)."""
    if maxiter == 0:
        return GoodLatticePointsDesign(n, s, local_random)
    return GoodLatticePointsDesignDecorrelation(n, s, local_random, maxiter)
