"""Oracle: exact integer hypervolumes (row A16 of SURVEY.md section 8a), by algorithms independent of the kernels.

Test infrastructure only (see oracle/__init__.py).

Points are integer vectors ``K`` (n, M) with an integer reference ``R``; a row counts only when it is strictly inside
``R`` in every objective (hv.py:159).  Volumes are Python or int64 integers, exact.

Mapped onto ``P = c + K * 2**-e`` (``c`` and ``e`` chosen so that every coordinate is exact), every difference a
hypervolume kernel forms is exact, and so is every product of differences; a sum is exact while each partial sum stays
an integer number of units (2**(-M e)) below 2**53.  So a float64 kernel whose partial sums are bounded that way must
return ``volume * 2**(-M e)`` bit for bit, whatever its summation order (``to_grid`` / ``chain_sum_bound``).

  * ``hv_cells``       any M: dominated cells of the compressed grid (``np.logical_or.accumulate`` along every axis).
  * ``hv_staircase2``  M = 2, O(n log n).
  * ``hv_sweep3``      M = 3: sweep along the last objective over a 2-D staircase kept in sorted lists.
  * ``hv_incl_excl``   the definition (inclusion-exclusion over subsets), n <= 12 rows inside R.
  * ``f32_tie_set``    rows that are mutually non-dominated in float64 and tie in objective 0 after a float32 rounding.
"""

import bisect
import itertools
import math

import numpy as np

EXACT = 1 << 53  # float64 holds every integer below this


def _ints(K, R):
    """Rows of K strictly inside R as int64 (K may be float with integer values, +-0.0 included), and R as int64."""
    K = np.asarray(K)
    R = np.asarray(R)
    M = R.shape[0]
    K = K.reshape(-1, M)
    with np.errstate(invalid="ignore"):
        inside = np.all(K < R, axis=1)
    P = K[inside]
    if P.dtype.kind == "f":
        assert np.all(np.isfinite(P)) and np.all(P == np.round(P)) and np.all(np.abs(P) < 2.0**62), "integer coordinates expected"
    assert np.all(R == np.round(R)), "integer reference expected"
    return P.astype(np.int64), R.astype(np.int64)


def hv_cells(K, R, max_cells=1 << 27):
    """Any M.  Axis j is cut at the distinct values of the points and at R_j; a point marks the cell it is the lower
    corner of, a prefix OR along every axis marks the dominated cells, and their widths multiply out exactly."""
    P, R = _ints(K, R)
    if P.shape[0] == 0:
        return 0
    M = R.shape[0]
    cuts, idx = [], []
    for j in range(M):
        v = np.unique(np.append(P[:, j], R[j]))
        cuts.append(v)
        idx.append(np.searchsorted(v, P[:, j]))
    shape = tuple(len(v) - 1 for v in cuts)
    assert math.prod(shape) <= max_cells, f"hv_cells: {math.prod(shape)} cells"
    grid = np.zeros(shape, dtype=bool)
    grid[tuple(idx)] = True
    for j in range(M):
        grid = np.logical_or.accumulate(grid, axis=j)
    big = math.prod(int(R[j] - cuts[j][0]) for j in range(M)) >= (1 << 63)  # bounds every partial sum below
    vol = grid.astype(object if big else np.int64)
    for j in range(M):
        w = np.diff(cuts[j]).astype(object if big else np.int64)
        vol = np.tensordot(w, vol, axes=([0], [0]))
    return int(vol)


def hv_staircase2(K, R):
    """M = 2: sort by (f0, f1), strips [x_p, x_{p+1}) under the running minimum of f1."""
    P, R = _ints(K, R)
    if P.shape[0] == 0:
        return 0
    o = np.lexsort((P[:, 1], P[:, 0]))
    x, y = P[o, 0], P[o, 1]
    ymin = np.minimum.accumulate(y)
    xn = np.append(x[1:], R[0])
    big = int(R[0] - x[0]) * int(R[1] - ymin[-1]) >= (1 << 63)
    dt = object if big else np.int64
    return int(np.sum((xn - x).astype(dt) * (R[1] - ymin).astype(dt)))


def hv_sweep3(K, R):
    """M = 3: points in ascending z; the xy-staircase of the points seen so far is kept as sorted Python lists (x
    ascending, y strictly descending).  Inserting a point adds its exclusive area and drops the steps it covers; the
    covered area times the gap to the next z is the volume of that slab."""
    P, R = _ints(K, R)
    if P.shape[0] == 0:
        return 0
    rx, ry, rz = (int(r) for r in R)
    P = P[np.argsort(P[:, 2], kind="stable")]
    pts = P.tolist()
    xs, ys = [], []
    area = 0
    total = 0
    for i, (x, y, z) in enumerate(pts):
        hi = bisect.bisect_right(xs, x)
        if not (hi > 0 and ys[hi - 1] <= y):  # not weakly dominated by a step at or left of x
            lo = bisect.bisect_left(xs, x)
            cap = ys[lo - 1] if lo > 0 else ry
            end = lo
            while end < len(xs) and ys[end] >= y:
                end += 1
            bounds = [x] + xs[lo:end] + [xs[end] if end < len(xs) else rx]
            heights = [cap] + ys[lo:end]
            area += sum((bounds[k + 1] - bounds[k]) * (heights[k] - y) for k in range(len(heights)))
            xs[lo:end] = [x]
            ys[lo:end] = [y]
        zn = pts[i + 1][2] if i + 1 < len(pts) else rz
        total += area * (zn - z)
    return total


def hv_incl_excl(K, R):
    """The definition: sum over non-empty subsets S of (-1)^(|S|+1) * prod_j (R_j - max_{i in S} K_ij)."""
    P, R = _ints(K, R)
    n = P.shape[0]
    assert n <= 12, "hv_incl_excl: at most 12 rows inside R"
    rows = P.tolist()
    Rl = [int(r) for r in R]
    total = 0
    for s in range(1, n + 1):
        for sub in itertools.combinations(rows, s):
            v = 1
            for j, r in enumerate(Rl):
                v *= r - max(p[j] for p in sub)
            total += v if s % 2 else -v
    return total


def hv_exact(K, R):
    """The integer volume by the cheapest algorithm above for the objective count."""
    M = np.asarray(R).shape[0]
    if M == 1:
        P, R = _ints(K, R)
        return int(R[0] - P[:, 0].min()) if P.shape[0] else 0
    if M == 2:
        return hv_staircase2(K, R)
    if M == 3:
        return hv_sweep3(K, R)
    return hv_cells(K, R)


# ------------------------------------------------------------------------------------------ dyadic grids
def from_grid(K, R, c, e):
    """P = c + K * 2**-e and ref = c + R * 2**-e in float64, checked to be exact (non-finite K rows pass through)."""
    K = np.asarray(K, dtype=np.float64)
    R = np.asarray(R, dtype=np.float64)
    P = c + np.ldexp(K, -e)
    ref = c + np.ldexp(R, -e)
    fin = np.isfinite(K)
    assert np.array_equal(np.ldexp(P[fin] - c, e), K[fin]) and np.array_equal(np.ldexp(ref - c, e), R), "grid not exact"
    return P, ref


def to_grid(P, ref, c, e):
    """Checks that every coordinate of the rows strictly inside ref, and ref itself, is exactly c + K * 2**-e, and
    returns (K of those rows, R, exact float64 hypervolume).  Asserts that the integer volume is below 2**53."""
    P = np.asarray(P, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    M = ref.shape[0]
    P = P.reshape(-1, M)
    with np.errstate(invalid="ignore"):
        P = P[np.all(P < ref, axis=1)]
    K = np.ldexp(P - c, e)
    R = np.ldexp(ref - c, e)
    assert np.all(K == np.round(K)) and np.all(R == np.round(R)), "coordinates off the grid"
    assert np.array_equal(c + np.ldexp(K, -e), P) and np.array_equal(c + np.ldexp(R, -e), ref), "grid not exact"
    vol = hv_exact(K, R)
    assert 0 <= vol < EXACT, vol
    return K.astype(np.int64), R.astype(np.int64), math.ldexp(float(vol), -M * e)


def chain_sum_bound(n, K, R):
    """n^(M-2) * G^M: a bound on the sum of the absolute terms of the M = 4, 5 chain sums over n rows (G = the extent of
    the integer box).  Below 2**53, every partial sum of those kernels is exact on the grid."""
    K = np.asarray(K, dtype=np.int64)
    R = np.asarray(R, dtype=np.int64)
    M = R.shape[0]
    G = max(int(R[j] - K[:, j].min()) for j in range(M)) if K.shape[0] else 0
    return n ** (M - 2) * G**M


# ------------------------------------------------------------------------------------------ integer fronts
def simplex(M, S):
    """All non-negative integer vectors with sum S: mutually non-dominated (a dominating point would have a smaller
    sum).  C(S + M - 1, M - 1) rows, in lexicographic order."""
    if M == 1:
        return np.array([[S]], dtype=np.int64)
    rows = [(k,) + r for k in range(S + 1) for r in map(tuple, simplex(M - 1, S - k))]
    return np.array(rows, dtype=np.int64)


def simplex_front(M, n, rng, S=None):
    """n distinct rows of the smallest integer simplex with at least n points (or of simplex(M, S)), in random order."""
    if S is None:
        S = 0
        while math.comb(S + M - 1, M - 1) < n:
            S += 1
    T = simplex(M, S)
    assert T.shape[0] >= n
    return T[rng.choice(T.shape[0], size=n, replace=False)]


def sphere_lattice(r):
    """For every (i, j) with i^2 + j^2 <= r^2: (i, j, ceil(sqrt(r^2 - i^2 - j^2))), the lattice points on or just
    outside a sphere octant of radius r: many distinct coordinates, a front that is not a simplex."""
    i, j = np.meshgrid(np.arange(r + 1), np.arange(r + 1), indexing="ij")
    ok = i * i + j * j <= r * r
    i, j = i[ok], j[ok]
    s = (r * r - i * i - j * j).tolist()
    k = [math.isqrt(v) + (math.isqrt(v) ** 2 < v) for v in s]
    return np.column_stack((i, j, k)).astype(np.int64)


# ------------------------------------------------------------------------------------------ float32 ties
def f32_tie_set(M, n_base, copies, rng, c=1.0, e=16):
    """Rows that are mutually non-dominated in float64, share objective 0 after rounding to float32, and carry the
    worse objective 1 at the later row index.

    The base front is g * (an integer simplex front), g = copies + 1.  Copy t (t = 0 .. copies - 1) of a base row K adds
    t units to objective 1 and subtracts t * 2**-30 from objective 0: within a copy group objective 0 falls as
    objective 1 rises (mutually non-dominated), and across groups the coordinate sums, multiples of g apart, rule
    dominance out.  With c + K * 2**-e in [1, 2) on a float32 grid (e <= 23) and |t * 2**-30| < 2**-25, rounding to
    float32 gives back c + K * 2**-e exactly.  Copies follow their base row in row order.

    Returns (Y64, Y32, K32): the float64 rows, their float32 rounding (as float64), and its integer grid coordinates."""
    assert M >= 2 and copies <= 32 and e <= 23 and abs(c) in (1.0, 2.0)
    g = copies + 1
    base = g * simplex_front(M, n_base, rng)
    K = np.repeat(base, copies, axis=0)
    t = np.tile(np.arange(copies), n_base)
    K[:, 1] += t
    assert K.max() < (1 << e)  # c + K * 2**-e stays in [1, 2) (c = 1) or [-2, -1) (c = -2)
    Y32 = c + np.ldexp(K.astype(np.float64), -e)
    Y64 = Y32.copy()
    Y64[:, 0] -= np.ldexp(t.astype(np.float64), -30)
    assert np.array_equal(Y64.astype(np.float32).astype(np.float64), Y32)
    return Y64, Y32, K


def mutually_nondominated(Y):
    """No row weakly dominates another distinct row (float64 comparisons)."""
    Y = np.asarray(Y, dtype=np.float64)
    le = np.all(Y[:, None, :] <= Y[None, :, :], axis=2)
    ne = np.any(Y[:, None, :] != Y[None, :, :], axis=2)
    return not np.any(le & ne)


def hv2_strips_unclipped(Y, ref):
    """The M = 2 strip sum of hv.cu before the running minimum: rows sorted by f0 (ties by row index), strip
    [x_p, x_{p+1}) under the row's own f1.  Valid for mutually non-dominated rows only."""
    Y = np.asarray(Y, dtype=np.float64)
    Y = Y[np.all(Y < ref, axis=1)]
    o = np.argsort(Y[:, 0], kind="stable")
    x, y = Y[o, 0], Y[o, 1]
    xn = np.append(x[1:], ref[0])
    return float(np.sum((xn - x) * (ref[1] - y)))
