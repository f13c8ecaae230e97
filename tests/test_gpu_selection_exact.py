"""The survival kernels every optimizer decides with, checked at their ties, non-finite values and thresholds:

  * crowding and Euclidean distance (csrc/sortmo.cu), bit for bit against oracle/indicators.py, for every M = 1 .. 16
    (both register templates, NumPy's pairwise sum at M = 8 and 16), n around the 256-thread blocks and past the grid of
    ``minmax_kernel`` (4 CTAs per SM), on tie-free data, heavy ties, constant columns, values that normalisation makes
    equal, +-0.0, subnormal ranges, float32-rounded rows over their float64 sources, and columns with +inf, +-inf or NaN;
  * the sortMO order (order_mo, remove_worst, remove_worst_pair) exactly against ``np.lexsort`` over the oracle ranks
    and distances, with 0, 1 and 8 extra descending keys holding ties, +-0.0, +-inf and NaN, on dominance chains whose
    ranks cross the rank-bit width of ``lexsort_device``, and on chains with tied ranks that the distance key orders
    (a NaN Euclidean distance among them);
  * EHVI selection (csrc/hv.cu) against an mpmath evaluation within ``oracle.hv.ehvi_bound`` (and scipy's float64 one
    within twice that), across the 64-box shared tile and the 128-candidate blocks, with f0 ties in the front, duplicate
    candidates, zero and negative variances and means far in both tails; the selection must be the stable descending
    order of the kernel's own scores, NaN last;
  * the duplicate scan (get_duplicates) on pairs whose difference is aligned with the projection weights, at magnitudes
    where the rounding of the projections, not eps, sets the scan window.

NaN sorts last everywhere, whatever its sign bit, as NumPy's sorts put it.  NaN objectives in the rank stay out of scope.
"""

import os

import numpy as np
import pytest

from oracle import dda, indicators, moea
from oracle import hv as ohv

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    for v in list(os.environ):
        if v.startswith("DMO_"):
            monkeypatch.delenv(v, raising=False)


# ------------------------------------------------------------------------------------------------ data generators
DIST_KINDS = ("free", "grid", "const", "merge", "zeros", "subnormal", "f32", "inf", "infs", "nan")


def distance_data(kind, n, M, seed):
    """(n, M) objectives of one data kind (the non-finite kinds put their values in one column)."""
    rng = np.random.default_rng(seed)
    j = (seed + M) % M
    if kind == "free":
        return rng.random((n, M))
    if kind == "grid":  # heavy ties
        return rng.integers(0, 4, size=(n, M)).astype(np.float64)
    if kind == "const":  # zero range -> 1.0
        Y = rng.random((n, M))
        Y[:, j] = 0.37
        return Y
    if kind == "merge":  # a few ulp apart on a large offset: distinct values the normalisation rounds together
        Y = rng.random((n, M))
        off = 1e6
        Y[:, j] = off + rng.integers(0, 8, size=n) * np.spacing(off)
        Y[0, j], Y[-1, j] = 0.1, 3.3e6
        return Y
    if kind == "zeros":
        return rng.choice(np.array([-0.0, 0.0, 0.5, 1.0]), size=(n, M))
    if kind == "subnormal":
        Y = rng.random((n, M))
        Y[:, j] = rng.integers(0, 40, size=n) * 5e-324
        return Y
    if kind == "f32":  # float32-rounded rows stacked on the float64 rows they came from
        c = rng.random((n - n // 2, M)) * 3.0
        return np.vstack((c, c[: n // 2].astype(np.float32).astype(np.float64)))
    Y = rng.random((n, M))
    if kind == "inf":
        Y[rng.integers(0, n), j] = np.inf
    elif kind == "infs":
        i = rng.permutation(n)[:2]
        Y[i[0], j] = np.inf
        Y[i[-1], j] = -np.inf
    elif kind == "nan":
        Y[rng.integers(0, n), j] = np.nan
    return Y


def chain(n, M, mixed, inf, seed):
    """Rows of a dominance chain, shuffled, and their ranks by construction.

    ``mixed``: a third of the levels hold a second point that trades objective 0 against objective 1 (unequally, so
    that the distances of the two differ) -- ties in rank, which the distance key and the extra keys decide.  The top
    level always holds one.  ``inf``: the top chain point holds +inf in objective M - 1.  That column's range is then
    infinite, so its finite rows normalise to 0 and the +inf row to NaN: that row's Euclidean distance is NaN and its
    rank partner's is finite.  Without ``mixed`` (all ranks distinct, the distances decide nothing) the first chain
    point also holds -inf in objective 0.
    """
    rng = np.random.default_rng(seed)
    a = 0.5 + rng.random(M)
    levels = n - n // 3 if mixed and M > 1 else n
    Y = (np.arange(levels)[:, None] + 1.0) * a
    rank = np.arange(levels)
    if levels < n:
        lv = np.concatenate(([levels - 1], rng.choice(levels - 1, size=n - levels - 1, replace=False)))
        extra = Y[lv].copy()
        extra[:, 0] += 0.25 * a[0]
        extra[:, 1] -= 0.15 * a[1]
        Y = np.vstack((Y, extra))
        rank = np.concatenate((rank, lv))
    if inf:
        Y[levels - 1, M - 1] = np.inf
        if levels == n:
            Y[0, 0] = -np.inf
    p = rng.permutation(n)
    return Y[p], rank[p]


def decided_pairs(r, dist):
    """(rank groups of two, how many of them the distance orders: unequal values, at most one of them NaN)."""
    _, inv, cnt = np.unique(r, return_inverse=True, return_counts=True)
    rows = np.flatnonzero(cnt[inv] == 2)
    a, b = rows[np.argsort(r[rows], kind="stable")].reshape(-1, 2).T
    return a.size, int(np.sum((dist[a] != dist[b]) & ~(np.isnan(dist[a]) & np.isnan(dist[b]))))


KEY_POOL = np.array([-1.0, -0.0, 0.0, 0.0, 1.0, 2.0, np.inf, -np.inf, np.nan, -np.nan])


def extra_keys(n, count, seed):
    """Descending keys with ties, +-0.0, +-inf and NaN of both signs."""
    rng = np.random.default_rng(seed)
    return [np.where(rng.random(n) < 0.5, rng.choice(KEY_POOL, size=n), rng.integers(0, 3, size=n).astype(np.float64)) for _ in range(count)]


def ehvi_front(M, nb, seed):
    """(F, ref) whose box decomposition (nds=False) has exactly nb boxes: a chain of nb - 1 points increasing in every
    objective below ref, plus points that tie a chain point's f0 and sit between it and the next chain point in every
    other objective.  Each tie turns one box into another, so the count holds while the boxes depend on the order
    of the tie.  nb = 1: one point beyond ref in f0."""
    rng = np.random.default_rng(seed)
    a = 0.5 + rng.random(M)
    if nb == 1:
        F = (1.0 + rng.random((1, M))) * a
        ref = F[0] + a
        F[0, 0] = ref[0] + a[0]
        return F, ref
    C = (np.arange(nb - 1)[:, None] + 1.0) * a
    t = rng.choice(nb - 1, size=(nb - 1) // 2 + 1, replace=False)
    Q = C[t].copy()
    Q[:, 1:] += (0.2 + 0.6 * rng.random((t.size, M - 1))) * a[1:]
    F = np.vstack((C, Q))
    return F[rng.permutation(F.shape[0])], C[-1] + 2.0 * a


def ehvi_candidates(F, ref, nc, seed):
    """nc candidates inside the front's range, with (when nc allows) duplicate rows, zero variance on a box bound
    (NaN) and off every bound (+-inf z), a negative variance (NaN) and means far in both tails."""
    rng = np.random.default_rng(seed)
    M = F.shape[1]
    fin = np.where(np.isfinite(F), F, 0.0)
    lo, hi = fin.min(axis=0), np.maximum(fin.max(axis=0), ref)
    span = np.maximum(hi - lo, 0.5)  # one point beyond ref: no range of its own
    mu = lo - 0.1 * span + 1.2 * span * rng.random((nc, M))
    var = (0.05 + rng.random((nc, M))) * (0.2 * span) ** 2
    if nc >= 10:
        p = F[rng.integers(0, F.shape[0])]
        mu[1], var[1] = p, 0.0  # on a box bound: z = 0 / 0
        mu[2], var[2] = p + 0.1 * span / np.sqrt(F.shape[0] + 7.0), 0.0  # off every bound: z = +-inf
        var[3, M - 1] = -var[3, M - 1]  # negative variance
        mu[4], var[4] = lo - 1e3 * span, 1e-4 * span**2  # far below
        mu[5], var[5] = hi + 1e3 * span, 1e-4 * span**2  # far above
        mu[6], var[6] = lo - 8.0 * span, span**2  # Phi within a few ulp of 1 at every bound
        d = rng.integers(0, nc, size=max(2, nc // 8))  # duplicates of earlier and later rows
        mu[nc - d.size :], var[nc - d.size :] = mu[d], var[d]
    return mu, var


# ------------------------------------------------------------------------------------------------ distances
def _nan_equal(a, b):
    return np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("kind", DIST_KINDS)
@pytest.mark.parametrize("M", range(1, 17))
def test_distances_bit_exact(L, M, kind):
    for n in (1, 2, 3, 255, 256, 257, 4097):
        Y = distance_data(kind, n, M, seed=1000 * M + n)
        c = L.crowding_distance(Y)
        assert np.array_equal(c, indicators.crowding_distance_metric(Y)), f"crowding n={n}"
        e = L.euclidean_distance(Y)
        assert _nan_equal(e, indicators.euclidean_distance_metric(Y)), f"euclidean n={n}"


@pytest.mark.parametrize("kind", ("free", "grid", "inf", "nan"))
@pytest.mark.parametrize("M", (3, 9))
def test_distances_past_the_minmax_grid(L, M, kind):
    n = 4 * L.sm_count() * 256 + 4097  # more rows than threads: minmax_kernel's grid-stride loop and its atomics
    Y = distance_data(kind, n, M, seed=M)
    assert np.array_equal(L.crowding_distance(Y), indicators.crowding_distance_metric(Y))
    assert _nan_equal(L.euclidean_distance(Y), indicators.euclidean_distance_metric(Y))


# ------------------------------------------------------------------------------------------------ sortMO order
METRICS = ("none", "crowding", "euclidean")


def _oracle_rank(Y, rank):
    # front peeling costs O(fronts * n^2): it pins the small chains, the longest-chain DP (itself pinned against peeling
    # in the CPU suite) the long ones; both must agree with the ranks the chain was built with
    r = dda.rank_canonical(Y) if Y.shape[0] <= 257 else dda.rank_chain_dp(Y)
    assert np.array_equal(r, rank)
    return r


def _oracle_order(L, Y, r, metric, keys):
    dist = None
    if metric != "none":
        dist = (indicators.crowding_distance_metric if metric == "crowding" else indicators.euclidean_distance_metric)(Y)
    cols = tuple(-k for k in keys) + ((-dist,) if dist is not None else ()) + (r,)
    return np.lexsort(cols), dist


def _metric(L, name):
    return {"none": L.METRIC_NONE, "crowding": L.METRIC_CROWDING, "euclidean": L.METRIC_EUCLIDEAN}[name]


@pytest.mark.parametrize("inf", (False, True))
@pytest.mark.parametrize("mixed", (False, True))
@pytest.mark.parametrize("n", (255, 256, 257, 4095, 4096, 4097))
def test_order_mo_exact(L, n, mixed, inf):
    M = 3
    Y, rank = chain(n, M, mixed, inf, seed=n)
    r = _oracle_rank(Y, rank)
    X = np.random.default_rng(n).random((n, 2))
    for metric in METRICS:
        for nk in (0, 1, 8):
            keys = extra_keys(n, nk, seed=n + nk)
            want, dist = _oracle_order(L, Y, r, metric, keys)
            if dist is not None and mixed:  # the distance key orders most tied ranks, and a NaN one among them
                pairs, decided = decided_pairs(r, dist)
                assert pairs == n // 3 and decided >= pairs // 2, (metric, pairs, decided)
                if metric == "euclidean":
                    nan = np.flatnonzero(np.isnan(dist))
                    assert nan.size == inf and (not inf or np.sum(r == r[nan[0]]) == 2)
            perm, rs, ds = L.order_mo(Y, _metric(L, metric), keys or None)
            assert np.array_equal(perm, want), (metric, nk)
            assert np.array_equal(rs, r[want])
            if dist is not None:
                assert _nan_equal(ds, dist[want])
            for keep in (1, n - 1, n, n + 5):
                Xo, Yo, ro, po = L.remove_worst(X, Y, keep, _metric(L, metric), keys or None)
                k = min(keep, n)
                assert np.array_equal(po, want[:k]), (metric, nk, keep)
                assert np.array_equal(ro, r[want[:k]])
                assert np.array_equal(Xo, X[want[:k]]) and np.array_equal(Yo, Y[want[:k]])
                if nk == 0:
                    h = n // 3
                    Xp, Yp, rp, pp = L.remove_worst_pair(X[:h], Y[:h], X[h:], Y[h:], keep, _metric(L, metric))
                    assert np.array_equal(pp, po) and np.array_equal(rp, ro)
                    assert np.array_equal(Xp, Xo) and np.array_equal(Yp, Yo)


# ------------------------------------------------------------------------------------------------ EHVI
MP_BUDGET = 2500  # mpmath (box, objective, candidate) terms per case


def check_ehvi(L, F, ref, mu, var, nds):
    nc, M = mu.shape
    front = F[dda.rank_canonical(F) == 0] if nds else F
    lo, up = ohv.decompose_boxes(front, ref)
    _, g = L.ehvi_select(F, mu, var, ref, nc, nds=nds, return_scores=True)
    with np.errstate(all="ignore"):
        o = ohv.batch_ehvi(lo, up, mu, var)
        B = ohv.ehvi_bound(lo, up, mu, var)
    nan = np.isnan(o)
    assert np.array_equal(np.isnan(g), nan), f"NaN pattern: gpu {np.flatnonzero(np.isnan(g))} oracle {np.flatnonzero(nan)}"
    assert np.array_equal(np.isnan(B), nan)
    bad = np.flatnonzero(np.abs(g - o)[~nan] > 2 * B[~nan])
    assert bad.size == 0, f"{bad.size} scores outside twice the bound, e.g. {g[~nan][bad[:3]]} vs {o[~nan][bad[:3]]}"
    rows = np.arange(min(nc, int(np.clip(MP_BUDGET // (lo.shape[0] * M), 3, 7))))  # the first rows hold the special cases
    m = ohv.ehvi_mp(lo, up, mu[rows], var[rows])
    assert np.array_equal(np.isnan(m), nan[rows])
    ok = np.isnan(m) | (np.abs(g[rows] - m) <= B[rows])
    assert ok.all(), f"gpu {g[rows][~ok]} mpmath {m[~ok]} bound {B[rows][~ok]}"
    # the selection: the stable descending order of the kernel's own scores, NaN last, as a prefix for every k
    order = np.argsort(-g, kind="stable")
    for k in (1, nc, nc + 3):
        sel = L.ehvi_select(F, mu, var, ref, k, nds=nds)
        assert np.array_equal(sel, order[: min(k, nc)]), k
    # and the oracle's order wherever two oracle scores differ by more than the two bounds allow
    fin = order[~np.isnan(g[order])]
    if fin.size > 1:
        hi_ = o[fin] + 2 * B[fin]
        lo_ = o[fin] - 2 * B[fin]
        assert np.all(lo_[1:] <= np.minimum.accumulate(hi_)[:-1])
    return lo.shape[0]


@pytest.mark.parametrize("nb", (1, 2, 63, 64, 65, 128, 129))
@pytest.mark.parametrize("M", (1, 2, 3, 8, 9, 16))
def test_ehvi_boxes_and_objectives(L, M, nb):
    F, ref = ehvi_front(M, nb, seed=100 * M + nb)
    mu, var = ehvi_candidates(F, ref, 129, seed=M + nb)
    assert check_ehvi(L, F, ref, mu, var, nds=False) == nb


@pytest.mark.parametrize("nc", (1, 127, 128, 129, 10000))
def test_ehvi_candidate_blocks(L, nc):
    for M, nb in ((2, 65), (9, 64)):
        F, ref = ehvi_front(M, nb, seed=nc + M)
        mu, var = ehvi_candidates(F, ref, nc, seed=nc)
        assert check_ehvi(L, F, ref, mu, var, nds=False) == nb


@pytest.mark.parametrize("nf", (1023, 1024))
@pytest.mark.parametrize("M", (3, 9))
def test_ehvi_nondominated_front_with_f0_ties(L, M, nf):
    rng = np.random.default_rng(nf + M)
    x = np.abs(rng.standard_normal((nf, M))) + 1e-3
    F = x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.2 * rng.integers(0, 3, size=(nf, 1)))
    F[:, 0] = np.round(F[:, 0] * 8) / 8  # f0 ties, the lowest ones among them
    front = F[dda.rank_canonical(F) == 0]
    assert np.unique(front[:, 0], return_counts=True)[1][0] > 1
    ref = F.max(axis=0) + 0.1
    mu, var = ehvi_candidates(F, ref, 300, seed=nf)
    check_ehvi(L, F, ref, mu, var, nds=True)


# ------------------------------------------------------------------------------------------------ duplicates
def dup_weight(c):
    """sortmo.cu's projection weight of column c, recomputed."""
    return 1.0 + float((((c * 2654435761) % 2**32) >> 8) & 0xFFFF) / 65536.0


def aligned_pairs(e, d, alpha, npair, seed):
    """Bases with every coordinate in the binade [2^e, 2^(e+1)) (either sign), and partners moved by k_c = round(alpha
    w_c) ulps in column c: a difference vector along the projection weights, and an exact distance."""
    rng = np.random.default_rng(seed)
    U = 2.0 ** (e - 52)
    k = np.rint(alpha * np.array([dup_weight(c) for c in range(d)]))
    m = rng.integers(64, 2**52 - 64, size=(npair, d)).astype(np.float64)
    x = rng.choice(np.array([-1.0, 1.0]), size=(npair, d)) * (2.0**e + m * U)
    y = x + k * U
    D = np.sqrt(np.sum((k * U) ** 2))
    assert np.all(np.sqrt(np.sum((y - x) ** 2, axis=1)) == D)
    return x, y, D


@pytest.mark.parametrize("d", (1, 2, 100))
@pytest.mark.parametrize("e", (20, 30, 40))  # magnitudes 1e6, 1e9, 1e12
def test_duplicates_projection_window(L, e, d):
    """Partners one or two ulps per column away (alpha = 1), so that the rounding term of dup_window dominates its reach
    2 sqrt(d) eps at every d.  Only at d = 100 do the projections actually round by more than the reach; with one or two
    columns their rounding stays inside it, and those cases check the eps cutoff on the same narrow windows."""
    npair = 200
    x, y, D = aligned_pairs(e, d, 1.0, npair, seed=e * 1000 + d)
    w = np.array([dup_weight(c) for c in range(d)])
    rng = np.random.default_rng(e + d)
    for s, flagged in ((0.99, True), (1.01, False)):
        eps = D / s
        reach = 2.0 * np.sqrt(d) * eps
        assert np.all(4.0 * d * 2.220446049250313e-16 * (np.abs(np.vstack((x, y))) @ w + reach) > reach)  # dup_window's terms
        X = np.vstack((x, y))[rng.permutation(2 * npair)]
        want = moea.get_duplicates(X, eps)
        assert want.sum() == (npair if flagged else 0)
        assert np.array_equal(L.get_duplicates(X, eps), want), (s, "self")
        Yb = x[rng.permutation(npair)]  # bases in another order: row i's base lies before it or not
        want = moea.get_duplicates(y, eps, Y=Yb)
        assert np.array_equal(L.get_duplicates(y, eps, Y=Yb), want), (s, "pair")
        if flagged:
            assert 0 < want.sum() < npair
