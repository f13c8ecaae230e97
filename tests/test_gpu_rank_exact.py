"""Every route of the non-dominated rank (csrc/rank.cu) and of the rank-0 filter, checked on EVERY row against the
brute-force float64 dominance test of oracle/dda.py (check_ranks / check_flags, run with torch on the same GPU).

The cases sit at the thresholds where the kernels switch:
  * 128-row block edges for every objective count (the dense-id route at M = 1, one chain template per M = 2 .. 16);
  * the segmented order (M <= 3, 16 .. 1024 blocks) switching on and off, its segment count, and the plain chain past
    1024 blocks;
  * the chain's double-buffered tile (M <= 7) and single-buffered one (M >= 8), its dynamic shared memory (M = 16), CTAs
    that loop over tickets (DMO_RANK_OCC=1) and the 32-bit fallback above 32000 fronts;
  * the filter's float64 scan (< 1024 rows), integer-id scan (>= 1024) and cell grid (M <= 3, >= 8192, up to 9-bit
    cells), through dmo_nondominated_flags;
  * front peeling for truncations (remove_worst, M = 3).
Route-selection variables are read on every call, so each case sets them for the calls it makes.

The data mixes uniform clouds, sphere shells (nearly one front), thick shells (a few fronts), integer grids with heavy
ties, exact duplicates, float32-rounded parents over float64 children, neighbours one ulp apart, and +-0.0 / +-inf /
subnormals / magnitudes near 1e+-300.  NaN is deliberately absent: what a NaN objective should rank is a separate
decision, not pinned down here.
"""

import numpy as np
import pytest

from oracle import dda, indicators

pytestmark = pytest.mark.gpu

ROUTE_VARS = ("DMO_RANK_SEGBITS", "DMO_RANK_NOSEG", "DMO_RANK_OCC", "DMO_ND_BRUTE", "DMO_RANK_PEEL", "DMO_RANK_PEEL_NOPROBE",
              "DMO_PEEL_GBITS")


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    for v in ROUTE_VARS:
        monkeypatch.delenv(v, raising=False)


DEV = "cuda"


def make(kind, n, M, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.random((n, M))
    if kind == "sphere":  # nearly one front
        x = np.abs(rng.standard_normal((n, M))) + 1e-12
        return x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 1e-3 * rng.random((n, 1)))
    if kind == "shells":  # a few thick fronts
        x = np.abs(rng.standard_normal((n, M))) + 1e-12
        return x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.05 * rng.integers(0, 6, size=(n, 1)) + 1e-4 * rng.random((n, 1)))
    if kind == "grid":  # heavy ties: six values per objective
        return rng.integers(0, 6, size=(n, M)).astype(np.float64)
    if kind == "coarse":  # ties, but enough distinct values to spread the segmented order's 8-bit bands
        return rng.integers(0, max(8, n // 16), size=(n, M)).astype(np.float64)
    if kind == "dup":  # exact duplicates: pairs, and one vector repeated across several 128-row blocks
        base = make("shells", max(1, n // 4), M, seed + 1)
        idx = rng.integers(0, base.shape[0], size=n)
        idx[: min(n, 300)] = 0
        return base[idx[rng.permutation(n)]]
    if kind == "f32":  # float32-rounded parents stacked on the float64 children they were rounded from
        nc = n - n // 2
        c = make("shells", nc, M, seed + 2)
        p = c[rng.integers(0, nc, size=n // 2)].astype(np.float32).astype(np.float64)
        return np.vstack((c, p))
    if kind == "ulp":  # neighbours one ulp apart on a sphere shell
        nb = n - n // 2
        base = make("sphere", nb, M, seed + 3)
        nbr = base[rng.integers(0, nb, size=n // 2)]
        step = rng.integers(-1, 2, size=nbr.shape)
        nbr = np.where(step > 0, np.nextafter(nbr, np.inf), np.where(step < 0, np.nextafter(nbr, -np.inf), nbr))
        return np.vstack((base, nbr))[rng.permutation(n)]
    if kind == "extreme":  # +-0.0, +-inf, subnormals, magnitudes near 1e+-300, mixed with ordinary values
        special = np.array([-np.inf, -1.7e308, -1e300, -1.0, -1e-300, -5e-324, -0.0, 0.0, 5e-324, 2.2e-310, 1e-300, 1.0, 1e300, 1.7e308, np.inf])
        y = rng.standard_normal((n, M)) * 10.0 ** rng.uniform(-300, 300, size=(n, M))
        pick = rng.random((n, M)) < 0.5
        y[pick] = rng.choice(special, size=int(pick.sum()))
        return y
    raise ValueError(kind)


def rank(L, Y, monkeypatch=None, **env):
    if not env:
        return L.rank_nd(Y)
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        return L.rank_nd(Y)


def flags(L, Y, monkeypatch=None, **env):
    if not env:
        return L.nondominated_flags(Y)
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        return L.nondominated_flags(Y)


def exact_rank(L, Y, monkeypatch=None, **env):
    r = rank(L, Y, monkeypatch, **env)
    assert r.shape == (Y.shape[0],)
    dda.check_ranks(Y, r, device=DEV)
    return r


# ------------------------------------------------------------------------------------------ block edges, every template
@pytest.mark.parametrize("M", list(range(1, 17)))
@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 255, 256, 257])
def test_block_edges_every_template(L, n, M):
    for kind in ("uniform", "grid", "dup", "ulp", "extreme"):
        Y = make(kind, n, M, 1000 * n + 10 * M + len(kind))
        exact_rank(L, Y)


# ------------------------------------------------------------------------------------------ segmented order on / off
@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("n", [1920, 1921, 2048, 2049])  # 15 blocks (plain chain), then 16, 16 and 17 (segmented)
def test_segmented_order_threshold(L, n, M):
    for kind in ("uniform", "sphere", "shells", "grid", "coarse", "dup", "f32", "ulp", "extreme"):
        exact_rank(L, make(kind, n, M, n + M + len(kind)))


def staircase_tie_set(seed):
    """M = 3, n = 2048: two segments of 1024 objective-1 ids.  The first tile of segment 0 is a chain of 128 points with
    ranks 0 .. 127; the first block of segment 1 lies above that tile's band in objective 2, so it reads the tile from its
    staircase, and every one of its 128 points ties the tile's largest objective-3 key.  All 128 tile points dominate
    each of them (rank 128 through the staircase's last entry, 127 if that entry were lost); no other row dominates them."""
    rng = np.random.default_rng(seed)
    i = np.arange(128.0)
    tile = np.column_stack((i, i, i))
    rest0 = np.column_stack((128.0 + rng.permutation(896), 3000.0 + rng.random(896) * 1000, 1000.0 + rng.random(896) * 1000))
    targets = np.column_stack((2047.0 - i, 200.0 + i, np.full(128, 127.0)))
    rest1 = np.column_stack((1024.0 + rng.permutation(896), 400.0 + rng.random(896) * 2000, rng.random(896) * 2000))
    Y = np.vstack((tile, rest0, targets, rest1))
    return Y, np.arange(1024, 1152)


def test_segmented_staircase_key_tie(L):
    Y, targets = staircase_tie_set(41)
    perm = np.random.default_rng(42).permutation(Y.shape[0])
    r = exact_rank(L, Y[perm])[np.argsort(perm)]
    assert np.all(r[targets] == 128)


@pytest.mark.parametrize("kind", ["uniform", "shells", "coarse", "ulp"])
def test_segment_count_overrides_give_identical_ranks(L, monkeypatch, kind):
    """n = 131072, M = 3: 1024 blocks, the last size of the segmented order (128 segments by default)."""
    n, M = 131072, 3
    Y = make(kind, n, M, 31 + len(kind))
    r = exact_rank(L, Y)
    for bits in (1, 4, 7):
        assert np.array_equal(rank(L, Y, monkeypatch, DMO_RANK_SEGBITS=bits), r), (kind, bits)
    assert np.array_equal(rank(L, Y, monkeypatch, DMO_RANK_NOSEG=1), r), kind


@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("kind", ["uniform", "coarse", "dup"])
def test_plain_chain_past_the_segmented_limit(L, M, kind):
    """n = 131073: 1025 blocks, one past the segmented order's band cache."""
    exact_rank(L, make(kind, 131073, M, 77 + M + len(kind)))


# ------------------------------------------------------------------------------------------ large plain chain
@pytest.mark.parametrize("M,n,kinds", [
    (4, 65536, ("uniform", "grid")),
    (5, 65536, ("shells", "dup")),
    (7, 32768, ("uniform", "f32")),   # last double-buffered tile
    (8, 32768, ("uniform", "grid")),  # first single-buffered tile
    (12, 16384, ("shells", "coarse")),
    (16, 16384, ("uniform", "grid")),  # dynamic shared memory
])
def test_large_plain_chain(L, M, n, kinds):
    for kind in kinds:
        exact_rank(L, make(kind, n, M, n + M + len(kind)))


# ------------------------------------------------------------------------------------------ CTAs that loop over tickets
@pytest.mark.parametrize("M", [3, 5])
@pytest.mark.parametrize("kind", ["uniform", "coarse"])
def test_cta_reuse(L, monkeypatch, M, kind):
    """DMO_RANK_OCC=1: one CTA per SM (132 on an H100 SXM) for 1024 blocks, so every CTA takes several tickets."""
    Y = make(kind, 131072, M, 500 + M + len(kind))
    r = exact_rank(L, Y)
    assert np.array_equal(rank(L, Y, monkeypatch, DMO_RANK_OCC=1), r)


# ------------------------------------------------------------------------------------------ more than 32000 fronts
@pytest.mark.parametrize("M", [3, 5])  # M = 3 takes the segmented order, M = 5 the plain chain
def test_more_than_32000_fronts(L, M):
    rng = np.random.default_rng(900 + M)
    # a total order of 33000 rows plus a cloud: only the later blocks leave the packed 16-bit path
    m = 33000
    base = np.arange(m, dtype=np.float64)
    chain = np.column_stack([base * (k + 1) + 0.5 * k for k in range(M)])
    Y = np.vstack((chain, rng.random((2000, M)) * np.array([m * (k + 1) for k in range(M)])))
    r = exact_rank(L, Y[rng.permutation(Y.shape[0])])
    assert r.max() > 32500 and np.count_nonzero(r > 32000) < Y.shape[0] // 2
    # a pure chain of 40000: every block above 32000 fronts
    m = 40000
    base = np.arange(m, dtype=np.float64)
    perm = rng.permutation(m)
    Y = np.column_stack([base * (k + 1) for k in range(M)])[perm]
    assert np.array_equal(exact_rank(L, Y), perm)


# ------------------------------------------------------------------------------------------ rank-0 flag routes
def exact_flags(L, Y, monkeypatch=None, **env):
    f = flags(L, Y, monkeypatch, **env)
    assert f.shape == (Y.shape[0],) and f.dtype == np.int32 and set(np.unique(f)) <= {0, 1}
    dda.check_flags(Y, f, device=DEV)
    return f


@pytest.mark.parametrize("M,n", [(M, n) for M in (2, 3) for n in (1023, 1024, 8191, 8192, 131072)]
                         + [(M, n) for M in (4, 8, 9, 16) for n in (1023, 1024, 5000)])
def test_flag_routes(L, monkeypatch, M, n):
    for kind in ("uniform", "sphere", "grid", "dup", "ulp", "extreme"):
        Y = make(kind, n, M, 7 * n + M + len(kind))
        f = exact_flags(L, Y)
        if M <= 3 and n >= 8192:  # the cell grid against the plain block scan
            assert np.array_equal(flags(L, Y, monkeypatch, DMO_ND_BRUTE=1), f), kind


@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("kind", ["sphere", "uniform", "coarse", "quantised"])
def test_flag_grid_extremes(L, monkeypatch, M, kind):
    """n = 2^18 + 5: the grid at its 9-bit cap; quantised data (40 distinct values, maxid << n): cell shift 0."""
    n = (1 << 18) + 5
    Y = np.round(make("sphere", n, M, 3 + M) * 40) / 40 if kind == "quantised" else make(kind, n, M, 11 + M + len(kind))
    f = exact_flags(L, Y)
    assert np.array_equal(flags(L, Y, monkeypatch, DMO_ND_BRUTE=1), f), kind


def test_flags_agree_with_the_hypervolume_filter(L):
    """The hypervolume of a set is the hypervolume of the rows flagged 0."""
    Y = make("shells", 3000, 3, 5)
    f = exact_flags(L, Y)
    ref = Y.max(axis=0) + 0.1
    assert abs(L.hypervolume(Y, ref) - L.hypervolume(Y[f == 0], ref)) <= 1e-12 * L.hypervolume(Y, ref)


# ------------------------------------------------------------------------------------------ front peeling (remove_worst)
def check_truncation(L, X, Y, keep, metric, r_ref, monkeypatch=None, **env):
    if env:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            Xo, Yo, rk, perm = L.remove_worst(X, Y, keep, metric)
    else:
        Xo, Yo, rk, perm = L.remove_worst(X, Y, keep, metric)
    if metric == L.METRIC_NONE:
        expect = np.argsort(r_ref, kind="stable")[:keep]
    else:
        expect = np.lexsort((-indicators.crowding_distance_metric(Y), r_ref))[:keep]
    assert np.array_equal(perm, expect), (metric, env)
    assert np.array_equal(rk, r_ref[perm]), (metric, env)
    assert np.array_equal(Yo, Y[perm]) and np.array_equal(Xo, X[perm])


@pytest.mark.parametrize("n", [20000, 131072])
@pytest.mark.parametrize("kind", ["shells", "sphere", "uniform"])
def test_truncation_by_peeling(L, monkeypatch, n, kind):
    """M = 3, n >= 8192: remove_worst peels the fronts it needs when they are few (shells, sphere) and runs the chain
    otherwise (uniform).  The kept rows, their order and their ranks are checked against the exact ranks."""
    M = 3
    Y = make(kind, n, M, n + len(kind))
    X = np.random.default_rng(n).random((n, 2))
    r_ref = exact_rank(L, Y)  # the chain, checked on every row: the exact rank
    for keep in (n // 4, n // 2):
        for metric in (L.METRIC_NONE, L.METRIC_CROWDING):
            check_truncation(L, X, Y, keep, metric, r_ref)
            if n <= 20000:  # peeling forced all the way, at both ends of the cell-grid size
                for gb in (4, 9):
                    check_truncation(L, X, Y, keep, metric, r_ref, monkeypatch, DMO_RANK_PEEL=100000, DMO_RANK_PEEL_NOPROBE=1,
                                     DMO_PEEL_GBITS=gb)
