"""Every exact hypervolume route (csrc/hv.cu, hv3_tree.cu, hv_many.cu) checked for EXACT equality with an integer volume
computed on the CPU by oracle/hv_exact.py, at the sizes where the kernels switch.

Each case builds an integer set K with an integer reference R and runs it twice: as integers, and mapped to
c + K * 2**-e with a negative c, so that the coordinates take both signs.  Every difference the kernels form is then
exact, and so is every product of differences; the sums are exact while every partial sum stays below 2**53 units
(asserted per case, with the chain-sum bound for M = 4, 5).  So the float64 result must equal volume * 2**(-M e) bit for
bit, whatever the summation order.

Every case also asserts the precondition of the route it claims: the number of rows inside ref (the filter's input) and
the front size from rank_nd (the kernel's input).  Route-selection variables are read on every call; the fixture clears
them and each case sets them only for the calls it makes.

The ranked entry (rank=...) skips the non-dominated filter, so it is checked on sets whose rank-0 rows are not mutually
non-dominated: float32-rounded tie sets ranked before the rounding (what dmo_nsga2_step hands it), and arbitrary integer
sets passed with rank 0 throughout.
"""

import ctypes
import math

import numpy as np
import pytest

from oracle import hv_exact as hx

pytestmark = pytest.mark.gpu

ROUTE_VARS = ("DMO_HV3_TREE", "DMO_HV_WFG", "DMO_ND_BRUTE")
GRIDS = ((0.0, 0), (-0.75, 6))  # plain integers; a negative offset on a finer grid (coordinates of both signs)
M3_ROUTES = ({}, {"DMO_HV3_TREE": 0}, {"DMO_HV3_TREE": 1})  # default switch at 4096, sweep forced, tree forced
M45_ROUTES = ({}, {"DMO_HV_WFG": 1})  # chain sums, limit-set recursion


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    for v in ROUTE_VARS:
        monkeypatch.delenv(v, raising=False)


def hv_env(L, monkeypatch, P, ref, env, rank=None):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        return L.hypervolume(P, ref, rank=rank)


def routes(M):
    return M3_ROUTES if M == 3 else (M45_ROUTES if M in (4, 5) else ({},))


def assert_exact_bounds(K, R, n_kernel):
    """The integer volume, and for M = 4, 5 the chain sums over the kernel's n_kernel rows, stay below 2**53."""
    M = R.shape[0]
    V = hx.hv_exact(K, R)
    assert 0 <= V < hx.EXACT
    if M in (4, 5):
        inside = K[np.all(K < R, axis=1)]
        assert hx.chain_sum_bound(n_kernel, inside, R) < hx.EXACT, (n_kernel, M)
    return V


def check(L, monkeypatch, K, R, envs, n_inside=None, front=None, extra_rows=True):
    """L.hypervolume on K and on its dyadic image equals the exact volume under every route in envs."""
    M = R.shape[0]
    inside = np.all(K < R, axis=1)
    if n_inside is not None:
        assert np.count_nonzero(inside) == n_inside
    nf = int(np.count_nonzero(L.rank_nd(K[inside].astype(np.float64)) == 0)) if M > 1 else 1
    if front is not None:
        assert nf == front, (nf, front)
    V = assert_exact_bounds(K, R, nf)
    for c, e in GRIDS:
        P, ref = hx.from_grid(K, R, c, e)
        target = math.ldexp(float(V), -M * e)
        for env in envs:
            v = hv_env(L, monkeypatch, P, ref, env)
            assert v == target, (env, c, e, v, target, (v - target) / target)
        if extra_rows:  # NaN, +inf, on ref, one coordinate on ref: outside the strict box, value unchanged
            edge = P[:1].copy()
            edge[0, M - 1] = ref[M - 1]
            bad = np.vstack((np.full(M, np.nan), np.full(M, np.inf), ref, edge))
            Pb = np.vstack((bad[:2], P, bad[2:]))
            v1 = L.hypervolume(Pb, ref)
            assert v1 == target, (c, e, v1, target)
            assert L.hypervolume(Pb, ref) == v1  # repeat call: bit-identical
    return V


def front_with_filler(M, f, n_dom, n_dup, rng, S=None, pad=3):
    """f distinct simplex rows, n_dup duplicates of them, n_dom rows each dominated by a front row; R = S + pad."""
    F = hx.simplex_front(M, f, rng, S)
    S = int(F.sum(axis=1)[0])
    dup = F[rng.integers(0, f, size=n_dup)]
    d = rng.integers(0, pad, size=(n_dom, M))
    d[np.arange(n_dom), rng.integers(0, M, size=n_dom)] += 1  # never all zero: strictly dominated
    d = np.minimum(d, pad - 1)
    dom = F[rng.integers(0, f, size=n_dom)] + d
    K = np.vstack((F, dup, dom))[rng.permutation(f + n_dup + n_dom)]
    return K, np.full(M, S + pad, dtype=np.int64)


# ------------------------------------------------------------------------------------------ the rank-0 filter in front
@pytest.mark.parametrize("M,n1", [(M, n1) for M in range(2, 9) for n1 in (1023, 1024)] + [(M, n1) for M in (2, 3) for n1 in (8191, 8192)])
def test_filter_thresholds(L, monkeypatch, M, n1):
    """n1 rows inside ref: float64 scan (< 1024), integer-id scan (>= 1024), cell grid (M <= 3, >= 8192); each
    against the plain block scan (DMO_ND_BRUTE=1) too."""
    rng = np.random.default_rng(100 * M + n1)
    f = {2: 500, 3: 500, 4: 120, 5: 60, 6: 120, 7: 100, 8: 80}[M]
    n_dup = f // 5
    K, R = front_with_filler(M, f, n1 - f - n_dup, n_dup, rng)
    outside = np.vstack((K[:7] + R, np.full((3, M), R[0])))
    K = np.vstack((K, outside))
    envs = [dict(r, DMO_ND_BRUTE=b) if b else dict(r) for r in routes(M) for b in (0, 1)]
    check(L, monkeypatch, K, R, envs, n_inside=n1, front=f + n_dup)


# ------------------------------------------------------------------------------------------ M = 1
@pytest.mark.parametrize("n", [1, 1025])
def test_one_objective(L, monkeypatch, n):
    rng = np.random.default_rng(n)
    K = rng.integers(-40, 60, size=(n, 1))
    K[: n // 2] = K[n // 2 : n // 2 + n // 2]  # ties
    R = np.array([50], dtype=np.int64)
    n_in = int(np.count_nonzero(K[:, 0] < 50))
    check(L, monkeypatch, K, R, ({},), n_inside=n_in, extra_rows=n_in > 0)


# ------------------------------------------------------------------------------------------ M = 2
@pytest.mark.parametrize("f", [1, 2, 255, 256, 257, 8192])
def test_two_objectives_block_edges(L, monkeypatch, f):
    """hv2_kernel's 256-row blocks, on fronts with dominated rows around them."""
    rng = np.random.default_rng(f)
    K, R = front_with_filler(2, f, 2 * f + 3, 0, rng)
    check(L, monkeypatch, K, R, ({},), front=f)


def test_two_objectives_anti_diagonal(L, monkeypatch):
    """2^20 points on the anti-diagonal (every row non-dominated), the volume at 2^39 units."""
    N = 1 << 20
    i = np.arange(N, dtype=np.int64)
    K = np.column_stack((i, N - 1 - i))[np.random.default_rng(1).permutation(N)]
    V = check(L, monkeypatch, K, np.array([N, N], dtype=np.int64), ({},), n_inside=N, front=N, extra_rows=False)
    assert V == N * (N + 1) // 2


# ------------------------------------------------------------------------------------------ M = 3
@pytest.mark.parametrize("f", [127, 128, 129, 1024, 1025, 4095, 4096])
def test_three_objectives_sweep_and_tree(L, monkeypatch, f):
    """HV_T = 128 tiles of the sweep, the tree's 1024-position shared-memory levels, the default switch at 4096; each
    under the default, the sweep forced and the tree forced."""
    rng = np.random.default_rng(3000 + f)
    K, R = front_with_filler(3, f, f // 3, 0, rng)
    check(L, monkeypatch, K, R, M3_ROUTES, front=f)


def test_three_objectives_large_simplex(L, monkeypatch):
    """The whole simplex of sum 373: 70 125 non-dominated points, past the tree's merge-path levels."""
    K = hx.simplex(3, 373)[np.random.default_rng(2).permutation(70125)]
    check(L, monkeypatch, K, np.full(3, 374, dtype=np.int64), M3_ROUTES, front=70125, extra_rows=False)


def test_three_objectives_sphere_lattice(L, monkeypatch):
    """Lattice points on a sphere octant of radius 256: many distinct coordinates, not a simplex (checked with the
    z-sweep oracle)."""
    K = hx.sphere_lattice(256)
    R = np.full(3, 257, dtype=np.int64)
    nf = int(np.count_nonzero(L.rank_nd(K.astype(np.float64)) == 0))
    assert nf > 4096  # the tree by default
    check(L, monkeypatch, K, R, M3_ROUTES, front=nf)


# ------------------------------------------------------------------------------------------ M = 4, 5
@pytest.mark.parametrize("M,f", [(M, f) for M in (4, 5) for f in (1, 2, 127, 128, 129, 256, 257)] + [(4, 600)])
def test_four_and_five_objectives_chain_sums(L, monkeypatch, M, f):
    """hv_slice_kernel's 128-row tiles along gridDim.y (256 -> 2, 257 -> 3 tiles) and the volume terms; each also
    through the limit-set recursion (DMO_HV_WFG=1)."""
    rng = np.random.default_rng(50 * M + f)
    K, R = front_with_filler(M, f, f // 2 + 1, 0, rng)
    check(L, monkeypatch, K, R, M45_ROUTES, front=f)


# ------------------------------------------------------------------------------------------ M = 6 .. 8
@pytest.mark.parametrize("M,f", [(6, 300), (7, 200), (8, 120)])
def test_six_to_eight_objectives_limit_sets(L, monkeypatch, M, f):
    rng = np.random.default_rng(60 * M + f)
    K, R = front_with_filler(M, f, f, f // 10, rng)
    check(L, monkeypatch, K, R, ({},), front=f + f // 10)


def test_six_objectives_front_limit(L):
    """2049 non-dominated rows at M = 6: refused with the 2048-point limit named, before the recursion runs."""
    K = hx.simplex_front(6, 2049, np.random.default_rng(6), S=10).astype(np.float64)
    assert np.count_nonzero(L.rank_nd(K) == 0) == 2049
    with pytest.raises(L.DmoError, match="2048"):
        L.hypervolume(K, np.full(6, 11.0))


# ------------------------------------------------------------------------------------------ the ranked entry
@pytest.mark.parametrize("M", list(range(2, 9)))
@pytest.mark.parametrize("c", [1.0, -2.0])
def test_ranked_float32_ties(L, monkeypatch, M, c):
    """(a) Rows mutually non-dominated in float64 that tie in objective 0 after rounding to float32, the worse
    objective 1 at the later row index, plus dominated rows.  Ranks come from the unrounded rows; the rounded rows must
    give the exact volume of the rounded set (before the running minimum, M = 2 came out too small)."""
    rng = np.random.default_rng(10 * M + (c < 0))
    n_base = {2: 300, 3: 300, 4: 100, 5: 40, 6: 40, 7: 40, 8: 40}[M]
    Y64, Y32, K = hx.f32_tie_set(M, n_base, 3, rng, c=c)
    R = np.full(M, K.max() + 3, dtype=np.int64)
    dom = K[rng.integers(0, K.shape[0], size=n_base)] + rng.integers(1, 3, size=(n_base, M))
    Kall = np.vstack((K, dom))
    Y64 = np.vstack((Y64, c + np.ldexp(dom.astype(np.float64), -16)))
    Y32 = np.vstack((Y32, c + np.ldexp(dom.astype(np.float64), -16)))
    _, ref = hx.from_grid(K[:1], R, c, 16)
    rk = L.rank_nd(Y64)
    assert np.count_nonzero(rk == 0) == K.shape[0] and np.all(rk[K.shape[0]:] > 0)
    assert not hx.mutually_nondominated(Y32[rk == 0])  # the rounding broke the front: the ranked entry must cope
    V = assert_exact_bounds(K, R, K.shape[0])  # the dominated rows add no volume (and too many cells)
    target = math.ldexp(float(V), -M * 16)
    assert hx.to_grid(Y32[: K.shape[0]], ref, c, 16)[2] == target
    assert np.array_equal(Y32[K.shape[0]:], c + np.ldexp(Kall[K.shape[0]:].astype(np.float64), -16))
    for env in routes(M):
        v = hv_env(L, monkeypatch, Y32, ref, env, rank=rk)
        assert v == target, (M, env, v, target, (v - target) / target, hx.hv2_strips_unclipped(Y32[rk == 0], ref) if M == 2 else None)
    assert L.hypervolume(Y32, ref) == target


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_ranked_arbitrary_sets_all_rank_zero(L, monkeypatch, M):
    """(b) Integer sets with strictly and weakly dominated rows and duplicates, every row passed with rank 0: whatever
    rows the ranked entry keeps, every route must give the exact volume."""
    rng = np.random.default_rng(800 + M)
    n = {1: 100, 2: 600, 3: 600, 4: 300, 5: 150, 6: 200, 7: 150, 8: 100}[M]
    Rv = 12 if M <= 5 else 6
    K = rng.integers(0, Rv, size=(n, M))
    K[: n // 5] = K[n // 2 : n // 2 + n // 5]  # duplicates
    K[n // 5 : n // 4] = K[n // 2 : n // 2 + n // 4 - n // 5]
    K[n // 5 : n // 4, 0] = np.minimum(K[n // 5 : n // 4, 0] + 1, Rv - 1)  # weakly dominated by the row they copy
    R = np.full(M, Rv, dtype=np.int64)
    if M > 1:
        assert not hx.mutually_nondominated(K.astype(np.float64))
    V = assert_exact_bounds(K, R, n)
    rk = np.zeros(n, dtype=np.int32)
    for c, e in GRIDS:
        P, ref = hx.from_grid(K, R, c, e)
        target = math.ldexp(float(V), -M * e)
        for env in routes(M):
            v = hv_env(L, monkeypatch, P, ref, env, rank=rk)
            assert v == target, (M, env, c, e, v, target)
        assert L.hypervolume(P, ref) == target


# ------------------------------------------------------------------------------------------ the fused step
def test_fused_step_float32_ties_two_objectives(L):
    """dmo_nsga2_step at M = 2 with round_to_f32=1, on a GP surrogate whose objective 0 varies by ~1e-10 around 1: the
    survivors rank in float64 on a trade-off front, and the float32 rounding collapses objective 0, so rank-0
    survivors tie with the worse objective 1 at a later index.  hv_out must equal the unranked (filtering) hypervolume
    of the rounded survivors, which is a single strip (r0 - 1) * (r1 - min f1)."""
    import dmosopt_b200 as b2

    rng = np.random.default_rng(21)
    d, M, pop = 5, 2, 2001
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((200, d))
    Ytr = np.column_stack((1.0 + 1e-10 * (Xtr[:, 0] + 0.3 * Xtr[:, 2]), 1.0 - Xtr[:, 0] + 0.2 * Xtr[:, 1] ** 2 + 0.1 * Xtr[:, 3]))
    sm = b2.GPR_Matern(Xtr, Ytr, d, M, xlb, xub, optimizer=None)
    x0 = rng.random((pop, d))
    y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
    ref = np.array([1.5, y0[:, 1].max() + 0.25])
    fx, fy, fr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    nch = np.zeros(1, dtype=np.int64)
    hv_f = ctypes.c_double(0.0)
    L._check(lib.dmo_nsga2_step(ctx, sm._gp._h, fx.ptr, fy.ptr, fr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr, dlb.ptr, dub.ptr,
                                31, 3, L.GP_FP64, 1, 0, 1, ref.ctypes.data, nch.ctypes.data, ctypes.byref(hv_f)), "nsga2_step")
    Yo, rk = fy.download(), fr.download()
    assert np.array_equal(Yo, Yo.astype(np.float32).astype(np.float64))
    z = np.flatnonzero(rk == 0)
    assert z.size >= 2 and np.all(Yo[:, 0] == 1.0), (z.size, np.unique(Yo[:, 0]))
    assert Yo[z[-1], 1] > Yo[z, 1].min()  # the worse objective 1 at the later index of the tie
    expect = (ref[0] - 1.0) * (ref[1] - Yo[:, 1].min())
    unclipped = hx.hv2_strips_unclipped(Yo[z], ref)
    assert L.hypervolume(Yo, ref) == expect
    assert hv_f.value == expect, (hv_f.value, expect, unclipped, (hv_f.value - expect) / expect)
