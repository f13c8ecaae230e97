"""oracle/hv_exact.py: the integer hypervolume algorithms agree with each other and with oracle/hv.py exactly, the value
moves with every front point, and the float32-tie sets meet their stated preconditions (CPU only)."""

import math
import time

import numpy as np
import pytest

from oracle import hv
from oracle import hv_exact as hx


def random_integer_set(M, n, rng, R=7):
    """Ties, duplicates, dominated rows, rows with a coordinate equal to R_j (outside: the filter is strict), +-0.0."""
    K = rng.integers(0, R, size=(n, M)).astype(np.float64)
    K[: n // 4] = K[n // 2 : n // 2 + n // 4]  # duplicates
    on = rng.random(n) < 0.15
    K[on, rng.integers(0, M, size=int(on.sum()))] = R
    K[K == 0] = np.where(rng.random(int((K == 0).sum())) < 0.5, -0.0, 0.0)
    return K, np.full(M, float(R))


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_algorithms_agree_on_random_integer_sets(M):
    rng = np.random.default_rng(40 + M)
    for trial in range(40):
        n = int(rng.integers(1, 13))
        K, R = random_integer_set(M, n, rng, R=int(rng.integers(2, 6)))
        v = hx.hv_cells(K, R)
        assert v == hx.hv_incl_excl(K, R), (M, trial)
        assert v == hx.hv_exact(K, R)
        assert float(v) == hv.hypervolume(K, R), (M, trial)
        if M == 2:
            assert v == hx.hv_staircase2(K, R)
        if M == 3:
            assert v == hx.hv_sweep3(K, R)
    for n in (40, 200):  # past inclusion-exclusion: cells against the sweep oracle of oracle/hv.py
        if M >= 6 and n > 40:
            continue
        K, R = random_integer_set(M, n, rng, R=6)
        assert float(hx.hv_cells(K, R)) == hv.hypervolume(K, R), (M, n)


def test_nothing_inside_and_boundary_rows_count_zero():
    R = np.array([3.0, 3.0, 3.0])
    assert hx.hv_cells(np.array([[3.0, 0.0, 0.0], [1.0, 3.0, 1.0]]), R) == 0
    assert hx.hv_sweep3(np.array([[3.0, 0.0, 0.0]]), R) == 0
    assert hx.hv_cells(np.array([[2.0, 2.0, 2.0]]), R) == 1
    assert hx.hv_cells(np.array([[-1.0, 0.0]]), np.array([1.0, 1.0])) == 2


@pytest.mark.parametrize("M,S", [(2, 300), (3, 40), (3, 89)])
def test_simplex_fronts_are_mutually_nondominated(M, S):
    T = hx.simplex(M, S)
    assert T.shape[0] == math.comb(S + M - 1, M - 1) and np.all(T.sum(axis=1) == S)
    if T.shape[0] <= 1000:
        assert hx.mutually_nondominated(T)


def test_staircase2_and_sweep3_agree_with_cells_at_the_gpu_sizes():
    rng = np.random.default_rng(3)
    N = 1 << 20  # the anti-diagonal front of the largest M = 2 case
    i = np.arange(N)
    K = np.column_stack((i, N - 1 - i))
    assert hx.hv_staircase2(K, np.array([N, N])) == N * (N + 1) // 2
    K2 = np.vstack((hx.simplex_front(2, 8192, rng, S=9000), rng.integers(0, 9001, size=(4000, 2))))
    assert hx.hv_staircase2(K2, np.array([9001, 9001])) == hx.hv_cells(K2, np.array([9001, 9001]))
    F3 = hx.simplex(3, 373)  # the ~70 000-point M = 3 front
    assert F3.shape[0] == 70125
    R3 = np.full(3, 374)
    assert hx.hv_sweep3(F3, R3) == hx.hv_cells(F3, R3)
    t0 = time.perf_counter()
    S = hx.sphere_lattice(256)
    v = hx.hv_cells(S, np.full(3, 257))
    elapsed = time.perf_counter() - t0
    assert S.shape[0] == 51722
    assert hx.hv_sweep3(S, np.full(3, 257)) == v
    assert elapsed < 30.0, elapsed
    perm = rng.permutation(S.shape[0])  # order-free
    assert hx.hv_sweep3(S[perm], np.full(3, 257)) == v


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_moving_any_front_point_down_one_unit_raises_the_value(M):
    """A front point moved one unit toward the origin along any axis gains a slab no other point covers: so a kernel
    that computes the volume of a perturbed set cannot pass an equality test by accident."""
    rng = np.random.default_rng(70 + M)
    K, R = random_integer_set(M, 10, rng, R=6)
    K = np.abs(K)
    v = hx.hv_cells(K, R)
    inside = np.all(K < R, axis=1)
    le = np.all(K[:, None, :] <= K[None, :, :], axis=2) & np.any(K[:, None, :] != K[None, :, :], axis=2)
    front = np.flatnonzero(inside & ~le.any(axis=0))
    assert front.size > 0
    for p in front:
        for j in range(M):
            K2 = K.copy()
            K2[p, j] -= 1
            w = hx.hv_cells(K2, R)
            assert w > v, (p, j)
            assert float(w) == hv.hypervolume(K2, R)


def test_grid_mapping_is_exact_and_checked():
    rng = np.random.default_rng(5)
    K = hx.simplex_front(3, 50, rng)
    R = np.full(3, K.max() + 2)
    for c, e in ((0.0, 0), (-0.75, 6), (-3.0, 20)):
        P, ref = hx.from_grid(K, R, c, e)
        K2, R2, target = hx.to_grid(P, ref, c, e)
        assert np.array_equal(np.sort(K2, axis=0), np.sort(K, axis=0)) and np.array_equal(R2, R)
        assert target == math.ldexp(float(hx.hv_exact(K, R)), -3 * e)
        assert abs(target - hv.hypervolume(P, ref)) <= 1e-12 * target
    with pytest.raises(AssertionError):
        hx.to_grid(np.array([[0.1, 0.2]]), np.array([1.0, 1.0]), 0.0, 4)
    assert hx.chain_sum_bound(257, np.zeros((1, 5)), np.full(5, 10)) == 257**3 * 10**5


@pytest.mark.parametrize("M", [2, 3, 5, 8])
@pytest.mark.parametrize("c", [1.0, -2.0])
def test_f32_tie_sets_meet_their_preconditions(M, c):
    rng = np.random.default_rng(M)
    Y64, Y32, K = hx.f32_tie_set(M, 40, 3, rng, c=c)
    assert hx.mutually_nondominated(Y64)
    assert np.array_equal(Y64.astype(np.float32).astype(np.float64), Y32)
    assert np.array_equal(Y32, c + np.ldexp(K.astype(np.float64), -16))
    # rounding makes rows tie in objective 0, and the worse objective 1 of a tie comes at the later row index
    later_worse = 0
    for i in range(Y32.shape[0] - 1):
        same = np.flatnonzero(Y32[i + 1 :, 0] == Y32[i, 0]) + i + 1
        later_worse += int(np.any(Y32[same, 1] > Y32[i, 1]))
    assert later_worse >= 40
    assert not hx.mutually_nondominated(Y32)


def test_the_unclipped_strip_sum_misses_float32_ties():
    """hv.cu's M = 2 strip sum as it stood before the running minimum: right on mutually non-dominated rows, too small
    on the rounded tie set (the ranked entry keeps every rank-0 row, rounded).  The running minimum is exact."""
    rng = np.random.default_rng(11)
    Y64, Y32, K = hx.f32_tie_set(2, 200, 4, rng)
    R = np.array([K[:, 0].max() + 3, K[:, 1].max() + 3])
    _, ref = hx.from_grid(K[:1], R, 1.0, 16)
    exact = hx.to_grid(Y32, ref, 1.0, 16)[2]
    assert abs(hx.hv2_strips_unclipped(Y64, ref) - hv.hypervolume(Y64, ref)) <= 1e-12 * exact
    wrong = hx.hv2_strips_unclipped(Y32, ref)
    assert wrong < exact * (1 - 1e-6), (wrong, exact)
    o = np.lexsort((np.arange(len(Y32)), Y32[:, 0]))
    x, ymin = Y32[o, 0], np.minimum.accumulate(Y32[o, 1])
    assert float(np.sum((np.append(x[1:], ref[0]) - x) * (ref[1] - ymin))) == exact
