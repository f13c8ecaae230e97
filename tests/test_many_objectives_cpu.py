"""Many-objective runs without a GPU: the NumPy restatement of the Monte-Carlo hypervolume estimators (oracle/hv_mc.py)
against exact volumes, and the optimizer plugins' objective limit."""

import itertools

import numpy as np
import pytest

from oracle import hv as ohv
from oracle import hv_mc


def exact_inclusion_exclusion(P, ref):
    """Volume of the union of the boxes [p, ref] by inclusion-exclusion (small n only)."""
    total = 0.0
    for k in range(1, len(P) + 1):
        for sub in itertools.combinations(range(len(P)), k):
            total += (-1) ** (k + 1) * np.prod(ref - P[list(sub)].max(axis=0))
    return total


def small_front(seed, n, M):
    rng = np.random.default_rng(seed)
    x = rng.random((n, M)) + 0.2
    return x / np.linalg.norm(x, axis=1, keepdims=True), np.full(M, 1.1)


@pytest.mark.parametrize("M", [3, 10])
def test_estimators_meet_epsilon_on_small_fronts(M):
    P, ref = small_front(M, 5, M)
    exact = exact_inclusion_exclusion(hv_mc.filtered_front(P, ref), ref)
    if M == 3:
        assert abs(exact - ohv.hypervolume(P, ref)) <= 1e-12 * exact
    eps = 0.1
    rng = np.random.default_rng(1)
    v, N, tests = hv_mc.fpras(P, ref, eps, 0.05, rng)
    assert abs(v - exact) <= eps * exact and tests == int(8 * (1 + eps) * 5 * np.log(2 / 0.05) / eps**2)
    v, N, S = hv_mc.mcm2rv(P, ref, eps, 0.05, rng)
    assert abs(v - exact) <= eps * exact and N >= S
    v = hv_mc.monte_carlo(P, ref, 20000, rng)
    assert abs(v - exact) <= 0.05 * exact


def test_single_point_and_filtering():
    ref = np.ones(10)
    p = np.full((1, 10), 0.5)
    rng = np.random.default_rng(0)
    assert hv_mc.fpras(p, ref, 0.2, 0.25, rng)[0] == pytest.approx(0.5**10, rel=0.0, abs=0.0)  # every xi is 1
    # dominated rows and rows outside ref do not reach the estimators
    F = np.vstack((p, p + 0.1, np.full((1, 10), 1.5)))
    assert np.array_equal(hv_mc.filtered_front(F, ref), p)


def test_moea_accepts_sixteen_sorted_objectives_and_refuses_seventeen():
    from dmosopt_b200 import MOEA

    assert MOEA.MAX_OBJECTIVES == 16

    class Probe(MOEA.MOEA):
        pass

    Probe("probe", 10, 3, 16)
    Probe("probe", 10, 3, 8, optimize_mean_variance=True)
    with pytest.raises(ValueError, match=r"17 objectives to sort .* at most 16"):
        Probe("probe", 10, 3, 17)
    with pytest.raises(ValueError, match=r"18 objectives to sort \(nOutput=9, doubled by optimize_mean_variance\)"):
        Probe("probe", 10, 3, 9, optimize_mean_variance=True)
