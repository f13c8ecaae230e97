"""DGSM and eFAST (oracle/sa.py and the host parts of dmosopt_b200/sa.py) on closed-form cases; no GPU needed."""

import math

import numpy as np
import pytest

from oracle import sa


def _dgsm(f, lb, ub, N=2048, R=100, seed=0):
    X = sa.dgsm_design(sa.dgsm_base(N, len(lb)), lb, ub)
    idx = np.random.default_rng(seed).integers(0, N, size=(R, N))
    return X, sa.dgsm_stats(X, f(X), lb, ub, idx)


def test_dgsm_linear_function_on_the_unit_box():
    a = np.array([3.0, -1.0, 0.5, 0.0, 2.0])
    d = a.shape[0]
    lb, ub = np.zeros(d), np.ones(d)
    X, st = _dgsm(lambda X: (X @ a)[:, None], lb, ub)
    # the difference quotient of a linear function is its slope: vi_j = a_j^2, vi_std = 0 up to rounding
    assert np.allclose(st["vi"][0], a**2, rtol=1e-10, atol=1e-12)
    assert np.all(st["vi_std"][0] <= 1e-9 * np.maximum(a**2, 1))
    var_f = np.var((X @ a).reshape(-1, d + 1)[:, 0])
    assert np.allclose(st["dgsm"][0], a**2 / (np.pi**2 * var_f), rtol=1e-10, atol=1e-14)
    assert st["dgsm"][0, 3] == 0.0 and st["conf"][0, 3] == 0.0
    assert np.all(st["conf"][0] >= 0) and np.all(np.isfinite(st["conf"]))


def test_dgsm_scales_with_the_bounds():
    """On the box [lb, ub] the slope of f = sum a_j x_j is a_j in x, and dgsm carries the squared range."""
    a = np.array([1.0, 2.0, -3.0])
    lb, ub = np.array([-1.0, 0.0, 2.0]), np.array([1.0, 10.0, 2.5])
    X, st = _dgsm(lambda X: np.column_stack([X @ a, np.sin(X[:, 0])]), lb, ub)
    assert np.allclose(st["vi"][0], a**2, rtol=1e-9)
    var_f = np.var((X @ a).reshape(-1, 4)[:, 0])
    assert np.allclose(st["dgsm"][0], a**2 * (ub - lb) ** 2 / (np.pi**2 * var_f), rtol=1e-9)
    # the second output depends on x0 only
    assert st["vi"][1, 0] > 0 and np.all(st["vi"][1, 1:] == 0)


def test_dgsm_bootstrap_confidence_is_the_replicate_spread():
    from scipy.stats import norm

    rng = np.random.default_rng(3)
    d, N, R = 3, 256, 50
    lb, ub = np.zeros(d), np.ones(d)
    X = sa.dgsm_design(sa.dgsm_base(N, d), lb, ub)
    Y = (np.sin(3 * X[:, 0]) + X[:, 1] ** 2)[:, None]
    idx = rng.integers(0, N, size=(R, N))
    st = sa.dgsm_stats(X, Y, lb, ub, idx)
    # replicate 0 by hand
    Xr, Yr = X.reshape(N, d + 1, d), Y.reshape(N, d + 1)
    for j in range(2):
        q2 = ((Yr[:, 1 + j] - Yr[:, 0]) / (Xr[:, 1 + j, j] - Xr[:, 0, j])) ** 2
        reps = [np.mean(q2[r]) / (np.var(Yr[r, 0]) * np.pi**2) for r in idx]
        assert math.isclose(st["conf"][0, j], norm.ppf(0.975) * np.std(reps, ddof=1), rel_tol=1e-12)
    # an index set equal to the identity in every replicate leaves no spread
    st0 = sa.dgsm_stats(X, Y, lb, ub, np.tile(np.arange(N), (R, 1)))
    assert np.all(st0["conf"] <= 1e-12 * st0["dgsm"])


def test_dgsm_design_rows():
    N, d = 5, 3
    lb, ub = np.array([0.0, -2.0, 1.0]), np.array([1.0, 2.0, 3.0])
    B = sa.dgsm_base(N, d)
    X = sa.dgsm_design(B, lb, ub)
    assert X.shape == (N * (d + 1), d)
    # the base rows are the unscrambled Sobol points 1024, 1025, ...
    from scipy.stats import qmc

    s = qmc.Sobol(d, scramble=False)
    s.fast_forward(1024)
    assert np.array_equal(B[0], s.random(1)[0])
    assert np.array_equal(X[0], B[0] * (ub - lb) + lb)
    assert np.array_equal(X[1], (B[0] + [0.01, 0, 0]) * (ub - lb) + lb)
    last = B[-1].copy()
    last[-1] += 0.01
    assert np.array_equal(X[-1], last * (ub - lb) + lb)
    Xr = X.reshape(N, d + 1, d)
    for j in range(d):
        step = Xr[:, 1 + j, :] - Xr[:, 0, :]
        assert np.allclose(step[:, j], 0.01 * (ub[j] - lb[j]), rtol=1e-12)
        assert np.all(np.delete(step, j, axis=1) == 0)


def test_fast_frequencies_hand_computed():
    # N 1000: omega_0 = floor(999 / 8) = 124, m = floor(124 / 8) = 15
    assert np.array_equal(sa.fast_frequencies(1000, 1), [124])
    assert np.array_equal(sa.fast_frequencies(1000, 4), [124, 1, 8, 15])  # m >= d - 1: floor(linspace(1, 15, 3))
    w = sa.fast_frequencies(1000, 20)  # m < d - 1: arange(19) % 15 + 1
    assert np.array_equal(w, [124] + list(range(1, 16)) + [1, 2, 3, 4])
    assert np.array_equal(sa.fast_frequencies(65, 3), [8, 1, 1])  # the smallest N: m = 1
    with pytest.raises(ValueError, match="N > 4 M"):
        sa.fast_frequencies(64, 3)


def test_fast_design_rows():
    N, d = 100, 3
    lb, ub = np.array([0.0, -1.0, 5.0]), np.array([1.0, 1.0, 6.0])
    w = sa.fast_frequencies(N, d)  # [12, 1, 1]
    phi = np.array([0.3, 1.7, 4.0])
    X = sa.fast_design(N, w, phi, lb, ub)
    assert X.shape == (N * d, d)
    # first row: s_0 = 0, every column is 0.5 + arcsin(sin(phi_0)) / pi
    x0 = 0.5 + np.arcsin(np.sin(phi[0])) / np.pi
    assert np.allclose(X[0], x0 * (ub - lb) + lb, rtol=0, atol=1e-15)
    # last row: block 2 (parameter 2 at omega_0 = 12), k = 99
    s = 2 * np.pi / N * 99
    wl = np.array([1.0, 1.0, 12.0])
    xl = 0.5 + np.arcsin(np.sin(wl * s + phi[2])) / np.pi
    assert np.allclose(X[-1], xl * (ub - lb) + lb, rtol=0, atol=1e-14)
    assert np.all(X >= lb) and np.all(X <= ub)


def test_triangle_wave_is_arcsin_of_sin():
    rng = np.random.default_rng(5)
    th = np.concatenate([rng.random(100000) * 1e4, (np.arange(1, 2000) * np.pi / 2)])  # and the peaks themselves
    lit = np.arcsin(np.sin(th))
    tri = sa.triangle(th)
    assert np.all(np.abs(tri) <= np.pi / 2)
    # as written, arcsin(sin(.)) amplifies sin's last-bit error as 1 / cos: within that conditioning bound everywhere
    bound = 4e-16 * np.maximum(th, 1) / np.maximum(np.abs(np.cos(th)), 1e-8) + 3e-8 * (np.abs(np.cos(th)) < 1e-7)
    assert np.all(np.abs(tri - lit) <= bound + 1e-15)
    assert np.median(np.abs(tri - lit)) <= 1e-15


def test_fast_additive_function_s1_equals_st():
    N, d = 4001, 4
    lb, ub = np.zeros(d), np.ones(d)
    w = sa.fast_frequencies(N, d)
    phi = 2 * np.pi * np.random.default_rng(0).random(d)
    X = sa.fast_design(N, w, phi, lb, ub)
    Y = (X[:, 0] + 2 * X[:, 1] + 0.5 * X[:, 2] ** 2)[:, None]  # parameter 3 does not enter
    S1, ST = sa.fast_indices(Y, N, d)
    assert np.all(np.abs(S1 - ST)[:, :3] < 1e-2), (S1, ST)
    assert S1[0, 3] < 1e-3
    # the closed-form first-order indices of the additive function (variances 1/12, 4/12 and 0.25 * 4/45)
    v = np.array([1 / 12, 4 / 12, 0.25 * 4 / 45])
    assert np.allclose(S1[0, :3], v / v.sum(), atol=2e-2)


def test_product_host_parts_follow_the_oracle():
    from dmosopt_b200.sa import SA_DGSM, SA_FAST

    names = ["a", "b", "c", "e"]
    lb, ub = np.zeros(4), np.ones(4)
    dg = SA_DGSM(lb, ub, names, ["y"])
    assert np.array_equal(dg.base_points(300), sa.dgsm_base(300, 4))
    fa = SA_FAST(lb, ub, names, ["y0", "y1"], seed=1)
    for N in (65, 1000, 10000):
        assert np.array_equal(fa.frequencies(N), sa.fast_frequencies(N, 4))
    N = 1001
    rng = np.random.default_rng(2)
    Y = rng.standard_normal((N * 4, 2)) + np.repeat(np.arange(4.0), N)[:, None]
    S1, ST = fa.indices(Y, N)
    o1, oT = sa.fast_indices(Y, N, 4)
    assert np.allclose(S1, o1, rtol=1e-12, atol=1e-15) and np.allclose(ST, oT, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("N", [1, 64])
def test_fast_sample_needs_more_than_4m2_points(N):
    from dmosopt_b200.sa import SA_FAST

    fa = SA_FAST([0, 0], [1, 1], ["a", "b"], ["y"])
    with pytest.raises(ValueError, match="4 M\\^2 = 64"):
        fa.sample(N)


def test_constructor_checks_the_bounds():
    from dmosopt_b200.sa import SA_DGSM

    with pytest.raises(ValueError, match="3 parameter names"):
        SA_DGSM([0, 0], [1, 1], ["a", "b", "c"], ["y"])
