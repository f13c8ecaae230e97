"""The host certificate of the feasibility fit (oracle/feasibility_exact.py) without a GPU: its score and margin bounds
against exact rational evaluations, including a literal replay of the kernels' FMA order, and its KKT test on the
oracle's optimum and on that optimum moved by 1e-6."""

from fractions import Fraction

import numpy as np
import pytest

from dmosopt_b200.feasibility import pca_components, stratified_test_folds
from oracle import feasibility as of
from oracle import feasibility_exact as fx

TOL = 1e-11  # LogisticFeasibilityModel's default


def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def warp_sum(v):
    """common.cuh warp_sum: the xor butterfly over 32 lanes (lane 0's value; every lane ends with the same sum)."""
    v = list(v)
    o = 16
    while o:
        v = [v[i] + v[i ^ o] for i in range(32)]
        o >>= 1
    return v[0]


def kernel_score(x, mean, V, sm, ss, c):
    """feas_scores_kernel then feas_standardise_kernel for one row and column: the FMA chain over l, then (u - m) / s."""
    u = 0.0
    for l in range(len(x)):
        u = fma(V[c, l], float(np.float64(x[l]) - np.float64(mean[l])), u)
    return (u - float(sm[c])) / float(ss[c])


def kernel_margin(z, w, b):
    """feas_margin: lane l chains columns l, l + 32, ... by FMA, the butterfly sums the lanes, then + b."""
    lanes = []
    for lane in range(32):
        t = 0.0
        for c in range(lane, len(w), 32):
            t = fma(z[c], w[c], t)
        lanes.append(t)
    return warp_sum(lanes) + float(b)


def setup(d, N=400, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    m, V = pca_components(X)
    V = V[: d - 1]
    sm, ss = of.scaler((X - m) @ V.T)
    return rng, X, m, V, sm, ss


@pytest.mark.parametrize("d", [2, 33, 90])
def test_score_and_margin_bounds_hold_against_exact_rationals(d):
    rng, X, m, V, sm, ss = setup(d)
    far = m + rng.standard_normal((4, d)) * 1e3  # rows far from the PCA mean
    rows = np.vstack((X[:4], far))
    sc = fx.Scores(rows, m, V, sm, ss)
    k = d - 1
    w = rng.standard_normal(k) * np.logspace(-3, 3, k)
    w[::3] = 0.0
    b = 0.37
    cert_rows = sc.Z[:, :k]
    bt = (sc.bz[:, :k] @ np.abs(w) + fx.gamma(k + 1) * (np.abs(cert_rows) @ np.abs(w) + abs(b))) * fx.SAFE
    t_host = cert_rows @ w + b
    for i, x in enumerate(rows):
        zx = []
        for c in range(k):
            D = [Fraction(float(xl)) - Fraction(float(ml)) for xl, ml in zip(x, m)]
            U = sum(Fraction(float(V[c, l])) * D[l] for l in range(d))
            zx.append((U - Fraction(float(sm[c]))) / Fraction(float(ss[c])))
            assert abs(Fraction(float(sc.Z[i, c])) - zx[c]) <= Fraction(float(sc.bz[i, c])), (i, c)
            kz = kernel_score(x, m, V, sm, ss, c)
            assert abs(Fraction(kz) - zx[c]) <= Fraction(float(sc.bz[i, c])), (i, c, "kernel order")
        # the margin of the exact scores, against the host margin of the host scores and the kernel's of its own
        t_exact = sum(zc * Fraction(float(wc)) for zc, wc in zip(zx, w)) + Fraction(b)
        assert abs(Fraction(float(t_host[i])) - t_exact) <= Fraction(float(bt[i])), i
        tk = kernel_margin([kernel_score(x, m, V, sm, ss, c) for c in range(k)], w, b)
        assert abs(Fraction(tk) - t_exact) <= Fraction(float(bt[i])), (i, "kernel order")
        # the bound is not vacuous: a few hundred ulps of the margin's terms at most
        assert bt[i] <= 1e-12 * (np.abs(cert_rows[i]) @ np.abs(w) + abs(b))


@pytest.mark.parametrize("d", [2, 33])
def test_scaler_bounds_hold_against_exact_rationals(d):
    rng, X, m, V, sm, ss = setup(d, N=300, seed=d)
    sc = fx.Scores(X, m, V, sm, ss)
    mh, bm, var, bvar, sd, bsd = fx.scaler(sc.U, sc.bU)
    for c in range(min(d - 1, 4)):
        U = [sum(Fraction(float(V[c, l])) * (Fraction(float(x[l])) - Fraction(float(m[l]))) for l in range(d)) for x in X]
        me = sum(U) / len(U)
        ve = sum((u - me) ** 2 for u in U) / len(U)
        assert abs(Fraction(float(mh[c])) - me) <= Fraction(float(bm[c]))
        # var about the exact mean is the smallest over centres, so the bound on var about m covers it from above
        assert abs(Fraction(float(var[c])) - ve) <= Fraction(float(bvar[c]))
    assert fx.scaler_agrees(sm, ss, sc.U, sc.bU).all()
    assert not fx.scaler_agrees(sm, ss * (1 + 1e-9), sc.U, sc.bU).any()
    assert not fx.scaler_agrees(sm + 1e-9 * ss, ss, sc.U, sc.bU).any()


def test_scaler_rule_on_a_constant_column():
    U = np.full((50, 1), 0.3)
    U[7] = np.nextafter(0.3, 1.0)  # constant to rounding: scale exactly 1
    bU = np.zeros_like(U)
    m, _, _, _, _, _ = fx.scaler(U, bU)
    assert fx.scaler_agrees(m, np.ones(1), U, bU).all()
    assert not fx.scaler_agrees(m, np.array([np.sqrt(np.var(U))]), U, bU).any()


def _problem(d=6, N=200, seed=1, k=4):
    rng = np.random.default_rng(seed)
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    a = X @ rng.standard_normal(d)
    c = (a > np.quantile(a, 0.4)) ^ (rng.random(N) < 0.1)
    folds = stratified_test_folds(c.astype(int))
    tr = folds != 2
    m, V = pca_components(X[tr])
    V = V[: d - 1]
    sm, ss = of.scaler(((X - m) @ V.T)[tr])
    sc = fx.Scores(X, m, V, sm, ss)
    return sc, c.astype(int), tr, k


@pytest.mark.parametrize("C,k", [(0.05, 5), (1.0, 4), (100.0, 4)])
def test_certificate_accepts_the_oracle_optimum_and_rejects_it_moved(C, k):
    sc, y, tr, _ = _problem(k=k)
    d = sc.Z.shape[1] + 1
    w, b, F = of.l1_logistic(sc.Z[tr, :k], y[tr], C)
    row = np.zeros(d)
    row[:k], row[d - 1] = w, b
    cert = fx.Certificate(sc, y, tr, ~tr, C, [k], row[None])
    assert cert.accepts(TOL)[0], (cert.kkt, cert.bk, cert.gtol_of(TOL))
    assert abs(cert.F[0] - F) <= 1e-12 * F
    cor = int(np.count_nonzero((sc.Z[~tr, :k] @ w + b > 0) == (y[~tr] > 0)))
    assert cert.lo[0] <= cor <= cert.lo[0] + cert.amb[0]
    assert cert.amb[0] == 0
    nz, z = np.flatnonzero(w != 0.0), np.flatnonzero(w == 0.0)
    assert nz.size, "the optimum has no non-zero coefficient to move"
    assert z.size or C > 0.05, "the small-C optimum has no zero coefficient to move"
    for c in nz:
        moved = row.copy()
        moved[c] *= 1 + 1e-6
        assert fx.Certificate(sc, y, tr, ~tr, C, [k], moved[None]).rejects(TOL)[0], ("non-zero", c)
    for c in z:
        moved = row.copy()
        moved[c] = 1e-6
        assert fx.Certificate(sc, y, tr, ~tr, C, [k], moved[None]).rejects(TOL)[0], ("zero", c)
    moved = row.copy()
    moved[d - 1] *= 1 + 1e-6
    assert fx.Certificate(sc, y, tr, ~tr, C, [k], moved[None]).rejects(TOL)[0], "intercept"


def test_certificate_at_w_zero_and_batched_over_k():
    """The batched certificate of several k equals the one-at-a-time certificate, and at w = 0 the objective is
    C n log 2 and the gradient C sum (1/2 - y) [z, 1]."""
    sc, y, tr, _ = _problem()
    d = sc.Z.shape[1] + 1
    ks = np.arange(1, d)
    rng = np.random.default_rng(3)
    rows = np.zeros((d - 1, d))
    for j, k in enumerate(ks):
        rows[j, :k] = rng.standard_normal(k)
        rows[j, d - 1] = rng.standard_normal()
    both = fx.Certificate(sc, y, tr, ~tr, 2.0, ks, rows)
    for j, k in enumerate(ks):
        one = fx.Certificate(sc, y, tr, ~tr, 2.0, [k], rows[j:j + 1])
        assert np.allclose(one.F, both.F[j], rtol=1e-14) and np.allclose(one.kkt, both.kkt[j], rtol=1e-12)
        assert one.lo[0] == both.lo[j] and one.amb[0] == both.amb[j]
    zero = fx.Certificate(sc, y, tr, None, 2.0, ks, np.zeros((d - 1, d)))
    n = np.count_nonzero(tr)
    assert np.allclose(zero.F, 2.0 * n * np.log(2.0), rtol=1e-14)
    assert np.allclose(zero.g[0][1], 2.0 * np.sum(0.5 - y[tr]), rtol=1e-12, atol=1e-12)
