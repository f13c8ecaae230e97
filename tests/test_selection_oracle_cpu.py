"""The selection oracles against themselves, without a GPU: the scipy EHVI against the mpmath one within
``oracle.hv.ehvi_bound`` (the bound the GPU scores are held to), the vectorised crowding distance against the literal
loops on every data kind of the GPU suite, NaN and +-inf included, and the stable box order of ``decompose_boxes``."""

import numpy as np
import pytest
from scipy.stats import norm

from oracle import hv as ohv
from oracle import indicators
from test_gpu_selection_exact import DIST_KINDS, distance_data, ehvi_candidates, ehvi_front


def term_magnitude(lower, upper, means, variances):
    """sum_b prod_j (s (phi_l + phi_u) + |mu| (Phi_l + Phi_u)): the size of each factor's terms before they cancel."""
    out = np.zeros(means.shape[0])
    for c in range(means.shape[0]):
        with np.errstate(all="ignore"):
            sd = np.sqrt(variances[c])
            zl, zu = (lower - means[c]) / sd, (upper - means[c]) / sd
        cl = np.where(np.isinf(lower), 0.0, norm.cdf(zl))
        cu = np.where(np.isinf(upper), 1.0, norm.cdf(zu))
        out[c] = np.sum(np.prod(sd * (norm.pdf(zl) + norm.pdf(zu)) + np.abs(means[c]) * (cl + cu), axis=1))
    return out


@pytest.mark.parametrize("M,nb", ((1, 1), (1, 65), (2, 2), (2, 64), (3, 65), (8, 9), (9, 3), (16, 2)))
def test_scipy_ehvi_within_the_bound_of_mpmath(M, nb):
    F, ref = ehvi_front(M, nb, seed=7 * M + nb)
    mu, var = ehvi_candidates(F, ref, 12, seed=M)
    lo, up = ohv.decompose_boxes(F, ref)
    assert lo.shape[0] == nb
    o = ohv.batch_ehvi(lo, up, mu, var)
    m = ohv.ehvi_mp(lo, up, mu, var)
    B = ohv.ehvi_bound(lo, up, mu, var)
    nan = np.isnan(m)
    assert nan[[1, 3]].all() and not nan[[0, 2, 4, 5, 6]].any()  # on a bound with zero variance, negative variance
    assert np.array_equal(np.isnan(o), nan) and np.array_equal(np.isnan(B), nan)
    assert np.all(np.abs(o - m)[~nan] <= B[~nan])
    # the bound is tight: at most 64 (nb + M) EPS times the size the terms have before any cancellation (room for the
    # 5-ulp Phi and the propagated z error), and scipy's actual error reaches a visible fraction of it
    S = term_magnitude(lo, up, mu, var)
    assert np.all(B[~nan] <= 64 * (nb + M) * ohv.EPS * S[~nan] + 1e-300)
    r = np.abs(o - m)[~nan & (B > 0)] / B[~nan & (B > 0)]
    assert r.max() >= 5e-4, r.max()


@pytest.mark.parametrize("kind", DIST_KINDS)
@pytest.mark.parametrize("M", (1, 2, 3, 8, 9, 16))
def test_crowding_metric_equals_the_loops(M, kind):
    for n in (1, 2, 3, 40, 257):
        Y = distance_data(kind, n, M, seed=1000 * M + n)
        assert np.array_equal(indicators.crowding_distance_metric(Y), indicators.crowding_distance_loops(Y)), n


def test_crowding_puts_nan_last():
    # an infinite objective normalises to NaN ((inf - lb) / inf) and the finite rows to 0; sorted last, the infinite row
    # gets an end contribution of 1.0, its sorted neighbour a NaN difference (a NaN sum counts as 0)
    Y = np.array([[0.0, 3.0], [1.0, 2.0], [np.inf, 1.0], [2.0, 0.0]])
    for f in (indicators.crowding_distance_metric, indicators.crowding_distance_loops):
        assert np.array_equal(f(Y), [1.0 + 1.0, 0.0 + (1.0 - 1.0 / 3.0), (2.0 / 3.0 - 0.0) + 1.0, 0.0])
        # a NaN objective makes its whole column NaN, whatever the NaN's sign
        P, N = Y.copy(), Y.copy()
        P[1, 0], N[1, 0] = np.nan, -np.nan
        assert np.array_equal(f(P), f(N))


def test_decompose_boxes_keeps_f0_ties_in_row_order():
    F = np.array([[1.0, 5.0], [2.0, 3.0], [1.0, 4.0], [2.0, 2.0], [3.0, 1.0]])
    ref = np.array([4.0, 6.0])
    lo, up = ohv.decompose_boxes(F, ref)
    o = np.array([0, 2, 1, 3, 4])  # rows by f0, equal f0 in row order
    low = np.vstack((np.full((1, 2), -np.inf), F[o]))
    upp = np.vstack((F[o], ref))
    keep = np.all(upp > low, axis=1)
    assert np.array_equal(lo, low[keep]) and np.array_equal(up, upp[keep])
    # the tie order matters: swapping the tied rows changes the boxes
    lo2, up2 = ohv.decompose_boxes(F[[2, 1, 0, 3, 4]], ref)
    assert not (lo2.shape == lo.shape and np.array_equal(lo2, lo) and np.array_equal(up2, up))
    # and on the generator's fronts (ties between a chain point and a point above it) the count is the chosen one
    for M in (1, 2, 3, 9):
        for nb in (1, 2, 63, 64, 65, 128, 129):
            F, ref = ehvi_front(M, nb, seed=M + nb)
            assert ohv.decompose_boxes(F, ref)[0].shape[0] == nb
