"""Good-lattice-point search and discrepancies, host side (dmosopt_b200/sampling.py, discrepancy.py, oracle/sampling.py):
candidate enumeration, branch choice, generator consumption and decorrelation against the reference's fixtures, and
the shortlist + exact-pass selection with the GPU's two entry points replaced by NumPy; no GPU needed."""

import math

import numpy as np
import pytest

from dmosopt_b200 import discrepancy, sampling
from oracle import sampling as osm

def _exact_terms(H, N, rows):
    """NumPy stand-in for dmo_glp_cd2_terms: D2, D3 of each lattice (reference order)."""
    out = np.array([osm.cd2_terms(osm.design(h, N, rows)) for h in H]).reshape(-1, 2)
    return out[:, 0].copy(), out[:, 1].copy()


def _exact_pairs(H, N, rows):
    """NumPy stand-in for dmo_glp_cd2_pairs: the reference's pair products, row-major."""
    P = []
    for h in H:
        X = osm.design(h, N, rows)
        p = np.ones((rows, rows))
        for i in range(X.shape[1]):
            x, y = X[:, i][:, None], X[:, i][None, :]
            p = p * (1 + 0.5 * np.abs(x - 0.5) + 0.5 * np.abs(y - 0.5) - 0.5 * np.abs(x - y))
        P.append(p.ravel())
    return np.array(P)


@pytest.fixture
def host_gpu(monkeypatch):
    """Route the two GPU entry points of the search to NumPy; ``perturb(d2, d3, H, N, rows)`` may disturb the
    screened terms."""
    state = {"perturb": None, "shortlists": []}

    def terms(H, N, rows):
        d2, d3 = _exact_terms(H, N, rows)
        return state["perturb"](d2, d3, H, N, rows) if state["perturb"] else (d2, d3)

    monkeypatch.setattr(sampling._lib, "glp_cd2_terms", terms)
    monkeypatch.setattr(sampling._lib, "glp_cd2_pairs", _exact_pairs)
    real = sampling.select

    def select(H, N, rows):
        best, short = real(H, N, rows)
        state["shortlists"].append(short)
        return best, short

    monkeypatch.setattr(sampling, "select", select)
    return state


def _cases(golden):
    g = golden("sampling")
    return g, [tuple(int(v) for v in c) for c in g["glp_cases"]]


# ------------------------------------------------------------------------------------------ enumeration and branch
def test_euler_phi_matches_the_oracle_float_totient():
    for n in range(2, 3000):
        assert sampling.euler_phi(n) == osm.euler(n), n


@pytest.mark.parametrize("n,s", [(13, 3), (12, 3), (12, 1), (2, 3), (60, 6), (61, 5), (90, 30), (100, 10), (299, 30), (800, 80), (600, 60), (1000, 100)])
def test_candidates_match_the_oracle(n, s):
    N, rows, H = sampling.candidates(n, s)
    oN, orows, oH = osm.candidates(n, s)
    assert (N, rows) == (oN, orows)
    assert H.dtype == np.int64 and np.array_equal(H, oH)


def test_branch_choice():
    assert sampling.candidates(13, 3)[:2] == (13, 13)  # phi 12 / 13 >= 0.9, column combinations
    N, rows, H = sampling.candidates(12, 3)  # phi 4 / 12 < 0.9: lattice 13 without its last point
    assert (N, rows) == (13, 12) and H.shape == (math.comb(12, 3), 3)
    N, rows, H = sampling.candidates(60, 6)  # plusone, power vectors of 61
    assert (N, rows) == (61, 60) and np.all(H[:, 0] == 1) and np.array_equal(H[:, 1], np.sort(H[:, 1]))
    assert sampling.candidates(90, 30)[2].shape == (0, 30)  # lattice 91 has group exponent 12 < 30
    assert sampling.candidates(1000, 100)[2].shape[0] == 0  # lattice 1001, exponent 60


def test_reference_modules_agree_where_present():
    from oracle import reference_build

    ref = reference_build.reference_path()
    if ref is None:
        pytest.skip("reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
    import sys

    sys.path.insert(0, ref)
    try:
        from dmosopt import GLP
    finally:
        sys.path.remove(ref)
    for n in range(2, 400):
        assert sampling.euler_phi(n) == GLP.EulerFunction(n)
    for N, s in [(61, 6), (101, 10), (91, 30), (301, 30), (97, 2)]:
        assert np.array_equal(sampling.power_vectors(N, s), GLP.PowerGenVector(N, s).astype(np.int64))
    for N in (11, 13, 20, 61):
        h = GLP.GenVector(N)
        assert np.array_equal(sampling.column_vectors(N, 1, len(h))[:, 0], h)


@pytest.mark.parametrize("n,s,why", [(1, 3, "n >= 2"), (0, 3, "n >= 2"), (61, 1, "s >= 2"), (100, 1, "s >= 2"), (13, 0, "at least one dimension")])
def test_inputs_the_reference_cannot_take_are_refused(n, s, why):
    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match=why):
        sampling.glp(n, s, rng)
    assert np.array_equal(rng.random(3), np.random.default_rng(0).random(3))  # nothing drawn


# ------------------------------------------------------------------------------------------ against the fixtures
def test_designs_draws_and_decorrelation_match_the_fixtures(golden, host_gpu):
    g, cases = _cases(golden)
    for c, (n, s, maxiter, seed) in enumerate(cases):
        if n * n * s > 150 * 150 * 10:
            continue
        rng = np.random.default_rng(seed)
        X = sampling.glp(n, s, rng, maxiter=maxiter)
        assert X.dtype == np.float64 and X.flags.c_contiguous
        assert X.shape == g[f"glp_{c}"].shape and np.array_equal(X, g[f"glp_{c}"]), (n, s, maxiter)
        assert np.array_equal(rng.random(4), g[f"glp_{c}_next"]), (n, s, maxiter)


def test_no_candidate_returns_the_discarded_draw(golden):
    g, cases = _cases(golden)
    c = cases.index((90, 30, 0, 13))
    X = sampling.glp(90, 30, np.random.default_rng(13))  # no candidate: no GPU call
    assert X.shape == (91, 30) and np.array_equal(X, g[f"glp_{c}"])
    c = cases.index((2, 3, 0, 6))
    assert np.array_equal(sampling.glp(2, 3, np.random.default_rng(6)), g[f"glp_{c}"])


def test_decorrelation_of_the_discarded_draw_matches(golden):
    g, cases = _cases(golden)
    c = cases.index((90, 30, 5, 14))
    rng = np.random.default_rng(14)
    assert np.array_equal(sampling.glp(90, 30, rng, maxiter=5), g[f"glp_{c}"])
    assert np.array_equal(rng.random(4), g[f"glp_{c}_next"])


def test_oracle_discrepancies_match_the_fixtures(golden):
    g = golden("sampling")
    for i in range(int(g["disc_count"])):
        X, ref = g[f"disc_{i}_X"], g[f"disc_{i}"]
        got = [osm.md2(X), osm.cd2(X), osm.sd2(X), osm.wd2(X)]
        assert got == list(ref[:4]), i  # the oracle keeps the reference's operation order: bit for bit
        assert discrepancy.MinDist(X) == ref[4]
        np.testing.assert_array_equal(discrepancy.corrscore(X), ref[5])


def test_oracle_glp_matches_the_fixtures(golden):
    g, cases = _cases(golden)
    for c, (n, s, maxiter, seed) in enumerate(cases):
        if maxiter == 0 and n * n * s <= 150 * 150 * 10:
            assert np.array_equal(osm.glp(n, s, np.random.default_rng(seed)), g[f"glp_{c}"]), (n, s)


def test_mindist_counts_the_zero_self_distance():
    X = np.random.default_rng(1).random((30, 4))
    assert discrepancy.MinDist(X) == 0.0
    assert discrepancy.MinDist(np.zeros((0, 3))) == 1e32


# ------------------------------------------------------------------------------------------ shortlist and exact pass
def test_screen_margin_covers_the_oracle_reordered_sums():
    """A different summation order (NumPy's pairwise sums) stays within half the margin."""
    N, rows, H = sampling.candidates(100, 10)
    D1 = (13.0 / 12.0) ** 10
    for h in H[:10]:
        X = osm.design(h, N, rows)
        d2, d3 = osm.cd2_terms(X)
        A = np.abs(X - 0.5)
        p2 = np.prod(1 + 0.5 * A - 0.5 * A * A, axis=1).sum()
        P = np.ones((rows, rows))
        for i in range(10):
            P *= 1 + 0.5 * A[:, i][:, None] + 0.5 * A[:, i][None, :] - 0.5 * np.abs(X[:, i][:, None] - X[:, i][None, :])
        p3 = P.sum()
        t2, t3 = 2 * d2 / rows, d3 / rows**2
        m = sampling.screen_margin(D1, t2, t3, rows, 10)
        assert abs((D1 - t2 + t3) - (D1 - 2 * p2 / rows + p3 / rows**2)) <= m / 2


@pytest.mark.parametrize("n,s", [(60, 6), (40, 5), (13, 3)])
def test_selection_survives_screening_errors_within_the_margin(host_gpu, n, s):
    """Screened terms disturbed adversarially within the margin: the exact pass still picks the oracle's index."""
    N, rows, H = sampling.candidates(n, s)
    best, d = osm.select(H, N, rows)
    D1 = (13.0 / 12.0) ** s

    def perturb(d2, d3, H, N, rows):
        t2, t3 = 2 * d2 / rows, d3 / rows**2
        m = sampling.screen_margin(D1, t2, t3, rows, s)
        sign = np.where(np.arange(d3.shape[0]) == best, 1.0, -1.0)  # the winner looks worse, every other better
        return d2, d3 + 0.45 * sign * m * rows**2

    host_gpu["perturb"] = perturb
    got, short = sampling.select(H, N, rows)
    assert got == best
    assert best in short and np.all(np.diff(short) > 0)


def test_exact_ties_keep_the_first_candidate(host_gpu):
    N, rows, H = sampling.candidates(60, 6)
    best, _ = osm.select(H[:8], N, rows)
    Hd = H[[best, 0, 1, 2, 3, 4, 5, 6, 7]]  # the winner twice: positions 0 and best + 1
    assert sampling.select(Hd, N, rows)[0] == 0
    Hd = H[list(range(8)) + [best]]
    assert sampling.select(Hd, N, rows)[0] == best


def test_exact_pass_is_the_reference_cd2(host_gpu):
    N, rows, H = sampling.candidates(60, 6)
    got = sampling._exact_cd2(H[:5], N, rows, 6)
    assert list(got) == [osm.cd2(osm.design(h, N, rows)) for h in H[:5]]
