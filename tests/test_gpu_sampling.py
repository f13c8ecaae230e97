"""Good-lattice-point search and L2 discrepancies on the GPU (csrc/design.cu, dmosopt_b200/sampling.py, discrepancy.py):
the designs bit for bit against the reference's fixtures, the screening kernel and the exact pass against
oracle/sampling.py at n 300 - 800 and s 30 - 80, the envelope refusals, and MOASMO.xinit of the unmodified reference."""

import sys

import numpy as np
import pytest

from oracle import sampling as osm

pytestmark = pytest.mark.gpu

METRICS = ("MD2", "CD2", "SD2", "WD2")
ORACLE = {"MD2": osm.md2, "CD2": osm.cd2, "SD2": osm.sd2, "WD2": osm.wd2}


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _reference():
    from oracle import reference_build

    return reference_build.reference_path()


def _import_ref(name):
    ref = _reference()
    sys.path.insert(0, ref)
    try:
        import importlib

        return importlib.import_module(f"dmosopt.{name}")
    finally:
        sys.path.remove(ref)


# ------------------------------------------------------------------------------------------ designs
def test_glp_is_bitwise_the_reference_on_every_fixture(L, golden):
    from dmosopt_b200 import sampling

    g = golden("sampling")
    for c, case in enumerate(g["glp_cases"]):
        n, s, maxiter, seed = (int(v) for v in case)
        rng = np.random.default_rng(seed)
        X = sampling.glp(n, s, rng, maxiter=maxiter)
        assert X.shape == g[f"glp_{c}"].shape and np.array_equal(X, g[f"glp_{c}"]), (n, s, maxiter)
        assert np.array_equal(rng.random(4), g[f"glp_{c}_next"]), (n, s, maxiter)


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("n,s,maxiter", [(30, 5, 0), (45, 4, 5), (16, 3, 0), (71, 7, 0), (18, 2, 5)])
def test_glp_is_bitwise_the_reference_package(L, n, s, maxiter):
    from dmosopt_b200 import sampling

    ref = _import_ref("sampling")
    a, b = np.random.default_rng(n), np.random.default_rng(n)
    assert np.array_equal(sampling.glp(n, s, a, maxiter=maxiter), ref.glp(n, s, b, maxiter=maxiter))
    assert np.array_equal(a.random(4), b.random(4))


def test_repeated_calls_are_bit_identical(L):
    from dmosopt_b200 import sampling

    N, rows, H = sampling.candidates(300, 30)
    first = L.glp_cd2_terms(H, N, rows)
    for _ in range(2):
        again = L.glp_cd2_terms(H, N, rows)
        assert all(np.array_equal(x, y) for x, y in zip(first, again))
    a = sampling.glp(300, 30, np.random.default_rng(1))
    assert np.array_equal(a, sampling.glp(300, 30, np.random.default_rng(1)))


# ------------------------------------------------------------------------------------------ screening and exact pass
@pytest.mark.parametrize("n,s,count", [(300, 30, 24), (400, 40, 10), (600, 60, 6), (640, 64, 5), (800, 80, 5)])
def test_screen_within_the_margin_and_the_pick_is_the_oracle_argmin(L, n, s, count):
    """On a slice of the candidates (the oracle's exact CD2 costs ~0.5 s per lattice at n 800), with the slice's
    winner repeated at the end: the screened D^2 lie within the margin of the reference-order values, and the
    selection is the oracle's first strict minimum."""
    from dmosopt_b200 import sampling

    N, rows, H = sampling.candidates(n, s)
    assert H.shape[0] >= count
    sub = H[np.linspace(0, H.shape[0] - 1, count).astype(int)]
    best, d = osm.select(sub, N, rows)
    sub = np.vstack([sub, sub[best]])
    d = np.append(d, d[best])
    d2, d3 = L.glp_cd2_terms(sub, N, rows)
    D1 = (13.0 / 12.0) ** s
    t2, t3 = 2 * d2 / rows, d3 / (float(rows) * rows)
    m = sampling.screen_margin(D1, t2, t3, rows, s)
    assert np.all(np.abs((D1 - t2 + t3) - d**2) <= m), np.max(np.abs((D1 - t2 + t3) - d**2) / m)
    got, short = sampling.select(sub, N, rows)
    assert got == best and best in short and sub.shape[0] - 1 in short
    assert np.array_equal(sampling._exact_cd2(sub[short], N, rows, s), d[short])  # the exact pass is bit-exact


def test_exact_pairs_are_the_reference_products(L):
    from dmosopt_b200 import sampling

    N, rows, H = sampling.candidates(100, 10)
    P = L.glp_cd2_pairs(H[:3], N, rows)
    for h, p in zip(H[:3], P):
        X = osm.design(h, N, rows)
        q = np.ones((rows, rows))
        for i in range(10):
            x, y = X[:, i][:, None], X[:, i][None, :]
            q = q * (1 + 0.5 * np.abs(x - 0.5) + 0.5 * np.abs(y - 0.5) - 0.5 * np.abs(x - y))
        assert np.array_equal(p, q.ravel())


# ------------------------------------------------------------------------------------------ envelope
def _raw_terms(L, H, C, s, lattice, rows):
    d2, d3 = np.empty(max(C, 1)), np.empty(max(C, 1))
    st = L.load_library().dmo_glp_cd2_terms(L.context(), H.ctypes.data, C, s, lattice, rows, d2.ctypes.data, d3.ctypes.data)
    msg = L.load_library().dmo_last_error(L.context()).decode()
    return st, msg


def test_envelope_edges_are_refused(L):
    H = np.ones((65536, 2), dtype=np.int64)
    assert _raw_terms(L, H, 65535, 2, 7, 7)[0] == 0  # the last admitted grid row count
    st, msg = _raw_terms(L, H, 65536, 2, 7, 7)
    assert st == 2 and "65535" in msg
    st, msg = _raw_terms(L, H, 4, 2, 2**31, 7)
    assert st == 2 and "lattice" in msg
    st, msg = _raw_terms(L, H, 4, 2, 7, 8)
    assert st == 2 and "rows" in msg
    st, msg = _raw_terms(L, np.full((4, 2), 7, dtype=np.int64), 4, 2, 7, 7)
    assert st == 2 and "multipliers" in msg
    big = np.array([[1, 2**31 - 2]], dtype=np.int64)  # the largest lattice: (k + 1) h near 2^62, still exact
    d2, d3 = L.glp_cd2_terms(big, 2**31 - 1, 3)
    X = osm.design(big[0], 2**31 - 1, 3)
    assert abs(d3[0] - osm.cd2_terms(X)[1]) <= 1e-12 * d3[0]
    with pytest.raises(ValueError, match="lattice"):
        L.glp_cd2_terms(big, 2**31, 3)
    with pytest.raises(L.DmoError, match="unknown metric"):
        _check_metric(L, 7)


def _check_metric(L, metric):
    X = np.random.default_rng(0).random((4, 2))
    d2, d3 = np.empty(1), np.empty(1)
    st = L.load_library().dmo_l2_discrepancy_terms(L.context(), metric, X.ctypes.data, 4, 2, d2.ctypes.data, d3.ctypes.data)
    L._check(st, "dmo_l2_discrepancy_terms")


# ------------------------------------------------------------------------------------------ discrepancies
def _d2_parts(metric, X, D2, D3):
    n, s = X.shape
    if metric == "MD2":
        return (4.0 / 3.0) ** s, D2 * 2 ** (1 - s) / n, D3 / n**2
    if metric == "CD2":
        return (13.0 / 12.0) ** s, 2 * D2 / n, D3 / n**2
    if metric == "SD2":
        return (4.0 / 3.0) ** s, 2 * D2 / n, D3 * 2**s / n**2
    return (4.0 / 3.0) ** s, 0.0, D3 / n**2


def _assert_close(L, metric, X, ref):
    from dmosopt_b200 import discrepancy

    got = getattr(discrepancy, metric)(X)
    D2, D3 = L.l2_discrepancy_terms(X, metric)
    bound = discrepancy.d2_bound(X.shape[0], X.shape[1], *_d2_parts(metric, X, D2, D3))
    assert abs(got**2 - ref**2) <= bound, (metric, X.shape, abs(got**2 - ref**2) / bound)


def test_discrepancies_match_the_fixtures(L, golden):
    from dmosopt_b200 import discrepancy

    g = golden("sampling")
    for i in range(int(g["disc_count"])):
        X, ref = g[f"disc_{i}_X"], g[f"disc_{i}"]
        for k, m in enumerate(METRICS):
            _assert_close(L, m, X, ref[k])
        r = discrepancy.all(X)
        assert r["MinDist"] == ref[4]
        np.testing.assert_array_equal(r["corrscore"], ref[5])


@pytest.mark.parametrize("n,s", [(1000, 3), (1500, 8), (1031, 20)])
def test_discrepancies_at_large_n_match_the_oracle(L, n, s):
    X = np.random.default_rng(n + s).random((n, s))
    for m in METRICS:
        _assert_close(L, m, X, ORACLE[m](X))


# ------------------------------------------------------------------------------------------ through the unmodified reference
@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("nInput,maxiter", [(4, 0), (6, 5), (3, 0)])
def test_moasmo_xinit_by_import_path_equals_glp(L, nInput, maxiter):
    MOASMO = _import_ref("MOASMO")
    xlb, xub = np.zeros(nInput), np.arange(1, nInput + 1, dtype=float)
    a, b = np.random.default_rng(5), np.random.default_rng(5)
    X = MOASMO.xinit(10, [f"x{i}" for i in range(nInput)], xlb, xub, method="dmosopt_b200.sampling.glp", maxiter=maxiter, local_random=a)
    Y = MOASMO.xinit(10, [f"x{i}" for i in range(nInput)], xlb, xub, method="glp", maxiter=maxiter, local_random=b)
    assert np.array_equal(X, Y)
    assert np.array_equal(a.random(4), b.random(4))
