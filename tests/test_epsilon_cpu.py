"""The epsilon-nondominated archive without a GPU: oracle/epsilon.py against the reference's fixture
(tests/golden/epsilon.npz), the batch form against one-by-one insertion, and the host logic of
dmosopt_b200.MOEA.EpsilonSort and dmosopt_b200.MOASMO.epsilon_get_best with ``_lib.epsilon_sort`` replaced by the
oracle."""

import ctypes

import numpy as np
import pytest

import fake_backend
from conftest import load_golden
from oracle import epsilon as oe

G = load_golden("epsilon")
CLASS_CASES = sorted(k[len("cls_") : -len("_idx")] for k in G.files if k.startswith("cls_") and k.endswith("_idx"))
GET_BEST_CASES = sorted(k[len("gb_") : -len("_by")] for k in G.files if k.startswith("gb_") and k.endswith("_by"))


def oracle_epsilon_sort(Y, eps):
    """Stand-in for _lib.epsilon_sort: the batch oracle on the first len(eps) columns."""
    return oe.batch(np.asarray(Y, dtype=np.float64)[:, : len(np.ravel(eps))], eps)


@pytest.fixture
def lib(monkeypatch):
    from dmosopt_b200 import _lib

    monkeypatch.setattr(_lib, "epsilon_sort", oracle_epsilon_sort)
    monkeypatch.setattr(_lib, "get_duplicates", fake_backend.get_duplicates)
    return _lib


def eps_arg(a):
    """The epsilons argument a get_best case gave the reference."""
    if a.dtype.kind == "U":
        return None if str(a) == "none" else str(a)
    return float(a) if a.ndim == 0 else [float(v) for v in a]


def test_fixture_covers_the_cases():
    for name in ("rand2", "rand3", "rand5", "rand10", "rand16", "front16", "dyadic3", "perm5", "naninf3", "eps_zero_nan",
                 "eps_negative", "eps_inf", "wide_rows", "n1"):
        assert name in CLASS_CASES
    assert {"default", "scalar", "auto", "list", "infeasible", "nofilter", "n1"} <= set(GET_BEST_CASES)


@pytest.mark.parametrize("name", CLASS_CASES)
def test_sequential_oracle_reproduces_the_reference(name):
    Y, eps = G[f"cls_{name}_Y"], G[f"cls_{name}_eps"]
    assert np.array_equal(oe.sequential(Y, eps), G[f"cls_{name}_idx"])


@pytest.mark.parametrize("name", CLASS_CASES)
def test_batch_oracle_reproduces_the_reference(name):
    Y, eps = G[f"cls_{name}_Y"], G[f"cls_{name}_eps"]
    assert np.array_equal(oe.batch(Y[:, : len(eps)], eps), G[f"cls_{name}_idx"])


def tie_heavy(rng, n, M):
    """Dyadic rows around a plane: shared boxes, equal distances, duplicates."""
    Y = rng.integers(0, 16, (n, M)) / 4.0
    Y[:, -1] = 2.0 * (M - 1) - Y[:, :-1].sum(axis=1) + rng.integers(0, 4, n) / 4.0
    Y[rng.integers(0, n, n // 5)] = Y[rng.integers(0, n, n // 5)]
    return Y


@pytest.mark.parametrize("M", [1, 2, 3, 4, 6])
@pytest.mark.parametrize("eps", [0.5, 1.0, np.inf])
def test_batch_equals_sequential_on_permuted_tie_heavy_sets(M, eps):
    rng = np.random.default_rng(M * 10 + int(np.isinf(eps)))
    Y = tie_heavy(rng, 160, M)
    e = [eps] * M if not np.isinf(eps) else [1.0] * (M - 1) + [np.inf]
    for _ in range(4):
        P = Y[rng.permutation(len(Y))]
        assert np.array_equal(oe.batch(P, e), oe.sequential(P, e))


def test_sequential_overflow_raises():
    with pytest.raises(OverflowError):
        oe.sequential(np.array([[1e300, 0.0]]), [1e-9, 1.0])
    with pytest.raises(OverflowError):
        oe.batch(np.array([[np.inf, 0.0]]), [0.5, 1.0])  # nan_to_num: the largest float / 0.5


@pytest.mark.parametrize("chunks", [[400], [1, 399], [37, 100, 1, 262], [100] * 4])
def test_lazy_class_in_chunks_equals_one_batch(lib, chunks):
    from dmosopt_b200.MOEA import EpsilonSort

    rng = np.random.default_rng(len(chunks))
    Y = tie_heavy(rng, 400, 3)
    s = EpsilonSort([0.5, 0.5, 0.5])
    i = 0
    for c in chunks:
        for _ in range(c):
            s.sortinto(Y[i], tagalong=f"row{i}")
            i += 1
        assert len(s.archive) == len(s.tagalongs) == len(s.boxes)  # a read resolves the buffer
    want = oe.batch(Y, [0.5] * 3)
    assert s.tagalongs == [f"row{j}" for j in want]
    assert all(np.array_equal(a, Y[j]) for a, j in zip(s.archive, want))
    assert s.boxes == [[int(v) for v in np.floor(Y[j] / 0.5)] for j in want]
    assert all(type(v) is int for b in s.boxes for v in b)


def test_lazy_class_add_remove_and_interface(lib):
    from dmosopt_b200.MOEA import EpsilonSort

    s = EpsilonSort([0.0, float("nan"), 0.25])
    assert s.epsilons == [1e-8, 1e-8, 0.25] and list(s.itobj) == [0, 1, 2]
    s.sortinto([1.0, 2.0, 0.3], "a")
    s.sortinto([np.nan, 3.0, 0.3, 99.0], "b")  # rows wider than the epsilons keep their extra columns
    assert s.tagalongs == ["a", "b"]
    assert np.array_equal(s.archive[1], [0.0, 3.0, 0.3, 99.0])
    s.remove(0)
    assert s.tagalongs == ["b"]
    s.sortinto([5.0, 5.0, 5.0], "c")  # dominated by b's box
    s.add(np.array([9.0, 9.0, 9.0]), "d", [0, 0, 0])
    assert s.tagalongs == ["b", "d"]
    with pytest.raises(OverflowError):
        s.sortinto([1e301, 0.0, 0.0])
    assert s.tagalongs == ["b", "d"]
    with pytest.raises(ValueError):
        EpsilonSort([0.1] * 17)


@pytest.mark.parametrize("name", GET_BEST_CASES)
def test_epsilon_get_best_host_logic_matches_the_reference(lib, name):
    from dmosopt_b200.MOASMO import epsilon_get_best

    p = f"gb_{name}_"
    get = lambda k: G[p + k] if p + k in G.files else None  # noqa: E731
    bx, by, bf, bc, be = epsilon_get_best(get("x"), get("y"), get("f"), get("c"), feasible=bool(G[p + "feasible"]),
                                          epsilons=eps_arg(G[p + "eps_arg"]))
    assert np.array_equal(bx, G[p + "bx"]) and np.array_equal(by, G[p + "by"])
    for got, key in ((bf, "bf"), (bc, "bc")):
        assert (got is None) == (get(key) is None) and (got is None or np.array_equal(got, get(key)))
    assert np.array_equal(np.asarray(be, dtype=np.float64), G[p + "beps"])


def test_epsilon_get_best_edges(lib):
    from dmosopt_b200.MOASMO import epsilon_get_best

    x, y = np.zeros((0, 2)), np.zeros((0, 3))
    out = epsilon_get_best(x, y, None, None)
    assert out[0] is x or out[0].shape == (0, 2)
    assert out[1].shape == (0, 3) and out[4] == [1e-9] * 3
    rng = np.random.default_rng(5)
    x, y = rng.random((50, 2)), rng.random((50, 3))
    e = np.array([0.1, 0.2, 0.05])  # an array of epsilons (the reference raises ValueError under NumPy 2)
    bx, by, _, _, be = epsilon_get_best(x, y, None, None, epsilons=e)
    assert be is e and np.array_equal(by, y[oe.batch(y, e)])
    bx, by, _, _, be = epsilon_get_best(x, y, None, None, epsilons=2)
    assert be == [2.0] * 3
    y[7, 1] = 1e300
    with pytest.raises(OverflowError):
        epsilon_get_best(x, y, None, None)


def test_overflow_status_becomes_overflow_error(monkeypatch):
    from dmosopt_b200 import _lib

    class FakeLib:
        def dmo_epsilon_sort(self, *args):
            return _lib.ERR_OVERFLOW

        def dmo_last_error(self, ctx):
            return b"epsilon_sort: y / eps overflows to infinity in row 3"

    monkeypatch.setattr(_lib, "_lib", FakeLib())
    monkeypatch.setattr(_lib, "load_library", lambda path=None: _lib._lib)
    monkeypatch.setattr(_lib, "context", lambda device=None: ctypes.c_void_p())
    with pytest.raises(OverflowError, match="row 3"):
        _lib.epsilon_sort(np.ones((4, 2)), [1e-9, 1e-9])
    with pytest.raises(ValueError):
        _lib.epsilon_sort(np.ones((4, 2)), [1.0, 1.0, 1.0])


def test_install_routes_epsilon_sort_by_width(monkeypatch, tmp_path):
    import sys

    from dmosopt_b200 import MOEA, patch

    pkg = tmp_path / "epsstub"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "MOEA.py").write_text("class EpsilonSort:\n    def __init__(self, epsilons):\n        self.epsilons = epsilons\n")
    for mod in ("indicators", "dda"):
        (pkg / f"{mod}.py").write_text("")
    (pkg / "hv.py").write_text("class AdaptiveHyperVolume:\n    def compute_hypervolume(self, *a, **k):\n        pass\n")
    sys.path.insert(0, str(tmp_path))
    try:
        import epsstub.MOEA as m

        original = m.EpsilonSort
        monkeypatch.setattr(patch, "_saved", [])
        for name in ("get_duplicates", "remove_duplicates", "sortMO", "orderMO", "remove_worst"):
            setattr(m, name, None)
        import epsstub.dda as d

        d.dda_ens = None
        patch.install("epsstub")
        try:
            assert isinstance(m.EpsilonSort([0.1] * 16), MOEA.EpsilonSort)
            assert type(m.EpsilonSort([0.1] * 17)) is original
        finally:
            patch.uninstall()
        assert m.EpsilonSort is original
    finally:
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "epsstub" or k.startswith("epsstub.")]:
            del sys.modules[k]
