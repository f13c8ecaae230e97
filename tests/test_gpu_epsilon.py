"""The epsilon-nondominated archive on the GPU (csrc/epsilon.cu): the reference's recorded archives, the reference's own
EpsilonSort and epsilon_get_best, every route of the box filter at its thresholds (grouping and winners against
oracle/epsilon.py, the filter row by row against oracle.dda.check_flags), the lazy class, install(), and the refusals."""

import ctypes

import numpy as np
import pytest

from conftest import load_golden
from oracle import dda
from oracle import epsilon as oe

pytestmark = pytest.mark.gpu

G = load_golden("epsilon")
CLASS_CASES = sorted(k[len("cls_") : -len("_idx")] for k in G.files if k.startswith("cls_") and k.endswith("_idx"))
GET_BEST_CASES = sorted(k[len("gb_") : -len("_by")] for k in G.files if k.startswith("gb_") and k.endswith("_by"))


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _reference():
    from oracle import reference_build

    return reference_build.reference_path()


def _import_reference():
    import sys

    path = _reference()
    sys.path.insert(0, path)
    try:
        from dmosopt import MOASMO, MOEA
    finally:
        sys.path.remove(path)
    return MOEA, MOASMO


def eps_arg(a):
    if a.dtype.kind == "U":
        return None if str(a) == "none" else str(a)
    return float(a) if a.ndim == 0 else [float(v) for v in a]


@pytest.mark.parametrize("name", CLASS_CASES)
def test_fixture_archives(L, name):
    Y, eps = G[f"cls_{name}_Y"], G[f"cls_{name}_eps"]
    assert np.array_equal(L.epsilon_sort(Y, eps), G[f"cls_{name}_idx"])


@pytest.mark.parametrize("name", GET_BEST_CASES)
def test_fixture_epsilon_get_best(L, name):
    from dmosopt_b200.MOASMO import epsilon_get_best

    p = f"gb_{name}_"
    get = lambda k: G[p + k] if p + k in G.files else None  # noqa: E731
    bx, by, bf, bc, be = epsilon_get_best(get("x"), get("y"), get("f"), get("c"), feasible=bool(G[p + "feasible"]),
                                          epsilons=eps_arg(G[p + "eps_arg"]))
    assert np.array_equal(bx, G[p + "bx"]) and np.array_equal(by, G[p + "by"])
    for got, key in ((bf, "bf"), (bc, "bc")):
        assert (got is None) == (get(key) is None) and (got is None or np.array_equal(got, get(key)))
    assert np.array_equal(np.asarray(be, dtype=np.float64), G[p + "beps"])


def near_front(rng, n, M, noise):
    x = np.abs(rng.standard_normal((n, M))) + 1e-3
    return x / np.linalg.norm(x, axis=1, keepdims=True) + noise * rng.random((n, M))


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("M", [3, 5, 16])
@pytest.mark.parametrize("eps", [None, 0.02, "auto"])
def test_reference_at_2000_rows(L, M, eps):
    from dmosopt_b200.MOASMO import epsilon_get_best

    rMOEA, rMOASMO = _import_reference()
    rng = np.random.default_rng(M)
    n = 2000
    x = rng.random((n, 4))
    y = near_front(rng, n, M, 0.03)
    f = rng.random((n, 1))
    c = rng.standard_normal((n, 2)) + 1.0
    want = rMOASMO.epsilon_get_best(x, y, f, c, epsilons=eps)
    got = epsilon_get_best(x, y, f, c, epsilons=eps)
    for a, b in zip(got[:4], want[:4]):
        assert np.array_equal(a, b)
    assert np.array_equal(np.asarray(got[4], dtype=np.float64), np.asarray(want[4], dtype=np.float64))
    e = [float(v) for v in np.ravel(want[4])]
    s = rMOEA.EpsilonSort(e)
    for i in range(n):
        s.sortinto(y[i], tagalong=i)
    assert np.array_equal(L.epsilon_sort(y, e), s.tagalongs)


def check_archive(L, Y, eps):
    """Exact check of one call: grouping and winners against the batch oracle, the box filter on every distinct box
    against check_flags, ascending output."""
    got = L.epsilon_sort(Y, eps)
    assert np.all(np.diff(got) > 0)
    uniq, win = oe.groups_and_winners(Y, eps)
    assert np.isin(got, win).all(), "a kept row is not its box's winner"
    dda.check_flags(uniq, (~np.isin(win, got)).astype(np.int32), device="cuda")
    return len(uniq), len(got)


@pytest.mark.parametrize("n,M", [(1023, 3), (1024, 3), (1023, 8), (1023, 9), (1024, 8), (1024, 9), (3000, 16)])
def test_box_filter_thresholds(L, n, M):
    """Default epsilon: every row its own box, so the filter sees n boxes (block kernel <8> / <16> below 1024, the id scan
    from 1024)."""
    rng = np.random.default_rng(n + M)
    Y = near_front(rng, n, M, 0.2)
    k, _ = check_archive(L, Y, [1e-9] * M)
    assert k == n


@pytest.mark.parametrize("brute", [False, True])
@pytest.mark.parametrize("M", [2, 3])
def test_box_filter_grid_route(L, monkeypatch, M, brute):
    if brute:
        monkeypatch.setenv("DMO_ND_BRUTE", "1")
    rng = np.random.default_rng(M)
    Y = rng.random((40000, M))
    k, _ = check_archive(L, Y, [1.0 / 128 if M == 2 else 1.0 / 24] * M)
    assert k >= 8192


@pytest.mark.parametrize("M,eps", [(2, 1.0 / 1024), (3, 1.0 / 40)])
def test_million_rows(L, M, eps):
    rng = np.random.default_rng(20 + M)
    Y = near_front(rng, 1 << 20, M, 0.05)
    k, kept = check_archive(L, Y, [eps] * M)
    assert k >= 8192 and kept > 1


def test_sixteen_objectives_at_2_17_rows(L):
    rng = np.random.default_rng(16)
    Y = rng.random((1 << 17, 16))
    Y[: 1 << 16] = near_front(rng, 1 << 16, 16, 0.01)
    check_archive(L, Y, [0.05] * 16)


def test_lazy_class_equals_the_reference_after_interleaved_calls(L):
    from dmosopt_b200.MOEA import EpsilonSort

    if _reference() is None:
        pytest.skip("reference package not built (oracle/_ref)")
    rMOEA, _ = _import_reference()
    rng = np.random.default_rng(4)
    Y = near_front(rng, 900, 3, 0.05)
    eps = [0.02, 0.03, 0.0]
    archives = []
    for cls in (rMOEA.EpsilonSort, EpsilonSort):
        s = cls(eps)
        for i in range(300):
            s.sortinto(Y[i], tagalong=i)
        first = list(s.tagalongs)
        s.remove(2)
        for i in range(300, 600):
            s.sortinto(Y[i], tagalong=i)
        s.add(np.array([-10.0, 100.0, 100.0]), "added", [-500, 3333, 10**10])
        for i in range(600, 900):
            s.sortinto(Y[i], tagalong=i)
        archives.append((first, list(s.tagalongs), [np.asarray(a) for a in s.archive], list(s.boxes)))
    (f0, t0, a0, b0), (f1, t1, a1, b1) = archives
    assert f0 == f1 and t0 == t1 and "added" in t1
    assert all(np.array_equal(a, b) for a, b in zip(a0, a1))
    assert [b for b, t in zip(b0, t0) if t != "added"] == [b for b, t in zip(b1, t1) if t != "added"]


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_install_keeps_the_reference_epsilon_get_best(L):
    from dmosopt_b200 import patch

    rMOEA, rMOASMO = _import_reference()
    rng = np.random.default_rng(9)
    x = rng.random((1500, 3))
    y = near_front(rng, 1500, 4, 0.05)
    c = rng.standard_normal((1500, 1)) + 0.5
    before = rMOASMO.epsilon_get_best(x, y, None, c, epsilons=0.03)
    original = rMOEA.EpsilonSort
    launches = L.launch_count()
    patch.install()
    try:
        after = rMOASMO.epsilon_get_best(x, y, None, c, epsilons=0.03)
        wide = rMOEA.EpsilonSort([0.1] * 17)
    finally:
        patch.uninstall()
    assert L.launch_count() > launches
    assert rMOEA.EpsilonSort is original and type(wide) is original
    for a, b in zip(before, after):
        assert (a is None and b is None) or np.array_equal(np.asarray(a), np.asarray(b))


def test_refusals_and_device_pointers(L):
    import torch

    with pytest.raises(OverflowError, match="row 5"):
        Y = np.ones((8, 2))
        Y[5, 1] = 1e301
        L.epsilon_sort(Y, [1e-9, 1e-9])
    lib = L.load_library()
    Y = np.random.default_rng(1).random((50, 17))
    eps = np.full(17, 0.1)
    idx = np.empty(50, dtype=np.int64)
    cnt = ctypes.c_int64(-1)
    assert lib.dmo_epsilon_sort(L.context(), Y.ctypes.data, 50, 17, eps.ctypes.data, idx.ctypes.data, ctypes.byref(cnt)) == 2
    assert cnt.value == 0
    # device inputs and output give the host result
    Y = near_front(np.random.default_rng(2), 5000, 4, 0.05)
    eps = np.array([0.01, 0.02, 0.0, 0.01])
    want = L.epsilon_sort(Y, eps)
    dY, de = torch.as_tensor(Y, device="cuda"), torch.as_tensor(eps, device="cuda")
    didx = torch.empty(5000, dtype=torch.int64, device="cuda")
    assert lib.dmo_epsilon_sort(L.context(), dY.data_ptr(), 5000, 4, de.data_ptr(), didx.data_ptr(), ctypes.byref(cnt)) == 0
    L.synchronize()
    assert np.array_equal(didx[: cnt.value].cpu().numpy(), want)
    # the same context still works after the refusals
    assert np.array_equal(L.epsilon_sort(G["cls_rand3_Y"], G["cls_rand3_eps"]), G["cls_rand3_idx"])
