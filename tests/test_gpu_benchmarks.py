"""WFG1 and the many-objective MaF1 / MaF2 / MaF4 on the GPU (dmo_benchmark_eval): against the reference's own
row-at-a-time outputs (tests/golden/benchmarks.npz), against the vectorised oracle at population size up to 16
objectives, from device-mirrored inputs, and driving NSGA-II and AGE-MOEA on MaF2 with ten objectives."""

import numpy as np
import pytest

from conftest import load_golden
from oracle import benchmarks_many as obm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def test_new_problems_against_reference_rows(L):
    from dmosopt_b200 import benchmarks as bm

    g = load_golden("benchmarks")
    for key in g["keys"]:
        key = str(key)
        nm, M, _ = key.split("_")
        fn, M = getattr(bm, nm), int(M)
        X = g[key + "_X"]
        Y = fn(X, M)
        np.testing.assert_allclose(Y, g[key + "_Y"], rtol=1e-12, atol=0, equal_nan=True, err_msg=key)
        for i in range(X.shape[0]):  # one decision vector, as the reference is called: the same bits as its row
            y1 = fn(X[i], M)
            assert y1.shape == (M,) and np.array_equal(y1, Y[i], equal_nan=True), (key, i)
    # the reference's defaults: n_obj 5 for MaF, 3 for WFG1
    for nm in ("maf1", "maf2", "maf4"):
        assert np.array_equal(getattr(bm, nm)(g["maf2_5_14_X"]), getattr(bm, nm)(g["maf2_5_14_X"], 5)), nm
    assert np.array_equal(bm.wfg1(g["wfg1_3_12_X"]), bm.wfg1(g["wfg1_3_12_X"], 3), equal_nan=True)


@pytest.mark.parametrize("name,M", [("maf1", 10), ("maf2", 10), ("maf4", 10), ("maf1", 16), ("maf2", 16), ("maf4", 16), ("wfg1", 3)])
def test_against_oracle_at_population_size(L, name, M):
    from dmosopt_b200 import benchmarks as bm

    d = M + 9
    X = np.random.default_rng(M * 7 + len(name)).random((65536, d))
    if name == "wfg1":
        X *= 2 * np.arange(1, d + 1)
    Y = getattr(bm, name)(X, M)
    R = getattr(obm, name)(X, M)
    assert Y.shape == (65536, M) and np.isfinite(Y).all()
    bar = 1e-12 * np.abs(R)  # relative, per objective: also for MaF4's 1 .. 1e30 scales
    if name == "maf1":
        # 1 + g cancels where g = sum (t^2 - cos(20 pi t)) nears -1: the sum's rounding (sequential here, pairwise in
        # NumPy) is relative to its terms, so the bar is scaled by the condition number of 1 + g
        t = X[:, M - 1 :] - 0.5
        terms = t**2 - np.cos(20 * np.pi * t)
        bar *= ((1 + np.abs(terms).sum(axis=1)) / np.abs(1 + terms.sum(axis=1)))[:, None]
    elif name == "wfg1":
        # 1 - sin(v pi / 2) cancels as the window maxima near 1 (and 1 - cos near 0): each factor is good to a few ulp
        # absolutely, so the bar adds 1e-14 of the objective's range [0, i + 2]
        bar += 1e-14 * (2 + np.arange(M))
    err = np.abs(Y - R)
    assert np.all(err <= bar), (np.argwhere(err > bar)[:5], float(np.max(err / np.maximum(np.abs(R), 1e-300))))


def test_device_mirrored_input_is_read_in_place(L):
    from dmosopt_b200 import benchmarks as bm

    X = np.random.default_rng(5).random((4096, 25))
    ref = {nm: getattr(bm, nm)(X, 16) for nm in ("maf1", "maf2", "maf4")}
    ref["wfg1"] = bm.wfg1(X[:, :12] * 2 * np.arange(1, 13), 3)
    Xm, base = L.mirrored_readonly(X)
    Xw, base_w = L.mirrored_readonly(X[:, :12] * 2 * np.arange(1, 13))
    assert base is not None and L.mirror_ptr(Xm) is not None
    h0, _ = L.transfer_bytes()
    got = {nm: getattr(bm, nm)(Xm, 16) for nm in ("maf1", "maf2", "maf4")}
    got["wfg1"] = bm.wfg1(Xw, 3)
    h1, _ = L.transfer_bytes()
    assert h1 == h0  # no upload
    for nm in ref:
        assert np.array_equal(got[nm], ref[nm]), nm
    bm.maf2(X, 16)
    assert L.transfer_bytes()[0] - h1 == X.nbytes  # the host array is uploaded once


def test_library_refuses_empty_wfg1_windows(L):
    X = np.random.default_rng(6).random((8, 12))
    with pytest.raises(L.DmoError, match="empty shape window"):
        L.benchmark_eval("wfg1", X, 4)
    assert L.benchmark_eval("wfg1", X[:, :5], 4).shape == (8, 4)  # (4 - 2) * 2 < 5: the windows [0, 2), [2, 4), [4, 5)
    with pytest.raises(L.DmoError, match="n_var must be at least n_obj"):
        L.benchmark_eval("maf2", X[:, :9], 10)


@pytest.mark.parametrize("algo", ["NSGA2", "AGEMOEA"])
def test_many_objective_run_on_maf2(L, algo):
    """The plugins run a real ten-objective problem end to end: MaF2, n_var 19, pop 2048, 30 generations.

    Convergence is not asserted.  At ten objectives nearly every point is non-dominated and the diversity terms favour
    extreme points, so Pareto-based selection lets the distance term g = sum (x_m - 0.5)^2 grow: it does here, and the
    reference's own NSGA-II does the same on this problem (the known dominance resistance of many-objective search)."""
    import dmosopt_b200 as b2
    from dmosopt_b200 import benchmarks as bm
    from dmosopt_b200.driver import optimize

    M, d, pop = 10, 19, 2048
    calls, first = [], {}

    class MaF2:
        def evaluate(self, x):
            mirrored = L.mirror_ptr(x) is not None
            h0 = L.transfer_bytes()[0]
            y = bm.maf2(x, M)
            calls.append((mirrored, L.transfer_bytes()[0] - h0))
            first.setdefault("y", y.copy())
            return y

    mdl = b2.Model(objective=MaF2())
    opt = getattr(b2, algo)(popsize=pop, nInput=d, nOutput=M, model=mdl)
    optimize(30, opt, mdl, d, M, np.zeros(d), np.ones(d), popsize=pop, local_random=np.random.default_rng(20261016))
    px, py = opt.population_objectives
    assert px.shape == (pop, d) and py.shape == (pop, M) and np.isfinite(py).all()
    # the stored objectives are the (float32) objectives of the stored rows, and their stored ranks the canonical ones
    assert np.array_equal(py, bm.maf2(px, M).astype(py.dtype))
    rank = np.asarray(opt.state.rank)
    assert np.array_equal(rank, L.rank_nd(py))
    # selection by rank: the share of mutually non-dominated rows does not fall below the initial sample's
    assert np.mean(rank == 0) >= np.mean(L.rank_nd(first["y"].astype(np.float32)) == 0)
    # every offspring matrix comes back with a device mirror and is evaluated without an upload
    assert len(calls) == 31 and all(m and h == 0 for m, h in calls[1:]), calls
