"""Sensitivity analysis on the GPU (csrc/sa.cu, dmosopt_b200/sa.py): the DGSM and eFAST designs and the DGSM statistics
against oracle/sa.py, SA_DGSM / SA_FAST through the surrogates, and the unmodified reference's analyze_sensitivity."""

import math

import numpy as np
import pytest

from oracle import sa as osa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _box(rng, d):
    lb = rng.uniform(-3, 1, d)
    return lb, lb + rng.uniform(0.5, 4, d)


def _grid_elems(L):
    return L.sm_count() * 16 * 256  # the design kernels' grid (csrc/sa.cu design_grid) in elements


# ------------------------------------------------------------------------------------------ designs
@pytest.mark.parametrize("N,d", [(1, 1), (257, 1), (300, 2), (100, 30), (61, 90), (120_000, 2), (800, 90)])
def test_dgsm_design_is_bitwise_numpy(L, N, d):
    rng = np.random.default_rng(N + d)
    lb, ub = _box(rng, d)
    B = osa.dgsm_base(N, d)
    ref = osa.dgsm_design(B, lb, ub)
    X = L.sa_dgsm_design(B, lb, ub)
    assert X.shape == ref.shape and not X.flags.writeable
    assert np.array_equal(X, ref)
    dev = np.empty_like(ref)  # the device copy is the same array
    L.memcpy(dev, L.mirror_ptr(X), dev.nbytes)
    assert np.array_equal(dev, ref)
    assert np.array_equal(L.sa_dgsm_design(B, lb, ub, mirror=False), ref)
    if N * (d + 1) * d > _grid_elems(L):
        assert N >= 800  # these shapes exercise the grid-stride loop


def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


@pytest.mark.parametrize("N,d", [(65, 1), (1001, 2), (300, 30), (200, 90), (10_000, 2), (150_000, 2)])
def test_fast_design_matches_the_oracle(L, N, d):
    rng = np.random.default_rng(N * 7 + d)
    lb, ub = _box(rng, d)
    w = osa.fast_frequencies(N, d)
    phi = 2 * math.pi * rng.random(d)
    ref = osa.fast_design(N, w, phi, lb, ub)
    X = L.sa_fast_design(N, w, phi, lb, ub)
    assert X.shape == (N * d, d) and not X.flags.writeable
    assert np.max(_ulps(X, ref)) <= 4
    assert np.max(_ulps(L.sa_fast_design(N, w, phi, lb, ub, mirror=False), ref)) <= 4
    if N == 150_000:
        assert N * d * d > _grid_elems(L)


def test_design_argument_errors(L):
    launches = L.launch_count()
    with pytest.raises(L.DmoError, match="outside"):
        L.sa_fast_design(64, [8.0, 1.0], [0.0, 0.0], [0, 0], [1, 1])
    with pytest.raises(ValueError, match="bounds"):
        L.sa_dgsm_design(np.zeros((3, 2)), [0], [1])
    with pytest.raises(L.DmoError, match="bootstrap indices"):
        L.sa_dgsm_stats(np.zeros((6, 2)), np.zeros((6, 1)), [0, 0], [1, 1], [[0, 2]])
    assert L.launch_count() == launches


# ------------------------------------------------------------------------------------------ DGSM statistics
def _outputs(X):
    return np.column_stack([np.sin(3 * X[:, 0]) + X[:, 1] ** 2 * X[:, -1], np.exp(0.3 * X.sum(axis=1)), X[:, 0] * X[:, -1] + 0.1 * X[:, 1]])


def _close(a, b, tol=1e-12, scale=None):
    s = np.maximum(np.abs(b), 0 if scale is None else scale)
    return np.all(np.abs(a - b) <= tol * s)


@pytest.mark.parametrize("N,d,R", [(300, 2, 100), (2000, 30, 100), (1000, 90, 7), (20_000, 3, 100)])
def test_dgsm_stats_match_the_oracle(L, N, d, R):
    """N 20 000 stages its columns in global memory (2 N doubles exceed a CTA's shared memory)."""
    import torch

    rng = np.random.default_rng(N + d)
    lb, ub = _box(rng, d)
    X = osa.dgsm_design(osa.dgsm_base(N, d), lb, ub)
    Y = _outputs(X)
    idx = rng.integers(0, N, size=(R, N), dtype=np.int32)
    ref = osa.dgsm_stats(X, Y, lb, ub, idx)
    host = L.sa_dgsm_stats(X, Y, lb, ub, idx)
    Xm = L.sa_dgsm_design(osa.dgsm_base(N, d), lb, ub)  # mirrored design, host outputs
    mir = L.sa_dgsm_stats(Xm, Y, lb, ub, idx)
    Xd, Yd = torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()
    dev = L.sa_dgsm_stats(Xd, Yd, lb, ub, idx)
    for k in ("vi", "dgsm", "conf"):
        assert _close(host[k], ref[k]), (k, np.max(np.abs(host[k] - ref[k]) / np.abs(ref[k])))
    assert _close(host["vi_std"], ref["vi_std"], scale=ref["vi"])
    for other in (mir, dev, L.sa_dgsm_stats(X, Y, lb, ub, idx)):
        for k in host:
            assert np.array_equal(other[k], host[k]), k  # the same fixed-order sums however the inputs arrive


def test_dgsm_stats_device_indices(L):
    import torch

    rng = np.random.default_rng(4)
    N, d = 500, 4
    lb, ub = np.zeros(d), np.ones(d)
    X = osa.dgsm_design(osa.dgsm_base(N, d), lb, ub)
    Y = _outputs(X)
    idx = rng.integers(0, N, size=(100, N), dtype=np.int32)
    a = L.sa_dgsm_stats(X, Y, lb, ub, idx)
    st = {k: np.empty_like(v) for k, v in a.items()}
    ti = torch.from_numpy(idx).cuda()
    from statistics import NormalDist

    L._check(L.load_library().dmo_sa_dgsm_stats(L.context(), X.ctypes.data, Y.ctypes.data, N, d, 3, lb.ctypes.data, ub.ctypes.data, ti.data_ptr(), 100,
                                                 NormalDist().inv_cdf(0.975), st["vi"].ctypes.data, st["vi_std"].ctypes.data,
                                                 st["dgsm"].ctypes.data, st["conf"].ctypes.data), "dmo_sa_dgsm_stats")
    for k in a:
        assert np.array_equal(a[k], st[k])


# ------------------------------------------------------------------------------------------ analyze through the surrogates
def _train(rng, n, d, M=2):
    X = rng.random((n, d))
    Y = np.column_stack([np.sin(3 * X[:, 0]) + X[:, 1] ** 2 + 0.1 * X[:, 2:].sum(axis=1) + k * X[:, 0] * X[:, 1] for k in range(M)])
    return X, Y


def _surrogate(name, X, Y, d, M, lb, ub):
    import dmosopt_b200 as b2
    from dmosopt_b200 import model_gpflow, model_gpytorch

    if name == "GPR_Matern":
        return b2.GPR_Matern(X, Y, d, M, lb, ub, optimizer=None)
    if name == "EGP_Matern":
        return model_gpytorch.EGP_Matern(X, Y, d, M, lb, ub, fit="gpu", n_iter=60, seed=2)
    if name == "MEGP_Matern":
        return model_gpytorch.MEGP_Matern(X, Y, d, M, lb, ub, fit="gpu", n_iter=60, seed=2)
    return model_gpflow.SVGP_Matern(X, Y, d, M, lb, ub, seed=3, fit="gpu", n_iter=30, inducing_fraction=0.2, min_inducing=50)


def _host_evaluate(model, X):
    Y = model.evaluate(np.array(X))  # an ordinary host copy: the surrogate's host path
    return np.asarray(Y[0] if isinstance(Y, tuple) else Y, dtype=np.float64)


@pytest.mark.parametrize("name", ["GPR_Matern", "EGP_Matern", "MEGP_Matern", "SVGP_Matern"])
def test_analyze_through_the_surrogates_matches_the_oracle(L, name):
    from dmosopt_b200.sa import SA_DGSM, SA_FAST

    rng = np.random.default_rng(21)
    d, M = 5, 2
    lb, ub = np.zeros(d), np.full(d, 2.0)
    X, Y = _train(rng, 150, d, M)
    sm = _surrogate(name, X * 2, Y, d, M, lb, ub)
    names, outs = [f"x{i}" for i in range(d)], ["f0", "f1"]
    N = 1000
    res = SA_DGSM(lb, ub, names, outs, seed=5).analyze(sm, num_samples=N)
    Xo = osa.dgsm_design(osa.dgsm_base(N, d), lb, ub)
    idx = np.random.default_rng(5).integers(0, N, size=(100, N), dtype=np.int32)
    ref = osa.dgsm_stats(Xo, _host_evaluate(sm, Xo), lb, ub, idx)
    for m, o in enumerate(outs):
        assert res["S1"][o].shape == (d,)
        assert _close(res["S1"][o], ref["dgsm"][m], 1e-10), (o, res["S1"][o], ref["dgsm"][m])
    res = SA_FAST(lb, ub, names, outs, seed=6).analyze(sm, num_samples=N)
    phi = 2 * math.pi * np.random.default_rng(6).random(d)
    Xo = osa.fast_design(N, osa.fast_frequencies(N, d), phi, lb, ub)
    S1, ST = osa.fast_indices(_host_evaluate(sm, Xo), N, d)
    for m, o in enumerate(outs):
        assert _close(res["S1"][o], S1[m], 1e-10, scale=1e-6) and _close(res["ST"][o], ST[m], 1e-10, scale=1e-6), o


def test_analyze_ranks_the_inputs_that_matter(L):
    import dmosopt_b200 as b2
    from dmosopt_b200.sa import SA_DGSM, SA_FAST

    rng = np.random.default_rng(8)
    d = 12
    lb, ub = np.zeros(d), np.ones(d)
    X = rng.random((300, d))
    Y = np.column_stack([np.sin(3 * X[:, 0]) + 2 * X[:, 1] ** 2, X[:, 0] - X[:, 1]])
    sm = b2.GPR_Matern(X, Y, d, 2, lb, ub, anisotropic=True, seed=0)
    names = [f"x{i}" for i in range(d)]
    for cls in (SA_DGSM, SA_FAST):
        res = cls(lb, ub, names, ["f0", "f1"], seed=1).analyze(sm, num_samples=2000)
        for o in ("f0", "f1"):
            assert set(np.argsort(res["S1"][o])[::-1][:2]) == {0, 1}, (cls.__name__, o, res["S1"][o])


def test_mirrored_design_is_predicted_without_upload(L):
    import dmosopt_b200 as b2
    from dmosopt_b200.sa import SA_DGSM

    rng = np.random.default_rng(9)
    d = 6
    lb, ub = np.zeros(d), np.ones(d)
    X, Y = _train(rng, 200, d)
    sm = b2.GPR_Matern(X, Y, d, 2, lb, ub, optimizer=None)
    D = SA_DGSM(lb, ub, [f"x{i}" for i in range(d)], ["f0", "f1"]).sample(4000)
    sm.evaluate(D)  # warm-up (calibration of the default precision)
    h0 = L.transfer_bytes()[0]
    a = sm.evaluate(D)
    h1 = L.transfer_bytes()[0]
    b = sm.evaluate(np.array(D))  # the same rows from pageable memory
    h2 = L.transfer_bytes()[0]
    assert np.array_equal(a, b)
    assert (h2 - h1) - (h1 - h0) == D.nbytes and h1 - h0 < D.nbytes


def test_mean_variance_models_use_the_mean(L):
    import dmosopt_b200 as b2
    from dmosopt_b200.sa import SA_DGSM

    rng = np.random.default_rng(10)
    d = 3
    lb, ub = np.zeros(d), np.ones(d)
    X, Y = _train(rng, 100, d)
    a = SA_DGSM(lb, ub, ["a", "b", "c"], ["f0", "f1"], seed=2).analyze(b2.GPR_Matern(X, Y, d, 2, lb, ub, optimizer=None), 500)
    b = SA_DGSM(lb, ub, ["a", "b", "c"], ["f0", "f1"], seed=2).analyze(
        b2.GPR_Matern(X, Y, d, 2, lb, ub, optimizer=None, return_mean_variance=True), 500)
    for o in ("f0", "f1"):
        assert np.array_equal(a["S1"][o], b["S1"][o])


# ------------------------------------------------------------------------------------------ through the unmodified reference
def _reference():
    from oracle import reference_build

    return reference_build.reference_path()


def _import_moasmo():
    import sys

    ref = _reference()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    return MOASMO


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("method", ["SA_DGSM", "SA_FAST"])
def test_reference_analyze_sensitivity(L, method):
    import dmosopt_b200 as b2

    MOASMO = _import_moasmo()
    rng = np.random.default_rng(12)
    d = 6
    xlb, xub = np.zeros(d), np.ones(d)
    X, Y = _train(rng, 120, d)
    sm = b2.GPR_Matern(X, Y, d, 2, xlb, xub, optimizer=None)
    di = MOASMO.analyze_sensitivity(sm, xlb, xub, [f"x{i}" for i in range(d)], ["f0", "f1"], sensitivity_method_name=f"dmosopt_b200.sa.{method}")
    for k in ("di_mutation", "di_crossover"):
        assert di[k].shape == (d,) and np.all(di[k] >= 1.0) and np.all(di[k] <= 20.0), di[k]
        assert di[k].max() == 20.0


@pytest.mark.skipif(_reference() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_reference_epoch_with_sensitivity(L):
    MOASMO = _import_moasmo()
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(11)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    g = 1 + 9 * X[:, 1:].mean(axis=1)
    Y = np.column_stack([X[:, 0], g * (1 - np.sqrt(X[:, 0] / g))])
    gen = MOASMO.epoch(
        4, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name="dmosopt_b200.NSGA2",
        optimizer_kwargs={}, surrogate_method_name="dmosopt_b200.GPR_Matern", surrogate_method_kwargs={"optimizer": None},
        sensitivity_method_name="dmosopt_b200.sa.SA_DGSM", local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
