"""Objectives that share a posterior covariance share one L^-1, one K_* and one variance contraction (dmo_gp_create
groups them).  Each objective's outputs must not depend on whether it shares: they are compared with a one-objective
model built from that objective alone."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _kernel(A, B, c, ls, kind):
    r2 = (((A[:, None, :] - B[None, :, :]) / ls) ** 2).sum(axis=2)
    if kind == "matern":
        r = np.sqrt(5.0 * r2)
        return c * (1.0 + r + r * r / 3.0) * np.exp(-r)
    return c * np.exp(-0.5 * r2)


def _model(rng, N, d, thetas, group_of, kind):
    """One posterior state per objective: objective m uses thetas[group_of[m]] = (c, length scales, noise) and its own
    targets.  Objectives on the same theta get the very same factor plane (one Cholesky per theta)."""
    X = rng.random((N, d))
    M = len(group_of)
    factors = {}
    for t, (c, ls, nz) in enumerate(thetas):
        K = _kernel(X, X, c, ls, kind) + (nz + 1e-10) * np.eye(N)
        factors[t] = (np.linalg.cholesky(K), K)
    st = dict(X=X, alpha=np.empty((M, N)), L=np.empty((M, N, N)), c=np.empty(M), ls=np.empty((M, d)), noise=np.empty(M),
              ymean=np.empty(M), ystd=np.empty(M))
    for m, t in enumerate(group_of):
        c, ls, nz = thetas[t]
        Lf, K = factors[t]
        y = np.sin(X @ rng.standard_normal(d)) + 0.1 * rng.standard_normal(N)
        ym, ys = y.mean(), y.std()
        st["alpha"][m] = np.linalg.solve(K, (y - ym) / ys)
        st["L"][m] = Lf
        st["c"][m], st["ls"][m], st["noise"][m], st["ymean"][m], st["ystd"][m] = c, ls, nz, ym, ys
    return st


def _handle(L, st, kind, idx):
    d = st["X"].shape[1]
    code = L.KERNEL_MATERN52 if kind == "matern" else L.KERNEL_RBF
    return L.GPHandle(st["X"], st["alpha"][idx], st["L"][idx], st["c"][idx], st["ls"][idx], st["noise"][idx], st["ymean"][idx],
                      st["ystd"][idx], np.zeros(d), np.ones(d), kernel=code)


def _check_against_single(L, st, kind, X, monkeypatch):
    """Every objective of the grouped model against its one-objective model: bit-identical on the tensor path (both
    K_* producer routes), within 1e-12 on the float64 path."""
    M = len(st["c"])
    h = _handle(L, st, kind, slice(None))
    singles = [_handle(L, st, kind, slice(m, m + 1)) for m in range(M)]
    for fused in ("1", "0"):
        monkeypatch.setenv("DMO_GP_FUSED", fused)
        mean, var = h.predict(X, precision=L.GP_TENSOR)
        for m, s in enumerate(singles):
            mo, vo = s.predict(X, precision=L.GP_TENSOR)
            assert np.array_equal(mean[:, m], mo[:, 0]), (kind, fused, m)
            assert np.array_equal(var[:, m], vo[:, 0]), (kind, fused, m)
    monkeypatch.delenv("DMO_GP_FUSED")
    mean, var = h.predict(X, precision=L.GP_FP64)
    for m, s in enumerate(singles):
        mo, vo = s.predict(X, precision=L.GP_FP64)
        prior = (st["c"][m] + st["noise"][m]) * st["ystd"][m] ** 2
        assert np.max(np.abs(var[:, m] - vo[:, 0])) <= 1e-12 * prior, (kind, m)
        assert np.max(np.abs(mean[:, m] - mo[:, 0]) / np.maximum(np.abs(mo[:, 0]), st["ystd"][m])) <= 1e-12, (kind, m)
    for s in singles:
        s.close()
    return h


@pytest.mark.parametrize("kind", ["matern", "rbf"])
def test_interleaved_groups(L, kind, monkeypatch):
    """M = 5 with objectives {0, 2, 4} on one theta and {1, 3} on another: two groups, and each objective predicts
    exactly what it predicts alone.  Isotropic Matern, and RBF with one length scale per dimension."""
    rng = np.random.default_rng(11 if kind == "matern" else 12)
    N, d, P = 700, 7, 900
    if kind == "matern":
        thetas = [(1.0, np.full(d, 0.5), 1e-6), (1.7, np.full(d, 0.8), 1e-4)]
    else:
        thetas = [(1.0, np.linspace(0.4, 0.9, d), 1e-6), (0.6, np.linspace(1.1, 0.5, d), 1e-5)]
    st = _model(rng, N, d, thetas, [0, 1, 0, 1, 0], kind)
    X = rng.random((P, d))
    h = _check_against_single(L, st, kind, X, monkeypatch)
    assert h.covariance_groups() == (2, [0, 1, 0, 1, 0])
    h.close()


@pytest.mark.parametrize("miss", ["factor", "constant"])
def test_near_misses_do_not_share(L, miss, monkeypatch):
    """A factor plane one ulp off in one element, or a constant one ulp off, makes a group of its own; its outputs still
    match its one-objective model."""
    rng = np.random.default_rng(13)
    N, d, P = 520, 5, 600
    st = _model(rng, N, d, [(1.0, np.full(d, 0.5), 1e-6)], [0, 0, 0], "matern")
    if miss == "factor":
        st["L"][1, N - 1, N // 2] = np.nextafter(st["L"][1, N - 1, N // 2], np.inf)
        want = (2, [0, 1, 0])
    else:
        st["c"][2] = np.nextafter(st["c"][2], np.inf)
        want = (2, [0, 0, 1])
    X = rng.random((P, d))
    h = _check_against_single(L, st, "matern", X, monkeypatch)
    assert h.covariance_groups() == want
    h.close()


def test_benchmarked_model_shares_one_covariance(L):
    """The bench.py model (N 4096, d 30, M 3, GPR_Matern at the fixed initial theta) fits its objectives in one batched
    call with the same theta: the factor planes come out bitwise equal, so the model holds one covariance.  AUTO still
    admits the tensor path for it."""
    import bench
    import dmosopt_b200 as b2

    N, d, M = 4096, 30, 3
    w = bench.workload(256, d, M, N)
    sm = b2.GPR_Matern(w["Xtr"], w["Ytr"], d, M, w["xlb"], w["xub"], optimizer=None)
    assert sm._gp.covariance_groups() == (1, [0, 0, 0])
    info = sm._gp.auto_info()
    assert info["mean_tensor"] and info["var_tensor"], info
