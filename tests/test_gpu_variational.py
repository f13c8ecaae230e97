"""The variational surrogates' posterior on the GPU (parity unpinned: gpflow is absent, so the state is given).

The five classes through dmo_svgp_create / dmo_svgp_predict against the dense float64 restatement in
oracle/variational.py, which applies q_sqrt by its dense product (no QR, no operator planes); a singular q_sqrt; the
optimal q against the oracle's Titsias optimum; VGP at the optimum against EGP_Matern; the unmodified reference
controller driving the plugins; and the argument checks.
"""

import functools

import numpy as np
import pytest

from oracle import variational as V

pytestmark = pytest.mark.gpu

N_TRAIN, N_CAND, N_IND = 300, 333, 141  # none a multiple of 128: padded inducing rows and candidate rows are exercised
KINDS = {"svgp": "SVGP_Matern", "vgp": "VGP_Matern", "siv": "SIV_Matern", "spv": "SPV_Matern", "crv": "CRV_Matern"}


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _lower(rng, L, Z, scale=0.3):
    q = np.tril(scale * rng.standard_normal((L, Z, Z)), -1)
    for l in range(L):
        q[l][np.diag_indices(Z)] = 0.2 + 0.5 * rng.random(Z)
    return q


@functools.lru_cache(maxsize=None)
def _case(kind, M, d):
    rng = np.random.default_rng(1000 * M + d + 7 * len(kind))
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    xub[0] = xlb[0]  # a degenerate input range: xrng = 1 there, as the reference's
    X = xlb + rng.random((N_TRAIN, d)) * (xub - xlb)
    Y = np.column_stack([np.sin(X @ rng.standard_normal(d)) + 0.1 * m for m in range(M)])
    xrng = np.where(np.isclose(xub - xlb, 0.0, rtol=1e-6, atol=1e-6), 1.0, xub - xlb)
    xn = (X - xlb) / xrng
    Lat = M
    Zn = N_TRAIN if kind == "vgp" else N_IND
    if kind == "vgp":
        Z = np.broadcast_to(xn, (Lat, N_TRAIN, d)).copy()
    elif kind == "svgp":
        Z = np.stack([xn[rng.choice(N_TRAIN, Zn, replace=False)] for _ in range(Lat)])
    else:
        Z = np.broadcast_to(xn[rng.choice(N_TRAIN, Zn, replace=False)], (Lat, Zn, d)).copy()
    ls = np.sqrt(d) * (0.4 + 0.6 * rng.random((Lat, d)))
    var = 0.5 + rng.random(Lat)
    if kind == "siv":
        ls[:] = ls[0]
        var[:] = var[0]
    hp = dict(lengthscales=ls, variance=var, likelihood_variance=1e-3, q_mu=rng.standard_normal((Lat, Zn)), q_sqrt=_lower(rng, Lat, Zn))
    if kind != "vgp":  # VGP's inducing points are the training inputs
        hp["Z"] = Z
    if kind == "crv":
        hp["W"] = rng.standard_normal((M, Lat))
    Xc = xlb + rng.random((N_CAND, d)) * (xub - xlb)
    Xc[:20] = X[rng.choice(N_TRAIN, 20, replace=False)] + 1e-7  # next to training (and for VGP inducing) points
    return X, Y, xlb, xub, hp, Xc


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("M,d", [(1, 2), (2, 12), (3, 40), (5, 12)])
def test_class_against_oracle(L, kind, M, d, precision):
    from dmosopt_b200 import model_gpflow

    X, Y, xlb, xub, hp, Xc = _case(kind, M, d)
    model = getattr(model_gpflow, KINDS[kind])(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision)
    mean, var = model.predict(Xc)
    om, ov = V.predict(kind, Xc, xlb, model.xrng, model.hyperparameters["Z"], hp["variance"], hp["lengthscales"], hp["q_mu"],
                       hp["q_sqrt"], model.y_train_mean, model.y_train_std, W=hp.get("W"))
    assert mean.dtype == om.dtype == np.float32 and var.dtype == ov.dtype and mean.shape == var.shape == (N_CAND, M)
    assert var.dtype == (np.float32 if kind in ("svgp", "vgp") else np.float64)
    ys = model.y_train_std.astype(np.float64)
    W = np.eye(M) if hp.get("W") is None else hp["W"]
    prior = ((W * W) @ hp["variance"]) * ys ** 2
    scale = np.maximum(np.abs(om).max(axis=0), ys)
    tol = 2e-6  # both paths take the mean from float64 kernel values
    assert np.all(np.abs(mean - om) <= tol * scale + np.spacing(np.abs(om))), np.abs(mean - om).max(axis=0) / scale
    # tensor path: the split-fp16 contraction's error follows the cancellation-free size of ||O1 k||^2; a random dense
    # q_sqrt makes that ~Z times the result, so the bound here is 1e-4 of max(|var|, prior), not GPR's 1e-5
    tol = 2e-6 if precision == "fp64" else 1e-4
    vscale = np.maximum(np.abs(ov).max(axis=0), prior)
    if var.dtype == np.float32 or precision == "tensor":
        assert np.all(np.abs(var - ov) <= tol * vscale), np.abs(var - ov).max(axis=0) / vscale
    else:
        assert np.all(np.abs(var - ov) <= 1e-9 * prior), np.abs(var - ov).max(axis=0) / prior
    assert model.evaluate(Xc[:3]).__class__ is (tuple if kind == "svgp" else np.ndarray)


@pytest.mark.parametrize("precision", [0, 1])
def test_singular_q_sqrt(L, precision):
    rng = np.random.default_rng(5)
    d, Zn, P = 4, 77, 200
    Z = rng.random((2, Zn, d))
    q = _lower(rng, 2, Zn)
    q[0][:, 10:] = 0.0  # rank 10: S singular
    q[1][:] = 0.0  # S = 0: the prior minus the explained part
    ls, s, qm = 0.5 + rng.random((2, d)), np.array([0.7, 1.3]), rng.standard_normal((2, Zn))
    h = L.SVGPHandle(Z, s, ls, qm, q, np.zeros(2), np.ones(2), np.zeros(d), np.ones(d))
    Xc = rng.random((P, d))
    mean, var = h.predict(Xc, precision=precision)
    for l in range(2):
        m, v = V.latent_predict(Xc, Z[l], s[l], ls[l], qm[l], q[l])
        tol = 1e-9 if precision == 0 else 1e-5
        np.testing.assert_allclose(var[:, l], v, atol=tol * s[l])
        np.testing.assert_allclose(mean[:, l], m, atol=tol * max(1.0, np.abs(m).max()))
    assert h.groups() == (2, 4)


def test_shared_planes_are_counted_once(L):
    rng = np.random.default_rng(2)
    Z1 = rng.random((50, 3))
    Z = np.stack([Z1, Z1, Z1])
    ls = np.broadcast_to(rng.random(3) + 0.5, (3, 3))
    q = _lower(rng, 3, 50)
    h = L.SVGPHandle(Z, np.ones(3), ls, rng.standard_normal((3, 50)), q, np.zeros(3), np.ones(3), np.zeros(3), np.ones(3))
    assert h.groups() == (1, 4)  # one K_* plane; one Lz^-1 and three q_sqrt operators


@pytest.mark.parametrize("Zn", [60, 300])
def test_optimal_q_against_oracle(L, Zn):
    rng = np.random.default_rng(Zn)
    N, d, Lat = 300, 5, 2
    X = rng.random((N, d))
    y = np.stack([np.sin(X @ rng.standard_normal(d)) for _ in range(Lat)])
    Z = np.stack([X[rng.choice(N, Zn, replace=False)] for _ in range(Lat)])
    s, ls, noise = np.array([0.9, 1.4]), 0.5 + rng.random((Lat, d)), np.array([1e-2, 3e-2])
    qm, qs = L.svgp_optimal_q(X, y, Z, s, ls, noise)
    for l in range(Lat):
        om, oS = V.optimal_q(X, y[l], Z[l], s[l], ls[l], noise[l])
        assert np.all(np.triu(qs[l], 1) == 0.0)
        np.testing.assert_allclose(qm[l], om, rtol=0, atol=1e-9 * np.abs(om).max())
        np.testing.assert_allclose(qs[l] @ qs[l].T, oS, rtol=0, atol=1e-9 * np.abs(oS).max())


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
def test_vgp_at_the_optimum_is_the_exact_gp(L, precision):
    """VGP_Matern with the optimal q (fixed kernel) against EGP_Matern with the same length scales and output scale,
    noise sigma^2 + 1e-2 (the reference's jitter) and zero linear mean: equal means, and the VGP's variance (latent f) is
    the exact GP's minus (sigma^2 + 1e-2) y_std^2.  GPflow's VGP sees the jitter in its data term too (f(X) = Lz v)."""
    from dmosopt_b200.model_gpflow import VGP_Matern
    from dmosopt_b200.model_gpytorch import EGP_Matern

    rng = np.random.default_rng(11)
    N, d, M, sig = 257, 6, 2, 1e-4
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(X @ rng.standard_normal(d)) + m for m in range(M)])
    ls, s = 0.6 + rng.random((M, d)), np.array([0.9, 1.3])
    vgp = VGP_Matern(X, Y, d, M, xlb, xub, precision=precision,
                     hyperparameters=dict(lengthscales=ls, variance=s, likelihood_variance=sig))
    egp = EGP_Matern(X, Y, d, M, xlb, xub, precision=precision,
                     hyperparameters=dict(lengthscale=ls, outputscale=s, noise=np.full(M, sig + 1e-2), weight=np.zeros((M, d)),
                                          bias=np.zeros(M)))
    Xc = np.vstack([rng.random((300, d)), X[:30] + 1e-6])
    mv, vv = vgp.predict(Xc)
    me, ve = egp.predict(Xc)
    ys = vgp.y_train_std
    tol = 2e-6 if precision == "fp64" else 1e-5
    scale = np.maximum(np.abs(me).max(axis=0), ys)
    assert np.all(np.abs(mv - me) <= tol * scale), np.abs(mv - me).max(axis=0) / scale
    noise_var = (sig + 1e-2) * ys ** 2
    assert np.all(np.abs(vv - (ve.astype(np.float64) - noise_var)) <= tol * (s * ys ** 2 + noise_var))


@pytest.mark.parametrize("precision", [0, 1])
def test_svgp_with_every_point_tends_to_the_exact_gp(L, precision):
    """SVGP's optimum with Z = X: its data term sees K(X, X) without the jitter, so it equals the exact GP with noise
    sigma^2 only as the jitter goes to 0 (here 1e-10)."""
    rng = np.random.default_rng(11)
    N, d, s, sig, jit = 257, 6, 0.9, 1e-2, 1e-10
    X, ls = rng.random((N, d)), 0.6 + rng.random(d)
    y = np.sin(X @ rng.standard_normal(d))
    qm, qs = L.svgp_optimal_q(X, y[None], X[None], [s], ls[None], [sig], jitter=jit)
    h = L.SVGPHandle(X[None], [s], ls[None], qm, qs, [0.25], [2.0], np.zeros(d), np.ones(d), jitter=jit)
    Xc = np.vstack([rng.random((300, d)), X[:30] + 1e-6])
    mean, var = h.predict(Xc, precision=precision)
    K = V.matern52(X, X, s, ls) + (sig + jit) * np.eye(N)
    ks = V.matern52(X, Xc, s, ls)
    me = ks.T @ np.linalg.solve(K, y)
    ve = s - np.sum(ks * np.linalg.solve(K, ks), axis=0)
    tol = 2e-6 if precision == 0 else 1e-5
    np.testing.assert_allclose(mean[:, 0], 2.0 * me + 0.25, atol=tol * 2.0 * max(1.0, np.abs(me).max()))
    np.testing.assert_allclose(var[:, 0], 4.0 * ve, atol=tol * 4.0 * s)


@pytest.mark.parametrize("kind", ["svgp", "spv", "vgp"])
def test_tensor_path_with_the_optimal_q_holds_1e5(L, kind):
    """A posterior as training leaves it (q at its optimum, S = B^-1 <= I), where the tensor path is held to 1e-5 of the
    column scale (mean) and of the prior (variance); the dense random q_sqrt above is the harder secondary case."""
    from dmosopt_b200 import model_gpflow

    X, Y, xlb, xub, hp, Xc = _case(kind, 3, 30)
    hp = {k: hp[k] for k in ("lengthscales", "variance", "likelihood_variance")}
    model = getattr(model_gpflow, KINDS[kind])(X, Y, 30, 3, xlb, xub, hyperparameters=hp, precision="tensor", seed=3)
    h = model.hyperparameters
    mean, var = model.predict(Xc)
    om, ov = V.predict(kind, Xc, xlb, model.xrng, h["Z"], hp["variance"], hp["lengthscales"], h["q_mu"], h["q_sqrt"],
                       model.y_train_mean, model.y_train_std)
    ys = model.y_train_std.astype(np.float64)
    scale = np.maximum(np.abs(om).max(axis=0), ys)
    prior = hp["variance"] * ys ** 2
    assert np.all(np.abs(mean - om) <= 1e-5 * scale + np.spacing(np.abs(om))), np.abs(mean - om).max(axis=0) / scale
    assert np.all(np.abs(var - ov) <= 1e-5 * prior), np.abs(var - ov).max(axis=0) / prior


def test_argument_errors(L):
    rng = np.random.default_rng(0)
    d, Zn = 2, 10
    Z, q = rng.random((1, Zn, d)), _lower(rng, 1, Zn)
    ok = dict(Zpts=Z, variance=[1.0], length_scale=np.ones((1, d)), q_mu=np.zeros((1, Zn)), q_sqrt=q, y_mean=[0.0], y_std=[1.0],
              xlb=np.zeros(d), xrng=np.ones(d))
    h = L.SVGPHandle(**ok)
    with pytest.raises(L.DmoError):
        h.predict(rng.random((5, d)), precision=L.GP_AUTO)
    bad = q.copy()
    bad[0, 0, 3] = 1e-3
    with pytest.raises(L.DmoError, match="lower triangular"):
        L.SVGPHandle(**dict(ok, q_sqrt=bad))
    with pytest.raises(L.DmoError):
        L.SVGPHandle(**dict(ok, Zpts=np.repeat(Z, 9, 0), variance=np.ones(9), length_scale=np.ones((9, d)), q_mu=np.zeros((9, Zn)),
                            q_sqrt=np.repeat(q, 9, 0), y_mean=np.zeros(9), y_std=np.ones(9)))
    with pytest.raises(L.DmoError):
        L.SVGPHandle(**dict(ok, W=np.ones((9, 1)), y_mean=np.zeros(9), y_std=np.ones(9)))
    with pytest.raises(L.DmoError, match="variance"):  # a non-positive kernel variance
        L.SVGPHandle(**dict(ok, variance=[-1.0]))
    # mismatched shapes
    for bad_kw in (dict(q_mu=np.zeros((1, Zn + 1))), dict(q_sqrt=q[:, :-1, :-1]), dict(length_scale=np.ones((1, d + 1))),
                   dict(variance=[1.0, 2.0]), dict(y_mean=np.zeros(2)), dict(W=np.ones((2, 3))), dict(xrng=np.ones(d + 1)),
                   dict(Zpts=Z[0])):
        with pytest.raises(L.DmoError):
            L.SVGPHandle(**dict(ok, **bad_kw))
    with pytest.raises(L.DmoError):  # VGP form: Z must equal N
        L._check(L.load_library().dmo_svgp_optimal_q(L.context(), 20, 10, d, 1, L._ptr(rng.random((20, d))), L._ptr(rng.random(20)), None,
                                                     L._ptr(np.ones(1)), L._ptr(np.ones(d)), L._ptr(np.ones(1)), 1e-2, 1,
                                                     L._ptr(np.zeros(10)), L._ptr(np.zeros(100))), "dmo_svgp_optimal_q")
    with pytest.raises(L.DmoError):
        L.svgp_optimal_q(rng.random((20, d)), rng.random((1, 20)), Z, [1.0], np.ones((1, d)), [0.0])


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


def _zdt1(x):
    g = 1.0 + 9.0 / (x.shape[1] - 1) * x[:, 1:].sum(axis=1)
    return np.column_stack((x[:, 0], g * (1.0 - np.sqrt(x[:, 0] / g))))


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("surrogate", ["SVGP_Matern", "CRV_Matern"])
def test_unmodified_moasmo_epoch_drives_the_variational_plugins(L, surrogate):
    """MOASMO.epoch resolves the surrogate by import path and builds it from kernel hyper-parameters (SVGP: q at its
    optimum; CRV: explicit Z, q and W), runs the generations and the resample step."""
    import sys

    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(11)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    Y = _zdt1(X)
    hp = dict(lengthscales=np.full((M, d), 0.8), variance=[1.0, 1.0], likelihood_variance=1e-3)
    if surrogate == "CRV_Matern":
        Zn = 40
        hp.update(Z=rng.random((Zn, d)), q_mu=0.3 * rng.standard_normal((M, Zn)), q_sqrt=_lower(rng, M, Zn, scale=0.02),
                  W=np.array([[1.0, 0.2], [-0.3, 0.9]]))
    launches0 = L.launch_count()
    gen = MOASMO.epoch(
        6, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name="dmosopt_b200.NSGA2",
        optimizer_kwargs={}, surrogate_method_name=f"dmosopt_b200.{surrogate}", surrogate_method_kwargs={"hyperparameters": hp},
        local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    assert L.launch_count() > launches0
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
    assert np.all(xr >= xlb) and np.all(xr <= xub)
