"""Training of the variational surrogates on the GPU (dmo_svgp_fit_*): the ELBO pieces and their hyper-parameter
gradient against the dense torch autograd oracle (oracle/variational_train.py) for every form; the natural-gradient step
against the oracle's autograd-derived step and, at gamma = 1 on the full batch, against dmo_svgp_optimal_q; determinism;
svgp_fit's loop against the oracle loop on the same batch stream; fitted models; and the unmodified reference controller
training the plugins with fit="gpu"."""

import numpy as np
import pytest

from oracle import variational as ov
from oracle import variational_train as vt

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _zdt1(x):
    d = x.shape[1]
    g = 1.0 + 9.0 / (d - 1) * x[:, 1:].sum(axis=1)
    return np.column_stack((x[:, 0], g * (1.0 - np.sqrt(x[:, 0] / g))))


def _data(rng, N, d, M):
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, (t + 1) % d] for t in range(M)])
    return X, (Y - Y.mean(0)) / Y.std(0)


def _q(rng, L, Zn, scale):
    qs = np.tril(rng.standard_normal((L, Zn, Zn))) * scale
    for l in range(L):
        qs[l][np.diag_indices(Zn)] = 0.5 + rng.random(Zn)
    return 0.5 * rng.standard_normal((L, Zn)), qs


def _set_q(L, st, X, Y, Z, b, s, ls, nz, W, vgp):
    """Drive the state to a non-trivial q: two natural-gradient steps on different batches."""
    st.natgrad(b[0], s, ls, nz, W, gamma=0.7)
    st.natgrad(b[1], s, ls, nz, W, gamma=0.4)
    return st.q()


# kind, N, Z, B, d, M
CASES = [("svgp", 120, 37, 50, 2, 1), ("svgp", 400, 256, 1, 12, 1), ("svgp", 350, 300, 350, 40, 1), ("vgp", 90, 90, 90, 12, 1),
         ("vgp", 300, 300, 300, 2, 1), ("siv", 200, 37, 50, 12, 3), ("spv", 300, 256, 50, 2, 5), ("crv", 300, 37, 300, 40, 3),
         ("crv", 400, 300, 50, 12, 4)]


@pytest.mark.parametrize("kind,N,Zn,B,d,M", CASES)
def test_elbo_grad_matches_the_autograd_oracle(L, kind, N, Zn, B, d, M):
    rng = np.random.default_rng(N + Zn + B + d)
    X, Y = _data(rng, N, d, M)
    vgp = kind == "vgp"
    Z = None if vgp else X[rng.choice(N, Zn, replace=False)]
    Lat = M
    s = 0.5 + rng.random(Lat)
    ls = np.exp(rng.uniform(np.log(0.3), np.log(2.0), (Lat, d))) * np.sqrt(d / 2)
    if kind == "siv":
        s[:], ls[:] = s[0], ls[0]
    nz = np.full(M, 0.05) if kind != "svgp" and kind != "vgp" else np.array([0.03])
    W = rng.standard_normal((M, Lat)) if kind == "crv" else None
    st = L.SVGPFitState(X, Y, Z, Lat, inducing_is_data=vgp)
    batches = [np.arange(N) if vgp else rng.permutation(N)[:B] for _ in range(3)]
    q_mu, q_sqrt = _set_q(L, st, X, Y, Z, batches, s, ls, nz, W, vgp)
    ell, kl, g = st.elbo_grad(batches[2], s, ls, nz, W)
    rell, rkl, rg = vt.elbo_and_grad(X, Y, Z, batches[2], s, ls, nz, W, q_mu, q_sqrt, vgp)
    np.testing.assert_allclose(ell, rell, rtol=1e-10, atol=1e-10 * np.abs(rell).max())
    np.testing.assert_allclose(kl, rkl, rtol=1e-10, atol=1e-10 * np.abs(rkl).max())
    for k, ref in (("variance", rg["variance"]), ("length_scale", rg["length_scale"]), ("noise", rg["noise"])):
        err = np.abs(g[k] - ref).max() / max(np.abs(ref).max(), 1e-300)
        assert err < 1e-8, (k, err)
    if W is not None:
        err = np.abs(g["W"] - rg["W"]).max() / np.abs(rg["W"]).max()
        assert err < 1e-8, ("W", err)
    # the logging evaluation (no gradient) gives the same pieces, and repeated calls are bit-identical
    ell2, kl2, _ = st.elbo_grad(batches[2], s, ls, nz, W, grad=False)
    _, _, g2 = st.elbo_grad(batches[2], s, ls, nz, W)
    assert np.array_equal(ell, ell2) and np.array_equal(kl, kl2)
    for k in g:
        assert (g[k] is None and g2[k] is None) or np.array_equal(g[k], g2[k])


@pytest.mark.parametrize("kind,N,Zn,B,d,M", [c for c in CASES if c[3] <= 300][:6])
def test_natgrad_step_matches_the_autograd_oracle(L, kind, N, Zn, B, d, M):
    rng = np.random.default_rng(7 + N + Zn)
    X, Y = _data(rng, N, d, M)
    vgp = kind == "vgp"
    Z = None if vgp else X[rng.choice(N, Zn, replace=False)]
    s, ls = 0.5 + rng.random(M), np.full((M, d), 0.8 * np.sqrt(d / 2))
    nz = np.full(M, 0.05)
    W = rng.standard_normal((M, M)) if kind == "crv" else None
    st = L.SVGPFitState(X, Y, Z, M, inducing_is_data=vgp)
    b = [np.arange(N) if vgp else rng.permutation(N)[:B] for _ in range(2)]
    st.natgrad(b[0], s, ls, nz, W, gamma=0.3)
    q0 = st.q()
    st.natgrad(b[1], s, ls, nz, W, gamma=0.3)
    q1 = st.q()
    r1 = vt.natgrad_step(X, Y, Z, b[1], s, ls, nz, W, q0[0], q0[1], 0.3, vgp)
    for a, r in zip(q1, r1):
        assert np.abs(a - r).max() / np.abs(r).max() < 1e-8
    assert np.all(q1[1][:, np.triu_indices(q1[1].shape[1], 1)[0], np.triu_indices(q1[1].shape[1], 1)[1]] == 0.0)


@pytest.mark.parametrize("vgp", [False, True])
def test_natgrad_at_gamma_one_on_the_full_batch_is_the_optimal_q(L, vgp):
    rng = np.random.default_rng(3)
    N, d, Zn = 200, 5, 60
    X, Y = _data(rng, N, d, 1)
    Z = None if vgp else X[rng.choice(N, Zn, replace=False)]
    s, ls, nz = np.array([0.9]), np.full((1, d), 0.7), np.array([0.02])
    st = L.SVGPFitState(X, Y, Z, 1, inducing_is_data=vgp)
    st.natgrad(np.arange(N), s, ls, nz, gamma=1.0)
    q_mu, q_sqrt = st.q()
    r_mu, r_sqrt = L.svgp_optimal_q(X, Y.T, None if vgp else Z[None], s, ls, nz, inducing_is_data=vgp)
    assert np.abs(q_mu - r_mu).max() / np.abs(r_mu).max() < 1e-9
    S, Sr = q_sqrt[0] @ q_sqrt[0].T, r_sqrt[0] @ r_sqrt[0].T
    assert np.abs(S - Sr).max() / np.abs(Sr).max() < 1e-9
    o_mu, o_S = ov.optimal_q(X, Y[:, 0], X if vgp else Z, s[0], ls[0], nz[0], inducing_is_data=vgp)
    assert np.abs(q_mu[0] - o_mu).max() / np.abs(o_mu).max() < 1e-8


def test_bad_arguments_are_refused(L):
    rng = np.random.default_rng(0)
    X, Y = _data(rng, 50, 3, 1)
    st = L.SVGPFitState(X, Y, X[:10], 1)
    s, ls, nz = np.array([1.0]), np.ones((1, 3)), np.array([0.1])
    with pytest.raises(L.DmoError, match="outside"):
        st.elbo_grad(np.array([0, 50]), s, ls, nz)
    with pytest.raises(L.DmoError, match="noise"):
        st.natgrad(np.arange(5), s, ls, np.array([0.0]))
    v = L.SVGPFitState(X, Y, None, 1, inducing_is_data=True)
    with pytest.raises(L.DmoError, match="full data"):
        v.natgrad(np.arange(10), s, ls, nz)


def test_svgp_fit_follows_the_oracle_loop(L):
    """100 iterations of SPV (two latents, minibatches of 50) and CRV against the oracle loop on the same batch stream.
    Both run the same float64 arithmetic up to summation order; the trajectories are compared at 1e-7 relative: each
    iteration adds rounding differences of ~1e-15 relative that Adam's normalised steps do not amplify beyond that."""
    from dmosopt_b200 import model_gpflow as mg

    rng = np.random.default_rng(5)
    N, d, M = 160, 4, 2
    X, Y = _data(rng, N, d, M)
    Z = X[:40].copy()
    for kind in ("spv", "crv"):
        W0 = np.array([[1.0, 0.3], [-0.2, 0.8]]) if kind == "crv" else None
        hp, info = mg.svgp_fit(kind, X, Y, Z, n_iter=100, seed=9, W0=W0)
        s = mg.MinibatchStream(N, 50, [9, 0])
        stream = (s.next() for _ in iter(int, 1))
        log, (rs, rls, rnz, rW, rqm, rqs) = vt.train(kind, X, Y, Z, stream, 100, gamma=0.1, W0=W0)
        assert info["iterations"] == [100]
        np.testing.assert_allclose(info["elbo"][0], log, rtol=1e-7)
        np.testing.assert_allclose(hp["lengthscales"], rls, rtol=1e-7)
        np.testing.assert_allclose(hp["variance"], rs, rtol=1e-7)
        np.testing.assert_allclose(hp["q_mu"], rqm, rtol=1e-6, atol=1e-9)
        if kind == "crv":
            np.testing.assert_allclose(hp["W"], rW, rtol=1e-7)


def test_lockstep_training_is_bitwise_that_of_one_output(L):
    from dmosopt_b200 import model_gpflow as mg

    rng = np.random.default_rng(8)
    X, Y = _data(rng, 150, 3, 3)
    Z = np.stack([X[rng.choice(150, 30, replace=False)] for _ in range(3)])
    hp, info = mg.svgp_fit("svgp", X, Y, Z, n_iter=30, seed=4)
    # output 2 alone: its own model with the same stream seed [seed, 2]
    m = mg._FitModel(X, Y, Z[2], [2], 1, 1, False, dict(lengthscale_bounds=(1e-6, 100.0), likelihood_sigma=1e-4, adam_lr=0.01, batch_size=50),
                     [4, 2], None)
    for it in range(30):
        m.step(0.1)
        if it % 10 == 0:
            m.elbo_log.append(m.elbo(m.batch()))
    assert np.array_equal(np.asarray(m.elbo_log), info["elbo"][2])
    q_mu, _ = m.state.q()
    assert np.array_equal(q_mu[0], hp["q_mu"][2])


@pytest.mark.parametrize("cls", ["SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern", "CRV_Matern"])
def test_fit_gpu_builds_every_class_from_raw_data(L, cls):
    from dmosopt_b200 import model_gpflow as mg

    rng = np.random.default_rng(21)
    d, N = 6, 300
    X = rng.random((N, d))
    Y = _zdt1(X)
    Xt = rng.random((200, d))
    Yt = _zdt1(Xt)
    n_iter = 300 if cls == "VGP_Matern" else 1500
    m = getattr(mg, cls)(X, Y, d, 2, np.zeros(d), np.ones(d), seed=3, fit="gpu", n_iter=n_iter, inducing_fraction=0.2, min_inducing=50)
    for e in m.fit_info["elbo"]:
        assert e[-1] > e[0]
    mean, var = m.predict(Xt)
    rel = np.sqrt(np.mean((mean - Yt) ** 2, axis=0)) / Yt.std(axis=0)
    assert np.all(rel < 0.25), rel
    assert np.all(np.isfinite(var)) and np.all(var > -1e-6)
    m2 = getattr(mg, cls)(X, Y, d, 2, np.zeros(d), np.ones(d), seed=3, hyperparameters=m.hyperparameters)
    mean2, var2 = m2.predict(Xt)
    assert np.array_equal(mean, mean2) and np.array_equal(var, var2)


def test_vgp_lands_near_the_exact_gp_at_its_noise(L):
    """At gamma = 1 q is the exact posterior of f(X) = Lz v, so the VGP predicts as the exact GP with noise
    sigma2 + jitter at the trained hyper-parameters."""
    from dmosopt_b200 import model_gpflow as mg

    rng = np.random.default_rng(2)
    d, N = 4, 200
    X, Y = _data(rng, N, d, 1)
    hp, info = mg.svgp_fit("vgp", X, Y, None, n_iter=200, seed=1)
    Xt = rng.random((100, d))
    ls, s, nz = hp["lengthscales"][0], hp["variance"][0], hp["likelihood_variance"][0]
    K = ov.matern52(X, X, s, ls) + (nz + mg.JITTER) * np.eye(N)
    ks = ov.matern52(Xt, X, s, ls)
    exact = ks @ np.linalg.solve(K, Y[:, 0])
    mean, _ = ov.latent_predict(Xt, X, s, ls, hp["q_mu"][0], hp["q_sqrt"][0])
    # q is the optimum for the hyper-parameters before the last Adam step; the last step moves them by ~lr
    assert np.abs(mean - exact).max() < 0.05 * np.abs(exact).max()


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("surrogate", ["SVGP_Matern", "CRV_Matern"])
def test_unmodified_moasmo_epoch_trains_the_variational_plugins_on_the_gpu(L, surrogate):
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
    gen = MOASMO.epoch(
        6, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name="dmosopt_b200.NSGA2",
        optimizer_kwargs={}, surrogate_method_name=f"dmosopt_b200.{surrogate}", surrogate_method_kwargs={"fit": "gpu", "n_iter": 50},
        local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
