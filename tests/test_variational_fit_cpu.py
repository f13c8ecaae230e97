"""Host side of the variational surrogates' training (no GPU): the oracle's autograd ELBO gradient against central
differences, its autograd-derived natural-gradient step at gamma = 1 on the full batch against the closed-form optimum
(oracle/variational.py), keras' Adam, the reference's stopping statistic, the minibatch stream, and argument errors."""

import numpy as np
import pytest

from oracle import variational as ov
from oracle import variational_train as vt

torch = pytest.importorskip("torch")


def _setup(rng, N=30, d=3, Zn=8, M=2):
    X = rng.random((N, d))
    Y = rng.standard_normal((N, M))
    Z = X[:Zn].copy()
    s = 0.7 + rng.random(M)
    ls = 0.5 + rng.random((M, d))
    nz = np.array([0.1, 0.2])[:M]
    W = rng.standard_normal((M, M))
    return X, Y, Z, s, ls, nz, W


@pytest.mark.parametrize("vgp", [False, True])
def test_autograd_gradient_matches_central_differences(vgp):
    rng = np.random.default_rng(0)
    X, Y, Z, s, ls, nz, W = _setup(rng)
    Zq = X.shape[0] if vgp else Z.shape[0]
    q_mu = rng.standard_normal((2, Zq))
    q_sqrt = np.tril(rng.standard_normal((2, Zq, Zq))) * 0.1 + np.eye(Zq)
    batch = np.arange(X.shape[0]) if vgp else rng.permutation(X.shape[0])[:11]

    def f(s_, ls_, nz_, W_):
        ell, kl, _ = vt.elbo_and_grad(X, Y, Z, batch, s_, ls_, nz_, W_, q_mu, q_sqrt, vgp)
        return ell.sum() - kl.sum()

    _, _, g = vt.elbo_and_grad(X, Y, Z, batch, s, ls, nz, W, q_mu, q_sqrt, vgp)
    h = 1e-6
    args = dict(s_=s, ls_=ls, nz_=nz, W_=W)
    for key, gk in (("s_", "variance"), ("ls_", "length_scale"), ("nz_", "noise"), ("W_", "W")):
        base = args[key]
        for idx in np.ndindex(base.shape):
            up, dn = base.copy(), base.copy()
            up[idx] += h
            dn[idx] -= h
            fd = (f(**dict(args, **{key: up})) - f(**dict(args, **{key: dn}))) / (2 * h)
            assert abs(fd - g[gk][idx]) <= 1e-5 * max(1.0, abs(fd)), (key, idx, fd, g[gk][idx])


@pytest.mark.parametrize("vgp", [False, True])
def test_oracle_natgrad_at_gamma_one_is_the_optimal_q(vgp):
    rng = np.random.default_rng(1)
    X, Y, Z, s, ls, nz, _ = _setup(rng, M=1)
    Zq = X.shape[0] if vgp else Z.shape[0]
    q_mu, q_sqrt = vt.natgrad_step(X, Y, Z, np.arange(X.shape[0]), s, ls, nz, None, np.zeros((1, Zq)), np.stack([np.eye(Zq)]), 1.0, vgp)
    r_mu, r_S = ov.optimal_q(X, Y[:, 0], X if vgp else Z, s[0], ls[0], nz[0], inducing_is_data=vgp)
    np.testing.assert_allclose(q_mu[0], r_mu, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(q_sqrt[0] @ q_sqrt[0].T, r_S, rtol=1e-8, atol=1e-10)


def test_keras_adam_matches_a_literal_restatement():
    from dmosopt_b200.model_gpflow import KerasAdam

    rng = np.random.default_rng(2)
    p = {"a": rng.standard_normal(4)}
    ref = p["a"].copy()
    m = np.zeros(4)
    v = np.zeros(4)
    adam = KerasAdam(lr=0.01)
    for t in range(1, 30):
        g = rng.standard_normal(4)
        adam.step(p, {"a": g})
        m = m + (g - m) * (1 - 0.9)
        v = v + (np.square(g) - v) * (1 - 0.999)
        ref = ref - 0.01 * np.sqrt(1 - 0.999**t) / (1 - 0.9**t) * m / (np.sqrt(v) + 1e-7)
        assert np.array_equal(p["a"], ref)


def test_stopping_statistic_is_the_literal_convolve_expression():
    from dmosopt_b200.model_gpflow import mean_elbo_pct_change

    rng = np.random.default_rng(3)
    log = list(-1000 + np.cumsum(rng.random(250)))
    diff_kernel = np.array([1, -1])
    elbo_change = np.convolve(log, diff_kernel, "same")[1:]
    elbo_pct_change = (elbo_change / np.abs(log[1:])) * 100
    assert mean_elbo_pct_change(np.asarray(log)) == np.mean(elbo_pct_change[-100:])


def test_minibatch_stream_is_reproducible_and_walks_permutations():
    from dmosopt_b200.model_gpflow import MinibatchStream

    a, b = MinibatchStream(23, 5, [4, 1]), MinibatchStream(23, 5, [4, 1])
    xa = np.concatenate([a.next() for _ in range(23)])
    xb = np.concatenate([b.next() for _ in range(23)])
    assert np.array_equal(xa, xb)
    for k in range(5):  # 115 indices: five whole permutations
        assert np.array_equal(np.sort(xa[23 * k : 23 * (k + 1)]), np.arange(23))
    assert not np.array_equal(xa[:23], MinibatchStream(23, 5, [4, 2]).next())


def test_argument_errors():
    from dmosopt_b200 import model_gpflow as mg

    X, Y = np.zeros((10, 2)), np.zeros((10, 2))
    with pytest.raises(ValueError, match="fit must be"):
        mg.SVGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="cpu")
    with pytest.raises(ValueError, match="num_latent_gps"):
        mg.CRV_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="gpu", num_latent_gps=1)
    with pytest.raises(ValueError, match="conflict"):
        mg.SPV_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="gpu", hyperparameters={"lengthscales": np.ones(2)})
