"""The variational surrogates without a GPU: the oracle against the exact GP, the read-out of gpflow posterior objects,
the inducing-point rule and the error without gpflow or hyper-parameters."""

import types

import numpy as np
import pytest

from oracle import gp as gp_oracle
from oracle import variational as V


def test_oracle_vgp_at_the_optimum_is_the_exact_gp_as_jitter_vanishes():
    """SVGP with every training point as inducing point (Z = X) and its optimal q is the exact GP with noise sigma^2 only
    once the jitter is negligible: its data term sees K(X, X), its prior K + j I.  (GPflow's VGP differs: its data term
    sees K + j I too, see the next test.)  The exact side is oracle/gp.py."""
    rng = np.random.default_rng(3)
    N, d, s, sig, jit = 70, 3, 0.8, 2e-2, 1e-11
    xlb, xub = np.zeros(d), np.ones(d)
    X, ls = rng.random((N, d)), np.array([0.5, 0.7, 0.9])
    y = np.sin(3 * X.sum(1))
    st = gp_oracle.fit_fixed(X, y.reshape(-1, 1), xlb, xub, constant=s, length_scale=ls, noise=sig + jit - 1e-10)
    ob = st.objectives[0]
    yn = (y - ob.y_mean) / ob.y_std
    qm, S = V.optimal_q(X, yn, X, s, ls, sig, jit)
    xs = rng.random((40, d))
    m, v = V.latent_predict(xs, X, s, ls, qm, np.linalg.cholesky(S), jit)
    me, ve = gp_oracle.predict(st, xs)
    ys = ob.y_std
    np.testing.assert_allclose(m * ys + ob.y_mean, me[:, 0], atol=1e-7 * ys)
    np.testing.assert_allclose(v * ys ** 2, ve[:, 0] - (sig + jit) * ys ** 2, atol=1e-7 * s * ys ** 2)


_Matern = type("Matern52", (), {})
_Zero = type("Zero", (), {})
_Linear = type("Linear", (), {})


def _kern(variance, ls):
    k = _Matern()
    k.variance, k.lengthscales = np.float64(variance), np.asarray(ls, dtype=np.float64)
    return k


def _posterior(kernel, X_data, q_mu, q_sqrt, whiten=True, mean_function=None):
    p = types.SimpleNamespace(kernel=kernel, X_data=X_data, whiten=whiten, mean_function=mean_function if mean_function is not None else _Zero())
    p.q_dist = types.SimpleNamespace(q_mu=q_mu, q_sqrt=q_sqrt)
    return p


def test_readout_of_gpflow_posteriors():
    from dmosopt_b200.model_gpflow import read_gpflow_posterior

    rng = np.random.default_rng(0)
    Zn, d, L = 7, 2, 3
    Z = rng.random((Zn, d))
    q_mu = rng.standard_normal((Zn, L))
    q_sqrt = np.tril(rng.standard_normal((L, Zn, Zn)))
    # SVGP: one output, InducingPoints
    st = read_gpflow_posterior(_posterior(_kern(0.7, [0.3, 0.4]), types.SimpleNamespace(Z=Z), q_mu[:, :1], q_sqrt[:1]), d)
    assert st["Z"].shape == (1, Zn, d) and st["W"] is None
    np.testing.assert_array_equal(st["q_mu"], q_mu[:, :1].T)
    np.testing.assert_array_equal(st["lengthscales"], [[0.3, 0.4]])
    # SIV: SharedIndependent + SharedIndependentInducingVariables, scalar length scale broadcast
    shared = types.SimpleNamespace(kernel=_kern(0.5, 0.2))
    st = read_gpflow_posterior(_posterior(shared, types.SimpleNamespace(inducing_variable=types.SimpleNamespace(Z=Z)), q_mu, q_sqrt), d)
    assert st["Z"].shape == (L, Zn, d) and np.all(st["variance"] == 0.5) and np.all(st["lengthscales"] == 0.2)
    np.testing.assert_array_equal(st["q_sqrt"], q_sqrt)
    # SPV: SeparateIndependent + SeparateIndependentInducingVariables
    sep = types.SimpleNamespace(kernels=[_kern(0.1 * (l + 1), [0.5, 0.6]) for l in range(L)])
    ivs = types.SimpleNamespace(inducing_variable_list=[types.SimpleNamespace(Z=Z + l) for l in range(L)])
    st = read_gpflow_posterior(_posterior(sep, ivs, q_mu, q_sqrt), d)
    np.testing.assert_allclose(st["variance"], [0.1, 0.2, 0.3])
    np.testing.assert_array_equal(st["Z"][2], Z + 2)
    # CRV: LinearCoregionalization carries W
    W = rng.standard_normal((2, L))
    crv = types.SimpleNamespace(kernels=sep.kernels, W=W)
    st = read_gpflow_posterior(_posterior(crv, types.SimpleNamespace(inducing_variable=types.SimpleNamespace(Z=Z)), q_mu, q_sqrt), d)
    np.testing.assert_array_equal(st["W"], W)
    # q_diag: (Z, L) standard deviations become diagonal q_sqrt
    qd = rng.random((Zn, L))
    st = read_gpflow_posterior(_posterior(shared, types.SimpleNamespace(inducing_variable=types.SimpleNamespace(Z=Z)), q_mu, qd), d)
    np.testing.assert_array_equal(st["q_sqrt"][1], np.diag(qd[:, 1]))


def test_readout_refuses_what_it_would_mis_predict():
    from dmosopt_b200.model_gpflow import read_gpflow_posterior

    Z = np.zeros((3, 2))
    args = (_kern(1.0, [1.0, 1.0]), types.SimpleNamespace(Z=Z), np.zeros((3, 1)), np.eye(3)[None])
    with pytest.raises(ValueError, match="whiten"):
        read_gpflow_posterior(_posterior(*args, whiten=False), 2)
    with pytest.raises(ValueError, match="zero mean"):
        read_gpflow_posterior(_posterior(*args, mean_function=_Linear()), 2)
    rbf = type("SquaredExponential", (), {})()
    rbf.variance, rbf.lengthscales = 1.0, 1.0
    with pytest.raises(ValueError, match="Matern52"):
        read_gpflow_posterior(_posterior(rbf, *args[1:]), 2)


def test_inducing_point_rule():
    from dmosopt_b200.model_gpflow import choose_inducing

    xn = np.random.default_rng(1).random((400, 3))
    np.testing.assert_array_equal(choose_inducing(xn, 0.2, 100, np.random.default_rng(0)), xn)  # round(80) < 100: all points
    Z = choose_inducing(xn, 0.2, 50, np.random.default_rng(0))
    assert Z.shape == (80, 3)
    rows = {tuple(r) for r in xn}
    assert all(tuple(r) in rows for r in Z) and len({tuple(r) for r in Z}) == 80
    np.testing.assert_array_equal(Z, choose_inducing(xn, 0.2, 50, np.random.default_rng(0)))  # seeded


@pytest.mark.parametrize("name", ["SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern", "CRV_Matern"])
def test_without_gpflow_and_hyperparameters_the_error_says_what_to_pass(name):
    from dmosopt_b200 import model_gpflow

    if model_gpflow._gpflow_available():
        pytest.skip("gpflow is importable here")
    cls = getattr(model_gpflow, name)
    with pytest.raises(RuntimeError, match="hyperparameters="):
        cls(np.zeros((10, 2)), np.zeros((10, 2)), 2, 2, np.zeros(2), np.ones(2))


def test_oracle_vgp_optimum_is_the_exact_gp_at_the_reference_jitter():
    """GPflow's VGP (f(X) = Lz v, Lz = chol(K + j I)) at its optimal q is the exact GP with noise sigma^2 + j, whose
    variance without the noise is the VGP's, at the reference's jitter 1e-2."""
    rng = np.random.default_rng(4)
    N, d, s, sig, jit = 90, 3, 0.8, 1e-4, V.JITTER
    xlb, xub = np.zeros(d), np.ones(d)
    X, ls = rng.random((N, d)), np.array([0.4, 0.6, 0.8])
    y = np.sin(3 * X.sum(1))
    st = gp_oracle.fit_fixed(X, y.reshape(-1, 1), xlb, xub, constant=s, length_scale=ls, noise=sig + jit - 1e-10)
    ob = st.objectives[0]
    yn = (y - ob.y_mean) / ob.y_std
    qm, S = V.optimal_q(X, yn, X, s, ls, sig, jit, inducing_is_data=True)
    xs = rng.random((40, d))
    m, v = V.latent_predict(xs, X, s, ls, qm, np.linalg.cholesky(S), jit)
    me, ve = gp_oracle.predict(st, xs)
    ys = ob.y_std
    np.testing.assert_allclose(m * ys + ob.y_mean, me[:, 0], atol=1e-9 * ys)
    np.testing.assert_allclose(v * ys ** 2, ve[:, 0] - (sig + jit) * ys ** 2, atol=1e-9 * s * ys ** 2)
    # the SVGP form of the optimum (data term without the jitter) is measurably different at this jitter
    qs, _ = V.optimal_q(X, yn, X, s, ls, sig, jit)
    assert np.abs(qs - qm).max() > 1e-4 * np.abs(qm).max()


def test_explicit_fit_with_hyperparameters_is_refused():
    from dmosopt_b200 import model_gpflow

    with pytest.raises(ValueError, match="conflict"):
        model_gpflow.SVGP_Matern(np.zeros((10, 2)), np.zeros((10, 2)), 2, 2, np.zeros(2), np.ones(2), fit="reference",
                                 hyperparameters=dict(lengthscales=np.ones((2, 2)), variance=[1.0, 1.0], likelihood_variance=1e-3))


def test_reference_fit_gets_the_reference_batch_size_default(monkeypatch):
    """Without an explicit batch_size the reference class keeps its own default (50 for the SVGP forms: its training
    minibatches), instead of receiving None."""
    from dmosopt_b200 import model_gpflow

    seen = {}

    def fake_fit(self, *args, **kw):
        seen.update(kw)
        raise RuntimeError("stop")

    monkeypatch.setattr(model_gpflow, "_gpflow_available", lambda: True)
    monkeypatch.setattr(model_gpflow._VariationalGP, "_fit_with_reference", fake_fit)
    for kw, expect in (({}, None), ({"batch_size": 20}, 20)):
        seen.clear()
        with pytest.raises(RuntimeError, match="stop"):
            model_gpflow.CRV_Matern(np.zeros((10, 2)), np.zeros((10, 2)), 2, 2, np.zeros(2), np.ones(2), **kw)
        assert seen.get("batch_size") == expect
