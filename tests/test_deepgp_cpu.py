"""CPU checks of the deep GP oracle (oracle/deepgp.py) and of MDSPP_Matern / MDGP_Matern's host side: the read-out of a
trained gpytorch model (on a stand-in with gpytorch's attribute names) and the constructor's refusals."""

from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import deepgp as DG
from oracle import variational as V


def problem(rng, d, H, T, Z1, Z2, J=3, quadrature=True):
    """A random deep GP in the ``hyperparameters=`` layout with q_sqrt holding junk above the diagonal (masked by every
    consumer), and its y statistics and input box."""
    def chol(n, m):
        L = 0.3 * rng.standard_normal((n, m, m)) + 3.0 * np.triu(rng.standard_normal((n, m, m)), 1)
        L[:, np.arange(m), np.arange(m)] = 0.2 + 0.5 * rng.random((n, m))
        return L

    hp = {
        "hidden_inducing_points": np.broadcast_to(rng.random((Z1, d)), (H, Z1, d)).copy(),
        "hidden_outputscale": 0.5 + rng.random(H), "hidden_lengthscale": np.sqrt(d) * (0.3 + 0.4 * rng.random((H, d))),
        "hidden_variational_mean": rng.standard_normal((H, Z1)), "hidden_chol_variational_covar": chol(H, Z1),
        "mean_weights": 0.5 * rng.standard_normal(d), "mean_bias": float(rng.standard_normal()),
        "last_inducing_points": 1.5 * rng.standard_normal((T, Z2, H)), "last_outputscale": 0.5 + rng.random(T),
        "last_lengthscale": 1.0 + rng.random((T, H)), "last_variational_mean": rng.standard_normal((T, Z2)),
        "last_chol_variational_covar": chol(T, Z2), "mean_constant": float(rng.standard_normal()),
        "task_noises": 1e-3 + 1e-2 * rng.random(T), "noise": 2e-3,
    }
    if quadrature:
        hp["quad_sites"] = rng.standard_normal((J, H))
    xlb, xrng = -1.0 - rng.random(d), 2.0 + rng.random(d)
    return hp, 3.0 * rng.standard_normal(T), 0.5 + 2.0 * rng.random(T), xlb, xrng


def test_layer_is_the_variational_latent_plus_prior_mean_and_jitter():
    rng = np.random.default_rng(0)
    hp, *_ = problem(rng, 4, 2, 1, 20, 10)
    xn = rng.random((30, 4))
    Z, s, ls = hp["hidden_inducing_points"][1], hp["hidden_outputscale"][1], hp["hidden_lengthscale"][1]
    qm, L = hp["hidden_variational_mean"][1], hp["hidden_chol_variational_covar"][1]
    m, v = DG.layer(xn, Z, s, ls, qm, L, 0.7, jitter=1e-4)
    m0, v0 = V.latent_predict(xn, Z, s, ls, qm, np.tril(L), jitter=1e-4)
    np.testing.assert_array_equal(m, m0 + 0.7)
    np.testing.assert_array_equal(v, v0 + 1e-4)


def test_mdgp_with_the_quadrature_sites_as_draws_is_mdspp():
    rng = np.random.default_rng(1)
    hp, ym, ys, xlb, xrng = problem(rng, 5, 3, 2, 25, 12, J=4)
    x = xlb + xrng * rng.random((40, 5))
    eps = np.broadcast_to(hp["quad_sites"][:, None, :], (4, 40, 3))
    a = DG.predict(x, xlb, xrng, hp, ym, ys)
    b = DG.predict(x, xlb, xrng, hp, ym, ys, eps=eps.copy())
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])


def test_identical_sites_equal_one_site():
    rng = np.random.default_rng(2)
    hp, ym, ys, xlb, xrng = problem(rng, 3, 2, 3, 15, 9, J=1)
    x = xlb + xrng * rng.random((25, 3))
    one = DG.predict(x, xlb, xrng, hp, ym, ys)
    hp5 = dict(hp, quad_sites=np.repeat(hp["quad_sites"], 5, axis=0))
    five = DG.predict(x, xlb, xrng, hp5, ym, ys)
    np.testing.assert_allclose(five[0], one[0], rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(five[1], one[1], rtol=1e-14)


def test_min_variance_floor_binds_where_it_should():
    rng = np.random.default_rng(3)
    hp, ym, ys, xlb, xrng = problem(rng, 3, 2, 2, 15, 9)
    x = xlb + xrng * rng.random((25, 3))
    xn = (x - xlb) / xrng
    _, sd_free = DG.hidden(xn, hp, min_variance=0.0)
    floor = float(np.median(sd_free**2))
    _, sd = DG.hidden(xn, hp, min_variance=floor)
    low = sd_free**2 < floor
    assert low.any() and (~low).any()
    np.testing.assert_array_equal(sd[low], np.sqrt(floor))
    np.testing.assert_array_equal(sd[~low], sd_free[~low])
    # a floor above every site's predictive variance: the output variance is y_std^2 times the floor
    _, var = DG.predict(x, xlb, xrng, hp, ym, ys, min_variance=1e3)
    np.testing.assert_allclose(var, np.broadcast_to(ys**2 * 1e3, var.shape), rtol=1e-15)
    _, var0 = DG.predict(x, xlb, xrng, hp, ym, ys, min_variance=0.0)
    _, var1 = DG.predict(x, xlb, xrng, hp, ym, ys, min_variance=1e-12)
    np.testing.assert_array_equal(var0, var1)  # far below every variance: no effect


def _stub_model(hp, d, H, T, wrapped, whitened=True, torch=None):
    t32 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)  # noqa: E731

    def layer(prefix, n_units, mean_module, extra=None):
        ls = hp[f"{prefix}_lengthscale"][:, :1].reshape(n_units, 1, 1)  # ard_num_dims=None: one length scale per unit
        scale = NS(outputscale=t32(hp[f"{prefix}_outputscale"]), base_kernel=NS(lengthscale=t32(ls)))
        dist = type("CholeskyVariationalDistribution", (), {})()
        dist.variational_mean = t32(hp[f"{prefix}_variational_mean"])
        dist.chol_variational_covar = t32(hp[f"{prefix}_chol_variational_covar"])
        strategy = type("VariationalStrategy" if whitened else "UnwhitenedVariationalStrategy", (), {})()
        Z = hp[f"{prefix}_inducing_points"]
        strategy.inducing_points = t32(Z[0] if prefix == "hidden" else Z)  # the hidden layer's one k-means set
        strategy._variational_distribution = dist
        lay = NS(variational_strategy=strategy, covar_module=NS(module=scale) if wrapped else scale, mean_module=mean_module,
                 output_dims=n_units, **(extra or {}))
        return lay

    hidden = layer("hidden", H, NS(weights=t32(hp["mean_weights"].reshape(d, 1)), bias=t32([hp["mean_bias"]])))
    last = layer("last", T, NS(constant=t32(hp["mean_constant"])), {"quad_sites": t32(hp["quad_sites"])} if "quad_sites" in hp else None)
    lik = NS(task_noises=t32(hp["task_noises"]), noise=t32([hp["noise"]]))
    return NS(hidden_layer=hidden, last_layer=last, likelihood=lik)


@pytest.mark.parametrize("wrapped", [False, True])
def test_read_out_of_a_trained_model(wrapped):
    torch = pytest.importorskip("torch")
    from dmosopt_b200.model_gpytorch import deepgp_check_hyperparameters, deepgp_hyperparameters

    rng = np.random.default_rng(4)
    d, H, T = 4, 3, 2
    hp, *_ = problem(rng, d, H, T, 11, 7, J=5)
    hp["hidden_lengthscale"] = np.repeat(hp["hidden_lengthscale"][:, :1], d, axis=1)
    hp["last_lengthscale"] = np.repeat(hp["last_lengthscale"][:, :1], H, axis=1)
    model = _stub_model(hp, d, H, T, wrapped, torch=torch)
    out = deepgp_hyperparameters(model, d, T, quadrature=True)
    f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731
    for k in hp:
        want = f32(hp[k])
        if k.endswith("chol_variational_covar"):
            want = np.tril(want)  # the junk above the diagonal is masked
            assert np.any(np.triu(hp[k], 1) != 0)
        got = np.asarray(out[k])
        assert got.dtype == np.float64, k
        np.testing.assert_array_equal(got, want, err_msg=k)
    assert out["quad_sites"].shape == (5, H)  # J from the parameter's shape
    deepgp_check_hyperparameters(out, d, T, True, "MDSPP_Matern")


def test_read_out_refuses_an_unwhitened_strategy():
    torch = pytest.importorskip("torch")
    from dmosopt_b200.model_gpytorch import deepgp_hyperparameters

    rng = np.random.default_rng(5)
    hp, *_ = problem(rng, 3, 2, 1, 6, 5)
    with pytest.raises(ValueError, match="whitened VariationalStrategy"):
        deepgp_hyperparameters(_stub_model(hp, 3, 2, 1, False, whitened=False, torch=torch), 3, 1, quadrature=True)


def _data(rng, N, d, T):
    return rng.random((N, d)), rng.standard_normal((N, T)), np.zeros(d), np.ones(d)


@pytest.mark.parametrize("cls", ["MDSPP_Matern", "MDGP_Matern"])
def test_constructor_refusals(cls):
    from dmosopt_b200 import _lib, model_gpytorch as mg

    C = getattr(mg, cls)
    rng = np.random.default_rng(6)
    x, y, lb, ub = _data(rng, 20, 3, 2)
    hp, *_ = problem(rng, 3, 2, 2, 8, 6)
    with pytest.raises(ValueError, match="not built yet"):
        C(x, y, 3, 2, lb, ub, fit="gpu")
    with pytest.raises(ValueError, match="precision"):
        C(x, y, 3, 2, lb, ub, precision="auto", hyperparameters=hp)
    bad = dict(hp)
    bad["last_variational_mean"] = bad["last_variational_mean"][:, :-1]
    with pytest.raises(ValueError, match="last_chol_variational_covar|last_inducing_points"):
        C(x, y, 3, 2, lb, ub, hyperparameters=bad)
    with pytest.raises(ValueError, match="missing mean_constant"):
        C(x, y, 3, 2, lb, ub, hyperparameters={k: v for k, v in hp.items() if k != "mean_constant"})
    if cls == "MDSPP_Matern":
        with pytest.raises(ValueError, match="quad_sites"):
            C(x, y, 3, 2, lb, ub, hyperparameters=dict(hp, quad_sites=np.zeros((3, 5))))
    d = _lib.GP_PREDICT_MAX_D + 1
    xd, yd, lbd, ubd = _data(rng, 20, d, 2)
    with pytest.raises(ValueError, match="precision='fp64'"):
        C(xd, yd, d, 2, lbd, ubd, precision="tensor", hyperparameters=problem(rng, d, 2, 2, 8, 6)[0])


def test_missing_gpytorch_without_hyperparameters_is_a_clear_error():
    from dmosopt_b200 import model_gpytorch as mg

    try:
        import dmosopt.model_gpytorch as ref

        if getattr(ref, "_has_gpytorch", False):
            pytest.skip("gpytorch is installed")
    except Exception:
        pass
    rng = np.random.default_rng(7)
    x, y, lb, ub = _data(rng, 20, 3, 2)
    with pytest.raises(RuntimeError, match="hyperparameters="):
        mg.MDSPP_Matern(x, y, 3, 2, lb, ub)
