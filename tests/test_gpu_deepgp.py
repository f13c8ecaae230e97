"""dmo_dgp (csrc/gp_deep.cu), the two-layer deep GP predict of MDSPP_Matern and MDGP_Matern, against oracle/deepgp.py.

Bars: float64, the mean within 1e-9 max(|mean|, y_std) and the variance within 1e-9 y_std^2 (s2 + noise); the tensor
hidden-layer variance within 1e-4 of the same scales.  MDGP is replayed from the draws the call returns (eps_out)."""

import numpy as np
import pytest

from oracle import deepgp as DG
from test_deepgp_cpu import problem

pytestmark = pytest.mark.gpu

SHAPES = [  # (d, H, T, Z1, Z2, J, P)
    (2, 1, 1, 5, 3, 1, 1),
    (12, 3, 2, 128, 128, 3, 1000),
    (30, 3, 3, 128, 128, 10, 4097),
    (40, 8, 8, 300, 37, 16, 513),
    (90, 2, 3, 64, 64, 3, 100),
]


def _handle(hp, ym, ys, xlb, xrng, quadrature, J, **kw):
    from dmosopt_b200 import _lib

    return _lib.DGPHandle(hp["hidden_inducing_points"], hp["hidden_outputscale"], hp["hidden_lengthscale"], hp["hidden_variational_mean"],
                          np.tril(hp["hidden_chol_variational_covar"]), hp["mean_weights"], hp["mean_bias"], hp["last_inducing_points"],
                          hp["last_outputscale"], hp["last_lengthscale"], hp["last_variational_mean"],
                          np.tril(hp["last_chol_variational_covar"]), hp["mean_constant"], hp["task_noises"] + hp["noise"], ym, ys, xlb, xrng,
                          quad_sites=hp["quad_sites"] if quadrature else None, n_sites=J, **kw)


def _case(seed, d, H, T, Z1, Z2, J, P, quadrature):
    rng = np.random.default_rng(seed)
    hp, ym, ys, xlb, xrng = problem(rng, d, H, T, Z1, Z2, J=J, quadrature=quadrature)
    x = xlb + xrng * (1.2 * rng.random((P, d)) - 0.1)
    return hp, ym, ys, xlb, xrng, x


def _assert_bars(hp, ys, mean, var, m_ref, v_ref, tol):
    ms = np.maximum(np.abs(m_ref), ys)
    vs = ys**2 * (hp["last_outputscale"] + hp["task_noises"] + hp["noise"])
    assert np.all(np.isfinite(mean)) and np.all(np.isfinite(var))
    assert np.max(np.abs(mean - m_ref) / ms) <= tol, np.max(np.abs(mean - m_ref) / ms)
    assert np.max(np.abs(var - v_ref) / vs) <= tol, np.max(np.abs(var - v_ref) / vs)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "d{}-H{}-T{}-Z{}-{}-J{}-P{}".format(*s))
@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
@pytest.mark.parametrize("precision", ["fp64", "tensor"])
def test_predict_matches_oracle(shape, quadrature, precision):
    from dmosopt_b200 import _lib

    d, H, T, Z1, Z2, J, P = shape
    if precision == "tensor" and d > _lib.GP_PREDICT_MAX_D:
        pytest.skip("the tensor path takes d <= 64")
    hp, ym, ys, xlb, xrng, x = _case(10 + d, *shape, quadrature)
    g = _handle(hp, ym, ys, xlb, xrng, quadrature, J)
    mean, var, eps = g.predict(x, seed=123, stream_id=4, return_eps=True,
                               precision=_lib.GP_FP64 if precision == "fp64" else _lib.GP_TENSOR)
    assert eps.shape == (J, P, H)
    if quadrature:
        np.testing.assert_array_equal(eps, np.broadcast_to(hp["quad_sites"][:, None, :], eps.shape))
    m_ref, v_ref = DG.predict(x, xlb, xrng, hp, ym, ys, eps=None if quadrature else eps)
    _assert_bars(hp, ys, mean, var, m_ref, v_ref, 1e-9 if precision == "fp64" else 1e-4)


@pytest.mark.parametrize("J", [3, 10])
@pytest.mark.parametrize("dP", [-1, 1])
def test_one_candidate_tile_plus_minus_one(J, dP):
    P = 64 // J + dP  # a CTA takes the J sites of 64 // J candidates
    hp, ym, ys, xlb, xrng, x = _case(20 + J, 5, 2, 2, 40, 30, J, P, False)
    mean, var, eps = _handle(hp, ym, ys, xlb, xrng, False, J).predict(x, seed=9, return_eps=True)
    m_ref, v_ref = DG.predict(x, xlb, xrng, hp, ym, ys, eps=eps)
    _assert_bars(hp, ys, mean, var, m_ref, v_ref, 1e-9)


def test_two_hidden_layer_chunks():
    from dmosopt_b200 import _lib

    P = (1 << 20) + 1  # GP_MAX_CHUNK + 1 candidates: the hidden layer runs two chunks
    hp, ym, ys, xlb, xrng, x = _case(30, 2, 1, 1, 16, 16, 3, P, True)
    mean, var = _handle(hp, ym, ys, xlb, xrng, True, 3).predict(x, precision=_lib.GP_FP64)
    m_ref, v_ref = DG.predict(x, xlb, xrng, hp, ym, ys)
    _assert_bars(hp, ys, mean, var, m_ref, v_ref, 1e-9)


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
def test_bit_identical_repeats_mean_only_and_device_buffers(quadrature):
    torch = pytest.importorskip("torch")
    from dmosopt_b200 import _lib

    hp, ym, ys, xlb, xrng, x = _case(40, 6, 3, 2, 200, 140, 5, 700, quadrature)  # Z2 140: two operator row blocks
    g = _handle(hp, ym, ys, xlb, xrng, quadrature, 5)
    m1, v1, e1 = g.predict(x, seed=77, stream_id=3, return_eps=True)
    m2, v2, e2 = g.predict(x, seed=77, stream_id=3, return_eps=True)
    np.testing.assert_array_equal(m1, m2)
    np.testing.assert_array_equal(v1, v2)
    np.testing.assert_array_equal(e1, e2)
    m3, v3 = g.predict(x, seed=77, stream_id=3, return_var=False)
    assert v3 is None
    np.testing.assert_array_equal(m1, m3)
    xd = torch.tensor(x, device="cuda")
    md = torch.empty((x.shape[0], 2), dtype=torch.float64, device="cuda")
    vd = torch.empty_like(md)
    ed = torch.empty((5, x.shape[0], 3), dtype=torch.float64, device="cuda")
    _lib._check(_lib.load_library().dmo_dgp_predict(_lib.context(), g._h, _lib._ptr(xd), x.shape[0], 77, 3, _lib._ptr(ed), _lib._ptr(md),
                                                    _lib._ptr(vd), _lib.GP_FP64), "dmo_dgp_predict")
    torch.cuda.synchronize()
    np.testing.assert_array_equal(md.cpu().numpy(), m1)
    np.testing.assert_array_equal(vd.cpu().numpy(), v1)
    np.testing.assert_array_equal(ed.cpu().numpy(), e1)
    m_ref, v_ref = DG.predict(x, xlb, xrng, hp, ym, ys, eps=None if quadrature else e1)
    _assert_bars(hp, ys, m1, v1, m_ref, v_ref, 1e-9)
    if not quadrature:
        m4, _, e4 = g.predict(x, seed=77, stream_id=4, return_eps=True)
        assert np.mean(e4 == e1) < 1e-3 and np.any(m4 != m1)
        _, _, e5 = g.predict(x, seed=78, stream_id=3, return_eps=True)
        assert np.mean(e5 == e1) < 1e-3


def test_draws_are_standard_normal():
    from scipy import stats

    hp, ym, ys, xlb, xrng, x = _case(50, 2, 1, 1, 8, 8, 64, 16384, False)
    _, _, eps = _handle(hp, ym, ys, xlb, xrng, False, 64).predict(x, seed=2024, stream_id=1, return_var=False, return_eps=True)
    e = eps.ravel()
    n = e.size
    assert n >= 10**6
    assert abs(e.mean()) < 5.0 / np.sqrt(n)
    assert abs(e.var() - 1.0) < 5.0 * np.sqrt(2.0 / n)
    assert stats.kstest(e, "norm").pvalue > 1e-3


def test_monte_carlo_mean_converges_to_the_gauss_hermite_expectation():
    hp, ym, ys, xlb, xrng, x = _case(60, 3, 1, 1, 30, 20, 64, 4096, False)
    mean, _, eps = _handle(hp, ym, ys, xlb, xrng, False, 64).predict(x, seed=5, stream_id=0, return_eps=True)
    nodes, weights = np.polynomial.hermite.hermgauss(20)
    expect = np.zeros_like(mean)
    for z, w in zip(nodes, weights):
        e = np.full((1, x.shape[0], 1), np.sqrt(2.0) * z)
        expect += w / np.sqrt(np.pi) * DG.predict(x, xlb, xrng, hp, ym, ys, eps=e)[0]
    per_site = np.stack([DG.predict(x, xlb, xrng, hp, ym, ys, eps=eps[j : j + 1])[0] for j in range(64)])
    se = per_site.std(axis=0, ddof=1) / np.sqrt(64)
    within = np.abs(mean - expect) <= 6.0 * se + 1e-12 * np.abs(expect)
    assert np.mean(within) >= 0.999, np.mean(within)


def test_argument_errors():
    from dmosopt_b200 import _lib

    hp, ym, ys, xlb, xrng, x = _case(70, 3, 2, 2, 10, 8, 3, 10, True)

    def create(h=hp, **kw):
        args = dict(hp=h, ym=ym, ys=ys, xlb=xlb, xrng=xrng)
        args.update(kw)
        return _handle(args["hp"], args["ym"], args["ys"], args["xlb"], args["xrng"], True, 3)

    def mk(name, fn):
        h = {k: np.array(v, copy=True) for k, v in hp.items()}
        fn(h)
        return h

    from dmosopt_b200._lib import DGPHandle

    with pytest.raises(_lib.DmoError, match="hidden layer.*q_sqrt\\[1\\] is not lower triangular"):
        h = {k: np.array(v, copy=True) for k, v in hp.items()}
        qs = np.tril(h["hidden_chol_variational_covar"])
        qs[1, 0, 3] = 0.5
        DGPHandle(h["hidden_inducing_points"], h["hidden_outputscale"], h["hidden_lengthscale"], h["hidden_variational_mean"], qs,
                  h["mean_weights"], h["mean_bias"], h["last_inducing_points"], h["last_outputscale"], h["last_lengthscale"],
                  h["last_variational_mean"], np.tril(h["last_chol_variational_covar"]), h["mean_constant"], h["task_noises"] + h["noise"],
                  ym, ys, xlb, xrng, quad_sites=h["quad_sites"])
    with pytest.raises(_lib.DmoError, match="xrng\\[1\\] must be > 0"):
        create(xrng=np.where(np.arange(3) == 1, 0.0, xrng))
    with pytest.raises(_lib.DmoError, match="last layer.*variance\\[1\\] must be finite and > 0"):
        create(h=mk("s2", lambda h: h["last_outputscale"].__setitem__(1, -1.0)))
    with pytest.raises(_lib.DmoError, match="hidden layer.*length_scale\\[0\\]\\[2\\] must be > 0"):
        create(h=mk("ls1", lambda h: h["hidden_lengthscale"].__setitem__((0, 2), np.nan)))
    with pytest.raises(_lib.DmoError, match="noise\\[0\\] must be finite and > 0"):
        create(h=mk("noise", lambda h: (h["task_noises"].__setitem__(0, -1.0), h.__setitem__("noise", 0.0))))
    with pytest.raises(_lib.DmoError, match="last layer.*latent 1 is not positive definite"):
        def dup(h):  # K(Z, Z) of task 1 is exactly the all-ones matrix: its second pivot is exactly 0
            h["last_inducing_points"][1] = h["last_inducing_points"][1, 0]
            h["last_outputscale"][1] = 1.0
        _handle(mk("Z2", dup), ym, ys, xlb, xrng, True, 3, jitter=0.0)
    with pytest.raises(_lib.DmoError, match="n_sites"):
        _handle(hp, ym, ys, xlb, xrng, False, 65)
    g = create()
    with pytest.raises(_lib.DmoError, match="precision"):
        g.predict(x, precision=_lib.GP_AUTO)


@pytest.mark.parametrize("cls", ["MDSPP_Matern", "MDGP_Matern"])
def test_plugin_classes_through_hyperparameters(cls):
    from dmosopt_b200 import model_gpytorch as mg

    quadrature = cls == "MDSPP_Matern"
    rng = np.random.default_rng(80)
    d, T = 6, 2
    hp, *_ = problem(rng, d, 3, T, 50, 40, J=3, quadrature=quadrature)
    xin = rng.random((60, d))
    yin = rng.standard_normal((60, T)) * [1.0, 5.0] + [0.0, 3.0]
    xlb, xub = np.zeros(d), np.ones(d)
    model = getattr(mg, cls)(xin, yin, d, T, xlb, xub, hyperparameters=hp, return_mean_variance=True)
    ym, ys = yin.mean(axis=0), yin.std(axis=0)
    np.testing.assert_array_equal(model.y_train_mean, ym)
    x = rng.random((300, d))
    mean, var = model.evaluate(x)
    assert mean.dtype == np.float64 and var.dtype == np.float64
    if quadrature:
        m_ref, v_ref = DG.predict(x, xlb, np.ones(d), hp, ym, ys)
        np.testing.assert_array_equal(model.predict(x)[0], mean)
    else:
        # call 0 drew with (seed, stream 0); replay it, and a second call draws afresh
        _, _, eps = model._gp.predict(x, seed=mg.MDGP_DEFAULT_SEED, stream_id=0, return_eps=True)
        m_ref, v_ref = DG.predict(x, xlb, np.ones(d), hp, ym, ys, eps=eps)
        assert model.num_samples == 10 and eps.shape[0] == 10
        assert np.any(model.predict(x)[0] != mean)
    _assert_bars(hp, ys, mean, var, m_ref, v_ref, 1e-9)
