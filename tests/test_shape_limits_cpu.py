"""Shape limits without a GPU.

  * The closed-form gradient reference (oracle/fit_grad_dense.py) against the torch autograd oracles.
    tests/test_gpu_shape_limits.py checks dmo_gp_lml_grad and dmo_mtgp_lml_grad at N 2048 against the closed form,
    where the autograd oracles' N x N x d graphs do not fit; here the closed form itself is checked against them at
    N 150, d 12, for one and three objectives (tasks), within 1e-10: the log marginal likelihood relative to itself,
    each gradient relative to max |ref| of its key.
  * The surrogate classes refuse a shape their GPU predict cannot take before any training starts: EGP_Matern and
    GPR_Matern / GPR_RBF past d 64 or M 16 (dmo_gp_create), MEGP_Matern and the variational classes with
    precision="tensor" past d 64 (the tensor-core predicts).  The trainers are replaced by a function that fails, so a
    refusal that came only after training would show as that failure.
"""

import numpy as np
import pytest

from oracle import egp, fit_grad_dense, megp

torch = pytest.importorskip("torch")


def refuse_training(monkeypatch):
    from dmosopt_b200 import model, model_gpflow, model_gpytorch

    def trained(*args, **kwargs):
        raise AssertionError("training started before the shape was refused")

    monkeypatch.setattr(model_gpytorch, "egp_fit", trained)
    monkeypatch.setattr(model_gpytorch, "megp_fit", trained)
    monkeypatch.setattr(model_gpflow, "svgp_fit", trained)
    monkeypatch.setattr(model._GPRBase, "_fit_on_gpu", trained)


def _make(module, cls, d, M, **kw):
    def make():
        import importlib

        rng = np.random.default_rng(d + M)
        X, Y = rng.random((40, d)), rng.standard_normal((40, M))
        return getattr(importlib.import_module(f"dmosopt_b200.{module}"), cls)(X, Y, d, M, np.zeros(d), np.ones(d), **kw)

    return make


_EXACT_D = r"the GPU predict takes at most 64 input dimensions \(got nInput=65\)"
_EXACT_M = r"the GPU predict takes at most 16 objectives \(got nOutput=17\)"
_TENSOR_D = r"the tensor-core predict takes at most 64 input dimensions \(got nInput=65\); use precision='fp64'"
REFUSALS = [
    (_make("model_gpytorch", "EGP_Matern", 65, 2, fit="gpu"), "EGP_Matern: " + _EXACT_D),
    (_make("model_gpytorch", "EGP_Matern", 4, 17, fit="gpu"), "EGP_Matern: " + _EXACT_M),
    (_make("model", "GPR_Matern", 65, 2), "GPR_Matern: " + _EXACT_D),
    (_make("model", "GPR_Matern", 4, 17, precision="fp64"), "GPR_Matern: " + _EXACT_M),
    (_make("model", "GPR_RBF", 65, 1, precision="tensor"), "GPR_RBF: " + _EXACT_D),
    (_make("model_gpytorch", "MEGP_Matern", 65, 2, fit="gpu", precision="tensor"), "MEGP_Matern: " + _TENSOR_D),
] + [(_make("model_gpflow", cls, 65, 2, fit="gpu", precision="tensor"), f"{cls}: " + _TENSOR_D)
     for cls in ("SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern", "CRV_Matern")]


@pytest.mark.parametrize("i", range(len(REFUSALS)))
def test_surrogate_classes_refuse_before_training(monkeypatch, i):
    refuse_training(monkeypatch)
    make, match = REFUSALS[i]
    with pytest.raises(ValueError, match=match):
        make()


def _data(rng, N, d, M):
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, (t + 2) % d] + 0.2 * t * X[:, -1] ** 2 for t in range(M)])
    yn, _, _ = egp.normalise_y(Y)
    return X, yn


def _close(g, rg, rel):
    assert set(g) == set(rg)
    for k in rg:
        assert np.shape(g[k]) == np.shape(rg[k]), k
        err, scale = np.abs(g[k] - rg[k]).max(), np.abs(rg[k]).max()
        assert err <= rel * scale, (k, err, scale)


@pytest.mark.parametrize("M", [1, 3])
def test_egp_closed_form_gradient_is_the_autograd_gradient(M):
    from oracle import egp_train

    rng = np.random.default_rng(150 + M)
    N, d = 150, 12
    X, yn = _data(rng, N, d, M)
    hp = (np.exp(rng.uniform(np.log(0.1), np.log(3.0), (M, d))), 0.3 + 1.2 * rng.random(M), np.geomspace(2e-3, 2e-2, M),
          0.3 * rng.standard_normal((M, d)), 0.2 * rng.standard_normal(M))
    lml, g = fit_grad_dense.egp_lml_and_grad(X, yn, *hp)
    ref, rg = egp_train.lml_and_grad_torch(X, yn, *hp)
    assert np.all(np.abs(lml - ref) <= 1e-10 * np.abs(ref)), (lml, ref)
    _close(g, rg, 1e-10)


@pytest.mark.parametrize("M", [1, 3])
def test_megp_closed_form_gradient_is_the_autograd_gradient(M):
    from oracle import megp_train

    rng = np.random.default_rng(1500 + M)
    N, d = 150, 12
    X, yn = _data(rng, N, d, M)
    ls = np.exp(rng.uniform(np.log(0.3), np.log(3.0), d))
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + 0.5 * rng.random(M))
    D = np.geomspace(5e-3, 2e-2, M)
    w, b = 0.2 * rng.standard_normal((M, d)), 0.1 * rng.standard_normal(M)
    lml, g = fit_grad_dense.megp_lml_and_grad(X, yn, ls, B, D, w, b)
    ref, rg = megp_train.lml_and_grad_torch(X, yn, ls, B, D, w, b)
    assert abs(lml - ref) <= 1e-10 * abs(ref), (lml, ref)
    _close(g, rg, 1e-10)
