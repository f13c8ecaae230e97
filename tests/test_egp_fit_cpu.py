"""Training of EGP_Matern without a GPU: the torch autograd oracle against scipy's Cholesky, finite differences and the
one-task multitask oracle, the host side of the GPU fit (chain rule to gpytorch's raw parameters, the initial draws)
against autograd, and the constructor's argument checks."""

import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky

from oracle import egp, egp_train, megp_train
from oracle.gp import MATERN52, kernel_matrix

torch = pytest.importorskip("torch")


def _problem(seed, N=40, d=3, M=3):
    rng = np.random.default_rng(seed)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, 0] + t) + 0.5 * X[:, (t + 1) % d] ** 2 for t in range(M)])
    yn, _, _ = egp.normalise_y(Y)
    hp = dict(length_scale=np.exp(rng.uniform(np.log(0.2), np.log(2.0), (M, d))), outputscale=0.5 + rng.random(M),
              noise=1e-2 * (1.0 + rng.random(M)), weight=0.3 * rng.standard_normal((M, d)), bias=0.1 * rng.standard_normal(M))
    return X, yn, hp


@pytest.mark.parametrize("M", [1, 2, 3])
def test_torch_oracle_lml_is_scipys_cholesky(M):
    X, yn, hp = _problem(20 + M, M=M)
    lml, _ = egp_train.lml_and_grad_torch(X, yn, *hp.values())
    N = X.shape[0]
    for m in range(M):
        K = hp["outputscale"][m] * kernel_matrix(X, X, hp["length_scale"][m], MATERN52)
        K[np.diag_indices_from(K)] += hp["noise"][m]
        L = cholesky(K, lower=True)
        r = yn[:, m] - (X @ hp["weight"][m] + hp["bias"][m])
        ref = -0.5 * r @ cho_solve((L, True), r) - np.log(np.diag(L)).sum() - 0.5 * N * np.log(2 * np.pi)
        assert abs(lml[m] - ref) <= 1e-12 * abs(ref), (m, lml[m], ref)


def test_torch_oracle_gradient_matches_finite_differences():
    X, yn, hp = _problem(3)
    _, g = egp_train.lml_and_grad_torch(X, yn, *hp.values())
    for k, v in hp.items():
        fd = np.zeros_like(v)
        for idx in np.ndindex(v.shape):
            h = 1e-6 * max(1.0, abs(v[idx]))
            up, dn = {kk: vv.copy() for kk, vv in hp.items()}, {kk: vv.copy() for kk, vv in hp.items()}
            up[k][idx] += h
            dn[k][idx] -= h
            m = idx[0]  # an objective's parameters only move its own lml
            fd[idx] = (egp_train.lml_and_grad_torch(X, yn, *up.values())[0][m] - egp_train.lml_and_grad_torch(X, yn, *dn.values())[0][m]) / (2 * h)
        assert np.abs(fd - g[k]).max() <= 1e-6 * np.abs(g[k]).max(), k


def test_torch_oracle_is_the_one_task_multitask_oracle():
    """One objective is an MEGP with one task: B = [[s]], D = [noise]."""
    X, yn, hp = _problem(5, M=2)
    lml, g = egp_train.lml_and_grad_torch(X, yn, *hp.values())
    for m in range(2):
        ref, rg = megp_train.lml_and_grad_torch(X, yn[:, m : m + 1], hp["length_scale"][m], np.array([[hp["outputscale"][m]]]),
                                                np.array([hp["noise"][m]]), hp["weight"][m : m + 1], hp["bias"][m : m + 1])
        assert abs(lml[m] - ref) <= 1e-12 * abs(ref)
        for k, rk in (("length_scale", "length_scale"), ("weight", "weight"), ("bias", "bias")):
            assert np.abs(g[k][m] - np.ravel(rg[rk])).max() <= 1e-11 * np.abs(rg[rk]).max(), k
        assert abs(g["outputscale"][m] - rg["B"][0, 0]) <= 1e-11 * abs(rg["B"][0, 0])
        assert abs(g["noise"][m] - rg["D"][0]) <= 1e-11 * abs(rg["D"][0])


@pytest.mark.parametrize("bounds", [None, (0.05, 5.0)])
def test_host_chain_rule_matches_autograd(bounds):
    from dmosopt_b200.model_gpytorch import egp_initial_raw, egp_natural, egp_raw_grad

    X, yn, _ = _problem(4, M=2)
    N, d = X.shape
    M = yn.shape[1]
    raw = egp_initial_raw(d, M, seed=7)
    rng = np.random.default_rng(8)
    raw["raw_lengthscale"] = rng.normal(0.0, 1.0, (M, d))
    raw["raw_outputscale"] = rng.normal(0.0, 1.0, M)
    raw["raw_noise"] = rng.normal(-4.0, 1.0, M)
    _, g = egp_train.lml_and_grad_torch(X, yn, *egp_natural(raw, bounds))
    got = egp_raw_grad(raw, g, bounds)
    for m in range(M):
        p = {k: torch.tensor(v[m : m + 1].copy(), requires_grad=True) for k, v in raw.items()}
        nat = egp_train.natural_torch(p, bounds)
        lml = egp_train._lml_torch(torch.tensor(X), torch.tensor(yn[:, m]), *nat)
        lml.backward()
        for k in raw:
            ref = p[k].grad.numpy()[0]
            assert np.abs(got[k][m] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300), (m, k)
        for u, v in zip(egp_natural({k: vv[m : m + 1] for k, vv in raw.items()}, bounds), nat):
            assert np.abs(np.ravel(u) - np.ravel(v.detach().numpy())).max() <= 1e-15 * np.abs(u).max()


def test_initial_draws_layout():
    from dmosopt_b200.model_gpytorch import egp_initial_raw, egp_natural

    d, M = 4, 3
    raw = egp_initial_raw(d, M, seed=11)
    rng = np.random.default_rng(11)
    for m in range(M):  # objective by objective: weights, then bias
        assert np.array_equal(raw["weights"][m], rng.standard_normal(d))
        assert raw["bias"][m] == rng.standard_normal()
    assert np.array_equal(raw["raw_lengthscale"], np.zeros((M, d)))
    assert np.array_equal(raw["raw_outputscale"], np.zeros(M)) and np.array_equal(raw["raw_noise"], np.zeros(M))
    assert np.array_equal(egp_initial_raw(d, M)["weights"], egp_initial_raw(d, M, seed=0)["weights"])
    ls, s, nz, _, _ = egp_natural(raw)
    assert np.allclose(ls, np.log(2.0)) and np.allclose(s, np.log(2.0)) and np.allclose(nz, 1e-4 + np.log(2.0))


def test_fit_argument_checks():
    from dmosopt_b200.model_gpytorch import EGP_Matern

    X, Y = np.random.default_rng(0).random((10, 2)), np.random.default_rng(1).random((10, 2))
    with pytest.raises(ValueError):
        EGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="bogus")
    with pytest.raises(ValueError, match="fit='reference'"):
        EGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="gpu", gp_likelihood_sigma=0.1)
    with pytest.raises(ValueError, match="batch_size"):
        EGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="gpu", batch_size=4)
