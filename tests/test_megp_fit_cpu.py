"""Training of MEGP_Matern without a GPU: the torch autograd oracle against the dense oracle and finite differences, the
host side of the GPU fit (chain rule to gpytorch's raw parameters, Adam, early stopping) against torch and the
reference's own early-stopping rule, and the constructor's argument checks."""

import os

import numpy as np
import pytest

from oracle import megp, megp_train

torch = pytest.importorskip("torch")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "early_stopping.npz")


def _problem(seed, N=40, d=3, M=3):
    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, 0] + t) + 0.5 * X[:, (t + 1) % d] ** 2 for t in range(M)])
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + rng.random(M))
    D = 1e-2 * (1.0 + rng.random(M))
    hp = dict(lengthscale=np.exp(rng.uniform(np.log(0.2), np.log(2.0), d)), B=B, D=D, weight=0.3 * rng.standard_normal((M, d)),
              bias=0.1 * rng.standard_normal(M))
    return X, Y, xlb, xub, hp


@pytest.mark.parametrize("M", [1, 2, 3])
def test_torch_oracle_lml_is_the_dense_oracle(M):
    X, Y, xlb, xub, hp = _problem(10 + M, M=M)
    st = megp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["B"], hp["D"], hp["weight"], hp["bias"])
    yn, _, _ = megp.normalise_y(Y)
    lml, _ = megp_train.lml_and_grad_torch(st.X_train, yn, hp["lengthscale"], hp["B"], hp["D"], hp["weight"], hp["bias"])
    assert abs(lml - st.lml) <= 1e-12 * abs(st.lml)


def test_torch_oracle_gradient_matches_finite_differences():
    X, Y, xlb, xub, hp = _problem(3)
    yn, _, _ = megp.normalise_y(Y)
    args = dict(length_scale=hp["lengthscale"], B=hp["B"], D=hp["D"], weight=hp["weight"], bias=hp["bias"])

    def f(a):
        return megp_train.lml_and_grad_torch(X, yn, a["length_scale"], a["B"], a["D"], a["weight"], a["bias"])[0]

    _, g = megp_train.lml_and_grad_torch(X, yn, *args.values())
    for k, v in args.items():
        fd, want = np.zeros_like(v), g[k].copy()
        for idx in np.ndindex(v.shape):
            h = 1e-6 * max(1.0, abs(v[idx]))
            up, dn = {kk: vv.copy() for kk, vv in args.items()}, {kk: vv.copy() for kk, vv in args.items()}
            up[k][idx] += h
            dn[k][idx] -= h
            if k == "B" and idx[0] != idx[1]:  # B stays symmetric: B_st and B_ts move together, d lml = g_st + g_ts
                up[k][idx[::-1]] += h
                dn[k][idx[::-1]] -= h
                want[idx] = g[k][idx] + g[k][idx[::-1]]
            fd[idx] = (f(up) - f(dn)) / (2 * h)
        assert np.abs(fd - want).max() <= 1e-6 * np.abs(want).max(), k
    assert np.abs(g["B"] - g["B"].T).max() <= 1e-12 * np.abs(g["B"]).max()  # the symmetric gradient


@pytest.mark.parametrize("bounds", [None, (0.05, 5.0)])
def test_host_chain_rule_matches_autograd(bounds):
    from dmosopt_b200.model_gpytorch import megp_initial_raw, megp_natural, megp_raw_grad

    X, Y, *_ = _problem(4)
    yn, _, _ = megp.normalise_y(Y)
    N, d = X.shape
    M = yn.shape[1]
    raw = megp_initial_raw(d, M, seed=7)
    rng = np.random.default_rng(8)
    raw["raw_lengthscale"] = rng.normal(0.0, 1.0, d)
    raw["raw_task_noises"] = rng.normal(-3.0, 1.0, M)
    raw["raw_noise"] = np.array([-4.0])
    raw["weights"] = raw["weights"] + 0.1 * rng.standard_normal((M, d))
    ls, B, D, w, b = megp_natural(raw, bounds)
    _, g = megp_train.lml_and_grad_torch(X, yn, ls, B, D, w, b)
    got = megp_raw_grad(raw, g, bounds)
    p = {k: torch.tensor(v, requires_grad=True) for k, v in raw.items()}
    lml = megp_train._lml_torch(torch.tensor(X), torch.tensor(yn), *megp_train.natural_torch(p, bounds))
    lml.backward()
    for k in raw:
        ref = p[k].grad.numpy()
        assert got[k].shape == ref.shape, k
        assert np.abs(got[k] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300), k
    for u, v in zip(megp_natural(raw, bounds), megp_train.natural_torch(p, bounds)):
        assert np.abs(u - v.detach().numpy()).max() <= 1e-15 * np.abs(u).max()


def test_numpy_adam_is_torch_adam():
    from dmosopt_b200.model_gpytorch import Adam

    rng = np.random.default_rng(9)
    shapes = {"a": (7,), "b": (3, 1), "c": (1,), "d": (3, 5)}
    p0 = {k: rng.standard_normal(s) for k, s in shapes.items()}
    grads = [{k: rng.standard_normal(s) * 10.0 ** rng.integers(-6, 3) for k, s in shapes.items()} for _ in range(500)]
    params = {k: v.copy() for k, v in p0.items()}
    opt = Adam(lr=0.01)
    tp = {k: torch.tensor(v.copy(), requires_grad=True) for k, v in p0.items()}
    topt = torch.optim.Adam(list(tp.values()), lr=0.01)
    for g in grads:
        opt.step(params, g)
        for k in tp:
            tp[k].grad = torch.tensor(g[k])
        topt.step()
    for k in shapes:
        ref = tp[k].detach().numpy()
        assert np.all(np.abs(params[k] - ref) <= 1e-15 * np.abs(ref)), (k, np.abs(params[k] - ref).max())


def test_early_stopping_restatement_reproduces_the_reference():
    from dmosopt_b200.model_gpytorch import EarlyStopping

    z = np.load(GOLDEN)
    for name, seq, at, why in zip(z["names"], z["losses"], z["stop_it"], z["reasons"]):
        es = EarlyStopping(threshold_pct=0.1)
        log, got, reason = [], -1, ""
        for it, v in enumerate(seq):
            log.append(float(v))
            if it >= es.warmup_iterations:
                stop, r = es.should_stop(it, np.array(log))
                if stop:
                    got, reason = it, r
                    break
        assert (got, reason) == (int(at), str(why)), name


def test_fit_argument_checks():
    from dmosopt_b200.model_gpytorch import MEGP_Matern

    X, Y = np.random.default_rng(0).random((10, 2)), np.random.default_rng(1).random((10, 2))
    with pytest.raises(ValueError):
        MEGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="bogus")
    with pytest.raises(ValueError, match="fit='reference'"):
        MEGP_Matern(X, Y, 2, 2, np.zeros(2), np.ones(2), fit="gpu", gp_likelihood_sigma=0.1)
