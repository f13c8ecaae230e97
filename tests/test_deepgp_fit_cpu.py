"""Deep GP training without a GPU: the autograd oracle (oracle/deepgp_train.py) against central finite differences, the
ReduceLROnPlateau restatement against torch's scheduler, the initial raw parameters, the stopping rules, raw <->
``hyperparameters=`` conversion and the fit="gpu-seeded" refusals."""

import logging

import numpy as np
import pytest

from oracle import deepgp_train as ot

torch = pytest.importorskip("torch")


def _problem(rng, N=30, d=2, T=2, H=2, Z=5, quadrature=True):
    from dmosopt_b200 import model_gpytorch as mg

    X = rng.random((N, d))
    Y = rng.standard_normal((N, T))
    raw = mg.deepgp_initial_raw(X, T, quadrature=quadrature, num_hidden_dims=H, num_inducing_points=Z, rng=rng)
    raw["hidden_variational_mean"] = 0.5 * rng.standard_normal(raw["hidden_variational_mean"].shape)
    raw["last_variational_mean"] = 0.5 * rng.standard_normal(raw["last_variational_mean"].shape)
    for k in ("hidden_chol_variational_covar", "last_chol_variational_covar"):
        raw[k] = raw[k] * 0.8 + 0.1 * rng.standard_normal(raw[k].shape)
    for k in ("hidden_raw_lengthscale", "hidden_raw_outputscale", "last_raw_lengthscale", "last_raw_outputscale", "raw_task_noises"):
        raw[k] = 0.3 * rng.standard_normal(raw[k].shape)
    if not quadrature:
        raw.pop("quad_sites", None)
    return X, Y, raw


def _fd_check(raw, X, Y, N, eps=None, bounds=None, jitter=ot.JITTER, entries=4, rng=None):
    _, g = ot.loss_grad(raw, X, Y, N, eps=eps, lengthscale_bounds=bounds, jitter=jitter)
    h = 1e-6
    for k, v in raw.items():
        flat = np.asarray(v, dtype=np.float64).reshape(-1)
        for idx in rng.choice(flat.size, min(entries, flat.size), replace=False):
            rp = {kk: np.array(vv, dtype=np.float64) for kk, vv in raw.items()}
            rm = {kk: np.array(vv, dtype=np.float64) for kk, vv in raw.items()}
            rp[k].reshape(-1)[idx] += h
            rm[k].reshape(-1)[idx] -= h
            lp = float(ot.loss(_torch(rp), X, Y, N, eps, bounds, jitter))
            lm = float(ot.loss(_torch(rm), X, Y, N, eps, bounds, jitter))
            fd = (lp - lm) / (2 * h)
            an = g[k].reshape(-1)[idx]
            assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (k, idx, fd, an)


def _torch(raw):
    return {k: torch.as_tensor(np.asarray(v, dtype=np.float64)) for k, v in raw.items()}


@pytest.mark.parametrize("quadrature", [True, False])
def test_oracle_gradient_matches_finite_differences(quadrature):
    rng = np.random.default_rng(1)
    X, Y, raw = _problem(rng, quadrature=quadrature)
    B = 7  # N = 30: a partial-batch size
    eps = None if quadrature else rng.standard_normal((B, B, 2))
    _fd_check(raw, X[:B], Y[:B], 30, eps=eps, rng=rng)
    _fd_check(raw, X[:B], Y[:B], 30, eps=eps, bounds=(0.1, 3.0), rng=rng)


def test_oracle_gradient_with_a_clamped_variance():
    """jitter 0 and the batch rows on the hidden inducing points: the hidden variance sits below min_variance, its
    gradient is blocked, and the finite differences agree."""
    rng = np.random.default_rng(2)
    X, Y, raw = _problem(rng, Z=5)
    raw["hidden_inducing_points"] = X[:5].copy()
    raw["hidden_chol_variational_covar"] = np.tile(1e-2 * np.eye(5), (2, 1, 1))
    raw["hidden_raw_outputscale"] = np.full(2, -6.0)
    xr = {k: torch.as_tensor(np.asarray(v)) for k, v in raw.items()}
    pm = None  # the hidden variance of the batch rows, recomputed as the oracle does
    with torch.no_grad():
        s = torch.nn.functional.softplus(xr["hidden_raw_outputscale"][0])
        ls = torch.nn.functional.softplus(xr["hidden_raw_lengthscale"][0])
        _, v, _ = ot._unit(torch.as_tensor(X[:5]), xr["hidden_inducing_points"], s, ls, xr["hidden_variational_mean"][0],
                           xr["hidden_chol_variational_covar"][0], 1e-12)
        pm = v.numpy()
    assert np.all(pm < ot.MIN_VARIANCE)
    _fd_check(raw, X[:5], Y[:5], 30, jitter=1e-12, rng=rng)


def _torch_lrs(losses, lr=0.1):
    p = torch.zeros(1, requires_grad=True)
    opt = torch.optim.Adam([p], lr=lr)
    sch = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, mode="min", patience=3, threshold=0.01)
    out = []
    for v in losses:
        sch.step(v)
        out.append(opt.param_groups[0]["lr"])
    return out


@pytest.mark.parametrize("losses", [
    [1.0] * 20,  # a plateau: repeated reductions
    [1.0, 0.99, 0.9801, 0.9703, 0.9606, 0.951, 0.9415],  # exactly at and around the rel threshold edge
    [1.0, 0.98, 0.97, 0.9702, 0.969, 0.968, 0.96, 0.95, 0.94, 0.94, 0.94, 0.94, 0.94, 0.5, 0.5, 0.5, 0.5, 0.5],
    list(np.linspace(1.0, 0.0, 30)) + [0.0] * 60,  # down to lr 1e-9 and past eps
    [-1.0, -1.005, -1.02, -1.02, -1.02, -1.02, -1.02, -2.0],  # negative losses
])
def test_reduce_lr_on_plateau_follows_torch(losses):
    from dmosopt_b200 import model_gpytorch as mg

    s = mg.ReduceLROnPlateau(0.1)
    assert [s.step(v) for v in losses] == _torch_lrs(losses)


def test_initial_raw_shapes_clipping_and_draw_order():
    from scipy.cluster.vq import kmeans2

    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(3)
    X = rng.random((90, 4))
    raw = mg.deepgp_initial_raw(X, 2, quadrature=True, num_hidden_dims=3, num_inducing_points=128, rng=np.random.default_rng(5))
    shapes = mg.deepgp_raw_shapes(4, 2, 3, 90, 90, True)  # Z clipped at N = 90 in both layers
    assert {k: v.shape for k, v in raw.items()} == shapes
    assert list(raw) == [k for k in mg.DEEPGP_RAW_KEYS if k in raw]
    g = np.random.default_rng(5)
    perm = g.permutation(90)
    assert np.array_equal(raw["hidden_inducing_points"], kmeans2(X, X[perm[:90]].copy(), minit="matrix")[0])
    assert np.array_equal(raw["mean_weights"], g.standard_normal(4)) and np.array_equal(raw["mean_bias"], g.standard_normal(1))
    assert np.array_equal(raw["hidden_variational_mean"], 1e-3 * g.standard_normal((3, 90)))
    assert np.array_equal(raw["last_variational_mean"], 1e-3 * g.standard_normal((2, 90)))
    assert np.array_equal(raw["last_inducing_points"], g.standard_normal((2, 90, 3)))
    assert np.array_equal(raw["quad_sites"], g.standard_normal((3, 3)))
    assert np.array_equal(raw["hidden_chol_variational_covar"], np.tile(np.eye(90), (3, 1, 1)))
    for k in ("hidden_raw_lengthscale", "hidden_raw_outputscale", "last_raw_lengthscale", "last_raw_outputscale", "raw_task_noises",
              "raw_noise", "mean_constant"):
        assert not np.any(raw[k]), k
    small = mg.deepgp_initial_raw(X, 2, quadrature=False, num_hidden_dims=3, num_inducing_points=16, rng=np.random.default_rng(5))
    assert small["hidden_inducing_points"].shape == (16, 4) and "quad_sites" not in small


def test_raw_hyperparameters_conversion():
    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(4)
    X, Y, raw = _problem(rng, N=30, d=3, T=2, H=2, Z=6)
    flat = mg.deepgp_flatten(raw)
    back = mg.deepgp_unflatten(flat, mg.deepgp_raw_shapes(3, 2, 2, 6, 6, True))
    assert all(np.array_equal(back[k], raw[k]) for k in raw)
    for bounds in (None, (0.2, 4.0)):
        hp = mg.deepgp_natural(raw, bounds)
        mg.deepgp_check_hyperparameters(hp, 3, 2, True, "test")
        assert hp["hidden_inducing_points"].shape == (2, 6, 3) and np.array_equal(hp["hidden_inducing_points"][1], raw["hidden_inducing_points"])
        ls = hp["hidden_lengthscale"]
        assert ls.shape == (2, 3) and np.all(ls == ls[:, :1])
        assert np.allclose(hp["hidden_outputscale"], np.log1p(np.exp(raw["hidden_raw_outputscale"])), rtol=1e-15)
        assert np.array_equal(hp["last_chol_variational_covar"], np.tril(raw["last_chol_variational_covar"]))
        assert np.allclose(hp["task_noises"], 1e-4 + np.log1p(np.exp(raw["raw_task_noises"])))
        assert hp["noise"] == 1e-4 + np.log(2.0)
        if bounds is not None:
            assert np.allclose(ls[:, 0], 0.2 + 3.8 / (1 + np.exp(-raw["hidden_raw_lengthscale"])))


class _Log(logging.Handler):
    def __init__(self):
        super().__init__()
        self.msgs = []

    def emit(self, record):
        self.msgs.append(record.getMessage())


def test_stopping_configurations_and_the_logger_only_break(monkeypatch):
    """DEEP_STOCHASTIC (MDSPP) from epoch 2000 and DEEP_GP (MDGP) from 1500, window 500, patience 3, warmup 200; a flat
    loss history stops the loop only when a logger is given, with the reference's log lines."""
    from dmosopt_b200 import model_gpytorch as mg

    for quadrature, first in ((True, 2000), (False, 1500)):
        st = mg.deepgp_stopper(quadrature, 1.0)
        assert (st.min_iterations, st.window, st.patience, st.warmup_iterations, st.threshold_pct) == (first, 500, 3, 200, 1.0)
        h = np.full(first + 10, 2.0)
        hits = [it for it in range(200, first + 10) if st.should_stop(it, h[: it + 1])[0]]
        assert hits[0] == first + 2  # the third successive call with two tests holding

    class FakeState:
        def __init__(self, X, Y, H, Z1, Z2, J, quadrature, B, **kw):
            self.n = len(mg.deepgp_flatten(mg.deepgp_initial_raw(X, Y.shape[1], quadrature=quadrature, num_hidden_dims=H,
                                                                  num_inducing_points=Z1, rng=np.random.default_rng(0))))

        def set_params(self, p):
            self.p = np.array(p)

        def get_params(self):
            return self.p

        def epoch(self, perm, B, lr, seed=0, step0=0):
            return np.full(-(-len(perm) // B), 1.5)

        def close(self):
            pass

    monkeypatch.setattr(mg._lib, "DGPFitState", FakeState)
    rng = np.random.default_rng(9)
    X, Y = rng.random((20, 2)), rng.standard_normal((20, 2))
    kw = dict(num_hidden_dims=2, num_inducing_points=4, n_iter=2100, batch_size=5)
    _, info = mg.deepgp_fit(X, Y, quadrature=False, **kw)
    assert info["iterations"] == 2100 and info["stop_reason"] == "n_iter"
    log = logging.getLogger("deepgp_fit_test")
    log.setLevel(logging.INFO)
    hd = _Log()
    log.addHandler(hd)
    _, info = mg.deepgp_fit(X, Y, quadrature=False, logger=log, **kw)
    assert info["iterations"] == 1503 and "Max absolute change" in info["stop_reason"]
    assert hd.msgs[0] == f"MDGP_Matern: iter 0/2100 - Loss: 1.500  noise:  {1e-4 + np.log(2.0):.3f}"
    assert hd.msgs[-1].startswith("MDGP_Matern: early stop at iteration 1503: ")
    hd.msgs.clear()
    _, info = mg.deepgp_fit(X, Y, quadrature=True, logger=log, **kw)
    assert info["iterations"] == 2003 and hd.msgs[0] == f"MDSPP_Matern: iter 0/2100 - Loss: 1.500  {1e-4 + np.log(2.0):.3f}"
    assert info["lr"][0] == 0.1 and info["lr"][5] == pytest.approx(0.01) and info["lr"][-1] <= 1.01e-8


@pytest.mark.parametrize("cls", ["MDSPP_Matern", "MDGP_Matern"])
def test_gpu_seeded_refusals(cls):
    from dmosopt_b200 import model_gpytorch as mg

    C = getattr(mg, cls)
    rng = np.random.default_rng(6)
    x, y = rng.random((200, 3)), rng.standard_normal((200, 2))
    lb, ub = np.zeros(3), np.ones(3)
    for kw, what in ((dict(gp_likelihood_sigma=0.1), "noise prior"), (dict(num_inducing_points=129), "inducing points"),
                     (dict(num_hidden_dims=9), "hidden units"), (dict(num_hidden_dims=0), "hidden units")):
        with pytest.raises(ValueError, match=f"{what}.*fit='reference'"):
            C(x, y, 3, 2, lb, ub, fit="gpu-seeded", **kw)
    with pytest.raises(ValueError, match="objectives.*fit='reference'"):
        C(x, rng.standard_normal((200, 9)), 3, 9, lb, ub, fit="gpu-seeded")
    xd = rng.random((200, 91))
    with pytest.raises(ValueError, match="input dimensions.*fit='reference'"):
        C(xd, y, 91, 2, np.zeros(91), np.ones(91), fit="gpu-seeded")
    with pytest.raises(ValueError, match="fit='gpu-seeded'"):
        C(x, y, 3, 2, lb, ub, fit="gpu")
