"""Training of the deep GPs on the GPU (dmo_dgp_fit_*): the minibatch loss and its full raw gradient against the dense
torch autograd oracle (oracle/deepgp_train.py) over a shape table, MDGP's draws, Adam against the host restatement,
epochs against their steps, deepgp_fit's loop against the oracle loop, fitted MDSPP_Matern / MDGP_Matern with
fit="gpu-seeded", the unmodified reference controller training them, and the argument errors."""

import numpy as np
import pytest

from oracle import deepgp_train as ot

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


def _data(rng, N, d, T):
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, : min(2, d)].sum(1) + t) + 0.4 * X[:, (t + 1) % d] for t in range(T)])
    return X, (Y - Y.mean(0)) / Y.std(0)


def _raw(rng, X, T, H, Z1, Z2, quadrature, bounds):
    """A non-trivial raw point: the seeded initial values, perturbed so that every block is away from its start."""
    from dmosopt_b200 import model_gpytorch as mg

    raw = mg.deepgp_initial_raw(X, T, quadrature=quadrature, num_hidden_dims=H, num_inducing_points=max(Z1, Z2), rng=rng)
    raw["hidden_inducing_points"] = raw["hidden_inducing_points"][:Z1] if len(raw["hidden_inducing_points"]) >= Z1 else rng.random((Z1, X.shape[1]))
    raw["hidden_variational_mean"] = 0.3 * rng.standard_normal((H, Z1))
    raw["last_variational_mean"] = 0.3 * rng.standard_normal((T, Z2))
    raw["last_inducing_points"] = rng.standard_normal((T, Z2, H))
    for k, Zn, U in (("hidden_chol_variational_covar", Z1, H), ("last_chol_variational_covar", Z2, T)):
        c = 0.1 * rng.standard_normal((U, Zn, Zn))  # junk above the diagonal is masked
        for u in range(U):
            c[u][np.diag_indices(Zn)] = 0.5 + 0.5 * rng.random(Zn)
        raw[k] = c
    for k in ("hidden_raw_lengthscale", "hidden_raw_outputscale", "last_raw_lengthscale", "last_raw_outputscale", "raw_task_noises"):
        raw[k] = 0.4 * rng.standard_normal(raw[k].shape) + (0.5 if "lengthscale" in k and bounds is None and "hidden" in k else 0.0)
    raw["raw_noise"] = np.array([-1.0])
    raw["mean_constant"] = np.array([0.2])
    return raw


def _state(L, X, Y, raw, quadrature, J, Bmax, bounds):
    from dmosopt_b200 import model_gpytorch as mg

    H = raw["hidden_raw_outputscale"].shape[0]
    st = L.DGPFitState(X, Y, H, raw["hidden_variational_mean"].shape[1], raw["last_variational_mean"].shape[1], J, quadrature, Bmax,
                       lengthscale_bounds=bounds)
    st.set_params(mg.deepgp_flatten(raw))
    return st


def _check_grad(gdev, graw, raw):
    from dmosopt_b200 import model_gpytorch as mg

    shapes = {k: np.shape(v) for k, v in raw.items()}
    gd = mg.deepgp_unflatten(gdev, shapes)
    for k in raw:
        ref = graw[k]
        scale = max(np.max(np.abs(ref)), 1e-300)
        err = np.max(np.abs(gd[k] - ref)) / scale
        assert err < 1e-8, (k, err, scale)


# quadrature, N, d, H, T, Z1, Z2, B, bounds
CASES = [(True, 40, 1, 1, 1, 1, 1, 1, None), (True, 120, 30, 3, 3, 37, 20, 10, None), (True, 200, 90, 8, 8, 128, 128, 50, (0.05, 5.0)),
         (True, 150, 30, 3, 1, 128, 37, 13, (0.1, 3.0)), (False, 60, 30, 3, 3, 37, 128, 10, None), (False, 80, 1, 8, 3, 20, 37, 1, None),
         (False, 130, 90, 1, 8, 128, 1, 50, (0.05, 5.0)), (False, 100, 8, 3, 2, 37, 37, 7, None)]


@pytest.mark.parametrize("quadrature,N,d,H,T,Z1,Z2,B,bounds", CASES)
def test_loss_grad_matches_the_autograd_oracle(L, quadrature, N, d, H, T, Z1, Z2, B, bounds):
    rng = np.random.default_rng(N + d + H + T + Z1 + Z2 + B)
    X, Y = _data(rng, N, d, T)
    raw = _raw(rng, X, T, H, Z1, Z2, quadrature, bounds)
    if not quadrature:
        raw.pop("quad_sites", None)
    J = 3 if quadrature else max(B, 2)
    st = _state(L, X, Y, raw, quadrature, J, max(B, 2), bounds)
    for b in (B, max(B - 3, 1)):  # a full and a partial batch
        batch = rng.choice(N, b, replace=False)
        loss, g, eps = st.loss_grad(batch, seed=5, step=3, return_eps=True)
        lo, go = ot.loss_grad(raw, X[batch], Y[batch], N, eps=None if quadrature else eps, lengthscale_bounds=bounds)
        assert abs(loss - lo) <= 1e-10 * abs(lo), (loss, lo)
        _check_grad(g, go, raw)


def test_clamped_variances_block_their_gradient(L):
    """With the jitter at 1e-9 the hidden variance at a batch row on an inducing point falls under min_variance (and so
    does the last layer's with a tiny output scale): device and oracle agree with the clamps active."""
    rng = np.random.default_rng(3)
    X, Y = _data(rng, 50, 2, 2)
    raw = _raw(rng, X, 2, 3, 12, 9, True, None)
    raw["hidden_inducing_points"] = X[:12].copy()
    raw["hidden_chol_variational_covar"] = np.tile(1e-3 * np.eye(12), (3, 1, 1))
    raw["hidden_raw_outputscale"] = np.full(3, -8.0)
    raw["last_raw_outputscale"] = np.array([-16.0, 0.3])
    raw["last_chol_variational_covar"] = np.tile(1e-3 * np.eye(9), (2, 1, 1))
    from dmosopt_b200 import model_gpytorch as mg

    st = L.DGPFitState(X, Y, 3, 12, 9, 3, True, 20, jitter=1e-9)
    st.set_params(mg.deepgp_flatten(raw))
    batch = np.arange(4, 24)
    loss, g = st.loss_grad(batch)
    lo, go = ot.loss_grad(raw, X[batch], Y[batch], 50, jitter=1e-9)
    assert abs(loss - lo) <= 1e-10 * abs(lo)
    _check_grad(g, go, raw)


def test_mdgp_draws_replay_and_statistics(L):
    rng = np.random.default_rng(4)
    X, Y = _data(rng, 300, 5, 2)
    raw = _raw(rng, X, 2, 3, 16, 16, False, None)
    raw.pop("quad_sites", None)
    st = _state(L, X, Y, raw, False, 50, 50, None)
    batch = rng.choice(300, 50, replace=False)
    l1, g1, e1 = st.loss_grad(batch, seed=9, step=4, return_eps=True)
    l2, g2, e2 = st.loss_grad(batch, seed=9, step=4, return_eps=True)
    assert l1 == l2 and np.array_equal(g1, g2) and np.array_equal(e1, e2)  # a fixed (seed, step) is bit-identical
    l3, _, e3 = st.loss_grad(batch, seed=9, step=5, return_eps=True)
    assert not np.array_equal(e1, e3)
    l4, g4 = st.loss_grad(batch, eps=e1)  # the draws replayed
    assert l4 == l1 and np.array_equal(g4, g1)
    lo, _ = ot.loss_grad(raw, X[batch], Y[batch], 300, eps=e1)
    assert abs(l1 - lo) <= 1e-10 * abs(lo)
    draws = np.concatenate([st.loss_grad(batch, seed=9, step=s, grad=False, return_eps=True)[2].ravel() for s in range(8)])
    n = draws.size  # 8 * 50 * 50 * 3 = 60 000
    assert abs(draws.mean()) < 5 / np.sqrt(n) and abs(draws.var() - 1.0) < 5 * np.sqrt(2.0 / n)
    assert abs(np.mean(draws**3)) < 5 * np.sqrt(15.0 / n) and abs(np.mean(draws**4) - 3.0) < 5 * np.sqrt(96.0 / n)


def test_adam_step_is_bit_equal_to_the_host_adam(L):
    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(5)
    X, Y = _data(rng, 60, 4, 2)
    raw = _raw(rng, X, 2, 2, 10, 8, True, None)
    st = _state(L, X, Y, raw, True, 3, 10, None)
    host = {"p": mg.deepgp_flatten(raw)}
    adam = mg.Adam(lr=0.1)
    for k, lr in enumerate((0.1, 0.1, 0.01, 0.01, 0.001)):
        adam.lr = lr
        _, g = st.loss_grad(rng.choice(60, 10, replace=False))
        st.adam_step(lr)
        adam.step(host, {"p": g})
        assert np.array_equal(st.get_params(), host["p"]), k


def test_epoch_equals_its_steps_and_fits_repeat(L):
    from dmosopt_b200 import model_gpytorch as mg

    for quadrature in (True, False):
        rng = np.random.default_rng(6)
        X, Y = _data(rng, 47, 3, 2)
        raw = _raw(rng, X, 2, 3, 12, 10, quadrature, None)
        if not quadrature:
            raw.pop("quad_sites", None)
        J, B = (3, 10) if quadrature else (10, 10)
        a = _state(L, X, Y, raw, quadrature, J, B, None)
        b = _state(L, X, Y, raw, quadrature, J, B, None)
        perm = rng.permutation(47)
        la = a.epoch(perm, B, 0.05, seed=2, step0=7)
        lb = []
        for k, b0 in enumerate(range(0, 47, B)):
            lb.append(b.loss_grad(perm[b0 : b0 + B], seed=2, step=7 + k, grad=False)[0])
            b.adam_step(0.05)
        assert la.shape == (5,) and np.array_equal(la, np.asarray(lb))
        assert np.array_equal(a.get_params(), b.get_params())
    rng = np.random.default_rng(7)
    X, Y = _data(rng, 64, 4, 2)
    kw = dict(num_hidden_dims=2, num_inducing_points=16, n_iter=6, batch_size=16, seed=3)
    for quadrature in (True, False):
        h1, i1 = mg.deepgp_fit(X, Y, quadrature=quadrature, **kw)
        h2, i2 = mg.deepgp_fit(X, Y, quadrature=quadrature, **kw)
        assert np.array_equal(i1["loss"], i2["loss"])
        assert all(np.array_equal(np.asarray(h1[k]), np.asarray(h2[k])) for k in h1)


def test_deepgp_fit_follows_the_oracle_loop(L):
    """20 epochs of MDSPP at N 60 on the same permutation stream and initial values: the epoch losses agree within 1e-6
    relative (float64 sums in a different order, compounded over 120 Adam steps, whose m / sqrt(v) amplifies rounding
    in the entries with near-zero gradients) and the lr history is identical."""
    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(8)
    X, Y = _data(rng, 60, 4, 2)
    n_iter, B, seed = 20, 10, 11
    hp, info = mg.deepgp_fit(X, Y, quadrature=True, num_hidden_dims=2, num_inducing_points=12, adam_lr=0.1, n_iter=n_iter, batch_size=B,
                             seed=seed)
    g = np.random.default_rng(seed)  # the same stream: initial draws first, then one permutation per epoch
    raw0 = mg.deepgp_initial_raw(X, 2, quadrature=True, num_hidden_dims=2, num_inducing_points=12, rng=g)
    perms = [g.permutation(60) for _ in range(n_iter)]
    losses, lrs, raw = ot.fit_loop(raw0, X, Y, perms, B, 0.1)
    assert np.max(np.abs(info["loss"] - losses) / np.abs(losses)) < 1e-6
    assert list(info["lr"]) == lrs


@pytest.mark.parametrize("cls", ["MDSPP_Matern", "MDGP_Matern"])
def test_gpu_seeded_surrogates_fit_zdt1(L, cls):
    from dmosopt_b200 import model_gpytorch as mg

    C = getattr(mg, cls)
    rng = np.random.default_rng(12)
    d = 30
    X = rng.random((640, d))
    Y = _zdt1(X)
    Xtr, Ytr, Xte, Yte = X[:512], Y[:512], X[512:], Y[512:]
    lb, ub = np.zeros(d), np.ones(d)
    kw = dict(n_iter=100, seed=1, num_inducing_points=64)
    m = C(Xtr, Ytr, d, 2, lb, ub, fit="gpu-seeded", **kw)
    assert m.fit_info["iterations"] == 100 and m.fit_info["loss"][-1] < m.fit_info["loss"][0]
    mean, var = m.predict(Xte)
    assert np.all(np.isfinite(mean)) and np.all(var > 0)
    mse = np.mean((mean - Yte) ** 2, axis=0)
    # held-out predictions beat the mean predictor over both objectives together.  Per objective MDSPP does not: its
    # hidden units have one isotropic length scale over the 30 inputs, and at this budget it leaves f1 = x0 at about
    # 1.6 times the variance of the held-out f1 while f2 falls to a fifth of its variance
    assert mse.sum() < np.var(Yte, axis=0).sum(), (mse, np.var(Yte, axis=0))
    # the fitted hyperparameters rebuild the same surrogate: the first predict of each (MDGP: the same (seed, call 0))
    m2 = C(Xtr, Ytr, d, 2, lb, ub, hyperparameters=m.hyperparameters, **kw)
    b = m2.predict(Xte)
    assert np.array_equal(mean, b[0]) and np.array_equal(var, b[1])


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
@pytest.mark.parametrize("surrogate", ["MDSPP_Matern", "MDGP_Matern"])
def test_unmodified_moasmo_epoch_trains_the_deep_gps_on_the_gpu(L, surrogate):
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
        optimizer_kwargs={}, surrogate_method_name=f"dmosopt_b200.model_gpytorch.{surrogate}",
        surrogate_method_kwargs={"fit": "gpu-seeded", "n_iter": 5, "num_inducing_points": 32}, local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))


def test_argument_errors(L):
    from dmosopt_b200 import model_gpytorch as mg

    rng = np.random.default_rng(13)
    X, Y = _data(rng, 40, 3, 2)
    launches = L.launch_count()
    with pytest.raises(L.DmoError, match="Z1, Z2 <= 128"):
        L.DGPFitState(X, Y, 2, 129, 8, 3, True, 10)
    with pytest.raises(L.DmoError, match="H, T <= 8"):
        L.DGPFitState(X, Y, 9, 8, 8, 3, True, 10)
    with pytest.raises(L.DmoError, match="batch_max"):
        L.DGPFitState(X, Y, 2, 8, 8, 3, True, 41)
    with pytest.raises(L.DmoError, match="X must be finite"):
        L.DGPFitState(np.where(X > 0.99, np.nan, X), Y, 2, 8, 8, 3, True, 10)
    with pytest.raises(L.DmoError, match="lengthscale_bounds"):
        L.DGPFitState(X, Y, 2, 8, 8, 3, True, 10, lengthscale_bounds=(2.0, 1.0))
    raw = _raw(rng, X, 2, 2, 8, 8, True, None)
    st = _state(L, X, Y, raw, True, 3, 10, None)
    with pytest.raises(L.DmoError, match="entries"):
        st.set_params(np.zeros(st.n_params + 1))
    with pytest.raises(L.DmoError, match="finite"):
        st.set_params(np.full(st.n_params, np.nan))
    with pytest.raises(L.DmoError, match="outside"):
        st.loss_grad([0, 40])
    with pytest.raises(L.DmoError, match="batch_max"):
        st.loss_grad(np.arange(11))
    with pytest.raises(L.DmoError, match="permutation"):
        st.epoch(np.zeros(40, np.int64), 10, 0.1)
    with pytest.raises(L.DmoError, match="lr"):
        st.adam_step(-1.0)
    assert L.launch_count() == launches  # every refusal came before any launch
    bad = dict(raw)
    bad["last_inducing_points"] = np.zeros_like(raw["last_inducing_points"])  # coincident points
    bad["last_raw_outputscale"] = np.full(2, 1e13)  # s = softplus(1e13) >> jitter: K(Z, Z) + jitter I is numerically singular
    st.set_params(mg.deepgp_flatten(bad))
    with pytest.raises(L.DmoError, match="last layer unit 0 is not positive definite"):
        st.loss_grad(np.arange(10))
