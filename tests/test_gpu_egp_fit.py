"""EGP_Matern training on the GPU (row A19): dmo_gp_lml_grad against the dense torch autograd oracle
(oracle/egp_train.py), against one-task dmo_mtgp_lml_grad calls (an independently derived gradient) and dmo_gp_fit's
log marginal likelihood; its per-objective determinism however the objectives are batched; egp_fit's Adam loop against
torch.optim.Adam on the oracle; the fitted surrogate against the hyper-parameters path and the dense posterior; and the
unmodified reference controller training the plugin without gpytorch."""

import sys

import numpy as np
import pytest

from oracle import egp, egp_train

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
    Y = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, (t + 2) % d] + 0.2 * t * X[:, -1] ** 2 for t in range(M)])
    yn, _, _ = egp.normalise_y(Y)
    return X, yn


def _hyper(rng, d, M, floor=False):
    hp = dict(length_scale=np.exp(rng.uniform(np.log(0.05), np.log(5.0), (M, d))), outputscale=0.3 + 1.2 * rng.random(M),
              noise=np.geomspace(2e-3, 2e-2, M), weight=0.3 * rng.standard_normal((M, d)), bias=0.2 * rng.standard_normal(M))
    if floor:  # the likelihood's GreaterThan(1e-4) floor, moderate length scales
        hp["length_scale"] = np.exp(rng.uniform(np.log(0.3), np.log(1.0), (M, d)))
        hp["noise"] = np.full(M, 1e-4)
    return hp


def _close(g, rg, rel):
    for k in rg:
        err, scale = np.abs(g[k] - rg[k]).max(), np.abs(rg[k]).max()
        assert err <= rel * scale, (k, err, scale)


def _check_against_oracle(L, X, yn, hp):
    lml, g = L.gp_lml_grad(X, yn, *hp.values())
    ref, rg = egp_train.lml_and_grad_torch(X, yn, *hp.values())
    assert np.all(np.abs(lml - ref) <= 1e-10 * np.abs(ref)), (lml, ref)
    _close(g, rg, 1e-8)
    return lml, g


@pytest.mark.parametrize("N", [150, 256, 333])
@pytest.mark.parametrize("d", [2, 12, 40])
@pytest.mark.parametrize("M", [1, 2, 3, 5])
def test_lml_grad_vs_autograd_oracle(L, M, d, N):
    rng = np.random.default_rng(1000 * M + 10 * d + N)
    X, yn = _data(rng, N, d, M)
    _check_against_oracle(L, X, yn, _hyper(rng, d, M))


def test_lml_grad_at_the_noise_floor(L):
    rng = np.random.default_rng(78)
    X, yn = _data(rng, 150, 12, 3)
    _check_against_oracle(L, X, yn, _hyper(rng, 12, 3, floor=True))


@pytest.mark.parametrize("N,d,M", [(150, 2, 1), (256, 12, 3), (333, 40, 5)])
def test_lml_grad_vs_one_task_multitask_calls(L, N, d, M):
    """Objective m as an MEGP with one task (B = [[s_m]], D = [noise_m]): the block route of dmo_mtgp_lml_grad."""
    rng = np.random.default_rng(7 * N + d + M)
    X, yn = _data(rng, N, d, M)
    hp = _hyper(rng, d, M)
    lml, g = L.gp_lml_grad(X, yn, *hp.values())
    for m in range(M):
        ref, rg = L.mtgp_lml_grad(X, yn[:, m], hp["length_scale"][m], np.array([[hp["outputscale"][m]]]), hp["noise"][m : m + 1],
                                  hp["weight"][m : m + 1], hp["bias"][m : m + 1])
        assert abs(lml[m] - ref) <= 1e-10 * abs(ref), (m, lml[m], ref)
        _close({"length_scale": g["length_scale"][m], "outputscale": g["outputscale"][m : m + 1], "noise": g["noise"][m : m + 1],
                "weight": g["weight"][m], "bias": g["bias"][m : m + 1]},
               {"length_scale": rg["length_scale"], "outputscale": rg["B"][0], "noise": rg["D"], "weight": rg["weight"][0], "bias": rg["bias"]},
               1e-10)


def test_lml_is_gp_fits_lml(L):
    rng = np.random.default_rng(31)
    N, d, M = 333, 9, 4
    X, yn = _data(rng, N, d, M)
    hp = _hyper(rng, d, M)
    lml, _ = L.gp_lml_grad(X, yn, *hp.values())
    res = yn.T - (hp["weight"] @ X.T + hp["bias"][:, None])
    _, _, ref = L.gp_fit(X, res, hp["outputscale"], list(hp["length_scale"]), hp["noise"], jitter=0.0, want_L=False, want_alpha=False)
    assert np.all(np.abs(lml - ref) <= 1e-12 * np.abs(ref)), (lml, ref)


def test_each_objective_is_bit_identical_however_batched(L):
    rng = np.random.default_rng(41)
    N, d, M = 333, 7, 5
    X, yn = _data(rng, N, d, M)
    hp = _hyper(rng, d, M)
    full = L.gp_lml_grad(X, yn, *hp.values())
    again = L.gp_lml_grad(X, yn, *hp.values())
    rev = L.gp_lml_grad(X, yn[:, ::-1], *(v[::-1] for v in hp.values()))

    def same(a, ia, b, ib):
        assert a[0][ia] == b[0][ib]
        for k in a[1]:
            assert np.array_equal(a[1][k][ia], b[1][k][ib]), k

    for m in range(M):
        alone = L.gp_lml_grad(X, yn[:, m : m + 1], *(v[m : m + 1] for v in hp.values()))
        same(full, m, alone, 0)
        same(full, m, again, m)
        same(full, m, rev, M - 1 - m)


def test_adam_trajectory_matches_torch(L):
    from dmosopt_b200.model_gpytorch import egp_fit, egp_initial_raw

    rng = np.random.default_rng(8)
    N, d, M = 200, 8, 2
    X, yn = _data(rng, N, d, M)
    raw0 = egp_initial_raw(d, M, seed=3)
    _, info = egp_fit(X, yn, n_iter=300, initial_raw=raw0)
    for m in range(M):
        raw_ref, loss_ref, _ = egp_train.train_adam_torch(X, yn[:, m], {k: v[m : m + 1] for k, v in raw0.items()}, n_iter=300)
        assert info[m]["iterations"] == 300 and len(loss_ref) == 300
        assert np.all(np.abs(info[m]["loss"] - loss_ref) <= 1e-9 * np.abs(loss_ref)), m
        for k in raw_ref:
            assert np.abs(info[m]["raw"][k] - raw_ref[k]).max() <= 1e-7, (m, k)


def test_default_fit_stops_like_the_oracle_trainer(L):
    """ZDT1's first objective is x_0 itself: the linear mean fits it exactly, and Adam then drives its output scale
    towards 0 with the noise at its floor.  There the loss is flat in most directions, Adam's normalised steps follow the
    sign of gradients that are mostly rounding, and the float64 trajectories of two correct implementations part after
    some 500 iterations (relative loss differences grow from 1e-15 to 1e-4).  Its trajectory is compared up to there, and
    it must stop for the same criteria within a few iterations; the second objective must stop at the same iteration."""
    from dmosopt_b200.model_gpytorch import egp_fit, egp_initial_raw, egp_natural

    rng = np.random.default_rng(9)
    N, d, M = 200, 6, 2
    X = rng.random((N, d))
    yn, _, _ = egp.normalise_y(_zdt1(X))
    hp, info = egp_fit(X, yn, seed=0)
    raw0 = egp_initial_raw(d, M, seed=0)

    def criteria(reason):  # the tests that held, without their formatted values
        return [r.split(" (")[0] for r in reason.split("; ")]

    for m in range(M):
        _, loss_ref, reason_ref = egp_train.train_adam_torch(X, yn[:, m], {k: v[m : m + 1] for k, v in raw0.items()})
        a = info[m]["loss"]
        assert np.all(np.abs(a[:500] - loss_ref[:500]) <= 1e-12 * np.abs(loss_ref[:500])), m
        assert criteria(info[m]["stop_reason"]) == criteria(reason_ref), (m, info[m]["stop_reason"], reason_ref)
        if m == 0:
            assert abs(info[m]["iterations"] - len(loss_ref)) <= 10, (m, info[m]["iterations"], len(loss_ref))
        else:
            assert info[m]["iterations"] == len(loss_ref), (m, info[m]["iterations"], len(loss_ref))
        assert info[m]["iterations"] < 5000
    lml0, _ = L.gp_lml_grad(X, yn, *egp_natural(raw0))
    lml1, _ = L.gp_lml_grad(X, yn, hp["lengthscale"], hp["outputscale"], hp["noise"], hp["weight"], hp["bias"])
    assert np.all(lml1 > lml0)
    hpb, _ = egp_fit(X, yn, lengthscale_bounds=(0.3, 2.0), n_iter=300)
    assert np.all(hpb["lengthscale"] >= 0.3) and np.all(hpb["lengthscale"] <= 2.0)


def test_lockstep_groups_are_bit_identical_to_single_objective_fits(L):
    """Ten objectives train in two groups of at most eight, and leave the batch when they stop; each one's result is
    the one of training it alone."""
    from dmosopt_b200.model_gpytorch import egp_fit, egp_initial_raw

    rng = np.random.default_rng(12)
    N, d, M = 64, 3, 10
    X = rng.random((N, d))
    Y = np.column_stack([np.sin((1 + 0.3 * t) * X[:, 0] + t) + 0.1 * t * X[:, 1] * X[:, 2] for t in range(M)])
    yn, _, _ = egp.normalise_y(Y)
    raw0 = egp_initial_raw(d, M, seed=5)
    hp, info = egp_fit(X, yn, n_iter=1100, min_loss_pct_change=1.0, initial_raw=raw0)
    for m in range(M):
        hpm, im = egp_fit(X, yn[:, m : m + 1], n_iter=1100, min_loss_pct_change=1.0, initial_raw={k: v[m : m + 1] for k, v in raw0.items()})
        assert im[0]["iterations"] == info[m]["iterations"] and im[0]["stop_reason"] == info[m]["stop_reason"], m
        assert np.array_equal(im[0]["loss"], info[m]["loss"]), m
        for k in hpm:
            assert np.array_equal(hpm[k][0], hp[k][m]), (m, k)


def test_fitted_surrogate_is_the_hyperparameter_path(L):
    from dmosopt_b200.model_gpytorch import EGP_Matern

    rng = np.random.default_rng(10)
    N, d, M = 180, 5, 3
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    X = xlb + rng.random((N, d)) * (xub - xlb)
    Y = np.column_stack([np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] for t in range(M)]) * (1.0 + np.arange(M))
    Xs = xlb + rng.random((250, d)) * (xub - xlb)
    sm = EGP_Matern(X, Y, d, M, xlb, xub, fit="gpu", n_iter=300, seed=2)
    assert len(sm.fit_info) == M and all(i["iterations"] == 300 and len(i["loss"]) == 300 for i in sm.fit_info)
    hp = sm.hyperparameters
    st = egp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["outputscale"], hp["noise"], hp["weight"], hp["bias"])
    em, ev = egp.predict(st, Xs)
    prior = np.array([(o.outputscale + o.noise) * o.y_std**2 for o in st.objectives])
    for precision, tol in (("fp64", 2e-6), ("tensor", 1e-5)):
        a = EGP_Matern(X, Y, d, M, xlb, xub, fit="gpu", n_iter=300, seed=2, precision=precision).predict(Xs)
        b = EGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision).predict(Xs)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.all(np.abs(a[0] - em).max(axis=0) <= tol * np.abs(em).max(axis=0))
        assert np.all(np.abs(a[1] - ev).max(axis=0) <= tol * prior)


def _reference_path():
    from oracle import reference_build

    return reference_build.reference_path()


@pytest.mark.skipif(_reference_path() is None, reason="reference package not built (oracle/_ref) nor given ($DMOSOPT_REF)")
def test_unmodified_moasmo_epoch_trains_egp_on_the_gpu(L):
    """surrogate_method_name EGP_Matern with no surrogate keywords: without gpytorch the plugin trains on the GPU."""
    ref = _reference_path()
    sys.path.insert(0, ref)
    try:
        from dmosopt import MOASMO
    finally:
        sys.path.remove(ref)
    d, M, pop = 8, 2, 64
    rng = np.random.default_rng(13)
    xlb, xub = np.zeros(d), np.ones(d)
    X = rng.random((120, d))
    Y = _zdt1(X)
    gen = MOASMO.epoch(
        4, [f"x{i}" for i in range(d)], ["y1", "y2"], xlb, xub, 0.25, X, Y, None, pop=pop, optimizer_name="dmosopt_b200.CMAES",
        optimizer_kwargs={}, surrogate_method_name="dmosopt_b200.model_gpytorch.EGP_Matern", surrogate_method_kwargs={},
        local_random=rng,
    )
    try:
        next(gen)
        raise AssertionError("epoch should finish without yielding when a surrogate is present")
    except StopIteration as ex:
        res = ex.args[0]
    xr, yp = res["x_resample"], res["y_pred"]
    assert xr.shape[1] == d and len(xr) > 0 and yp.shape == (len(xr), M) and np.all(np.isfinite(yp))
    from dmosopt_b200.model_gpytorch import EGP_Matern

    sm = EGP_Matern(X, Y, d, M, xlb, xub)
    assert sm.fit_info is not None and all(i["iterations"] >= 51 for i in sm.fit_info)
    mean, _ = sm.predict(xr)
    assert np.allclose(yp, mean, rtol=1e-4, atol=1e-4 * np.abs(mean).max())
