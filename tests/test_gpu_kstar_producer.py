"""The K_* producer of the tensor predict with variance (kstar_mean_kernel: K_* hi / lo planes and the K_* alpha mean from
one kernel) at the shapes it takes that the other parity tests do not reach: per-dimension length scales (M <= 2), d = 32
and M = 6, ragged N and P, training-set slices that start inside a 64-point chunk.  Against the CPU oracle at the tensor path's bars, and against the two-kernel route
(DMO_GP_FUSED=0: kstar_tensor_kernel + mean_split_kernel), whose K_* planes carry the same bits: the variances, which
depend on K_* only through the contraction, must agree exactly."""

import numpy as np
import pytest

from oracle import gp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


# (1000, 12, 2, 33792): 132 candidate blocks of 256 on a 1024-point padded training set; with the slice choice for 132 SMs
# (pick_slices) the training set falls into slices of 352 points, so the 64-point chunks at the slice boundaries are
# shared by two blocks, each storing its half of the lines and folding only its own 16-point groups into the mean
@pytest.mark.parametrize("N,d,M,P,ard,kind", [(700, 16, 1, 300, True, "rbf"), (600, 32, 6, 700, False, "matern"), (513, 32, 2, 1030, True, "matern"),
                                               (1000, 12, 2, 33792, True, "matern")])
def test_kstar_producer_shapes(L, monkeypatch, N, d, M, P, ard, kind):
    rng = np.random.default_rng(7 * N + P)
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, : min(4, d)].sum(axis=1) + k) + Xtr[:, (1 + k) % d] ** 2 for k in range(M)])
    ls = [(0.4 + 0.6 * rng.random(d)) if ard else 0.5 + 0.05 * m for m in range(M)]
    knd = gp.MATERN52 if kind == "matern" else gp.RBF
    st = gp.fit_fixed(Xtr, Ytr, xlb, xub, [1.0 + 0.5 * m for m in range(M)], ls, 1e-3, kind=knd)  # well conditioned at any d
    h = L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                   [np.broadcast_to(np.asarray(o.length_scale, dtype=np.float64), (d,)) for o in st.objectives], [o.noise for o in st.objectives],
                   [o.y_mean for o in st.objectives], [o.y_std for o in st.objectives], xlb, xub, kernel=L.KERNEL_MATERN52 if kind == "matern" else L.KERNEL_RBF)
    X = rng.random((P, d))
    X[:5] = np.clip(Xtr[:5] + 1e-2 * rng.standard_normal((5, d)), 0, 1)
    mean_o, var_o = gp.predict(st, X)
    ystd = np.array([o.y_std for o in st.objectives])
    prior = np.array([(o.constant + o.noise) * o.y_std**2 for o in st.objectives])
    monkeypatch.setenv("DMO_GP_FUSED", "1")
    mean_f, var_f = h.predict(X, precision=L.GP_TENSOR)
    monkeypatch.setenv("DMO_GP_FUSED", "0")
    mean_s, var_s = h.predict(X, precision=L.GP_TENSOR)
    h.close()
    err_v = np.max(np.abs(var_f - var_o) / prior)
    err_m = np.max(np.abs(mean_f - mean_o) / np.maximum(np.abs(mean_o), ystd))
    print(f"K_* producer N={N} d={d} M={M} ard={ard} {kind}: var err/prior {err_v:.2e}, mean rel err {err_m:.2e}")
    assert err_v < 1e-5, err_v
    assert err_m < 1e-5, err_m
    assert np.array_equal(var_f, var_s)  # same K_* bits from both producers
    assert np.max(np.abs(mean_f - mean_s) / np.maximum(np.abs(mean_s), ystd)) < 1e-5  # fp32 kernel values vs stored hi + lo
