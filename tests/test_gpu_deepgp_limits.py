"""The deep GPs (MDSPP_Matern, MDGP_Matern) at the edges of their shape envelope and on both sides of every blocking
constant of their kernels: the predict (csrc/gp_deep.cu) against oracle/deepgp.py and the training (csrc/gp_deep_fit.cu)
against the torch autograd oracle oracle/deepgp_train.py.

Bars, those of test_gpu_deepgp.py and test_gpu_deepgp_fit.py: predict float64, the mean within 1e-9 of max(|mean|,
y_std) and the variance within 1e-9 of y_std^2 (s2 + noise); with the tensor hidden layer 1e-4 of the same scales;
training, the loss within 1e-10 relative and every gradient block within 1e-8 of its max |ref|.  Models past 128
inducing points keep K(Z, Z) + jitter well conditioned (_spread: last-layer points N(0, 1.5^2) in H = 8 dimensions with
length scales 0.9 .. 1.1, hidden points in [0, 1]^8 with length scales 0.2 .. 0.25; cond(K) measured at most ~300 at
Z = 8192), and their q_sqrt's off-diagonal scaled by sqrt(128 / Z) so that S = q_sqrt q_sqrt' stays O(1) instead of
growing with Z.  Otherwise the bar would measure the conditioning of the model, not the kernel.

What each case straddles (gp_deep.cu unless named):

Predict, dgp_layer2_kernel:
  * Z2 in {1, 15, 16, 17, 127, 128, 129, 255, 256, 257, 1000, 8192}, H 8, T 2, J 3, P 100 (PT = 21: the last CTA holds
    16 candidates), MDSPP and MDGP, float64 and tensor hidden layer (test_layer2_blocking):
      - DG_KS = 16 staged operator columns (:36, :133-139): 15 / 16 / 17;
      - DG_IB = DG_KC = 128 operator-row blocks and K_* chunks (:34-35, :103-106, :112): 127 / 128 / 129, 255 / 256 / 257,
        and the warp's skip of column steps above the diagonal (:141) in every block past the first;
      - GpVarOps Npad (gp.cu:407, rows rounded up to 256): 256 / 257 pad to 256 / 512;
      - DG_ZMAX = 8192 (:32, :252), at T 1, J 2, P 45.
    At every Z2 the mean-only call (dgp_layer2_kernel<false>, one block over every chunk) equals the full call's mean
    (<true>, the mean summed on each chunk's first visit, :130-131) bit for bit.
  * J in {1, 2, 21, 22, 31, 32, 33, 63, 64}, P in {1, PT - 1, PT, PT + 1, 300} with PT = DG_ROWS / J (:33, :356):
    PT = 64, 32, 3, 2, 2, 2, 1, 1, 1; idle CTA rows at J 21, 22, 31, 33, 63; J 64 = DG_MAX_SITES (:31)
    (test_sites_per_candidate).
  * The MDGP draws replayed on the host from Philox4x32-10, counter (p, (stream_id << 10) | (j H + h)) (:91) and
    Box-Muller (:93), at T = H = 8 = DG_MAX_HT (:30, the full us[64][9] row :73 and DgTasks table :46-48), J = 64 and a
    stream_id near 2^54 (:337), and at J = 3, where a CTA holds 21 candidates; only task 0 writes eps_out (:95), and
    every task's mean and variance against the oracle fed those draws shows that each task's CTAs drew the same
    (test_predict_draws_replay).
  * H = T = 8 with Z2 in {129, 257}; Z1 in {255, 256, 257} at H = T = 8; Z1 = 8192 = DG_ZMAX with H = 1
    (test_widest_layers).
  * d in {1, 64, 65, 90}: 64 the tensor hidden layer's limit, 65 and 90 float64 only (the tensor request refused,
    gp_multitask.cu:327), 90 = MT_FIT_DMAX (gp.cuh:159) (test_input_dimension).
  * The hidden layer's candidate chunk (GpUnitPredict::alloc, gp_multitask.cu:331-338) at Z1 = 2048: P = chunk + 1,
    the rows around the seam against the oracle and against a predict of just those rows (test_hidden_layer_chunk_seam).
  * Refusals one past each limit, before any launch: Z1 or Z2 = 8193, d = 91, H or T = 9 (:250-254) (test_create_refusals).

Training, dmo_dgp_fit_* (gp_deep_fit.cu), each case at batch_max = B (row stride RS = J batch_max equal to the call's
R2 = J B) and at batch_max = B + 7 (RS != R2; the row-capacity case runs B - 7 instead) (test_fit_thresholds):
  * DF_RT = 32 rows per CTA (:39, :214-215, :332-333, :730): hidden rows B in {31, 32, 33} (J 1, so R2 too); last-layer
    rows R2 = J B in {31, 32, 33} as 31 x 1, 32 x 1 (MDGP) and 3 x 11 (MDSPP).
  * DF_RC = 512 rows per Gram chunk (:40, :465, :730, the chunk sums :522, :610): R2 = 7 x 73, 8 x 64, 3 x 171; hidden
    B in {511, 512, 513} with J 1.
  * 32 x 32 Gram tiles, nt = ceil(ZS / 32) (:457-461, :472-476): ZS in {32, 33, 64, 65, 96, 97, 128}, with Z1 != Z2
    both ways, (33, 128) and (128, 1), so that one unit leaves partial and absent tiles below ZS.
  * DF_MAX_ROWS = 65536 (:41, :818): n_sites x batch_max = 16 x 4096 computes correctly; 16 x 4097 and 1 x 65537 are
    refused before any launch (test_fit_row_capacity_refusal).
  * The largest layout: H = T = 8, Z1 = Z2 = 128 = DF_ZMAX (:37-38), d = 90, the rows kernels at df_rows_smem(128) =
    192 KB (:705), MDSPP and MDGP; there two loss_grad calls are bit-identical (the file's fixed sum orders, :25-26).
  * Epochs with N = 513, B = 512 (a last batch of one row, :1014-1016): epoch() equals its steps bit for bit
    (test_epoch_with_a_one_row_last_batch).
  * The training draws replayed from Philox4x32-10, counter (step, (i << 32) | (j H + h)) (:284) (test_fit_draws_replay).

Box-Muller bound (both replays): e = sqrt(-2 log1p(-u1)) cospi(2 u2) with u1, u2 the same doubles on both sides.  CUDA
documents log1p to 1 ulp and cospi to 2 ulp, and sqrt and the products round correctly (1/2 ulp).  An ulp of x is at
most 2^-52 |x|, so the relative error is at most 1/2 (log1p, halved by the square root) + 1/2 (sqrt) + 2 (cospi) + 1/2
(product) = 3.5 times 2^-52, to first order.  The host evaluates in long double with cospi reduced exactly to
[-1/4, 1/4] (its own error is below 2^-60 relative); the bound used is 3.6 * 2^-52 |e|.

Cost: the file ran in 87 s on one H100 80GB HBM3 (700 W power limit), most of it the host side of the four cases at
8192 inducing points (building the model and the oracle's float64 Cholesky factors, 10-16 s each); the oracle needs no
cached factor at that size.
"""

import functools

import numpy as np
import pytest

from oracle import deepgp as DG
from oracle import deepgp_train as ot
from oracle import philox
from test_deepgp_cpu import problem
from test_gpu_deepgp import _assert_bars, _handle
from test_gpu_deepgp_fit import _check_grad, _data, _raw, _state

pytestmark = pytest.mark.gpu

LD = np.longdouble
DG_ROWS = 64  # gp_deep.cu:33
DG_ZMAX = 8192  # gp_deep.cu:32
DF_MAX_ROWS = 1 << 16  # gp_deep_fit.cu:41
MAX_CHUNK = 1 << 20  # gp.cuh: GP_MAX_CHUNK


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _tol(precision):
    return 1e-9 if precision == "fp64" else 1e-4


def _prec(L, precision):
    return L.GP_FP64 if precision == "fp64" else L.GP_TENSOR


def _spread(hp, rng):
    """Past 128 inducing points: well-conditioned K(Z, Z) + jitter and S = q_sqrt q_sqrt' of order one (see the module
    docstring)."""
    for layer in ("hidden", "last"):
        ch = hp[f"{layer}_chol_variational_covar"]
        U, Z = ch.shape[:2]
        if Z <= 128:
            continue
        if layer == "last":
            hp["last_lengthscale"] = 0.9 + 0.2 * rng.random(hp["last_lengthscale"].shape)
        else:
            hp["hidden_lengthscale"] = 0.2 + 0.05 * rng.random(hp["hidden_lengthscale"].shape)
        f = np.sqrt(128.0 / Z)
        for u in range(U):
            dg = np.diagonal(ch[u]).copy()
            ch[u] *= f  # the junk above the diagonal is masked either way
            ch[u][np.diag_indices(Z)] = dg
    return hp


def _model(seed, d, H, T, Z1, Z2, J, P):
    """A random model (with J quadrature sites, unused by MDGP) and P candidates around its input box."""
    rng = np.random.default_rng(seed)
    hp, ym, ys, xlb, xrng = problem(rng, d, H, T, Z1, Z2, J=J, quadrature=True)
    _spread(hp, rng)
    x = xlb + xrng * (1.2 * rng.random((P, d)) - 0.1)
    return hp, ym, ys, xlb, xrng, x


def _oracle(x, xlb, xrng, hp, ym, ys, eps, quadrature):
    return DG.predict(x, xlb, xrng, hp, ym, ys, eps=None if quadrature else eps)


# ------------------------------------------------------------------------------------------ predict
Z2S = [1, 15, 16, 17, 127, 128, 129, 255, 256, 257, 1000, DG_ZMAX]


@functools.lru_cache(maxsize=1)
def _largest_z2_model():
    return _model(8192, 4, 8, 1, 40, DG_ZMAX, 2, 45)


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
@pytest.mark.parametrize("Z2", Z2S)
def test_layer2_blocking(L, Z2, quadrature):
    if Z2 == DG_ZMAX:  # its q_sqrt plane alone is 512 MB: one task, J 2 (PT 32), P 45
        J = 2
        hp, ym, ys, xlb, xrng, x = _largest_z2_model()
    else:
        J = 3
        hp, ym, ys, xlb, xrng, x = _model(100 + Z2, 4, 8, 2, 40, Z2, J, 100)
    assert x.shape[0] % (DG_ROWS // J) != 0  # the last CTA is ragged
    g = _handle(hp, ym, ys, xlb, xrng, quadrature, J)
    ref = None
    for precision in ("fp64", "tensor"):
        mean, var, eps = g.predict(x, seed=31, stream_id=7, return_eps=True, precision=_prec(L, precision))
        if ref is None:
            ref = _oracle(x, xlb, xrng, hp, ym, ys, eps, quadrature)
        _assert_bars(hp, ys, mean, var, *ref, _tol(precision))
        m0, v0 = g.predict(x, seed=31, stream_id=7, return_var=False, precision=_prec(L, precision))
        assert v0 is None
        assert np.array_equal(m0, mean), (precision, np.max(np.abs(m0 - mean)))


def _pt_sizes(J):
    PT = DG_ROWS // J
    return sorted({p for p in (1, PT - 1, PT, PT + 1, 300) if p >= 1})


SITES = [(J, P) for J in (1, 2, 21, 22, 31, 32, 33, 63, 64) for P in _pt_sizes(J)]


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
@pytest.mark.parametrize("J,P", SITES, ids=[f"J{J}-P{P}" for J, P in SITES])
def test_sites_per_candidate(L, J, P, quadrature):
    hp, ym, ys, xlb, xrng, x = _model(200 + J, 3, 2, 2, 20, 30, J, P)
    mean, var, eps = _handle(hp, ym, ys, xlb, xrng, quadrature, J).predict(x, seed=3, stream_id=1, return_eps=True)
    assert eps.shape == (J, P, 2)
    _assert_bars(hp, ys, mean, var, *_oracle(x, xlb, xrng, hp, ym, ys, eps, quadrature), 1e-9)


def _cospi(x):
    """cos(pi x) in long double for doubles x in [0, 2): x = k / 2 + y with |y| <= 1/4 exactly (Sterbenz)."""
    k = np.rint(2.0 * x)
    y = (x - 0.5 * k).astype(LD)
    pi = 4 * np.arctan(LD(1))
    c, s = np.cos(pi * y), np.sin(pi * y)
    k = k.astype(np.int64) % 4
    return np.select([k == 0, k == 1, k == 2], [c, -s, -c], s)


def box_muller(seed, ctr_lo, ctr_hi):
    """The draws of Philox(seed)(ctr_lo, ctr_hi) through the kernels' Box-Muller, in long double, and their bound."""
    w = philox.philox4x32_10(seed, ctr_lo, ctr_hi)
    u1, u2 = philox.u01_53(w[0], w[1]), philox.u01_53(w[2], w[3])
    e = np.sqrt(LD(-2) * np.log1p(-u1.astype(LD))) * _cospi(2.0 * u2)
    return e, 3.6 * 2.0**-52 * np.abs(e)


def _within(got, ref, bound):
    err = np.abs(got.astype(LD) - ref)
    assert np.all(err <= bound), (np.argwhere(err > bound)[:5], float(np.max(err / np.maximum(bound, LD(1e-300)))))


@pytest.mark.parametrize("J,H,T,P", [(64, 8, 8, 37), (3, 8, 2, 100)], ids=["J64-PT1", "J3-PT21"])
def test_predict_draws_replay(L, J, H, T, P):
    """J 64: PT 1, 37 CTAs per task and 8 task rows.  J 3: PT 21, where a CTA's index is not its candidates' index."""
    stream_id = (1 << 53) + 12345
    hp, ym, ys, xlb, xrng, x = _model(300 + J, 5, H, T, 30, 40, J, P)
    mean, var, eps = _handle(hp, ym, ys, xlb, xrng, False, J).predict(x, seed=0xDEADBEEF12345, stream_id=stream_id, return_eps=True)
    j, p, h = np.meshgrid(np.arange(J), np.arange(P), np.arange(H), indexing="ij")
    ctr_hi = (np.uint64(stream_id) << np.uint64(10)) | (j * H + h).astype(np.uint64)
    ref, bound = box_muller(0xDEADBEEF12345, p.astype(np.uint64), ctr_hi)
    _within(eps, ref, bound)
    # every task against the oracle fed task 0's draws: a task whose CTAs drew differently would be far off
    _assert_bars(hp, ys, mean, var, *DG.predict(x, xlb, xrng, hp, ym, ys, eps=eps), 1e-9)


WIDE = [  # (d, H, T, Z1, Z2, J, P)
    (4, 8, 8, 40, 129, 3, 50),
    (4, 8, 8, 40, 257, 3, 50),
    (8, 8, 8, 255, 37, 3, 50),
    (8, 8, 8, 256, 37, 3, 50),
    (8, 8, 8, 257, 37, 3, 50),
    (8, 1, 1, DG_ZMAX, 20, 2, 45),
]


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
@pytest.mark.parametrize("shape", WIDE, ids=lambda s: "d{}-H{}-T{}-Z{}-{}-J{}-P{}".format(*s))
def test_widest_layers(L, shape, quadrature):
    d, H, T, Z1, Z2, J, P = shape
    hp, ym, ys, xlb, xrng, x = _model(400 + Z1 + Z2, *shape)
    g = _handle(hp, ym, ys, xlb, xrng, quadrature, J)
    mean, var, eps = g.predict(x, seed=4, stream_id=2, return_eps=True)
    ref = _oracle(x, xlb, xrng, hp, ym, ys, eps, quadrature)
    _assert_bars(hp, ys, mean, var, *ref, 1e-9)
    mt, vt = g.predict(x, seed=4, stream_id=2, precision=L.GP_TENSOR)
    _assert_bars(hp, ys, mt, vt, *ref, 1e-4)


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
@pytest.mark.parametrize("d", [1, 64, 65, 90])
def test_input_dimension(L, d, quadrature):
    hp, ym, ys, xlb, xrng, x = _model(500 + d, d, 3, 2, 50, 40, 3, 70)
    g = _handle(hp, ym, ys, xlb, xrng, quadrature, 3)
    mean, var, eps = g.predict(x, seed=5, return_eps=True)
    ref = _oracle(x, xlb, xrng, hp, ym, ys, eps, quadrature)
    _assert_bars(hp, ys, mean, var, *ref, 1e-9)
    if d <= L.GP_PREDICT_MAX_D:
        _assert_bars(hp, ys, *g.predict(x, seed=5, precision=L.GP_TENSOR), *ref, 1e-4)
    else:
        launches = L.launch_count()
        with pytest.raises(L.DmoError, match=r"dgp_predict\(tensor\): at most 64 input dimensions"):
            g.predict(x, seed=5, precision=L.GP_TENSOR)
        assert L.launch_count() == launches


def unit_chunk(Z, tensor):
    """GpUnitPredict::alloc (gp_multitask.cu:331-338): the K_* plane of a chunk (Npad float64, or fp16 hi + lo) within
    6 GiB, at most GP_MAX_CHUNK candidates, a multiple of the 128-candidate tile."""
    npad = -(-Z // 256) * 256
    pc = min((6 << 30) // (npad * (4 if tensor else 8)), MAX_CHUNK)
    return max(pc // 128 * 128, 128)


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
def test_hidden_layer_chunk_seam(L, precision):
    """Z1 = 2048: chunks of 393 216 (float64) and 786 432 (tensor) candidates; P = chunk + 1.  The rows [chunk - 256, P)
    (a start on a multiple of 256, so each row keeps its place in its 128- and 256-candidate tiles) against the oracle,
    and against a predict of just those rows: the tensor hidden variance bit for bit (fixed n_q partial sums), the
    float64 one within 1e-12 of the scales (its n_vp partial sums follow the chunk length), as test_gpu_predict_chunks.py
    holds the variational predict.  MDSPP, whose sites do not depend on the row's index."""
    Z1 = 2048
    chunk = unit_chunk(Z1, precision == "tensor")
    assert chunk == ((6 << 30) // (Z1 * (4 if precision == "tensor" else 8)))
    P = chunk + 1
    hp, ym, ys, xlb, xrng, x = _model(600, 8, 1, 1, Z1, 16, 1, P)
    g = _handle(hp, ym, ys, xlb, xrng, True, 1)
    mean, var = g.predict(x, precision=_prec(L, precision))
    assert np.all(np.isfinite(mean)) and np.all(np.isfinite(var))
    w = np.arange(chunk - 256, P)
    ma, va = g.predict(x[w], precision=_prec(L, precision))
    if precision == "tensor":
        assert np.array_equal(ma, mean[w]) and np.array_equal(va, var[w])
    else:
        _assert_bars(hp, ys, mean[w], var[w], ma, va, 1e-12)
    _assert_bars(hp, ys, mean[w], var[w], *DG.predict(x[w], xlb, xrng, hp, ym, ys), _tol(precision))


def _zeros_handle(d, H, T, Z1, Z2, J=3):
    """A create call with arrays of the requested shape; the shape checks come before any value is read."""
    from dmosopt_b200 import _lib

    z = np.zeros
    return _lib.DGPHandle(z((H, Z1, d)), np.ones(H), np.ones((H, d)), z((H, Z1)), z((H, Z1, Z1)), z(d), 0.0, z((T, Z2, H)), np.ones(T),
                          np.ones((T, H)), z((T, Z2)), z((T, Z2, Z2)), 0.0, np.ones(T), z(T), np.ones(T), z(d), np.ones(d), n_sites=J)


@pytest.mark.parametrize("shape,msg", [((2, 1, 1, DG_ZMAX + 1, 4), "unsupported shape"), ((2, 1, 1, 4, DG_ZMAX + 1), "unsupported shape"),
                                       ((91, 2, 2, 4, 4), "unsupported shape"), ((2, 9, 2, 4, 4), r"H, T <= 8"),
                                       ((2, 2, 9, 4, 4), r"H, T <= 8")],
                         ids=["Z1-8193", "Z2-8193", "d-91", "H-9", "T-9"])
def test_create_refusals(L, shape, msg):
    launches = L.launch_count()
    with pytest.raises(L.DmoError, match=msg):
        _zeros_handle(*shape)
    assert L.launch_count() == launches


# ------------------------------------------------------------------------------------------ training
FIT = [  # id, quadrature, d, H, T, Z1, Z2, J, B
    ("rt-hidden-31", True, 5, 2, 2, 20, 12, 1, 31),
    ("rt-hidden-32", True, 5, 2, 2, 20, 12, 1, 32),
    ("rt-hidden-33", True, 5, 2, 2, 20, 12, 1, 33),
    ("rt-last-31x1", False, 4, 2, 2, 12, 20, 31, 1),
    ("rt-last-32x1", False, 4, 2, 2, 12, 20, 32, 1),
    ("rt-last-3x11", True, 4, 2, 2, 12, 20, 3, 11),
    ("rc-last-7x73", False, 4, 2, 2, 16, 20, 7, 73),
    ("rc-last-8x64", True, 4, 2, 2, 16, 20, 8, 64),
    ("rc-last-3x171", True, 4, 2, 2, 16, 20, 3, 171),
    ("rc-hidden-511", True, 4, 2, 2, 20, 16, 1, 511),
    ("rc-hidden-512", True, 4, 2, 2, 20, 16, 1, 512),
    ("rc-hidden-513", True, 4, 2, 2, 20, 16, 1, 513),
    ("zs-32", True, 30, 3, 2, 32, 32, 2, 40),
    ("zs-33", False, 30, 3, 2, 33, 17, 2, 40),
    ("zs-64", True, 30, 3, 2, 64, 64, 2, 40),
    ("zs-65", False, 30, 3, 2, 17, 65, 2, 40),
    ("zs-96", True, 30, 3, 2, 96, 96, 2, 40),
    ("zs-97", False, 30, 3, 2, 97, 64, 2, 40),
    ("zs-33-128", True, 30, 3, 2, 33, 128, 2, 40),
    ("zs-128-1", False, 30, 3, 2, 128, 1, 2, 40),
    ("rows-65536", True, 2, 1, 1, 8, 8, 16, 4096),
    ("largest-mdspp", True, 90, 8, 8, 128, 128, 3, 64),
    ("largest-mdgp", False, 90, 8, 8, 128, 128, 4, 48),
]


@pytest.mark.parametrize("slack", [0, 7], ids=["rs-eq-r2", "rs-ne-r2"])
@pytest.mark.parametrize("case", FIT, ids=[c[0] for c in FIT])
def test_fit_thresholds(L, case, slack):
    name, quadrature, d, H, T, Z1, Z2, J, B = case
    Bmax = B + slack
    if J * Bmax > DF_MAX_ROWS:  # the row-capacity case: batch_max stays at the limit and the batch shrinks
        Bmax, B = B, B - slack
    N = Bmax + 7
    rng = np.random.default_rng(sum(map(ord, name)))
    X, Y = _data(rng, N, d, T)
    raw = _raw(rng, X, T, H, Z1, Z2, quadrature, None)
    raw.pop("quad_sites", None)
    if quadrature:
        raw["quad_sites"] = rng.standard_normal((J, H))
    st = _state(L, X, Y, raw, quadrature, J, Bmax, None)
    assert st.J * st.batch_max <= DF_MAX_ROWS
    batch = rng.choice(N, B, replace=False)
    loss, g, eps = st.loss_grad(batch, seed=17, step=9, return_eps=True)
    lo, go = ot.loss_grad(raw, X[batch], Y[batch], N, eps=None if quadrature else eps)
    assert abs(loss - lo) <= 1e-10 * abs(lo), (loss, lo)
    _check_grad(g, go, raw)
    if name.startswith("largest"):  # fixed sum orders, no atomics
        l2, g2, e2 = st.loss_grad(batch, seed=17, step=9, return_eps=True)
        assert l2 == loss and np.array_equal(g2, g) and np.array_equal(e2, eps)


def test_fit_row_capacity_refusal(L):
    rng = np.random.default_rng(21)
    launches = L.launch_count()
    X, Y = _data(rng, DF_MAX_ROWS + 1, 2, 1)
    with pytest.raises(L.DmoError, match="n_sites \\* batch_max <= 65536"):
        L.DGPFitState(X, Y, 1, 8, 8, 1, True, DF_MAX_ROWS + 1)
    with pytest.raises(L.DmoError, match="n_sites \\* batch_max <= 65536"):
        L.DGPFitState(X[:4097], Y[:4097], 1, 8, 8, 16, True, 4097)
    assert L.launch_count() == launches


@pytest.mark.parametrize("quadrature", [True, False], ids=["mdspp", "mdgp"])
def test_epoch_with_a_one_row_last_batch(L, quadrature):
    N, B = 513, 512
    J = 3 if quadrature else 2
    rng = np.random.default_rng(22)
    X, Y = _data(rng, N, 3, 2)
    raw = _raw(rng, X, 2, 2, 12, 10, quadrature, None)
    if not quadrature:
        raw.pop("quad_sites", None)
    a = _state(L, X, Y, raw, quadrature, J, B, None)
    b = _state(L, X, Y, raw, quadrature, J, B, None)
    perm = rng.permutation(N)
    la = a.epoch(perm, B, 0.05, seed=6, step0=11)
    lb = []
    for k, b0 in enumerate(range(0, N, B)):
        lb.append(b.loss_grad(perm[b0 : b0 + B], seed=6, step=11 + k, grad=False)[0])
        b.adam_step(0.05)
    assert la.shape == (2,) and np.array_equal(la, np.asarray(lb))
    assert np.array_equal(a.get_params(), b.get_params())


def test_fit_draws_replay(L):
    N, d, H, T, Z1, Z2, J, B = 80, 4, 8, 1, 12, 10, 16, 33
    rng = np.random.default_rng(23)
    X, Y = _data(rng, N, d, T)
    raw = _raw(rng, X, T, H, Z1, Z2, False, None)
    raw.pop("quad_sites", None)
    st = _state(L, X, Y, raw, False, J, B, None)
    seed, step = 0x123456789ABC, (1 << 40) + 3
    batch = rng.choice(N, B, replace=False)
    loss, g, eps = st.loss_grad(batch, seed=seed, step=step, return_eps=True)
    j, i, h = np.meshgrid(np.arange(J), np.arange(B), np.arange(H), indexing="ij")
    ctr_hi = (i.astype(np.uint64) << np.uint64(32)) | (j * H + h).astype(np.uint64)
    ref, bound = box_muller(seed, np.full(ctr_hi.shape, step, np.uint64), ctr_hi)
    _within(eps, ref, bound)
    lo, go = ot.loss_grad(raw, X[batch], Y[batch], N, eps=eps)
    assert abs(loss - lo) <= 1e-10 * abs(lo), (loss, lo)
    _check_grad(g, go, raw)
