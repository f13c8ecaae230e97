"""The GP predicts across their candidate chunks and at their launch-grid limits.

Every GP predict splits its candidates into chunks (a memory budget for the K_* planes, capped at GP_MAX_CHUNK = 2^20
rows so that no producer grid exceeds the 65535 limit of its y extent) and walks them on the host.  Each model below
runs at a size where it takes more than one chunk on every path it has, and each test checks

  1. that every row is written and sane: the outputs are device buffers pre-filled with NaN, so a row that no chunk
     writes stays NaN; all rows are finite and 0 <= var <= prior;
  2. that no row depends on the chunk it fell into: 512-row windows (the first rows, both sides of every seam of the
     path, the ragged tail), each predicted on its own, against the same rows of the big call;
  3. the windows against the CPU oracle at the bars of the existing parity tests;
  4. (exact GP) the chunked mean against the mean-only predict, an independent code path, on every row.

Windows start at multiples of 256, so a row keeps its position within its 128- and 256-candidate tiles when its window is
predicted alone.  Every window holds training (or inducing) points displaced by 1e-4 .. 1e-2: posterior variances near
zero, where a row read from the wrong K_* is furthest off.  A launch-count guard proves that each big call ran more
than one chunk.

Which rows must agree bit for bit in check 2 (from the kernels' summation orders):
  * exact GP, float64 mean: bitwise.  mean_kernel reduces one row's own K_* values in one warp, whatever the chunk.
  * exact GP, float64 variance: 1e-12 of the prior.  var_kernel splits L^-1's row blocks over nsplit CTAs, and nsplit
    follows Pc_alloc; var_finish_kernel adds those partial sums.
  * exact GP, tensor variance: bitwise.  The K_* hi / lo bits are per element.  The n_q work items of a 128-row block own
    fixed row blocks of L^-1, and var_finish_tc_kernel adds the n_q planes in a fixed order.
  * exact GP, tensor mean: the fused producer (kstar_mean_kernel) takes its training-set slices from pick_slices(Pcpad /
    256, ...), so 1e-12 of max(|mean|, y_std); the two-kernel route's mean_split_kernel reduces one row in one warp: bitwise.
  * exact GP, AUTO: the rows it recomputes in float64 go through a float64 predict whose nsplit follows their count,
    so 1e-12 as for the float64 path.
  * MEGP and variational means: bitwise (n_mp = Npad / producer span partial sums, fixed).  Their tensor variance:
    bitwise (n_q fixed).  Their float64 variance: 1e-12 of the prior (n_vp follows Pc_alloc).
"""

import functools

import numpy as np
import pytest

from oracle import gp, megp
from oracle import variational as V
from test_gpu_parity import _assert_gp_bars

pytestmark = pytest.mark.gpu

MAX_CHUNK = 1 << 20  # gp.cuh: GP_MAX_CHUNK
WIN = 512


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


# ------------------------------------------------------------------------------------------ chunk budgets
def _npad(n):
    return -(-n // 256) * 256  # GpVarOps::alloc (gp.cu:416)


def exact_fp64_chunk(G, N):
    """gp.cu:439-443 (gp_predict_fp64): Ks (G x Pc x Npad float64) within 8 GiB, at most GP_MAX_CHUNK, multiple of 128."""
    pc = min((8 << 30) // (G * _npad(N) * 8), MAX_CHUNK)
    return max(pc // 128 * 128, 128)


def exact_tensor_chunk(G, N):
    """gp_tensor.cu:1061-1064 (gp_predict_tensor): K_* hi + lo (G x Pc x Npad x 4 bytes) within 6 GiB, at most GP_MAX_CHUNK,
    multiple of 256."""
    pc = min((6 << 30) // (G * _npad(N) * 4), MAX_CHUNK)
    return max(pc // 256 * 256, 256)


def unit_chunk(N, tensor):
    """gp_multitask.cu:333-336 (GpUnitPredict::alloc, MEGP and variational): one K_* plane within 6 GiB, at most
    GP_MAX_CHUNK, multiple of 128."""
    pc = min((6 << 30) // (_npad(N) * (4 if tensor else 8)), MAX_CHUNK)
    return max(pc // 128 * 128, 128)


def mean_only_chunk():
    """gp_tensor.cu:952-953 (gp_mean_direct)."""
    return MAX_CHUNK


def _n_chunks(P, chunk):
    return -(-P // chunk)


# ------------------------------------------------------------------------------------------ windows and candidates
def _windows(P, chunks):
    """Row ranges [w0, w1): the first rows, rows on both sides of every seam of every chunk size in `chunks`, the ragged
    tail.  Starts are multiples of 256; overlapping windows are merged."""
    starts = {0, max(0, -(-(P - WIN) // 256) * 256)}
    for c in chunks:
        starts.update((s - WIN // 2) // 256 * 256 for s in range(c, P, c))
    out = []
    for w0 in sorted(starts):
        w1 = min(w0 + WIN, P)
        if out and w0 <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], w1))
        else:
            out.append((w0, w1))
    return out


def _rows(windows):
    return np.concatenate([np.arange(w0, w1) for w0, w1 in windows])


def _plant(rng, X, windows, anchors, per_window=24):
    """Points of `anchors` displaced by 1e-4 .. 1e-2 (log-uniform) at random rows of every window (inputs in the unit cube)."""
    d = X.shape[1]
    for w0, w1 in windows:
        at = w0 + rng.choice(w1 - w0, per_window, replace=False)
        scale = 10.0 ** rng.uniform(-4.0, -2.0, size=(per_window, 1))
        X[at] = np.clip(anchors[rng.integers(0, len(anchors), per_window)] + scale * rng.uniform(-1, 1, size=(per_window, d)), 0, 1)


# ------------------------------------------------------------------------------------------ predict into NaN
def _predict(L, fn, h, M, X, precision, want_var=True):
    """dmo_<model>_predict writing straight into device buffers pre-filled with NaN: a row that no chunk writes stays
    NaN.  Returns (mean, var, kernel launches of the call)."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    P = X.shape[0]
    nan = np.full((P, M), np.nan)
    dm = L.DeviceArray((P, M)).upload(nan)
    dv = L.DeviceArray((P, M)).upload(nan) if want_var else None
    n0 = L.launch_count()
    L._check(getattr(L.load_library(), fn)(L.context(), h._h, L._ptr(X), P, dm.ptr, dv.ptr if dv else None, int(precision)), fn)
    launches = L.launch_count() - n0
    mean, var = dm.download(), dv.download() if dv else None
    dm.free()
    if dv:
        dv.free()
    return mean, var, launches


def _assert_chunked(what, launches_big, launches_one, chunks):
    """The big call repeated its per-chunk launches chunks - 1 more times than a one-chunk call of the same model (made
    after the model's one-off preparation, so that both calls carry the same fixed launches)."""
    extra = launches_big - launches_one
    print(f"{what}: {chunks} chunks, {launches_big} launches against {launches_one} for one chunk")
    assert chunks > 1 and extra > 0 and extra % (chunks - 1) == 0, (what, launches_big, launches_one, chunks)


def _assert_sane(what, mean, var, prior, slack=1e-9):
    assert np.isfinite(mean).all(), (what, np.argwhere(~np.isfinite(mean))[:5])
    if var is not None:
        assert np.isfinite(var).all(), (what, np.argwhere(~np.isfinite(var))[:5])
        assert (var >= 0).all(), (what, var.min())
        assert (var <= prior * (1 + slack)).all(), (what, np.max(var / prior))


def _assert_windows_alone(what, out_big, outs_alone, windows, scale, tol):
    """The windows' rows of the big call against each window predicted alone: bitwise (tol None) or within tol * scale."""
    for (w0, w1), alone in zip(windows, outs_alone):
        big = out_big[w0:w1]
        if tol is None:
            assert np.array_equal(big, alone), (what, w0, np.argwhere(big != alone)[:5] + [w0, 0])
        else:
            err = np.max(np.abs(big - alone) / scale)
            assert err <= tol, (what, w0, err)


def _run_windows(L, fn, h, M, X, windows, precision, want_var=True):
    """Each window predicted on its own: [(mean, var)], and the launches of the last (a one-chunk call after the model's
    one-off preparation, which the first call of a path makes)."""
    outs = []
    for w0, w1 in windows:
        m, v, n = _predict(L, fn, h, M, X[w0:w1], precision, want_var)
        outs.append((m, v))
    return outs, n


# ------------------------------------------------------------------------------------------ exact GP
EXACT = {  # N, d, M, per-dimension length scales, objectives sharing their covariance in pairs
    "isotropic_G6": (2048, 24, 6, False, False),
    "per_dimension_G6": (2048, 40, 6, True, False),
    "grouped_G3": (2048, 24, 6, False, True),
}


@functools.lru_cache(maxsize=None)
def _exact_case(name):
    N, d, M, ard, paired = EXACT[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, :4].sum(axis=1) + k) + Xtr[:, 4 + k] ** 2 for k in range(M)])
    theta = [m // 2 if paired else m for m in range(M)]  # objective m takes the hyper-parameters theta[m]
    # length scales no longer than the benchmarked model's (0.5 at d = 30): AUTO's calibration admits the tensor path
    ls_t = [(0.6 + 0.4 * rng.random(d)) if ard else 0.4 + 0.02 * t for t in range(M)]
    const = [1.0 + 0.2 * theta[m] for m in range(M)]
    noise = np.array([1e-6 * (1 + theta[m]) for m in range(M)])
    st = gp.fit_fixed(Xtr, Ytr, xlb, xub, const, [ls_t[theta[m]] for m in range(M)], noise)
    for m in range(M):  # objectives with the same hyper-parameters share one factor plane, bit for bit
        st.objectives[m].L = st.objectives[theta.index(theta[m])].L
    h = _gp_handle(st, d)
    G = len(set(theta))
    chunks = (exact_fp64_chunk(G, N), exact_tensor_chunk(G, N))
    P = max(chunks) + 1000  # a full chunk of either path plus a ragged tail (1000 = 7 x 128 + 104)
    X = rng.random((P, d))
    windows = _windows(P, chunks)
    _plant(rng, X, windows, Xtr)
    rows = _rows(windows)
    mean_o, var_o = gp.predict(st, X[rows])
    ystd = np.array([o.y_std for o in st.objectives])
    prior = np.array([(o.constant + o.noise) * o.y_std * o.y_std for o in st.objectives])
    return st, h, G, chunks, X, windows, rows, mean_o, var_o, ystd, prior


def _gp_handle(st, d):
    from dmosopt_b200 import _lib

    return _lib.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]),
                         [o.constant for o in st.objectives], [np.broadcast_to(np.asarray(o.length_scale, dtype=np.float64), (d,)) for o in st.objectives],
                         [o.noise for o in st.objectives], [o.y_mean for o in st.objectives], [o.y_std for o in st.objectives], st.xlb, st.xub)


def _exact_path(L, name, precision, label, chunk):
    """Checks 1 -- 3 on one path of an exact GP; returns the big call's (mean, var)."""
    st, h, G, chunks, X, windows, rows, mean_o, var_o, ystd, prior = _exact_case(name)
    M = len(st.objectives)
    alone, n_one = _run_windows(L, "dmo_gp_predict", h, M, X, windows, precision)
    mean, var, n_big = _predict(L, "dmo_gp_predict", h, M, X, precision)
    what = f"{name} {label}"
    if chunk:
        _assert_chunked(what, n_big, n_one, _n_chunks(len(X), chunk))
    _assert_sane(what, mean, var, prior)
    if precision == L.GP_FP64:
        mean_rule, var_rule = None, 1e-12
    elif precision == L.GP_TENSOR:
        fused = label == "tensor"
        mean_rule, var_rule = (1e-12 if fused else None), None
    else:
        mean_rule, var_rule = 1e-12, 1e-12
    _assert_windows_alone(what + " mean", mean, [m for m, _ in alone], windows, np.maximum(np.abs(mean_o).max(axis=0), ystd), mean_rule)
    _assert_windows_alone(what + " var", var, [v for _, v in alone], windows, prior, var_rule)
    em = np.max(np.abs(mean[rows] - mean_o) / np.maximum(np.abs(mean_o), ystd))
    ev = np.max(np.abs(var[rows] - var_o) / prior)
    print(f"{what}: windows {len(rows)} rows, mean rel err {em:.2e}, var err/prior {ev:.2e}")
    if precision == L.GP_FP64:
        assert em < 1e-8 and ev < 1e-8, (what, em, ev)
    elif precision == L.GP_TENSOR:
        assert em < 1e-5 and ev < 1e-5, (what, em, ev)
    else:
        _assert_gp_bars(mean[rows], var[rows], mean_o, var_o, ystd, prior, what)
    return mean, var


def _assert_mean_matches_mean_only(L, name, means):
    """Check 4: the chunked means against the mean-only predict on every row."""
    st, h, G, chunks, X, windows, rows, mean_o, var_o, ystd, prior = _exact_case(name)
    mean_only, none, _ = _predict(L, "dmo_gp_predict", h, len(st.objectives), X, L.GP_TENSOR, want_var=False)
    assert none is None
    _assert_sane(f"{name} mean-only", mean_only, None, prior)
    for label, mean in means.items():
        err = np.max(np.abs(mean - mean_only) / np.maximum(np.abs(mean_only), ystd))
        print(f"{name} {label}: chunked mean against the mean-only predict on all {len(X)} rows: {err:.2e}")
        assert err < 1e-5, (name, label, err)


def test_exact_gp_isotropic_six_covariances_across_chunks(L, monkeypatch):
    """G = 6 (distinct constants and length scales), d = 24: the fused K_* + mean producer with MT = 6, not grouped.
    float64, tensor (fused and two-kernel) and AUTO, which must admit the tensor path and refine rows past its first chunk."""
    name = "isotropic_G6"
    st, h, G, (c64, ctc), X, windows, rows, mean_o, var_o, ystd, prior = _exact_case(name)
    assert h.covariance_groups()[0] == 6
    m64, _ = _exact_path(L, name, L.GP_FP64, "fp64", c64)
    monkeypatch.setenv("DMO_GP_FUSED", "1")
    mt, vt = _exact_path(L, name, L.GP_TENSOR, "tensor", ctc)
    monkeypatch.setenv("DMO_GP_FUSED", "0")
    ms, vs = _exact_path(L, name, L.GP_TENSOR, "tensor two-kernel", ctc)
    monkeypatch.delenv("DMO_GP_FUSED")
    assert np.array_equal(vt, vs)  # the two producers write the same K_* bits
    assert np.max(np.abs(mt - ms) / np.maximum(np.abs(ms), ystd)) < 1e-5
    ma, va = _exact_path(L, name, L.GP_AUTO, "auto", None)
    info = h.auto_info()
    print("auto:", info)
    assert info["mean_tensor"] and info["var_tensor"], info
    # AUTO recomputes in float64 the rows whose tensor variance is below theta * prior (flag_small_var_kernel, same
    # arithmetic); the tensor variance does not depend on the chunking, so the flagged rows are known exactly
    c = np.array([o.constant for o in st.objectives])
    nz = np.array([o.noise for o in st.objectives])
    small = ~np.all(vt >= info["theta"] * ((c + nz) * ystd * ystd), axis=1)
    print(f"auto refined {info['last_refined']} rows, {int(small[ctc:].sum())} of them past the first tensor chunk")
    assert info["last_refined"] == int(small.sum()) > 0, (info["last_refined"], int(small.sum()))
    assert small[ctc:].any()
    assert np.array_equal(va[~small], vt[~small]) and np.array_equal(ma[~small], mt[~small])
    _assert_mean_matches_mean_only(L, name, {"fp64": m64, "tensor": mt, "tensor two-kernel": ms, "auto": ma})


def test_exact_gp_per_dimension_length_scales_across_chunks(L):
    """G = 6 with per-dimension length scales, d = 40: kstar_kernel<false> and the DMAX = 64 two-kernel tensor route."""
    name = "per_dimension_G6"
    st, h, G, (c64, ctc), *_ = _exact_case(name)
    assert h.covariance_groups()[0] == 6
    m64, _ = _exact_path(L, name, L.GP_FP64, "fp64", c64)
    mt, _ = _exact_path(L, name, L.GP_TENSOR, "tensor two-kernel", ctc)
    _assert_mean_matches_mean_only(L, name, {"fp64": m64, "tensor": mt})


def test_exact_gp_grouped_covariances_across_chunks(L):
    """Six objectives sharing their covariance in pairs (G = 3): the grouped fused producer, chunks twice as long."""
    name = "grouped_G3"
    st, h, G, (c64, ctc), *_ = _exact_case(name)
    assert h.covariance_groups() == (3, [0, 0, 1, 1, 2, 2])
    m64, _ = _exact_path(L, name, L.GP_FP64, "fp64", c64)
    mt, _ = _exact_path(L, name, L.GP_TENSOR, "tensor", ctc)
    _assert_mean_matches_mean_only(L, name, {"fp64": m64, "tensor": mt})


# ------------------------------------------------------------------------------------------ MEGP
@functools.lru_cache(maxsize=None)
def _megp_case():
    N, d, M = 1000, 12, 3
    rng = np.random.default_rng(1000)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] + 0.1 * t * X[:, -1] ** 2 for t in range(M)])
    # shorter length scales and more noise than test_gpu_megp.py's model: twice the training points there, and rows
    # planted 1e-4 from them, would otherwise put the tensor variance at its 1e-5 bar
    ls = 0.4 + 0.4 * rng.random(d)
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + 0.5 * rng.random(M))
    D = np.geomspace(1e-3, 8e-3, M) + 1e-2
    w, b = 0.2 * rng.standard_normal((M, d)), 0.1 * rng.standard_normal(M)
    xlb, xub = np.zeros(d), np.ones(d)
    st = megp.fit_fixed(X, Y, xlb, xub, ls, B, D, w, b)
    yn, ym, ys = megp.normalise_y(Y)
    P = MAX_CHUNK + 300
    Xc = rng.random((P, d))
    windows = _windows(P, (unit_chunk(N, False), unit_chunk(N, True)))
    _plant(rng, Xc, windows, X)
    rows = _rows(windows)
    mean_o, var_o = megp.predict(st, Xc[rows])
    return N, M, (X, yn, ls, B, D, w, b, ym, ys, xlb, xub), Xc, windows, rows, mean_o, var_o, (np.diag(B) + D) * ys**2


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
def test_megp_across_chunks(L, precision):
    """N = 1000 (Npad 1024), d = 12, M = 3, P = 2^20 + 300: float64 chunks of 786432 rows, tensor chunks at the 2^20 cap."""
    N, M, args, Xc, windows, rows, mean_o, var_o, prior = _megp_case()
    tensor = precision == "tensor"
    prec = L.GP_TENSOR if tensor else L.GP_FP64
    h = L.MTGPHandle(*args)
    alone, n_one = _run_windows(L, "dmo_mtgp_predict", h, M, Xc, windows, prec)
    mean, var, n_big = _predict(L, "dmo_mtgp_predict", h, M, Xc, prec)
    h.close()
    what = f"MEGP {precision}"
    _assert_chunked(what, n_big, n_one, _n_chunks(len(Xc), unit_chunk(N, tensor)))
    _assert_sane(what, mean, var, prior)
    scale = np.abs(mean_o).max(axis=0).astype(np.float64)
    _assert_windows_alone(what + " mean", mean, [m for m, _ in alone], windows, scale, None)
    _assert_windows_alone(what + " var", var, [v for _, v in alone], windows, prior, None if tensor else 1e-12)
    tol = 1e-5 if tensor else 2e-6  # test_gpu_megp.py (the oracle returns float32)
    em = np.abs(mean[rows] - mean_o).max(axis=0) / scale
    ev = np.abs(var[rows] - var_o).max(axis=0) / prior
    print(f"{what}: windows {len(rows)} rows, mean err/scale {em.max():.2e}, var err/prior {ev.max():.2e}")
    assert np.all(em <= tol) and np.all(ev <= tol), (what, em, ev)


# ------------------------------------------------------------------------------------------ variational
@functools.lru_cache(maxsize=None)
def _svgp_case(kind):
    Lat, Zn, d = 3, 819, 8
    rng = np.random.default_rng(819 + len(kind))
    Z = rng.random((Lat, Zn, d))
    ls = np.sqrt(d) * (0.4 + 0.6 * rng.random((Lat, d)))
    s = 0.5 + rng.random(Lat)
    q_mu = rng.standard_normal((Lat, Zn))
    # S = q_sqrt q_sqrt' <= I, so that the variance s - ||O0 k||^2 + ||O1 k||^2 stays within [0, s]
    q_sqrt = np.tril(0.05 / np.sqrt(Zn) * rng.standard_normal((Lat, Zn, Zn)), -1)
    for l in range(Lat):
        q_sqrt[l][np.diag_indices(Zn)] = 0.2 + 0.4 * rng.random(Zn)
        assert np.linalg.norm(q_sqrt[l], 2) < 1.0
    W = rng.standard_normal((3, Lat)) if kind == "crv" else None
    Wm = np.eye(Lat) if W is None else W
    M = Wm.shape[0]
    ym, ys = rng.standard_normal(M), 0.5 + rng.random(M)
    P = MAX_CHUNK + 300
    Xc = rng.random((P, d))
    windows = _windows(P, (unit_chunk(Zn, False), unit_chunk(Zn, True)))
    _plant(rng, Xc, windows, Z.reshape(-1, d))
    rows = _rows(windows)
    g = [V.latent_predict(Xc[rows], Z[l], s[l], ls[l], q_mu[l], q_sqrt[l]) for l in range(Lat)]
    mean_o = ys * (np.stack([m for m, _ in g], axis=1) @ Wm.T) + ym
    var_o = (np.stack([v for _, v in g], axis=1) @ (Wm * Wm).T) * ys**2
    prior = ((Wm * Wm) @ s) * ys**2
    args = (Z, s, ls, q_mu, q_sqrt, ym, ys, np.zeros(d), np.ones(d))
    return Zn, M, args, W, Xc, windows, rows, mean_o, var_o, ys, prior


@pytest.mark.parametrize("precision", ["fp64", "tensor"])
@pytest.mark.parametrize("kind", ["svgp", "crv"])
def test_variational_across_chunks(L, kind, precision):
    """Z = 819 (Npad 1024), three latents with their own inducing points and length scales (three K_* groups, each
    with its own chunk loop), identity or CRV mixing W, P = 2^20 + 300."""
    Zn, M, args, W, Xc, windows, rows, mean_o, var_o, ys, prior = _svgp_case(kind)
    tensor = precision == "tensor"
    prec = L.GP_TENSOR if tensor else L.GP_FP64
    h = L.SVGPHandle(*args, W=W)
    assert h.groups()[0] == 3
    alone, n_one = _run_windows(L, "dmo_svgp_predict", h, M, Xc, windows, prec)
    mean, var, n_big = _predict(L, "dmo_svgp_predict", h, M, Xc, prec)
    h.close()
    what = f"{kind} {precision}"
    _assert_chunked(what, n_big, n_one, _n_chunks(len(Xc), unit_chunk(Zn, tensor)))
    # test_gpu_variational.py's bars: mean 2e-6 of max(|mean|, y_std); variance 1e-9 of the prior (float64), 1e-4 of
    # max(|var|, prior) (tensor).  s - v0 + v1 is not a prior minus a sum of squares, so its upper bound carries that bar.
    tol_v = 1e-4 if tensor else 1e-9
    _assert_sane(what, mean, var, prior, slack=tol_v)
    scale = np.maximum(np.abs(mean_o).max(axis=0), ys)
    _assert_windows_alone(what + " mean", mean, [m for m, _ in alone], windows, scale, None)
    _assert_windows_alone(what + " var", var, [v for _, v in alone], windows, prior, None if tensor else 1e-12)
    em = np.abs(mean[rows] - mean_o).max(axis=0) / scale
    vscale = np.maximum(np.abs(var_o).max(axis=0), prior) if tensor else prior
    ev = np.abs(var[rows] - var_o).max(axis=0) / vscale
    print(f"{what}: windows {len(rows)} rows, mean err/scale {em.max():.2e}, var err {ev.max():.2e}")
    assert np.all(em <= 2e-6) and np.all(ev <= tol_v), (what, em, ev)


# ------------------------------------------------------------------------------------------ launch-grid limits
def _small_case(P):
    """N = 200 (Npad 256), d = 2, M = 1: the budgets alone would allow chunks of millions of rows."""
    N, d = 200, 2
    rng = np.random.default_rng(P)
    Xtr = rng.random((N, d))
    Ytr = np.sin(3 * Xtr.sum(axis=1))[:, None] + Xtr[:, :1] ** 2
    st = gp.fit_fixed(Xtr, Ytr, np.zeros(d), np.ones(d), 1.0, 0.2, 1e-2)  # 200 points in the unit square: noise keeps alpha small
    X = rng.random((P, d))
    return st, Xtr, X, _gp_handle(st, d)


@pytest.mark.parametrize("route", ["fp64", "tensor two-kernel"])
def test_exact_gp_past_the_launch_grid_limit(L, monkeypatch, route):
    """P = 2 100 000 at N = 200: without the GP_MAX_CHUNK cap, one chunk would put 65628 (kstar_kernel) or 65632
    (kstar_tensor_kernel) blocks on the K_* grid's y extent, past its limit of 65535.  That launch failed without the
    predict reporting it: the call returned success after one chunk, its rows computed from a K_* nobody wrote."""
    P = 2_100_000
    st, Xtr, X, h = _small_case(P)
    tensor = route != "fp64"
    chunk = exact_tensor_chunk(1, 200) if tensor else exact_fp64_chunk(1, 200)
    assert chunk == MAX_CHUNK
    windows = _windows(P, (chunk,))
    X = X.copy()
    _plant(np.random.default_rng(1), X, windows, Xtr)
    rows = _rows(windows)
    mean_o, var_o = gp.predict(st, X[rows])
    ystd = np.array([st.objectives[0].y_std])
    prior = np.array([(st.objectives[0].constant + st.objectives[0].noise) * ystd[0] * ystd[0]])
    prec = L.GP_TENSOR if tensor else L.GP_FP64
    if tensor:
        monkeypatch.setenv("DMO_GP_FUSED", "0")
    alone, n_one = _run_windows(L, "dmo_gp_predict", h, 1, X, windows, prec)
    mean, var, n_big = _predict(L, "dmo_gp_predict", h, 1, X, prec)
    monkeypatch.delenv("DMO_GP_FUSED", raising=False)
    _assert_chunked(route, n_big, n_one, _n_chunks(P, chunk))
    _assert_sane(route, mean, var, prior)
    _assert_windows_alone(route + " mean", mean, [m for m, _ in alone], windows, None, None)
    _assert_windows_alone(route + " var", var, [v for _, v in alone], windows, prior, None if tensor else 1e-12)
    em = np.max(np.abs(mean[rows] - mean_o) / np.maximum(np.abs(mean_o), ystd))
    ev = np.max(np.abs(var[rows] - var_o) / prior)
    print(f"{route} P={P}: mean rel err {em:.2e}, var err/prior {ev:.2e}")
    bar = 1e-5 if tensor else 1e-8
    assert em < bar and ev < bar, (route, em, ev)
    mean_only, _, _ = _predict(L, "dmo_gp_predict", h, 1, X, L.GP_TENSOR, want_var=False)
    assert np.max(np.abs(mean - mean_only) / np.maximum(np.abs(mean_only), ystd)) < 1e-5


def test_mean_only_predict_past_the_launch_grid_limit(L):
    """P = 2^24 + 1 at N = 200, d = 2, M = 1: gp_mean_direct puts ceil(P / 256) = 65537 candidate blocks on its grid's y
    extent unless it walks the candidates in chunks; the float64 mean-only predict needs its chunk cap as well."""
    P = (1 << 24) + 1
    st, Xtr, X, h = _small_case(P)
    windows = _windows(P, (mean_only_chunk(),))
    _plant(np.random.default_rng(2), X, windows, Xtr)
    rows = _rows(windows)
    mean_o, _ = gp.predict(st, X[rows])
    ystd = np.array([st.objectives[0].y_std])
    prior = np.array([(st.objectives[0].constant + st.objectives[0].noise) * ystd[0] * ystd[0]])
    means = {}
    for label, prec, chunk in (("mean-only tensor", L.GP_TENSOR, mean_only_chunk()), ("mean-only fp64", L.GP_FP64, exact_fp64_chunk(1, 200))):
        alone, n_one = _run_windows(L, "dmo_gp_predict", h, 1, X, windows, prec, want_var=False)
        mean, _, n_big = _predict(L, "dmo_gp_predict", h, 1, X, prec, want_var=False)
        _assert_chunked(label, n_big, n_one, _n_chunks(P, chunk))
        _assert_sane(label, mean, None, prior)
        # the float64 mean is bitwise; the direct kernel's slices follow pick_slices(chunk blocks, ...)
        _assert_windows_alone(label, mean, [m for m, _ in alone], windows, np.maximum(np.abs(mean_o).max(), ystd),
                              1e-12 if prec == L.GP_TENSOR else None)
        em = np.max(np.abs(mean[rows] - mean_o) / np.maximum(np.abs(mean_o), ystd))
        print(f"{label} P={P}: windows {len(rows)} rows, mean rel err {em:.2e}")
        assert em < (1e-5 if prec == L.GP_TENSOR else 1e-8), (label, em)
        means[label] = mean
    err = np.max(np.abs(means["mean-only tensor"] - means["mean-only fp64"]) / np.maximum(np.abs(means["mean-only fp64"]), ystd))
    print(f"mean-only tensor against float64 on all {P} rows: {err:.2e}")
    assert err < 1e-5, err
