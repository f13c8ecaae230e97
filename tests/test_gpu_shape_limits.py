"""Every GP entry point at the edges of its shape envelope and on both sides of its kernel-dispatch thresholds.

Each case compares the GPU result with the CPU oracle of the same operation (oracle/gp.py, megp.py, variational.py for
the predicts; egp_train.py, megp_train.py, variational_train.py and the closed-form fit_grad_dense.py for the
gradients), at the bars the existing files use for the same path:
  * exact-GP float64 predict 1e-8; forced tensor predict 1e-5 of max(|mean|, y_std) and of the prior, AUTO
    _assert_gp_bars (test_gpu_parity.py, test_gpu_predict_chunks.py).  The forced tensor variance is not held to
    _assert_gp_bars' 1e-5 of its own value for variances just above 1e-3 of the prior: on these cases with length
    scales 0.15 sqrt(d) (here 0.1 sqrt(d)) and nuggets 1e-6 it measured 2.6e-4 .. 2.3e-3 of the value there, absolute
    errors of at most 2.5e-6 of the prior, and 5.7e-5 at N 2.  That bar is what AUTO's float64 refinement of
    small-variance rows is for, and AUTO meets it in every case;
  * MEGP 2e-6 (float64; the oracle returns float32) and 1e-5 (tensor) of max |mean| and of the prior (test_gpu_megp.py);
  * variational mean 2e-6 of max(|mean|, y_std), variance 1e-9 of the prior (float64) or 1e-4 of max(|var|, prior)
    (tensor) (test_gpu_variational.py);
  * log marginal likelihoods 1e-10 relative; gradients and natural-gradient steps 1e-8 of max |ref|; ELBO pieces 1e-10.
Candidate sets hold displaced training (inducing) points, as _candidates_with_near_training_rows makes them, so that
posterior variances near zero are exercised.  Where a path has a twin, the twins are compared as well: tensor against
float64, and the two-kernel tensor route (DMO_GP_FUSED=0) against the fused one (the same K_* bits, so the same
variance bit for bit).  Which route a case takes follows from the thresholds in the code.

What each case straddles (file:line of the threshold or limit it guards):

Exact GP (gp.cu, gp_tensor.cu), float64 + tensor (fused and two-kernel) + AUTO + mean-only (tensor and float64):
  * d in {1, 16, 17, 32, 33, 64}, isotropic, M = 3:
      - gp_tensor.cu:964 mean-direct NJ = 4 (d <= 16) against NJ = 8: d 16 / 17;
      - gp_tensor.cu:1056 mean-direct and :1078 fused K_* + mean, d <= KM_D = 32: d 32 / 33;
      - gp_tensor.cu:1134-1149 two-kernel K_* producer DMAX 32 (d <= 32) against 64: d 32 / 33;
      - gp.cu:663 d <= KS_DMAX = 64 (gp_create) and kstar_kernel's register-held coordinates: d 64; d 1 the smallest.
  * per-dimension length scales at d in {32, 33, 64} with G = 2 and G = 3 of M = 3: gp_tensor.cu:1078 admits the fused
    producer for per-dimension length scales only when G <= 2 and d <= 32, so d 32 takes the fused route at G 2 and the
    two-kernel route at G 3; d 33 and 64 take the two-kernel route at both, with DMAX 64 (:1146).
  * M in {6, 7, 8, 16}, G = M: the fused / mean-direct gate M <= 6 (gp_tensor.cu:1056, :1078) and the MT template
    switches (:972-979, :1112-1119); M 16 = GP_MAX_M (gp.cu:357, :663).
  * M = 16 with 6 covariances shared in an irregular pattern over objectives 1 - 16, two of them first appearing at
    objectives 9 and 12 with the constant and length scales of group 0 but their own noises (so their own factors):
    covariance_groups() must equal the expected grouping, which needs factor_diff_kernel (gp.cu:358-376) to compare all
    16 planes with each other.
  * M = 7 with G = 4 < M: past the fused gate, the grouped (G < M) layout of K_* planes on the two-kernel route.
  * N in {1, 2, 255, 256, 257}: Npad steps of 256 (GpVarOps::alloc, gp.cu) and a model with one training point.
  * P in {1, 127, 129}: one candidate, ragged 128-candidate tiles.

MEGP (gp_multitask.cu), M = 8 = MT_MAX (gp.cuh:137, the MT_MAX-wide loops of mt_mix_kernel, gp_multitask.cu:212-251):
  * d in {33, 64} on both precisions: mt_kstar_tensor_kernel DMAX 32 against 64 (gp_multitask.cu:309);
  * d in {65, 90} on float64: past the tensor limit (gp_multitask.cu:326), up to MT_FIT_DMAX = 90 (gp.cuh:138);
  * N in {1, 63, 64, 65} on both precisions: the 64-row Cholesky blocks of the fit;
  * dmo_mtgp_lml_grad at M 8, d 90, N in {63, 64, 65} (gp_multitask.cu:375).

EGP / exact fit (gp_multitask_fit.cu, gp_fit.cu):
  * dmo_gp_lml_grad at M = 8 (one lockstep call, gp_multitask_fit.cu:414) with d = 90, N in {1, 63, 64, 65};
  * dmo_gp_fit at d = 90 (gp_fit.cu:347; kernel_matrix_kernel's dynamic shared memory is then 46 592 B, under the 48 KB
    default) at N in {63, 127} (the augmented target row is the last row of the padded factor, with no identity tail)
    and N = 64.

Variational (gp_variational.cu, gp_variational_fit.cu):
  * create / predict at L = M = 8 = SV_MAX (gp_variational.cu:263) for CRV (a dense W) and SPV, and at d = 90
    (gp_variational.cu:264) on float64;
  * Z in {1, 64, 65, 257}: Npad steps and the smallest model;
  * dmo_svgp_optimal_q at Z = 1 and Z = 1100 (gp_linv_from_factor_batched then runs with Np = 2048, gp.cu:382);
  * SVGPFitState natgrad + elbo_grad at L = M = 8 = SVF_MAX with a CRV W; at d = 90, where svf_fold_kernel (one block of
    128 threads over d + 1 outputs, gp_variational_fit.cu:663) and svf_grad_pass_kernel (:221, one coordinate per
    thread) cover every length scale; at B = 1; at Z in {1, 64, 65}; VGP at N = Z = 65.

Training sizes (one case each): dmo_gp_lml_grad at N 2048, d 30, M 3 (32 x 32 tile rows of the gradient kernels, the
Np = 2048 batched L^-1) and dmo_mtgp_lml_grad at N 2048, d 30, M 2 against the closed form (oracle/fit_grad_dense.py,
itself checked against the autograd oracles in test_shape_limits_cpu.py); elbo_grad + natgrad at Z 1100, B 256, L 3.

Refusals: the first shape past each limit fails with its DmoError message and the refused call counts no launch:
d 65 for dmo_gp_create (gp.cu:663); d 65 with tensor precision for MEGP and variational predicts (gp_multitask.cu:326);
d 91 for every fit (MT_FIT_DMAX); M 17 (gp.cu:663); M 9 for MEGP and dmo_gp_lml_grad (MT_MAX); L 9 and Z 8193 for the
variational entry points (SV_MAX / SV_ZMAX, SVF_MAX / SVF_ZMAX).  The Python classes refuse a shape their predict
cannot take before any training (test_python_classes_refuse_before_training_without_a_launch, and without a GPU
test_shape_limits_cpu.py).
"""

import functools

import numpy as np
import pytest

from oracle import egp_train, fit_grad_dense, gp, megp, megp_train
from oracle import variational as V
from test_gpu_parity import _assert_gp_bars, _candidates_with_near_training_rows, _state_scales

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
from oracle import variational_train as vt  # noqa: E402  (imports torch)


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _rel(a, ref):
    return np.abs(np.asarray(a) - ref).max() / max(np.abs(ref).max(), 1e-300)


# ------------------------------------------------------------------------------------------ exact GP
def _exact_model(N, d, theta, ard=False, seed=0, noise_of=None):
    """An exact GP of M = len(theta) objectives: objective m takes hyper-parameter set theta[m] (objectives with the same
    set share one factor plane bit for bit).  noise_of: {set: set whose constant and length scales it copies, with its
    own noise}.  Length scales grow with sqrt(d), so that kernel values stay away from 0 and 1 at every d."""
    rng = np.random.default_rng(seed)
    M, T = len(theta), max(theta) + 1
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, : min(d, 4)].sum(axis=1) + k) + Xtr[:, k % d] ** 2 for k in range(M)])
    base = 0.1 * np.sqrt(max(d, 4))  # 0.4 at d 16, as the parity tests' models
    ls_t = [base * (0.75 + 0.5 * rng.random(d)) if ard else base * (1.0 + 0.02 * t) for t in range(T)]
    c_t = [1.0 + 0.2 * t for t in range(T)]
    nz0 = 1e-3 if d == 1 else 1e-6  # d 1: training points 1 / N apart, a larger nugget keeps K well conditioned
    nz_t = [nz0 * (1 + t) for t in range(T)]
    for t, src in (noise_of or {}).items():
        ls_t[t], c_t[t] = ls_t[src], c_t[src]
    st = gp.fit_fixed(Xtr, Ytr, np.zeros(d), np.ones(d), [c_t[theta[m]] for m in range(M)], [ls_t[theta[m]] for m in range(M)],
                      np.array([nz_t[theta[m]] for m in range(M)]))
    for m in range(M):
        st.objectives[m].L = st.objectives[theta.index(theta[m])].L
    return st, rng


def _gp_handle(L, st, d):
    return L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]),
                      [o.constant for o in st.objectives], [np.broadcast_to(np.asarray(o.length_scale, dtype=np.float64), (d,)) for o in st.objectives],
                      [o.noise for o in st.objectives], [o.y_mean for o in st.objectives], [o.y_std for o in st.objectives], st.xlb, st.xub)


def _pred(h, X, precision, var=True):
    m, v = h.predict(X, return_var=var, precision=precision)
    return np.array(m), (np.array(v) if var else None)


def _assert_tensor_bar(mean, var, mean_o, var_o, ystd, prior, what):
    """The forced tensor path's bar (test_gpu_parity.py, test_gpu_predict_chunks.py): mean 1e-5 of max(|mean|, y_std),
    variance 1e-5 of the prior.  _assert_gp_bars also holds variances above 1e-3 of the prior to 1e-5 of their own
    value; that is what AUTO's float64 refinement of small-variance rows provides, and AUTO is held to it."""
    em = np.max(np.abs(mean - mean_o) / np.maximum(np.abs(mean_o), ystd))
    ev = np.max(np.abs(var - var_o) / prior)
    print(f"{what}: mean rel err {em:.2e}, var err/prior {ev:.2e}")
    assert em < 1e-5 and ev < 1e-5, (what, em, ev)


def _exact_all_paths(L, monkeypatch, st, h, X, what):
    """float64, tensor fused (the default route), tensor two-kernel, AUTO and both mean-only predicts against the oracle,
    and the twins against each other."""
    mean_o, var_o = gp.predict(st, X)
    ystd, prior = _state_scales(st)
    monkeypatch.delenv("DMO_GP_FUSED", raising=False)
    m64, v64 = _pred(h, X, L.GP_FP64)
    em = np.max(np.abs(m64 - mean_o) / np.maximum(np.abs(mean_o), ystd))
    ev = np.max(np.abs(v64 - var_o) / prior)
    print(f"{what} fp64: mean rel err {em:.2e}, var err/prior {ev:.2e}")
    assert em < 1e-8 and ev < 1e-8, (what, em, ev)
    mt, vt_ = _pred(h, X, L.GP_TENSOR)
    _assert_tensor_bar(mt, vt_, mean_o, var_o, ystd, prior, what + " tensor")
    _assert_tensor_bar(mt, vt_, m64, v64, ystd, prior, what + " tensor against fp64")
    monkeypatch.setenv("DMO_GP_FUSED", "0")
    ms, vs = _pred(h, X, L.GP_TENSOR)
    mso, _ = _pred(h, X, L.GP_TENSOR, var=False)
    monkeypatch.delenv("DMO_GP_FUSED")
    _assert_tensor_bar(ms, vs, mean_o, var_o, ystd, prior, what + " tensor two-kernel")
    assert np.array_equal(vs, vt_), (what, "the two K_* producers write the same K_* bits")
    assert np.max(np.abs(ms - mt) / np.maximum(np.abs(mt), ystd)) < 1e-5, what
    ma, va = _pred(h, X, L.GP_AUTO)
    _assert_gp_bars(ma, va, mean_o, var_o, ystd, prior, what + " auto")
    for label, prec, bar in (("mean-only tensor", L.GP_TENSOR, 1e-5), ("mean-only fp64", L.GP_FP64, 1e-8)):
        mo, _ = _pred(h, X, prec, var=False)
        err = np.max(np.abs(mo - mean_o) / np.maximum(np.abs(mean_o), ystd))
        print(f"{what} {label}: mean rel err {err:.2e}")
        assert err < bar, (what, label, err)
    # the mean-only predict ignores DMO_GP_FUSED (the direct kernel, or the K_* route past its gate)
    assert np.max(np.abs(mso - mean_o) / np.maximum(np.abs(mean_o), ystd)) < 1e-5, what


@pytest.mark.parametrize("d", [1, 16, 17, 32, 33, 64])
def test_exact_gp_input_dimension_thresholds(L, monkeypatch, d):
    st, rng = _exact_model(300, d, [0, 1, 2], seed=d)
    h = _gp_handle(L, st, d)
    assert h.covariance_groups() == (3, [0, 1, 2])
    X = _candidates_with_near_training_rows(rng, st.X_train, 400, d)
    _exact_all_paths(L, monkeypatch, st, h, X, f"exact d={d}")


@pytest.mark.parametrize("d", [32, 33, 64])
@pytest.mark.parametrize("G", [2, 3])
def test_exact_gp_per_dimension_length_scales(L, monkeypatch, d, G):
    theta = [0, 1, 0] if G == 2 else [0, 1, 2]
    st, rng = _exact_model(300, d, theta, ard=True, seed=100 + d + G)
    h = _gp_handle(L, st, d)
    assert h.covariance_groups() == (G, theta)
    X = _candidates_with_near_training_rows(rng, st.X_train, 400, d)
    _exact_all_paths(L, monkeypatch, st, h, X, f"exact per-dimension d={d} G={G}")


@pytest.mark.parametrize("M", [6, 7, 8, 16])
def test_exact_gp_objective_count_thresholds(L, monkeypatch, M):
    d = 12
    st, rng = _exact_model(200, d, list(range(M)), seed=200 + M)
    h = _gp_handle(L, st, d)
    assert h.covariance_groups() == (M, list(range(M)))
    X = _candidates_with_near_training_rows(rng, st.X_train, 300, d)
    _exact_all_paths(L, monkeypatch, st, h, X, f"exact M={M}")


# objective -> covariance: sets 4 and 5 have the constant and length scales of set 0 but their own noises, so only the
# factor planes tell them apart from set 0 and from each other.  Set 4 first appears at objective 9 (index 8): the planes
# past the first eight must be compared with the earlier ones; set 5 first appears at objective 12 (index 11), after
# set 4's leader: planes past the first eight must be compared with each other as well.
IRREGULAR_16 = [0, 1, 0, 2, 1, 0, 3, 2, 4, 3, 1, 5, 4, 2, 5, 0]


def test_exact_gp_sixteen_objectives_sharing_covariances_irregularly(L, monkeypatch):
    d = 10
    st, rng = _exact_model(200, d, IRREGULAR_16, seed=16, noise_of={4: 0, 5: 0})
    h = _gp_handle(L, st, d)
    assert h.covariance_groups() == (6, IRREGULAR_16)
    X = _candidates_with_near_training_rows(rng, st.X_train, 300, d)
    _exact_all_paths(L, monkeypatch, st, h, X, "exact M=16 G=6")


def test_exact_gp_seven_objectives_on_four_covariances(L, monkeypatch):
    d, theta = 12, [0, 1, 1, 2, 0, 3, 2]
    st, rng = _exact_model(200, d, theta, seed=7)
    h = _gp_handle(L, st, d)
    assert h.covariance_groups() == (4, theta)
    X = _candidates_with_near_training_rows(rng, st.X_train, 300, d)
    _exact_all_paths(L, monkeypatch, st, h, X, "exact M=7 G=4")


@pytest.mark.parametrize("N", [1, 2, 255, 256, 257])
def test_exact_gp_training_set_sizes(L, monkeypatch, N):
    d = 8
    st, rng = _exact_model(N, d, [0, 1], seed=300 + N)
    h = _gp_handle(L, st, d)
    X = _candidates_with_near_training_rows(rng, st.X_train, 300, d)
    X[-1] = st.X_train[0]  # a candidate on a training point
    _exact_all_paths(L, monkeypatch, st, h, X, f"exact N={N}")


@functools.lru_cache(maxsize=None)
def _candidate_model():
    return _exact_model(300, 20, [0, 1, 2], seed=400)


@pytest.mark.parametrize("P", [1, 127, 129])
def test_exact_gp_candidate_counts(L, monkeypatch, P):
    st, _ = _candidate_model()
    h = _gp_handle(L, st, 20)
    rng = np.random.default_rng(P)
    X = _candidates_with_near_training_rows(rng, st.X_train, P, 20)
    X[0] = np.clip(st.X_train[5] + 1e-4, 0, 1)
    _exact_all_paths(L, monkeypatch, st, h, X, f"exact P={P}")


# ------------------------------------------------------------------------------------------ MEGP
def _megp_model(N, d, M, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(X[:, :2].sum(1) + t) + 0.3 * X[:, (t + 2) % d] + 0.1 * t * X[:, -1] ** 2 for t in range(M)])
    ls = np.sqrt(d / 4.0) * (0.4 + 0.4 * rng.random(d))
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + 0.5 * rng.random(M))
    D = np.geomspace(1e-3, 8e-3, M) + 1e-2
    w, b = 0.2 * rng.standard_normal((M, d)), 0.1 * rng.standard_normal(M)
    st = megp.fit_fixed(X, Y, np.zeros(d), np.ones(d), ls, B, D, w, b)
    yn, ym, ys = megp.normalise_y(Y)
    args = (X, yn, ls, B, D, w, b, ym, ys, np.zeros(d), np.ones(d))
    return st, args, (np.diag(B) + D) * ys**2, rng


def _megp_check(L, N, d, precisions, seed):
    M = 8
    st, args, prior, rng = _megp_model(N, d, M, seed)
    h = L.MTGPHandle(*args)
    Xc = _candidates_with_near_training_rows(rng, args[0], 300, d)
    mean_o, var_o = megp.predict(st, Xc)
    scale = np.abs(mean_o).max(axis=0).astype(np.float64)
    out = {}
    for precision in precisions:
        tensor = precision == "tensor"
        m, v = _pred(h, Xc, L.GP_TENSOR if tensor else L.GP_FP64)
        tol = 1e-5 if tensor else 2e-6
        em, ev = np.abs(m - mean_o).max(axis=0) / scale, np.abs(v - var_o).max(axis=0) / prior
        print(f"MEGP N={N} d={d} {precision}: mean err/scale {em.max():.2e}, var err/prior {ev.max():.2e}")
        assert np.all(em <= tol) and np.all(ev <= tol), (N, d, precision, em, ev)
        out[precision] = (m, v)
    if len(out) == 2:
        (m64, v64), (mt, vt_) = out["fp64"], out["tensor"]
        assert np.all(np.abs(mt - m64).max(axis=0) <= 1e-5 * scale) and np.all(np.abs(vt_ - v64).max(axis=0) <= 1e-5 * prior)
    h.close()


@pytest.mark.parametrize("d,precisions", [(33, ("fp64", "tensor")), (64, ("fp64", "tensor")), (65, ("fp64",)), (90, ("fp64",))])
def test_megp_eight_tasks_input_dimensions(L, d, precisions):
    _megp_check(L, 300, d, precisions, seed=500 + d)


@pytest.mark.parametrize("N", [1, 63, 64, 65])
def test_megp_eight_tasks_training_set_sizes(L, N):
    _megp_check(L, N, 12, ("fp64", "tensor"), seed=600 + N)


def _close(g, rg, rel, what):
    for k in rg:
        err, scale = np.abs(np.asarray(g[k]) - rg[k]).max(), np.abs(rg[k]).max()
        print(f"{what} {k}: err/max|ref| {err / max(scale, 1e-300):.2e}")
        assert err <= rel * scale, (what, k, err, scale)


@pytest.mark.parametrize("N", [63, 64, 65])
def test_mtgp_lml_grad_eight_tasks_ninety_dimensions(L, N):
    d, M = 90, 8
    rng = np.random.default_rng(700 + N)
    X = rng.random((N, d))
    yn = rng.standard_normal((N, M))
    ls = np.sqrt(d / 4.0) * np.exp(rng.uniform(np.log(0.5), np.log(2.0), d))
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + 0.5 * rng.random(M))
    D = np.geomspace(5e-3, 3e-2, M)
    w, b = 0.2 * rng.standard_normal((M, d)), 0.1 * rng.standard_normal(M)
    lml, g = L.mtgp_lml_grad(X, yn, ls, B, D, w, b)
    ref, rg = megp_train.lml_and_grad_torch(X, yn, ls, B, D, w, b)
    assert abs(lml - ref) <= 1e-10 * abs(ref), (lml, ref)
    _close(g, rg, 1e-8, f"mtgp_lml_grad N={N}")


# ------------------------------------------------------------------------------------------ EGP / exact fit
def _egp_hyper(rng, d, M):
    return (np.sqrt(d / 4.0) * np.exp(rng.uniform(np.log(0.3), np.log(3.0), (M, d))), 0.3 + 1.2 * rng.random(M),
            np.geomspace(2e-3, 2e-2, M), 0.3 * rng.standard_normal((M, d)) / np.sqrt(d), 0.2 * rng.standard_normal(M))


@pytest.mark.parametrize("N", [1, 63, 64, 65])
def test_gp_lml_grad_eight_objectives_ninety_dimensions(L, N):
    d, M = 90, 8
    rng = np.random.default_rng(800 + N)
    X = rng.random((N, d))
    yn = rng.standard_normal((N, M))
    hp = _egp_hyper(rng, d, M)
    lml, g = L.gp_lml_grad(X, yn, *hp)
    ref, rg = egp_train.lml_and_grad_torch(X, yn, *hp)
    assert np.all(np.abs(lml - ref) <= 1e-10 * np.abs(ref)), (lml, ref)
    _close(g, rg, 1e-8, f"gp_lml_grad N={N}")


@pytest.mark.parametrize("N", [63, 64, 127])
def test_gp_fit_ninety_dimensions(L, N):
    from scipy.linalg import cho_solve, cholesky

    d, M = 90, 2
    rng = np.random.default_rng(900 + N)
    X = rng.random((N, d))
    y = rng.standard_normal((M, N))
    c, nz, jit = np.array([1.3, 0.7]), np.array([1e-3, 5e-3]), 1e-10
    ls = [np.sqrt(d / 4.0) * (0.5 + rng.random(d)) for _ in range(M)]
    Lg, ag, lg = L.gp_fit(X, y, c, ls, nz, jitter=jit)
    for m in range(M):
        K = c[m] * gp.kernel_matrix(X, X, ls[m])
        K[np.diag_indices(N)] += nz[m] + jit
        Lr = cholesky(K, lower=True)
        ar = cho_solve((Lr, True), y[m])
        lr = -0.5 * y[m] @ ar - np.log(np.diag(Lr)).sum() - 0.5 * N * np.log(2 * np.pi)
        print(f"gp_fit N={N} objective {m}: L {_rel(Lg[m], Lr):.2e}, alpha {_rel(ag[m], ar):.2e}, lml {abs(lg[m] - lr) / abs(lr):.2e}")
        assert abs(lg[m] - lr) <= 1e-10 * abs(lr), (m, lg[m], lr)
        assert _rel(np.tril(Lg[m]), Lr) < 1e-12 and _rel(ag[m], ar) < 1e-8, m
    # the fit's lml is the lml_grad's (zero linear mean, no jitter)
    _, _, l0 = L.gp_fit(X, y, c, ls, nz, jitter=0.0, want_L=False, want_alpha=False)
    l1, _ = L.gp_lml_grad(X, y.T, np.stack(ls), c, nz, np.zeros((M, d)), np.zeros(M))
    assert np.all(np.abs(l0 - l1) <= 1e-12 * np.abs(l1)), (l0, l1)


# ------------------------------------------------------------------------------------------ training sizes
def test_gp_lml_grad_at_a_training_size(L):
    """N 2048, d 30, M 3: the gradient kernels' 32 x 32 tile rows and the Np = 2048 batched L^-1 of a real EGP fit."""
    N, d, M = 2048, 30, 3
    rng = np.random.default_rng(2048)
    X = rng.random((N, d))
    yn = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, t + 2] for t in range(M)])
    yn = (yn - yn.mean(0)) / yn.std(0)
    hp = _egp_hyper(rng, d, M)
    lml, g = L.gp_lml_grad(X, yn, *hp)
    ref, rg = fit_grad_dense.egp_lml_and_grad(X, yn, *hp)
    assert np.all(np.abs(lml - ref) <= 1e-10 * np.abs(ref)), (lml, ref)
    _close(g, rg, 1e-8, "gp_lml_grad N=2048")


def test_mtgp_lml_grad_at_a_training_size(L):
    N, d, M = 2048, 30, 2
    rng = np.random.default_rng(2049)
    X = rng.random((N, d))
    yn = np.column_stack([np.sin(3 * X[:, :2].sum(1) + t) + 0.4 * X[:, t + 2] for t in range(M)])
    yn = (yn - yn.mean(0)) / yn.std(0)
    ls = np.sqrt(d / 4.0) * np.exp(rng.uniform(np.log(0.5), np.log(2.0), d))
    B = megp.task_covariance(rng.standard_normal((M, 1)), 0.2 + 0.5 * rng.random(M))
    D = np.array([1e-2, 2e-2])
    w, b = 0.3 * rng.standard_normal((M, d)) / np.sqrt(d), 0.1 * rng.standard_normal(M)
    lml, g = L.mtgp_lml_grad(X, yn, ls, B, D, w, b)
    ref, rg = fit_grad_dense.megp_lml_and_grad(X, yn, ls, B, D, w, b)
    assert abs(lml - ref) <= 1e-10 * abs(ref), (lml, ref)
    _close(g, rg, 1e-8, "mtgp_lml_grad N=2048")


# ------------------------------------------------------------------------------------------ variational predict
def _sv_model(kind, Lat, Zn, d, seed):
    rng = np.random.default_rng(seed)
    Zp = rng.random((Lat, Zn, d))
    if kind == "spv":
        Zp[:] = Zp[0]
    ls = np.sqrt(d) * (0.4 + 0.6 * rng.random((Lat, d)))
    s = 0.5 + rng.random(Lat)
    q_mu = rng.standard_normal((Lat, Zn))
    q_sqrt = np.tril(0.05 / np.sqrt(Zn) * rng.standard_normal((Lat, Zn, Zn)), -1)
    for l in range(Lat):
        q_sqrt[l][np.diag_indices(Zn)] = 0.2 + 0.4 * rng.random(Zn)
    W = rng.standard_normal((Lat, Lat)) if kind == "crv" else None
    Wm = np.eye(Lat) if W is None else W
    ym, ys = rng.standard_normal(Lat), 0.5 + rng.random(Lat)
    Xc = _candidates_with_near_training_rows(rng, Zp.reshape(-1, d), 300, d)
    g = [V.latent_predict(Xc, Zp[l], s[l], ls[l], q_mu[l], q_sqrt[l]) for l in range(Lat)]
    mean_o = ys * (np.stack([m for m, _ in g], axis=1) @ Wm.T) + ym
    var_o = (np.stack([v for _, v in g], axis=1) @ (Wm * Wm).T) * ys**2
    prior = ((Wm * Wm) @ s) * ys**2
    return (Zp, s, ls, q_mu, q_sqrt, ym, ys, np.zeros(d), np.ones(d)), W, Xc, mean_o, var_o, ys, prior


def _sv_check(L, kind, Lat, Zn, d, precisions, seed):
    args, W, Xc, mean_o, var_o, ys, prior = _sv_model(kind, Lat, Zn, d, seed)
    h = L.SVGPHandle(*args, W=W)
    scale = np.maximum(np.abs(mean_o).max(axis=0), ys)
    out = {}
    for precision in precisions:
        tensor = precision == "tensor"
        m, v = _pred(h, Xc, L.GP_TENSOR if tensor else L.GP_FP64)
        vscale = np.maximum(np.abs(var_o).max(axis=0), prior) if tensor else prior
        em, ev = np.abs(m - mean_o).max(axis=0) / scale, np.abs(v - var_o).max(axis=0) / vscale
        tol_v = 1e-4 if tensor else 1e-9
        print(f"{kind} L={Lat} Z={Zn} d={d} {precision}: mean err/scale {em.max():.2e}, var err {ev.max():.2e}")
        assert np.all(em <= 2e-6) and np.all(ev <= tol_v), (kind, Lat, Zn, d, precision, em, ev)
        out[precision] = (m, v)
    if len(out) == 2:
        (m64, v64), (mt, vt_) = out["fp64"], out["tensor"]
        assert np.all(np.abs(mt - m64).max(axis=0) <= 2e-6 * scale)
        assert np.all(np.abs(vt_ - v64).max(axis=0) <= 1e-4 * np.maximum(np.abs(v64).max(axis=0), prior))
    h.close()


@pytest.mark.parametrize("kind", ["crv", "spv"])
def test_variational_eight_latents(L, kind):
    _sv_check(L, kind, 8, 64, 10, ("fp64", "tensor"), seed=1000 + len(kind))


@pytest.mark.parametrize("kind", ["svgp", "crv"])
def test_variational_ninety_dimensions(L, kind):
    _sv_check(L, kind, 2, 100, 90, ("fp64",), seed=1090 + len(kind))


@pytest.mark.parametrize("Zn", [1, 64, 65, 257])
def test_variational_inducing_point_counts(L, Zn):
    _sv_check(L, "svgp", 2, Zn, 8, ("fp64", "tensor"), seed=1100 + Zn)


@pytest.mark.parametrize("Zn,N", [(1, 50), (1100, 1500)])
def test_svgp_optimal_q_inducing_point_counts(L, Zn, N):
    d = 4
    rng = np.random.default_rng(1200 + Zn)
    X = rng.random((N, d))
    y = np.sin(3 * X.sum(1))[None]
    Z = X[rng.choice(N, Zn, replace=False)]
    s, ls, nz = np.array([0.9]), np.full((1, d), 0.6), np.array([0.05])
    q_mu, q_sqrt = L.svgp_optimal_q(X, y, Z[None], s, ls, nz)
    o_mu, o_S = V.optimal_q(X, y[0], Z, s[0], ls[0], nz[0])
    S = q_sqrt[0] @ q_sqrt[0].T
    print(f"optimal_q Z={Zn}: q_mu {_rel(q_mu[0], o_mu):.2e}, S {_rel(S, o_S):.2e}")
    assert _rel(q_mu[0], o_mu) < 1e-8 and _rel(S, o_S) < 1e-8
    assert np.all(np.triu(q_sqrt[0], 1) == 0.0)


# ------------------------------------------------------------------------------------------ variational training
def _fit_data(rng, N, d, M):
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, : min(d, 2)].sum(1) + t) + 0.4 * X[:, (t + 1) % d] for t in range(M)])
    return X, (Y - Y.mean(0)) / Y.std(0)


def _fit_check(L, kind, N, Zn, B, d, M, seed):
    """natgrad against the autograd-derived step, then elbo_grad at that q against the autograd ELBO."""
    rng = np.random.default_rng(seed)
    X, Y = _fit_data(rng, N, d, M)
    vgp = kind == "vgp"
    Z = None if vgp else X[rng.choice(N, Zn, replace=False)]
    Lat = M
    s = 0.5 + rng.random(Lat)
    ls = np.exp(rng.uniform(np.log(0.5), np.log(2.0), (Lat, d))) * np.sqrt(d / 2)
    nz = np.geomspace(0.03, 0.08, M)
    W = rng.standard_normal((M, Lat)) if kind == "crv" else None
    st = L.SVGPFitState(X, Y, Z, Lat, inducing_is_data=vgp)
    b = [np.arange(N) if vgp else rng.permutation(N)[:B] for _ in range(3)]
    st.natgrad(b[0], s, ls, nz, W, gamma=0.6)
    q0 = st.q()
    st.natgrad(b[1], s, ls, nz, W, gamma=0.4)
    q1 = st.q()
    r1 = vt.natgrad_step(X, Y, Z, b[1], s, ls, nz, W, q0[0], q0[1], 0.4, vgp)
    what = f"{kind} N={N} Z={Zn} B={B} d={d} L={Lat}"
    for name, a, r in zip(("q_mu", "q_sqrt"), q1, r1):
        print(f"{what} natgrad {name}: {_rel(a, r):.2e}")
        assert _rel(a, r) < 1e-8, (what, name, _rel(a, r))
    ell, kl, g = st.elbo_grad(b[2], s, ls, nz, W)
    rell, rkl, rg = vt.elbo_and_grad(X, Y, Z, b[2], s, ls, nz, W, q1[0], q1[1], vgp)
    np.testing.assert_allclose(ell, rell, rtol=1e-10, atol=1e-10 * np.abs(rell).max())
    np.testing.assert_allclose(kl, rkl, rtol=1e-10, atol=1e-10 * np.abs(rkl).max())
    keys = ("variance", "length_scale", "noise") + (("W",) if W is not None else ())
    _close({k: g[k] for k in keys}, {k: rg[k] for k in keys}, 1e-8, what)
    st.close()


@pytest.mark.parametrize("kind,N,Zn,B,d,M", [
    ("crv", 200, 40, 50, 6, 8),     # L = M = 8 = SVF_MAX with a dense W
    ("svgp", 150, 30, 60, 90, 1),   # d = 90: svf_fold_kernel's d + 1 outputs, svf_grad_pass_kernel's coordinates
    ("crv", 120, 25, 40, 90, 2),
    ("svgp", 100, 20, 1, 4, 1),     # B = 1
    ("svgp", 150, 1, 50, 5, 1),     # Z = 1
    ("svgp", 150, 64, 50, 5, 1),
    ("spv", 150, 65, 50, 5, 2),
    ("vgp", 65, 65, 65, 5, 1),      # VGP, N = Z = 65
])
def test_variational_fit_at_the_limits(L, kind, N, Zn, B, d, M):
    _fit_check(L, kind, N, Zn, B, d, M, seed=N + Zn + B + d + M)


def test_variational_fit_at_a_training_size(L):
    """Z 1100 (the Np = 2048 batched L^-1), B 256, three latents on shared inducing points."""
    _fit_check(L, "spv", 3000, 1100, 256, 5, 3, seed=1100)


# ------------------------------------------------------------------------------------------ refusals
def _refused(L, call, match):
    n0 = L.launch_count()
    with pytest.raises(L.DmoError, match=match):
        call()
    assert L.launch_count() == n0, match


def test_exact_gp_refuses_past_its_limits(L):
    rng = np.random.default_rng(0)

    def create(d, M, N=10):
        X = rng.random((N, d))
        return L.GPHandle(X, np.zeros((M, N)), np.stack([np.eye(N)] * M), np.ones(M), [np.ones(d)] * M, np.full(M, 1e-6),
                          np.zeros(M), np.ones(M), np.zeros(d), np.ones(d))

    create(64, 16).close()
    _refused(L, lambda: create(65, 1), "gp_create: unsupported shape N=10 d=65 M=1")
    _refused(L, lambda: create(8, 17), "gp_create: unsupported shape N=10 d=8 M=17")


def test_multitask_refuses_past_its_limits(L):
    rng = np.random.default_rng(1)

    def args(N, d, M):
        return (rng.random((N, d)), rng.standard_normal((N, M)), np.ones(d), np.eye(M), np.full(M, 0.1), np.zeros((M, d)), np.zeros(M))

    h = L.MTGPHandle(*args(20, 65, 2), np.zeros(2), np.ones(2), np.zeros(65), np.ones(65))
    X = rng.random((5, 65))
    h.predict(X, precision=L.GP_FP64)
    _refused(L, lambda: h.predict(X, precision=L.GP_TENSOR), r"mtgp_predict\(tensor\): at most 64 input dimensions \(got 65\)")
    h.close()
    _refused(L, lambda: L.MTGPHandle(*args(20, 91, 2), np.zeros(2), np.ones(2), np.zeros(91), np.ones(91)),
             r"mtgp_create: unsupported shape N=20 d=91 M=2 \(1 <= M <= 8, d <= 90\)")
    _refused(L, lambda: L.MTGPHandle(*args(20, 4, 9), np.zeros(9), np.ones(9), np.zeros(4), np.ones(4)),
             r"mtgp_create: unsupported shape N=20 d=4 M=9")
    _refused(L, lambda: L.mtgp_lml_grad(*args(20, 91, 2)), r"mtgp_lml_grad: unsupported shape N=20 d=91 M=2")
    _refused(L, lambda: L.mtgp_lml_grad(*args(20, 4, 9)), r"mtgp_lml_grad: unsupported shape N=20 d=4 M=9")


def test_exact_fits_refuse_past_their_limits(L):
    rng = np.random.default_rng(2)
    X91 = rng.random((20, 91))
    _refused(L, lambda: L.gp_fit(X91, rng.standard_normal((1, 20)), [1.0], [np.ones(91)], [1e-3]), "gp_fit: bad arguments")

    def lml_grad(d, M):
        return L.gp_lml_grad(rng.random((20, d)), rng.standard_normal((20, M)), np.ones((M, d)), np.ones(M), np.full(M, 1e-2),
                             np.zeros((M, d)), np.zeros(M))

    _refused(L, lambda: lml_grad(91, 1), r"gp_lml_grad: unsupported shape N=20 d=91 M=1 \(1 <= M <= 8, d <= 90\)")
    _refused(L, lambda: lml_grad(4, 9), r"gp_lml_grad: unsupported shape N=20 d=4 M=9")


def test_variational_refuses_past_its_limits(L):
    rng = np.random.default_rng(3)

    def create(Lat, Zn, d, W=None):
        return L.SVGPHandle(rng.random((Lat, Zn, d)), np.ones(Lat), np.ones((Lat, d)), np.zeros((Lat, Zn)),
                            np.broadcast_to(np.eye(Zn), (Lat, Zn, Zn)), np.zeros(Lat if W is None else W.shape[0]),
                            np.ones(Lat if W is None else W.shape[0]), np.zeros(d), np.ones(d), W=W)

    h = create(1, 10, 65)
    X = rng.random((5, 65))
    h.predict(X, precision=L.GP_FP64)
    _refused(L, lambda: h.predict(X, precision=L.GP_TENSOR), r"svgp_predict\(tensor\): at most 64 input dimensions \(got 65\)")
    h.close()
    _refused(L, lambda: create(1, 10, 91), r"svgp_create: unsupported shape Z=10 d=91 \(Z <= 8192, d <= 90\)")
    _refused(L, lambda: create(9, 10, 4), r"svgp_create: 1 <= L, M <= 8 \(got L=9 M=9\)")
    _refused(L, lambda: create(2, 10, 4, W=np.ones((9, 2))), r"svgp_create: 1 <= L, M <= 8 \(got L=2 M=9\)")
    # Z = 8193: q_sqrt is an untouched (lazily zero) array; the shape is refused before it is read
    _refused(L, lambda: L.SVGPHandle(np.zeros((1, 8193, 1)), np.ones(1), np.ones((1, 1)), np.zeros((1, 8193)), np.zeros((1, 8193, 8193)),
                                     np.zeros(1), np.ones(1), np.zeros(1), np.ones(1)), r"svgp_create: unsupported shape Z=8193 d=1")
    X, Y = rng.random((30, 91)), rng.standard_normal((30, 1))
    _refused(L, lambda: L.SVGPFitState(X, Y, X[:10], 1), r"svgp_fit_create: unsupported shape")
    _refused(L, lambda: L.SVGPFitState(X[:, :4], rng.standard_normal((30, 2)), X[:10, :4], 9), r"svgp_fit_create: 1 <= L, M <= 8 \(got L=9 M=2\)")
    Xz = rng.random((9000, 1))
    _refused(L, lambda: L.SVGPFitState(Xz, rng.standard_normal((9000, 1)), Xz[:8193], 1), r"svgp_fit_create: unsupported shape")
    _refused(L, lambda: L.svgp_optimal_q(X, Y.T, X[None, :10], np.ones(1), np.ones((1, 91)), np.full(1, 0.1)),
             r"svgp_optimal_q: unsupported shape N=30 Z=10 d=91")
    _refused(L, lambda: L.svgp_optimal_q(Xz, rng.standard_normal((1, 9000)), Xz[None, :8193], np.ones(1), np.ones((1, 1)), np.full(1, 0.1)),
             r"svgp_optimal_q: unsupported shape N=9000 Z=8193 d=1")
    _refused(L, lambda: L.svgp_optimal_q(X[:, :4], rng.standard_normal((9, 30)), rng.random((9, 10, 4)), np.ones(9), np.ones((9, 4)),
                                         np.full(9, 0.1)), r"svgp_optimal_q: 1 <= L <= 8 \(got 9\)")


def test_python_classes_refuse_before_training_without_a_launch(L, monkeypatch):
    """A shape the class's predict cannot take is refused with a ValueError before any training: no launch, and the
    trainers are never entered."""
    from test_shape_limits_cpu import REFUSALS, refuse_training

    refuse_training(monkeypatch)
    for make, match in REFUSALS:
        n0 = L.launch_count()
        with pytest.raises(ValueError, match=match):
            make()
        assert L.launch_count() == n0, match
