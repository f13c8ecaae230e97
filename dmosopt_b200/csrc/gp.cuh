// GP posterior state shared by gp.cu (float64 path) and gp_tensor.cu (wgmma path), and the variance operators that the
// exact, multitask (gp_multitask.cu) and variational (gp_variational.cu) posteriors contract against.
#pragma once
#include <vector>

#include "common.cuh"

// G lower-triangular float64 planes Linv_g: a posterior's variance terms are the column sums of squares ||Linv_g k_*||^2
// against a K_* plane.  The exact GP's planes are the L^-1 of its covariances; MEGP's the L_j^-1 of its blocks; the
// variational posterior's the operators s Lz^-1 and s T.  h_kscale[g] is the output scale of the K_* plane that plane g
// is contracted against; it fixes that plane's K_* scaling exponent on the tensor path.
struct GpVarOps {
  int64_t Npad = 0;  // rows and columns of a plane: N rounded up to the float64 (128) and wgmma (256) tiles
  int G = 0;
  std::vector<double> h_kscale;  // (G,)
  DevBuf<double> Linv;           // (G, Npad, Npad), zero above the diagonal and in the padding
  // tensor path (built lazily by gp_prepare_tensor)
  bool tensor_ready = false;
  DevBuf<uint16_t> Lhi, Llo;  // (G, Npad, Npad) fp16 split of the row-scaled Linv
  DevBuf<float> Lscale;       // (G, Npad) 1 / (row scale * K_* scale), powers of two
  DevBuf<int> Kexp;           // (G,) K_* scaling exponents
  // G zeroed planes for N points, K_* scales 1
  int alloc(dmo_ctx* ctx, int64_t N, int G);
};

struct dmo_gp {
  int64_t N = 0;  // training points
  int d = 0, M = 0, kernel = 0;
  bool isotropic = true;
  // Objectives that share a posterior covariance (bitwise equal constant, length scales and factor plane; noise may
  // differ, it only enters the final subtraction) share one L^-1, one K_* and one variance contraction.  Decided once
  // by dmo_gp_create: ops.G groups numbered in order of first appearance, cov[m] the group of objective m, lead[g] the
  // first objective of group g.  Every per-covariance array below has ops.G planes.
  GpVarOps ops;                    // the L^-1 of each group, K_* scales the group constants
  std::vector<int> h_cov, h_lead;  // (M,), (G,)
  DevBuf<int> cov;                 // (M,) device copy of h_cov
  DevBuf<double> Xt;        // (N, d) normalised training inputs
  DevBuf<double> alpha;     // (M, N)
  DevBuf<double> inv_ls;    // (M, d) 1 / length_scale
  DevBuf<double> g_inv_ls, g_constant;  // (G, d), (G,) 1 / length_scale and constant of each group (its first objective)
  DevBuf<double> constant, noise, ymean, ystd;  // (M,)
  DevBuf<double> xlb, xrg;  // (d,)
  std::vector<double> h_constant, h_noise, h_ystd;
  // optional linear prior mean m(x) = w . x_n + b in the normalised-output space (gpytorch LinearMean, A19)
  bool has_linear_mean = false;
  DevBuf<double> lin_w, lin_b;  // (M, d), (M,)
  DevBuf<float> Xtf;          // (Npad, 32) float copy of Xt, zero padded (mean-only direct kernel, d <= 32); built lazily
  DevBuf<float> CAf;          // (M, Npad) c_m * alpha_m as float, zero padded (fused K_* + mean kernel); built with Xtf
  // DMO_GP_AUTO: per-model calibration of the tensor path against the float64 path on probe candidates (gp.cu)
  bool calibrated = false;
  bool auto_mean_tensor = false;  // the tensor-path mean (K_* alpha pass) holds 1e-5 on the probes (with margin)
  bool auto_var_tensor = false;   // split-fp16 variance holds 1e-5 * prior on the probes (with margin)
  double cal_mean_err = 0.0;      // max |mean_t - mean_64| / max(|mean_64|, y_std) over the probes
  bool auto_mean_only = false;    // the mean-only tensor-path call (direct kernel where it applies) holds 1e-5 on the probes
  double cal_mean_err_only = 0.0; // its probe error
  double cal_var_err = 0.0;       // max |var_t - var_64| / prior over the probes
  double refine_theta = 1.0;      // rows with var_t < theta * prior are recomputed in float64
  int64_t last_refined = 0;       // rows recomputed by the last DMO_GP_AUTO predict
};

// The float64 covariance at the squared scaled distance s2 = r^2: Matern-5/2 (1 + K + K^2 / 3) exp(-K) with K = sqrt(s2)
// sqrt(5), or RBF exp(-s2 / 2).  gp_deep_fit.cu keeps its own Matern: it forms sqrt(5 s2), which rounds differently.  The
// float32 helpers of the tensor paths are not this function either.
__device__ __forceinline__ double stationary(double s2, int kind) {
  if (kind == DMO_KERNEL_MATERN52) {
    const double K = sqrt(s2) * 2.23606797749978969641;
    return (1.0 + K + K * K / 3.0) * exp(-K);
  }
  return exp(-0.5 * s2);
}

// Candidates per chunk of any predict, whatever its memory budget allows: the K_* producers put chunk / 32 blocks on
// the grid's y extent (at most 65535), so 2^20 keeps it at 32768.
constexpr int64_t GP_MAX_CHUNK = (int64_t)1 << 20;

int gp_predict_fp64(dmo_ctx* ctx, dmo_gp* gp, const double* dXn, int64_t P, double* d_mean, double* d_var);

// Building blocks shared with the multitask posterior (gp_multitask.cu).  All pointers are device pointers.
// L^-1 of the lower Cholesky factor L (N, N) into dst (rows of ldo doubles, lower triangle; the rest is left untouched)
int gp_linv_from_factor(dmo_ctx* ctx, const double* L, int64_t N, int64_t ldo, double* dst);
// the same for nbat factors L + b * sL (rows of ldl doubles) into dst + b * sdst, in one pass; not synchronised.  Scratch:
// 2.5 nbat Np^2 doubles, Np the power of two >= max(N, 128)
int gp_linv_from_factor_batched(dmo_ctx* ctx, const double* L, int64_t ldl, int64_t sL, int64_t N, int nbat, int64_t ldo,
                                int64_t sdst, double* dst);
// nbat independent exact-GP factorisations in one pass of the blocked Cholesky (gp_fit.cu; see its definition)
int gp_fit_batched(dmo_ctx* ctx, int64_t N, int d, int nbat, int kernel, const double* X, const double* inv_ls, const double* constant,
                   const double* diag_add, const double* y, double* A, int64_t ld, int* info, double* work, double* alpha, double* lml);
// in-place lower Cholesky factorisation of nbat symmetric matrices A + b * ld^2 (lower triangles read, row-major, ld a
// multiple of 64; pad with an identity tail); info[b] (zeroed by the caller) receives a non-positive pivot + 1.  Not
// synchronised.
int gp_potrf_batched(dmo_ctx* ctx, double* A, int64_t ld, int nbat, int* info);
// float64 variance contraction (var_kernel) over the ops.G planes: vnorm[z][g][p] = partial sums over the row blocks z
// (mod nsplit) of ||Linv_g Ks_g[p]||^2, Ks_g = Ks + g * kplane with rows of ops.Npad doubles (kplane = 0: one K_* plane
// for every g); Pcpad is a multiple of GP_F64_TILE
constexpr int GP_F64_TILE = 128;
int gp_var_contract_fp64(dmo_ctx* ctx, const GpVarOps& ops, const double* Ks, int64_t kplane, int64_t Pcpad, int nsplit,
                         double* vnorm, int64_t vn_ld);
// the fp16 hi / lo split of the planes and its row scales, and the K_* scaling exponents ops.Kexp (built once)
int gp_prepare_tensor(dmo_ctx* ctx, GpVarOps& ops);
// wgmma variance contraction (gp_var_wgmma_kernel, paired schedule) over K_* hi / lo rows of ops.Npad fp16 values:
// k_alloc rows are allocated, plane g < ops.G reads rows g * k_rows + [0, Pcpad) (k_rows = 0: one K_* plane for every
// g); Pcpad is a multiple of GP_TC_TILE.  vnorm[q][g][p], q < gp_tensor_var_planes(ops.Npad), holds the partial sums.
// abort_flag (device int, zeroed by the caller) is set when the pipeline watchdog trips.  The grid is the smallest one
// with as many work items per CTA as sm_count - free_sms CTAs would take; every item writes its own vnorm slot, so the
// grid does not change a bit.
constexpr int GP_TC_TILE = 128;
int gp_tensor_var_planes(int64_t Npad);
int gp_var_contract_tensor(dmo_ctx* ctx, const GpVarOps& ops, const uint16_t* Kh, const uint16_t* Kl, int64_t k_alloc,
                           int64_t k_rows, int64_t Pcpad, double* vnorm, int64_t vn_ld, int* abort_flag, int free_sms = 0);
// SMs the overlapped contraction leaves to the fused step's lane (the truncation and the hypervolume, step.cu).  Each SM
// taken from the contraction costs it about 0.034 ms at the bench shape (H100 80GB HBM3, 700 W); the value is the one
// scripts/step_phases.py --free-sms picked (README, "Resident step by phase").  -DDMO_GP_LANE_SMS=F builds another.
#ifndef DMO_GP_LANE_SMS
#define DMO_GP_LANE_SMS 14
#endif
constexpr int GP_LANE_SMS = DMO_GP_LANE_SMS;
// A caller that runs its own work beside the variance contraction (the fused step's lane, step.cu) passes this to the
// tensor route: mean_ready is recorded on the stream once the last chunk's mean is written, and the contraction runs on
// the context's high-priority stream (joined back before var_finish_tc_kernel) with a grid that leaves at least
// GP_LANE_SMS SMs to the caller's work.  The caller creates those streams first (dmo_lane_streams).
struct GpOverlap {
  cudaEvent_t mean_ready = nullptr;
};
// abort_flag null: the call reads the contraction's watchdog back and fails when it tripped.  Otherwise the call zeroes
// *abort_flag (device) and the watchdog lands there; the caller reads it back and fails the same way (gp_predict_auto folds
// it into its own read-back).  The mean-only route writes no flag.  var_route_mean (d_var null): the mean is the one a
// call with d_var writes, bit for bit, without the variance contraction and with no read-back.
int gp_predict_tensor(dmo_ctx* ctx, dmo_gp* gp, const double* dXn, int64_t P, double* d_mean, double* d_var,
                      int* abort_flag = nullptr, const GpOverlap* ov = nullptr, bool var_route_mean = false);
extern const char* const GP_WATCHDOG_MSG;
// An AUTO predict whose one read-back (watchdog, rows to refine) is left pending, so the caller can enqueue work behind it
// while the GP runs; gp_predict_finish waits for it, fails on a tripped watchdog and refines the rows the check flags
// (after that work: *refined tells the caller to redo it).  Only the AUTO variance route of models without a linear mean
// defers; other calls finish inside gp_predict_device and leave `active` false.  A caller that sets ov.mean_ready before
// the call gets the overlapped contraction of GpOverlap; once `active`, the event has been recorded.
struct GpPending {
  GpOverlap ov;
  bool active = false;
  int64_t P = 0;
  const double* dXn = nullptr;
  double *d_mean = nullptr, *d_var = nullptr;
  DevBuf<double> xn;
  DevBuf<int32_t> flag, pos;
};
// dmo_gp_predict on device arrays: X (P, d) un-normalised, mean / var (P, M); var may be null.  var_route_mean (var null,
// DMO_GP_FP64 or DMO_GP_TENSOR): the mean of dmo_gp_predict with a variance buffer, bit for bit, without its variance
// (float64: the mean never depends on it; tensor: gp_predict_tensor's var_route_mean).
int gp_predict_device(dmo_ctx* ctx, dmo_gp* gp, const double* dX, int64_t P, double* d_mean, double* d_var, int precision,
                      GpPending* pending = nullptr, bool var_route_mean = false);
int gp_predict_finish(dmo_ctx* ctx, dmo_gp* gp, GpPending& pending, bool* refined);

// Candidate chunks and variance scratch of the unit-scale posteriors (MEGP, variational; gp_multitask.cu): one K_* plane
// per chunk (float64 Ks, or fp16 Kh / Kl) contracted against up to `planes` operator planes, partial sums in vnorm (rows
// of Pc_alloc).  Messages are prefixed by `who`.
struct GpUnitPredict {
  const char* who = "";
  bool tensor = false;
  int64_t tile = 0;      // candidate padding of a chunk
  int64_t Pc_alloc = 0;  // candidates per chunk
  int n_vp = 0;          // vnorm partial-sum planes per operator plane
  DevBuf<double> vnorm, Ks;
  DevBuf<uint16_t> Kh, Kl;
  DevBuf<int> abort_flag;
  // precision is DMO_GP_FP64 or DMO_GP_TENSOR, and d fits the tensor path
  int check(dmo_ctx* ctx, const char* who, int precision, int d);
  // chunk size and scratch for P candidates against Npad-row planes
  int alloc(dmo_ctx* ctx, int64_t P, int64_t Npad, int planes, bool want_var);
  // the variance partial sums of one chunk of Pcpad candidates, its K_* plane already produced
  int contract(dmo_ctx* ctx, const GpVarOps& ops, int64_t Pcpad);
  // fails when the tensor pipeline's watchdog tripped (synchronises)
  int watchdog(dmo_ctx* ctx);
};

template <typename T>
int upload(dmo_ctx* ctx, DevBuf<T>& dst, const std::vector<T>& src) {
  DMO_TRY(dst.alloc(ctx, src.size()));
  DMO_CUDA(cudaMemcpyAsync(dst.p, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return DMO_OK;
}

// ---- dense float64 helpers of the variational posterior (gp_variational.cu), shared with its training (gp_variational_fit.cu)
// C[i][j] = alpha sum_k A(i, k) B(k, j) + (i == j ? diag : 0), i < m, j < n (rows of ldc), A(i, k) = A[i sai + k sak],
// B(k, j) = B[k sbk + j sbj]; every output one fixed-order chain.  Not synchronised.
int sv_gemm(dmo_ctx* ctx, int64_t m, int64_t n, int64_t K, double alpha, const double* A, int64_t sai, int64_t sak, const double* B,
            int64_t sbk, int64_t sbj, double diag, double* C, int64_t ldc);
// O = s J C' J (rows of ldo) for a row-major n x n lower-triangular C (J reverses the order): lower triangular
int sv_flip(dmo_ctx* ctx, const double* C, int64_t n, double s, double* O, int64_t ldo);
// dmo_svgp_predict before its output mix: the latent moments fm (L,P) and fv (L,P) (fv NULL: means only) of the DEVICE
// inputs X (P,d), with up checked by the caller (GpUnitPredict::check).  Not synchronised; the caller runs up.watchdog.
int svgp_latent_moments(dmo_ctx* ctx, dmo_svgp* sv, GpUnitPredict& up, const double* X, int64_t P, double* fm, double* fv);
// dmo_svgp_predict on DEVICE arrays without its trailing waits: X (P, d), mean / var (P, M), var may be null.  The mean
// does not depend on whether var is given.  up checked by the caller, which runs up.watchdog.
int svgp_predict_device(dmo_ctx* ctx, dmo_svgp* sv, GpUnitPredict& up, const double* X, int64_t P, double* mean, double* var);
// input dimensions and outputs of a variational or deep-GP posterior
void svgp_dims(const dmo_svgp* sv, int* d, int* M);
void dgp_dims(const dmo_dgp* g, int* d, int* T);
// dmo_dgp_predict on DEVICE arrays without its trailing waits (eps / var may be null; the mean does not depend on var:
// the last layer's mean-only kernel accumulates it in the same order).  up checked by the caller, which runs
// up.watchdog; stream_id < 2^54 checked by the caller.
int dgp_predict_device(dmo_ctx* ctx, dmo_dgp* g, GpUnitPredict& up, const double* X, int64_t P, uint64_t seed, uint64_t stream_id,
                       double* eps, double* mean, double* var);

// The surrogate posterior of a resident step (step.cu, smpso.cu).  DMO_POSTERIOR_GP with var_route_mean: the mean of the
// predict with variance, without the variance (gp_predict_device); the variational and deep-GP means never depend on the
// variance, which these steps do not form (the deep GP's hidden layer still contracts its own: its spread places the last
// layer's inputs).  mean_f32: the offspring's mean is rounded to float32 before the truncation and the record.
struct StepPosterior {
  int kind = DMO_POSTERIOR_GP;
  dmo_gp* gp = nullptr;
  dmo_svgp* sv = nullptr;
  dmo_dgp* dg = nullptr;
  uint64_t draw_seed = 0, draw_stream = 0;  // the deep GP's Philox key (Monte Carlo draws)
  bool var_route_mean = false;
  bool mean_f32 = false;
};
// The posterior given by kind and handle to a recorded step, checked against the population's d and M: an unknown kind, a
// null handle, a precision other than DMO_GP_FP64 / DMO_GP_TENSOR when var_route_mean (AUTO's refinement follows the
// variance), a posterior of other dimensions and a deep GP's draw_stream >= 2^54 are refused with DMO_ERR_ARG.  Messages
// are prefixed by `who`.
int step_posterior(dmo_ctx* ctx, const char* who, int kind, void* posterior, uint64_t draw_seed, uint64_t draw_stream, bool var_route_mean,
                   bool mean_f32, int precision, int d, int M, StepPosterior* post);
// the posterior mean (and, for the exact GP only, variance) of the P rows of the device array X; only the exact GP's AUTO
// route with a variance may leave its read-back pending in gpp.  The variational and deep-GP routes wait only for the
// tensor pipeline's watchdog, when a contraction ran.  Messages are prefixed by `who`.
int step_predict(dmo_ctx* ctx, const char* who, const StepPosterior& post, const double* X, int64_t P, double* mean, double* var,
                 int precision, GpPending* gpp);
// Latent l's device operands, for a caller that forms its own K_*: the operator planes O0 = s Lz^-1 and O1 = s T (rows
// of Npad, zero padded), the mean vector a_l (Npad,), the scaled inducing points XtT (d, Npad) and 1 / ell (d,).
struct SvLatentView {
  const double *O0, *O1, *A, *XtT, *inv_ls;
  int64_t Npad;
};
int svgp_latent_view(const dmo_svgp* sv, int l, SvLatentView* v);

// ---- multitask model (gp_multitask.cu): the block factorisation shared by dmo_mtgp_create and dmo_mtgp_lml_grad --
constexpr int MT_MAX = 8;        // tasks per model
constexpr int MT_FIT_DMAX = 90;  // input dimensions dmo_gp_fit takes
struct MtBlocks {
  std::vector<double> hx, ls, hB, hD, hw, hb;  // the inputs, copied to the host
  std::vector<double> sqD, lam, Q;             // sqrt(D_s); D^-1/2 B D^-1/2 = Q diag(lam) Q' (Q row-major, Q[s * M + j])
  std::vector<double> xs;                      // (N, d) x_n / l
  std::vector<double> blk_lml;                 // (M,) per-block log marginal likelihoods
  double lml = 0.0;                            // log p(Y)
  DevBuf<double> Lf;                           // (M, N, N) lower Cholesky factors of lambda_j K_x + I
};
// Argument checks (messages prefixed by `who`), Jacobi, rotated residuals and dmo_gp_fit on the M blocks; alpha_out
// ((M, N), host or device) receives the block alphas a_j.  Returns after dmo_gp_fit's synchronisation.
int mtgp_blocks_fit(dmo_ctx* ctx, const char* who, int64_t N, int d, int M, const double* X_train, const double* Y,
                    const double* length_scale, const double* B, const double* D, const double* weight, const double* bias,
                    MtBlocks& mb, double* alpha_out);

// The multitask producers (gp_multitask.cu), also used by the variational posterior (gp_variational.cu).
// xs = ((X - xlb) / xrg) * inv_ls, (P, d)
int mt_scale_inputs(dmo_ctx* ctx, const double* X, int64_t P, int d, const double* xlb, const double* xrg, const double* inv_ls,
                    double* xs);
// training points per producer block: mpart has Npad / mt_kstar_span(tensor) row-block planes
int64_t mt_kstar_span(bool tensor);
// the producer's (d, Npad) training inputs: XtT[k][n] = x(n, k), the scaled coordinate k of point n < N; zero padded
template <typename F>
std::vector<double> mt_xt_transposed(int64_t N, int d, int64_t Npad, F x) {
  std::vector<double> xtT((size_t)d * Npad, 0.0);
  for (int64_t n = 0; n < N; ++n)
    for (int k = 0; k < d; ++k) xtT[(size_t)k * Npad + n] = x(n, k);
  return xtT;
}
// One unit-scale Matern-5/2 K_* plane k(xs_p, XtT[:, n]) for the candidates p_base + [0, Pcpad) (float64 Ks, or fp16 hi / lo
// Kh / Kl scaled by 2^k_exp[0]; NULL: not written) and the partial sums mpart[z][j][p] of k' A_j, j < M <= MT_MAX.
// tensor: d <= 64.
int mt_kstar_produce(dmo_ctx* ctx, bool tensor, const double* xs, int64_t P, int64_t p_base, int64_t Pcpad, const double* XtT, int64_t N,
                     int64_t Npad, int d, int M, const double* A, const int* k_exp, double* Ks, uint16_t* Kh, uint16_t* Kl,
                     double* mpart, int64_t mp_ld);
