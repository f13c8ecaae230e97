/*
 * dmosopt_b200 -- C ABI of the H100-native surrogate-generation hot path.
 *
 * The reference (dmosopt @ 5cd63e4c) is pure Python and has NO foreign-function
 * interface; this header is new surface that sits directly under the Python
 * plugin classes (dmosopt_b200.NSGA2 / AGEMOEA / SMPSO / CMAES, GPR_Matern ...)
 * which dmosopt loads by import path (dmosopt/config.py:5-11,
 * dmosopt/MOASMO.py:256-259,516-519).  Every entry point names the reference
 * function it replaces (file:line relative to the reference checkout).
 *
 * Conventions
 *   - plain C, no C++ / torch types; every function returns an int status
 *     (DMO_OK == 0) and never throws; dmo_last_error(ctx) gives the message.
 *   - matrices are row-major (C order), double unless stated; index outputs
 *     are int64 (numpy intp), ranks int32.
 *   - every array pointer may be HOST memory (pageable or pinned) or DEVICE
 *     memory of the context's GPU; the library detects which
 *     (cudaPointerGetAttributes) and stages host buffers through the
 *     context's stream.  The caller owns all buffers; the library owns only
 *     its context, its stream-ordered scratch memory and the objects it
 *     creates (dmo_gp).
 *   - one context per GPU and per calling thread (not re-entrant); all work is
 *     issued on the context's own stream and calls return after the results
 *     are in the caller's buffers (host outputs) or enqueued (device outputs;
 *     call dmo_synchronize before reading them from another stream).
 */
#ifndef DMOSOPT_B200_H
#define DMOSOPT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMO_OK 0
#define DMO_ERR_CUDA 1        /* a CUDA runtime call or kernel failed           */
#define DMO_ERR_ARG 2         /* bad shape / null pointer / unsupported size    */
#define DMO_ERR_STATE 3       /* object used before it was initialised          */
#define DMO_ERR_UNSUPPORTED 4 /* valid request that this build does not cover   */
#define DMO_ERR_INTERNAL 5    /* watchdog / consistency check tripped           */

/* distance metrics of MOEA.sortMO (dmosopt/MOEA.py:256-266) */
#define DMO_METRIC_NONE 0
#define DMO_METRIC_CROWDING 1  /* indicators.crowding_distance_metric  */
#define DMO_METRIC_EUCLIDEAN 2 /* indicators.euclidean_distance_metric */

/* stationary kernels of the sklearn surrogates (dmosopt/model.py:1227-1229, 1318-1320) */
#define DMO_KERNEL_MATERN52 0
#define DMO_KERNEL_RBF 1

/* arithmetic used for the GP posterior variance contraction */
#define DMO_GP_FP64 0   /* CUDA-core float64 everywhere: matches sklearn to ~1e-10               */
#define DMO_GP_TENSOR 1 /* wgmma split-fp16 (3 MMAs / product), fp32 accumulate in registers     */
#define DMO_GP_AUTO 2   /* tensor path where a per-model calibration against the float64 path   *
                         * holds 1e-5, float64 for the rest (rows with small variance, badly   *
                         * conditioned models): see dmo_gp_auto_info                            */

typedef struct dmo_ctx dmo_ctx;
typedef struct dmo_gp dmo_gp;
typedef struct dmo_mtgp dmo_mtgp;
typedef struct dmo_svgp dmo_svgp;
typedef struct dmo_feas dmo_feas;

/* ---- context ----------------------------------------------------------- */
int dmo_version(void);
int dmo_create(int device, dmo_ctx** out);
int dmo_destroy(dmo_ctx* ctx);
const char* dmo_last_error(dmo_ctx* ctx);
int dmo_synchronize(dmo_ctx* ctx);
void* dmo_stream(dmo_ctx* ctx);             /* the context's cudaStream_t */
int64_t dmo_launch_count(dmo_ctx* ctx);     /* kernels launched by this context so far */
int dmo_sm_count(dmo_ctx* ctx);
/* CUDA-event stopwatch on the context's stream (bench.py times kernels with it) */
int dmo_timer_begin(dmo_ctx* ctx);
int dmo_timer_end(dmo_ctx* ctx, float* elapsed_ms);
/* pinned host memory for callers that want asynchronous staging */
int dmo_host_alloc(void** out, uint64_t bytes);
int dmo_host_free(void* p);
/* device memory for callers that keep populations resident */
int dmo_device_alloc(dmo_ctx* ctx, void** out, uint64_t bytes);
int dmo_device_free(dmo_ctx* ctx, void* p);
int dmo_memcpy(dmo_ctx* ctx, void* dst, const void* src, uint64_t bytes); /* any direction, stream ordered + sync */
/* bytes staged so far between host buffers and the GPU by this context */
int dmo_transfer_bytes(dmo_ctx* ctx, uint64_t* h2d, uint64_t* d2h);
/* per-kernel CUDA-event timers: enable(1) clears and starts recording, report() writes "name ms count" lines */
int dmo_profile_enable(dmo_ctx* ctx, int on);
int dmo_profile_report(dmo_ctx* ctx, char* buf, uint64_t cap);
/* in-place float64 -> float32 -> float64 rounding of a device array (the reference's float32 state arrays,
 * dmosopt/NSGA2.py:228-230 + dmosopt/MOASMO.py:64), for callers that keep the population resident */
int dmo_round_f32(dmo_ctx* ctx, double* a, int64_t n);
/* writes zeros through a scratch buffer larger than L2 (bench L2 flush) */
int dmo_flush_l2(dmo_ctx* ctx);

/* ---- A1/A2: non-dominated rank ------------------------------------------
 * replaces dda.dda_ens (dmosopt/dda.py:97-152), the rank used by every sortMO.
 * Y (n, M) -> rank (n,), the canonical Pareto front index; identical vectors are
 * mutually non-dominating (dda.py:108-115).  Equal to dda_ens whenever
 * objective 0 is tie-free.  1 <= M <= 16. */
int dmo_rank_nd(dmo_ctx* ctx, const double* Y, int64_t n, int M, int32_t* rank);

/* ---- A3/A4: distance metrics ---------------------------------------------
 * replace indicators.crowding_distance_metric (dmosopt/indicators.py:12-51) and
 * indicators.euclidean_distance_metric (:54-62).  Bit-identical float64. */
int dmo_crowding_distance(dmo_ctx* ctx, const double* Y, int64_t n, int M, double* D);
int dmo_euclidean_distance(dmo_ctx* ctx, const double* Y, int64_t n, int M, double* D);

/* ---- A5: sortMO / orderMO / remove_worst ----------------------------------
 * dmosopt/MOEA.py:242-347, 398-423.
 * dmo_order_mo: perm = np.lexsort((-extra_k..., -ydist, rank)); outputs are in sorted
 *   order.  extra_desc_keys: n_extra host-evaluated x-metrics (feasibility rank,
 *   NSGA2.py:47-49), each (n,), least-significant first; may be NULL.
 *   rank_sorted / dist_sorted may be NULL.
 * dmo_remove_worst: the first `keep` rows of that order gathered from X (n,d) / Y (n,M). */
int dmo_order_mo(dmo_ctx* ctx, const double* Y, int64_t n, int M, int metric,
                 const double* const* extra_desc_keys, int n_extra,
                 int64_t* perm, int32_t* rank_sorted, double* dist_sorted);
int dmo_remove_worst(dmo_ctx* ctx, const double* X, const double* Y, int64_t n, int d, int M,
                     int metric, const double* const* extra_desc_keys, int n_extra, int64_t keep,
                     double* X_out, double* Y_out, int32_t* rank_out, int64_t* perm_out);

/* dmo_remove_worst on the row-wise concatenation [A (na rows); B (nb rows)] without building it on the host
 * (NSGA2.update_strategy stacks the children over the parents, dmosopt/NSGA2.py:205-214). Outputs may alias B. */
int dmo_remove_worst_pair(dmo_ctx* ctx, const double* Xa, const double* Ya, int64_t na, const double* Xb,
                          const double* Yb, int64_t nb, int d, int M, int metric, int64_t keep,
                          double* X_out, double* Y_out, int32_t* rank_out, int64_t* perm_out);
/* dmo_remove_worst_pair with the feasibility rank of `key` (dmo_feas_create) evaluated on the device over [Xa; Xb] as
 * the least significant descending key: np.lexsort((-key, -ydist, rank)), MOEA.remove_worst with
 * x_distance_metrics = [feasibility.rank] (dmosopt/NSGA2.py:54-55).  key's d must equal d. */
int dmo_remove_worst_pair_keys(dmo_ctx* ctx, const double* Xa, const double* Ya, int64_t na, const double* Xb,
                               const double* Yb, int64_t nb, int d, int M, int metric, const dmo_feas* key,
                               int64_t keep, double* X_out, double* Y_out, int32_t* rank_out, int64_t* perm_out);

/* ---- A6: tournament selection ---------------------------------------------
 * replaces MOEA.tournament_selection (dmosopt/MOEA.py:375-395): candidates ordered by
 * lexsort(metrics) (rank primary; AGE-MOEA adds -crowd_dist as secondary,
 * AGEMOEA.py:140-142), P(i-th best) ~ p (1-p)^i, poolsize draws WITHOUT replacement.
 * Implemented in log space (Gumbel-top-k), so it does not underflow for pop > 2150.
 * crowd may be NULL.  u_out (pop,) optionally receives the uniforms used, in candidate
 * order position (for distribution / replay tests). */
int dmo_tournament(dmo_ctx* ctx, const int32_t* rank, const double* crowd, int64_t pop,
                   int64_t poolsize, uint64_t seed, uint64_t stream_id,
                   int64_t* pool_idx, double* u_out);

/* ---- A7/A8: variation operators with explicit uniforms (kernel-level parity) ----
 * MOEA.mutation (dmosopt/MOEA.py:191-212) and MOEA.crossover_sbx (:215-239) applied
 * row-wise: parents / u / children (n, d); di_* / xlb / xub (d,). */
int dmo_mutation_u(dmo_ctx* ctx, const double* parents, const double* u, int64_t n, int d,
                   const double* di_mutation, const double* xlb, const double* xub,
                   double mutation_rate, double* children);
int dmo_sbx_u(dmo_ctx* ctx, const double* parent1, const double* parent2, const double* u,
              int64_t n, int d, const double* di_crossover, const double* xlb, const double* xub,
              double* child1, double* child2);

/* ---- A9: NSGA-II / AGE-MOEA offspring generation ----------------------------
 * replaces the serial loop of NSGA2.generate_strategy (dmosopt/NSGA2.py:142-178; same
 * loop in AGEMOEA.py:144-180): iteration t emits an SBX pair w.p. crossover_prob and
 * then a mutant w.p. mutation_prob, until count >= popsize-1.  The control flow is
 * planned in parallel from counter-based Philox4x32-10 draws (seed, stream_id).
 * pop_x (npop, d); pool_idx (poolsize,) rows of pop_x forming the mating pool.
 * x_gen has room for popsize+1 rows; child_kind (popsize+1,) gets 0/1 = SBX child 1/2,
 * 2 = mutant; n_children the number of rows produced.
 * draws (optional, may be NULL): receives the random draws actually used so the CPU
 * oracle can replay them: T * (5 + 2 d) doubles, T = dmo_nsga2_plan_length(...) planned
 * iterations, layout documented in dmosopt_b200/_lib.py (nsga2_generate).
 * dmo_nsga2_plan_length: the number of loop iterations planned for the given rates
 * (>= 2 popsize + 64; grows as 1 / (2 crossover_prob + mutation_prob) so that mutation-only
 * and low-rate configurations terminate like the reference's while-loop); -1 if the rates
 * are too small to plan. */
int64_t dmo_nsga2_plan_length(int64_t popsize, double crossover_prob, double mutation_prob);
int dmo_nsga2_generate(dmo_ctx* ctx, const double* pop_x, int64_t npop, int d,
                       const int64_t* pool_idx, int64_t poolsize, int64_t popsize,
                       double crossover_prob, double mutation_prob, double mutation_rate,
                       const double* di_crossover, const double* di_mutation,
                       const double* xlb, const double* xub, uint64_t seed, uint64_t stream_id,
                       double* x_gen, int32_t* child_kind, int64_t* n_children, double* draws);

/* ---- A10 + A20: one resident NSGA-II surrogate generation ----------------------
 * the body of MOASMO.optimize's loop (dmosopt/MOASMO.py:105-116) for NSGA2 (dmosopt/NSGA2.py:116-236) with a
 * GP surrogate, population resident in HBM: tournament -> variation -> GP posterior mean [+ variance] ->
 * vstack(children, parents) -> rank + stable truncation -> float32 rounding of the stored objectives
 * (NSGA2.py:228-230) -> optional hypervolume of the survivors (hv_ref / hv_out host pointers, may be NULL).
 * pop_x (pop,d), pop_y (pop,M), rank (pop,) are DEVICE buffers, updated in place; Philox streams
 * stream_id (tournament) and stream_id + 1 (variation) are consumed; n_children (host) receives P.
 * distance_metric: DMO_METRIC_* used to break rank ties in the truncation (NSGA2's own default is
 * "crowding", NSGA2.py:25; MOASMO.epoch constructs it with distance_metric=None, MOASMO.py:370). */
int dmo_nsga2_step(dmo_ctx* ctx, dmo_gp* gp, double* pop_x, double* pop_y, int32_t* rank, int64_t pop,
                   int d, int M, double crossover_prob, double mutation_prob, double mutation_rate,
                   const double* di_crossover, const double* di_mutation, const double* xlb,
                   const double* xub, uint64_t seed, uint64_t stream_id, int precision,
                   int distance_metric, int with_variance, int round_to_f32, const double* hv_ref,
                   int64_t* n_children, double* hv_out);

/* ---- A18: exact-GP posterior (GPR_Matern / GPR_RBF predict) -------------------
 * replaces GPR_Matern.predict / .evaluate (dmosopt/model.py:1254-1275; GPR_RBF :1343-1364),
 * i.e. per objective sklearn GaussianProcessRegressor.predict(return_std=True) ** 2.
 * dmo_gp_create uploads the posterior state once per epoch:
 *   X_train (N,d) normalised inputs; alpha (M,N); L (M,N,N) lower Cholesky factors of
 *   K + noise I (factor_is_inverse = 0) or their inverses L^-1 (factor_is_inverse = 1);
 *   constant (M,), length_scale (M,d) (isotropic = the scalar repeated), noise (M,),
 *   y_mean (M,), y_std (M,), xlb / xub (d,) raw input bounds.
 * dmo_gp_predict: X (P,d) raw inputs -> mean (P,M), var (P,M) (var may be NULL). */
int dmo_gp_create(dmo_ctx* ctx, int64_t N, int d, int M, int kernel, const double* X_train,
                  const double* alpha, const double* factor, int factor_is_inverse,
                  const double* constant, const double* length_scale, const double* noise,
                  const double* y_mean, const double* y_std, const double* xlb, const double* xub,
                  dmo_gp** out);
int dmo_gp_destroy(dmo_ctx* ctx, dmo_gp* gp);
/* N1: the exact-GP fit for given hyper-parameters, per objective m: K = c_m k(X, X; l_m) + (noise_m + jitter) I,
 * L = chol(K), alpha = K^-1 y_m, lml = log p(y_m | theta) -- what GaussianProcessRegressor.fit /
 * .log_marginal_likelihood compute behind GPR_Matern.__init__ (dmosopt/model.py:1214-1251) and what every trial of the
 * SCE-UA hyper-parameter search evaluates (dmosopt/model.py:1419-1753).  X_train (N,d) normalised inputs, y (M,N)
 * normalised targets; scikit-learn's jitter is 1e-10 (its alpha parameter).  L_out (M,N,N), alpha_out (M,N), lml_out (M,)
 * may each be NULL (an SCE-UA trial needs lml only).  Fails with DMO_ERR_ARG when K is not positive definite. */
int dmo_gp_fit(dmo_ctx* ctx, int64_t N, int d, int M, int kernel, const double* X_train, const double* y,
               const double* constant, const double* length_scale, const double* noise, double jitter,
               double* L_out, double* alpha_out, double* lml_out);
/* A19: prior mean of the gpytorch exact GPs (model_gpytorch.EGP_Matern.predict,
 * dmosopt/model_gpytorch.py:2188-2228; GPyTorchExactGPModelMatern with LinearMean, :455-508):
 * after this call dmo_gp_predict returns y_std * (K_* alpha + weight_m . x_n + bias_m) + y_mean,
 * x_n the normalised input; alpha must then be (K + noise I)^-1 (y_n - X_n weight - bias).
 * weight (M,d), bias (M,); both NULL removes the term.  The variance is unaffected. */
int dmo_gp_set_linear_mean(dmo_ctx* ctx, dmo_gp* gp, const double* weight, const double* bias);
int dmo_gp_predict(dmo_ctx* ctx, dmo_gp* gp, const double* X, int64_t P, double* mean,
                   double* var, int precision);
/* What DMO_GP_AUTO decided for this model (runs the one-off calibration if it has not run yet):
 * both arithmetic paths predict 512 probe candidates; mean_tensor bit 0 = the fp32-K_* alpha pass is
 * admitted (predicts with variance), bit 1 unused (0), bit 2 = the mean-only kernel (K_* never written, fp32 kernel values, float64 partial sums) is admitted
 * for predicts without variance; var_tensor = 1 when the wgmma variance is admitted; errors relative to max(|mean|, y_std) and to
 * the prior variance, margins documented in csrc/gp.cu; theta: rows whose tensor variance is
 * below theta * prior are recomputed in float64; last_refined: rows the last AUTO predict recomputed
 * (= P when the whole call ran in float64).  Any output pointer may be NULL. */
int dmo_gp_auto_info(dmo_ctx* ctx, dmo_gp* gp, int* mean_tensor, int* var_tensor, double* mean_err,
                     double* var_err, double* theta, int64_t* last_refined);
/* Objectives that share a posterior covariance: dmo_gp_create puts objective m in the group of an earlier
 * objective l when their constant, length scales and uploaded factor planes are bitwise equal (noise may differ).
 * Each group's L^-1, K_* and variance contraction are computed once and the variance is scaled per objective.
 * n_groups receives the number of groups G; group_of (M,) host array, may be NULL, receives each objective's
 * group, numbered 0 .. G-1 in order of first appearance. */
int dmo_gp_covariance_groups(dmo_ctx* ctx, dmo_gp* gp, int* n_groups, int* group_of);

/* ---- A19: multitask exact-GP posterior (MEGP_Matern predict) -------------------
 * replaces model_gpytorch.MEGP_Matern.predict (dmosopt/model_gpytorch.py:1872-1919; model :510-571): one
 * ExactGP over N points x M tasks, covariance K_x (x) B with K_x the ARD Matern-5/2 kernel (no output scale)
 * and B = F F' + diag(v) (IndexKernel), noise I_N (x) D (MultitaskGaussianLikelihood, D_t = task noise t +
 * global noise), prior mean w_t . x_n + b_t per task (MultitaskMean(LinearMean)).
 * dmo_mtgp_create uploads the posterior state once per epoch:
 *   X_train (N,d) normalised inputs; Y (N,M) normalised targets; length_scale (d,); B (M,M) symmetric positive
 *   semi-definite; D (M,) > 0; weight (M,d), bias (M,); y_mean, y_std (M,); xlb / xub (d,) raw input bounds.
 *   1 <= M <= 8, d <= 90.  The posterior splits exactly into M single-output GPs over the eigenvectors of
 *   D^-1/2 B D^-1/2 (host Jacobi, deterministic), each factorised in float64 as dmo_gp_fit does.
 *   lml_out (may be NULL) receives the exact log marginal likelihood log p(Y).
 * dmo_mtgp_predict: X (P,d) raw inputs -> mean (P,M), var (P,M) (var may be NULL; it includes D):
 *   precision DMO_GP_FP64 or DMO_GP_TENSOR (d <= 64); DMO_GP_AUTO is not offered (DMO_ERR_ARG). */
int dmo_mtgp_create(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* Y,
                    const double* length_scale, const double* B, const double* D, const double* weight,
                    const double* bias, const double* y_mean, const double* y_std, const double* xlb,
                    const double* xub, double* lml_out, dmo_mtgp** out);
int dmo_mtgp_predict(dmo_ctx* ctx, dmo_mtgp* mt, const double* X, int64_t P, double* mean, double* var,
                     int precision);
int dmo_mtgp_destroy(dmo_ctx* ctx, dmo_mtgp* mt);
/* dmo_mtgp_lml_grad: the exact log marginal likelihood of the same model and its gradient, for training.
 *   Arguments and limits as dmo_mtgp_create (host or device pointers).  lml_out (scalar) is bit-identical to what
 *   dmo_mtgp_create reports for the same inputs; the gradients are d lml / d length_scale (d,), d lml / d B (M,M,
 *   entries treated as independent), d lml / d D (M,), d lml / d weight (M,d), d lml / d bias (M,).  Float64,
 *   deterministic (fixed-order reductions); returns when the outputs are filled. */
int dmo_mtgp_lml_grad(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* Y,
                      const double* length_scale, const double* B, const double* D, const double* weight,
                      const double* bias, double* lml_out, double* g_length_scale, double* g_B, double* g_D,
                      double* g_weight, double* g_bias);
/* dmo_gp_lml_grad: training of M independent exact GPs (EGP_Matern): per objective m the exact log marginal
 *   likelihood of y_m under K_m = s_m Matern52(X / l_m) + sigma2_m I (no jitter) with the linear prior mean
 *   X w_m + b_m, and its gradient.  X_train (N,d) normalised inputs, y (M,N) normalised targets (as dmo_gp_fit),
 *   length_scale and weight (M,d), outputscale, noise and bias (M,); host or device pointers; 1 <= M <= 8, d <= 90.
 *   Outputs, same shapes: lml_out (M,), d lml_m / d length_scale_m (M,d), / d outputscale_m, / d noise_m (M,),
 *   / d weight_m (M,d), / d bias_m (M,).  A K_m that is not positive definite gives DMO_ERR_ARG naming the objective.
 *   Float64, deterministic: objective m's outputs are bit-identical whichever other objectives are evaluated with it,
 *   in any order, and on repeated calls.  Returns when the outputs are filled. */
int dmo_gp_lml_grad(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* y,
                    const double* length_scale, const double* outputscale, const double* noise, const double* weight,
                    const double* bias, double* lml_out, double* g_length_scale, double* g_outputscale,
                    double* g_noise, double* g_weight, double* g_bias);

/* ---- variational GP posterior (SVGP_Matern / VGP_Matern / SIV_Matern / SPV_Matern / CRV_Matern predict) --------
 * replaces predict_f of the GPflow posteriors behind dmosopt/model.py's variational surrogates (:290-318, 509-537,
 * 730-757, 953-981, 1143-1172): per latent GP l a whitened variational posterior q(v) = N(q_mu_l, q_sqrt_l q_sqrt_l')
 * over inducing points Z_l with kernel variance_l Matern52(. / length_scale_l) (ARD), zero mean, and jitter added to
 * K(Z, Z); the variance is that of the latent f (no likelihood noise) and is not clamped.
 * dmo_svgp_create: 1 <= L, M <= 8 latents and outputs, 1 <= Z <= 8192 inducing points per latent, 1 <= d <= 90;
 *   Zpts (L,Z,d) normalised inputs; variance (L,) > 0; length_scale (L,d) > 0; q_mu (L,Z); q_sqrt (L,Z,Z) lower
 *   triangular (a non-zero above the diagonal is DMO_ERR_ARG), any rank; W (M,L) output mixing (NULL: identity, M == L);
 *   y_mean, y_std (M,); y_var_scale (M,) multiplies the variance (NULL: y_std^2); xlb, xrng (d,) with xrng > 0:
 *   x_n = (x - xlb) / xrng.  Latents with bitwise equal Z planes and length scales share one K_* plane per predict.
 * dmo_svgp_predict: X (P,d) raw inputs -> mean (P,M) = y_std (W g_mean) + y_mean, var (P,M) = ((W o W) g_var) y_var_scale
 *   (var may be NULL); precision DMO_GP_FP64 or DMO_GP_TENSOR (d <= 64); DMO_GP_AUTO is not offered (DMO_ERR_ARG).
 * dmo_svgp_groups: the number of distinct K_* planes and of operator planes the variance contracts per candidate.
 * dmo_svgp_optimal_q: the closed-form optimum of q for a Gaussian likelihood (Titsias 2009) in whitened coordinates, per
 *   latent: A = Lz^-1 K(Z, X), B = I + A A' / noise, q_mu = B^-1 A y / noise, q_sqrt q_sqrt' = B^-1 (q_sqrt lower
 *   triangular).  X (N,d) normalised inputs, y (L,N) normalised targets, Zpts / variance / length_scale as above, noise
 *   (L,) > 0; outputs q_mu (L,Z), q_sqrt (L,Z,Z).  Not defined for coupled latents (CRV).
 *   inducing_is_data != 0 (GPflow's VGP): the inducing points are X itself (Zpts ignored, may be NULL; Z == N) and
 *   f(X) = Lz v, so A = Lz' -- the data term sees K(X, X) + jitter I, and the posterior is the exact GP with noise
 *   noise + jitter.  With inducing_is_data = 0 and Z = X (SVGP with every point) the data term sees K(X, X) without the
 *   jitter; that posterior equals the exact GP only as the jitter goes to 0.
 *   Cost: dmo_svgp_create runs a Householder QR per latent (2 (Z - 1) launches, ~4/3 Z^3 flop) whatever q is. */
int dmo_svgp_create(dmo_ctx* ctx, int L, int M, int64_t Z, int d, const double* Zpts, const double* variance,
                    const double* length_scale, const double* q_mu, const double* q_sqrt, const double* W, double jitter,
                    const double* y_mean, const double* y_std, const double* y_var_scale, const double* xlb,
                    const double* xrng, dmo_svgp** out);
int dmo_svgp_predict(dmo_ctx* ctx, dmo_svgp* sv, const double* X, int64_t P, double* mean, double* var, int precision);
int dmo_svgp_groups(dmo_ctx* ctx, dmo_svgp* sv, int* n_groups, int* n_planes);
int dmo_svgp_destroy(dmo_ctx* ctx, dmo_svgp* sv);
int dmo_svgp_optimal_q(dmo_ctx* ctx, int64_t N, int64_t Z, int d, int L, const double* X, const double* y,
                       const double* Zpts, const double* variance, const double* length_scale, const double* noise,
                       double jitter, int inducing_is_data, double* q_mu_out, double* q_sqrt_out);

/* ---- training of the variational surrogates (gp_variational_fit.cu) ------------------------------------------------
 * A dmo_svgp_fit is the device-resident training state of one GPflow model: L <= 8 whitened latents over one set of
 * inducing points, mixed into M <= 8 outputs by W (M,L) (NULL: the identity, M == L).  SVGP_Matern and VGP_Matern are
 * one state per output (L = M = 1), SIV / SPV / CRV one state for the whole model.  q_l is held in natural
 * parameters (Lambda_l = S_l^-1, theta1_l = Lambda_l m_l) with its factor kept current; it starts at N(0, I).
 * dmo_svgp_fit_create: X (N,d) normalised inputs, Y (M,N) normalised targets, Zpts (Z,d) the inducing points shared by
 *   the latents (1 <= Z <= 8192, d <= 90); inducing_is_data != 0 is GPflow's VGP: Z = X (Zpts ignored, Z == N),
 *   f(X) = Lz v, and every call takes the full data.  jitter is added to K(Z, Z).
 * Every call takes the model's hyper-parameters -- variance (L,) > 0, length_scale (L,d) > 0, noise (M,) > 0 (one
 * likelihood variance per output; a model with one variance passes copies), W (M,L) or NULL -- and one minibatch:
 * batch (B,) int64 indices into [0, N), 1 <= B <= N (VGP: a permutation of [0, N)); the data term is scaled by N / B.
 * A K(Z, Z) + jitter I that is not positive definite gives DMO_ERR_ARG naming the latent.
 * dmo_svgp_fit_natgrad: one natural-gradient step on q with step gamma in (0, 1] (GPflow's NaturalGradient, XiNat
 *   parameters, Gaussian likelihood), in place: Lambda_l <- (1 - g) Lambda_l + g (I + (N / B) c_l A_l A_l'),
 *   theta1_l <- (1 - g) theta1_l + g (N / B) A_l r~_l, c_l = sum_m W_ml^2 / noise_m, r~_l = sum_m W_ml (y_m - sum_{l' != l}
 *   W_ml' mu_l') / noise_m.  At gamma = 1 on the full batch with one latent this is dmo_svgp_optimal_q's optimum.
 * dmo_svgp_fit_elbo_grad: the ELBO pieces at the current q -- ell_out (M,) the expected log likelihood of each output
 *   over the batch times N / B, kl_out (L,) KL(q_l || N(0, I)) -- and, when g_variance, g_length_scale and g_noise are
 *   not NULL, d ELBO / d variance (L,), d length_scale (L,d), d noise (M,) and (g_W, needs W) d W (M,L) at fixed q.
 * dmo_svgp_fit_q: q_mu (L,Z) and lower-triangular q_sqrt (L,Z,Z), the input of dmo_svgp_create.
 * Host or device pointers; float64; deterministic (fixed-order reductions, no atomics): repeated calls are
 * bit-identical.  Each call returns when its outputs are filled. */
typedef struct dmo_svgp_fit dmo_svgp_fit;
int dmo_svgp_fit_create(dmo_ctx* ctx, int64_t N, int d, int M, int L, int64_t Z, const double* X, const double* Y,
                        const double* Zpts, int inducing_is_data, double jitter, dmo_svgp_fit** out);
int dmo_svgp_fit_destroy(dmo_ctx* ctx, dmo_svgp_fit* st);
int dmo_svgp_fit_natgrad(dmo_ctx* ctx, dmo_svgp_fit* st, const int64_t* batch, int64_t B, const double* variance,
                         const double* length_scale, const double* noise, const double* W, double gamma);
int dmo_svgp_fit_elbo_grad(dmo_ctx* ctx, dmo_svgp_fit* st, const int64_t* batch, int64_t B, const double* variance,
                           const double* length_scale, const double* noise, const double* W, double* ell_out,
                           double* kl_out, double* g_variance, double* g_length_scale, double* g_noise, double* g_W);
int dmo_svgp_fit_q(dmo_ctx* ctx, dmo_svgp_fit* st, double* q_mu_out, double* q_sqrt_out);

/* ---- two-layer deep GP posterior (MDSPP_Matern / MDGP_Matern predict) ------------------------------------------------
 * replaces the predict of gpytorch's DSPP / DeepGP behind dmosopt/model_gpytorch.py's MDSPP_Matern (:991-1306) and
 * MDGP_Matern (:1308-1620): two whitened variational GP layers with Matern-5/2 kernels (csrc/gp_deep.cu).
 * dmo_dgp_create: hidden layer of H units over d inputs -- Z1pts (H,Z1,d) normalised inducing points, s1 (H,) output
 *   scales, ls1 (H,d) length scales, q_mu1 (H,Z1), q_sqrt1 (H,Z1,Z1) lower triangular, prior mean w1 . x_n + b1 (w1 (d,))
 *   shared by every unit; last layer of T tasks over the H hidden outputs -- Z2pts (T,Z2,H), s2 (T,), ls2 (T,H), q_mu2
 *   (T,Z2), q_sqrt2 (T,Z2,Z2), constant prior mean c2; noise (T,) the task noise plus the global noise; jitter is added to
 *   K(Z, Z) and k(x, x) in both layers; min_variance floors the hidden variance and every site's predictive variance.
 *   quad_sites (n_sites,H) non-NULL: quadrature sites (DSPP); NULL: n_sites Monte Carlo draws per predict (DeepGP).
 *   y_mean, y_std (T,); xlb, xrng (d,), x_n = (x - xlb) / xrng.  1 <= H, T <= 8, 1 <= n_sites <= 64, Z1, Z2 <= 8192,
 *   d <= 90.  DMO_ERR_ARG names the problem: a q_sqrt that is not lower triangular, xrng <= 0, a non-finite or
 *   non-positive scale, length scale or noise, or a K(Z, Z) + jitter I that is not positive definite (with its layer and
 *   unit).
 * dmo_dgp_predict: X (P,d) raw inputs -> mean (P,T), var (P,T) (may be NULL) averaged over the n_sites sites:
 *   u_j = mean1 + e_j o sqrt(var1), e_j the quadrature sites or N(0, I) draws from Philox4x32-10 keyed by seed with the
 *   counter (candidate, site * H + h, stream_id < 2^54) -- independent of chunking and of T.  eps_out (n_sites,P,H), may
 *   be NULL, receives the e_j used.  precision DMO_GP_FP64, or DMO_GP_TENSOR (d <= 64: the hidden variance through the
 *   split-fp16 contraction); the last layer is always float64.  DMO_GP_AUTO is refused.
 * Host or device pointers; deterministic (fixed-order sums): repeated calls are bit-identical. */
typedef struct dmo_dgp dmo_dgp;
int dmo_dgp_create(dmo_ctx* ctx, int d, int H, int T, int64_t Z1, int64_t Z2, const double* Z1pts, const double* s1,
                   const double* ls1, const double* q_mu1, const double* q_sqrt1, const double* w1, double b1,
                   const double* Z2pts, const double* s2, const double* ls2, const double* q_mu2, const double* q_sqrt2,
                   double c2, const double* noise, double jitter, double min_variance, int n_sites,
                   const double* quad_sites, const double* y_mean, const double* y_std, const double* xlb,
                   const double* xrng, dmo_dgp** out);
int dmo_dgp_predict(dmo_ctx* ctx, dmo_dgp* g, const double* X, int64_t P, uint64_t seed, uint64_t stream_id,
                    double* eps_out, double* mean, double* var, int precision);
int dmo_dgp_destroy(dmo_ctx* ctx, dmo_dgp* g);

/* ---- two-layer deep GP training (MDSPP_Matern / MDGP_Matern fit) ---------------------------------------------------
 * A dmo_dgp_fit is the device-resident training state of gpytorch's DSPP / DeepGP model behind MDSPP_Matern and
 * MDGP_Matern (csrc/gp_deep_fit.cu): X (N,d) normalised inputs, Y (N,T) normalised targets, a flat float64 vector of raw
 * parameters, its gradient and the Adam moments.  The raw vector, in order: hidden inducing points Z1 (Z1,d) shared by
 * the H units, raw length scales (H,), raw output scales (H,), variational means (H,Z1), chol_variational_covar
 * (H,Z1,Z1), linear-mean weights (d,) and bias (1); last-layer inducing points (T,Z2,H), raw length scales (T,), raw
 * output scales (T,), variational means (T,Z2), chol_variational_covar (T,Z2,Z2), constant mean (1); raw task noises
 * (T,), raw global noise (1); with quadrature the sites (n_sites,H).  Transforms: output scale softplus; length scale
 * softplus, or lo + (hi - lo) sigmoid with lengthscale_bounds (2,) non-NULL; noises 1e-4 + softplus; the rest
 * untransformed (chol masked to its lower triangle).
 * dmo_dgp_fit_create: 1 <= H, T <= 8, 1 <= Z1, Z2 <= 128, d <= 90, 1 <= batch_max <= N, n_sites * batch_max <= 65536
 *   (n_sites: the quadrature sites, or MDGP's draws per row).  The raw vector starts at zero.
 * dmo_dgp_fit_set_params / get_params: the raw vector (n its length).
 * dmo_dgp_fit_loss_grad: the minibatch loss -ELBO / B of the rows batch (B,) at the current parameters into *loss_out and
 *   its gradient by the raw vector into grad_out (may be NULL; kept for adam_step).  Without quadrature the draws are
 *   eps_in (n_sites,B,H) when given, else N(0,1) from Philox4x32-10 keyed by seed with the counter (step, row, site *
 *   H + h); eps_out (n_sites,B,H), may be NULL, receives the draws used.
 * dmo_dgp_fit_adam_step: one torch.optim.Adam step (betas 0.9 / 0.999, eps 1e-8) with the last gradient.
 * dmo_dgp_fit_epoch: every step of one epoch -- batches perm[b B : (b + 1) B] of the permutation perm (N,) of
 *   range(N), the last one partial, draws keyed by step step0 + b -- each a loss_grad and an Adam step with lr, with no
 *   host synchronisation in between; losses_out (ceil(N / B),) the batch losses.
 * A K(Z, Z) + jitter I that is not positive definite is DMO_ERR_ARG naming its layer and unit.  Host or device
 * pointers; deterministic (fixed-order sums, no atomics): repeated calls are bit-identical. */
typedef struct dmo_dgp_fit dmo_dgp_fit;
int dmo_dgp_fit_create(dmo_ctx* ctx, int64_t N, int d, int H, int T, int64_t Z1, int64_t Z2, int n_sites, int quadrature,
                       int64_t batch_max, const double* X, const double* Y, const double* lengthscale_bounds, double jitter,
                       double min_variance, dmo_dgp_fit** out);
int dmo_dgp_fit_destroy(dmo_ctx* ctx, dmo_dgp_fit* st);
int dmo_dgp_fit_set_params(dmo_ctx* ctx, dmo_dgp_fit* st, const double* raw, int64_t n);
int dmo_dgp_fit_get_params(dmo_ctx* ctx, dmo_dgp_fit* st, double* raw, int64_t n);
int dmo_dgp_fit_loss_grad(dmo_ctx* ctx, dmo_dgp_fit* st, const int64_t* batch, int64_t B, uint64_t seed, uint64_t step,
                          const double* eps_in, double* eps_out, double* loss_out, double* grad_out);
int dmo_dgp_fit_adam_step(dmo_ctx* ctx, dmo_dgp_fit* st, double lr);
int dmo_dgp_fit_epoch(dmo_ctx* ctx, dmo_dgp_fit* st, const int64_t* perm, int64_t B, double lr, uint64_t seed, uint64_t step0,
                      double* losses_out);

/* ---- A16: exact hypervolume ---------------------------------------------------
 * replaces hv.AdaptiveHyperVolume.compute_hypervolume(..., 'box') (dmosopt/hv.py:123-189)
 * -> HyperVolumeBoxDecomposition.compute_hypervolume (dmosopt/hv_box_decomposition.py:86-304)
 * and indicators.Hypervolume._do (dmosopt/indicators.py:244-256).  Minimisation; points not
 * strictly inside ref are ignored (hv.py:159).  True hypervolume (see DESIGN.md for the
 * reference's <=0-coordinate defect).  1 <= M <= 8: chain sums for M <= 5 (M >= 4 is
 * O(n^(M-1))), limit-set recursion for 6 .. 8 objectives (fronts of up to 2048 points; exponential in the worst case, as
 * every exact algorithm, cheap on the mostly non-dominated fronts an optimizer produces). */
int dmo_hypervolume(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref, double* out);
/* The same for a set that carries its non-dominated ranks within the superset it was selected from by rank
 * (the survivors of dmo_remove_worst / MOEA.remove_worst, dmosopt/MOEA.py:398-423): rows with rank > 0 are dominated
 * by a rank-0 row of the same set and add no volume, so the non-dominated filter pass is skipped.  rank (n,) int32. */
int dmo_hypervolume_ranked(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref,
                           const int32_t* rank, double* out);
/* The non-dominated filter in front of the hypervolume and EHVI, on its own: flags (n,) int32, 0 for a rank-0 row,
 * 1 for a dominated one (identical vectors are mutually non-dominating).  The same route as the filter: a float64 scan
 * below 1024 rows, the integer-id scan from 1024 rows, the cell grid for M <= 3 from 8192 rows.  1 <= M <= 16. */
int dmo_nondominated_flags(dmo_ctx* ctx, const double* Y, int64_t n, int M, int32_t* flags);

/* ---- A16: Monte-Carlo hypervolume (2 <= M <= 16) -----------------------------
 * replaces the non-'box' branches of hv.AdaptiveHyperVolume.compute_hypervolume (dmosopt/hv.py:123-241) and
 * compute_hypervolume_fpras / _mcm2rv / _hybrid (dmosopt/hv_adaptive.py:188-855).  F (n,M) host or device, ref (M,).
 * Estimates the volume of the rows strictly inside ref, after their non-dominated filter (the reference passes the
 * unfiltered front; see DESIGN.md section 4.3).  algorithm: DMO_HVMC_HYBRID / _FPRAS / _MCM2RV (epsilon, delta in (0, 1))
 * or _MONTE_CARLO (n_samples uniform points).  Random numbers: Philox keyed by seed and stream_id (< 2^24); the result
 * is bit-identical for the same (front, seed, stream_id).  samples_out: N (successful samples; monte_carlo: points
 * drawn), tests_out: dominance tests (point against one front row) performed: for fpras the budget M1, as the
 * reference counts; for mcm2rv and monte_carlo the rows scanned up to the first dominator of each point, plus one per
 * eta (the reference counts n rows per point, or one per point with its k-d tree); algorithm_out: the estimator that ran
 * (a DMO_HVMC_* code, _HYBRID_FPRAS / _HYBRID_MCM2RV when the hybrid decided after its FPRAS rounds); each may be NULL.
 * FPRAS budgets M1 = 8 (1 + epsilon) n ln(2 / delta) / epsilon^2 must stay below 2^34 tests (DMO_ERR_ARG otherwise). */
#define DMO_HVMC_HYBRID 0
#define DMO_HVMC_FPRAS 1
#define DMO_HVMC_MCM2RV 2
#define DMO_HVMC_MONTE_CARLO 3
#define DMO_HVMC_HYBRID_FPRAS 4
#define DMO_HVMC_HYBRID_MCM2RV 5
int dmo_hypervolume_mc(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref, int algorithm, double epsilon,
                       double delta, int64_t n_samples, uint64_t seed, uint64_t stream_id, double* out,
                       int64_t* samples_out, int64_t* tests_out, int* algorithm_out);

/* ---- A17: HV-improvement (EHVI) candidate selection -----------------------------
 * replaces indicators.HypervolumeImprovement._do (dmosopt/indicators.py:295-313) ->
 * HyperVolumeBoxDecomposition.select_candidates / _compute_batch_ehvi /
 * _decompose_dominated_space (dmosopt/hv_box_decomposition.py:306-437).
 * F (nf,M): the chosen set (its rank-0 subset is taken when nds != 0); means / variances (nc,M);
 * sel (k,) indices of the k largest scores (ties by index); score (nc,) may be NULL. */
int dmo_ehvi_select(dmo_ctx* ctx, const double* F, int64_t nf, const double* means,
                    const double* variances, int64_t nc, int M, const double* ref, int nds,
                    int64_t k, int64_t* sel, double* score);

/* ---- A21: duplicate rows ---------------------------------------------------------
 * replaces MOEA.get_duplicates (dmosopt/MOEA.py:426-437) at its default eps = 1e-16:
 * is_dup[i] = 1 iff an earlier row j < i has ||x_i - x_j||_2 <= eps. */
int dmo_get_duplicates(dmo_ctx* ctx, const double* X, int64_t n, int d, double eps, uint8_t* is_dup);
/* the two-set form MOASMO's resample step uses (dmosopt/MOASMO.py:442, MOEA.get_duplicates(best_x, x_0)):
 * is_dup[i] = 1 when some row j < i of Y (ny, d) lies within eps of row i of X (n, d) -- the reference masks
 * the upper triangle of cdist(X, Y) including the diagonal (MOEA.py:430). */
int dmo_get_duplicates_pair(dmo_ctx* ctx, const double* X, int64_t n, const double* Y, int64_t ny, int d,
                            double eps, uint8_t* is_dup);

/* ---- A11: AGE-MOEA survival score (greedy part) -------------------------------------
 * replaces the O(m^2) greedy loop of AGEMOEA.survival_score (dmosopt/AGEMOEA.py:398-428):
 * yn (m,M) normalised front, nn (m,) = ||yn_i||_p, extreme (n_ext,) pre-selected corner solutions;
 * crowd (m,): inf for the extremes, else the sum of the two smallest distances
 * ||yn_s - yn_r||_p / nn[s] to the already selected set at the moment r is selected. */
int dmo_age_survival(dmo_ctx* ctx, const double* yn, const double* nn, int64_t m, int M, double p,
                     const int32_t* extreme, int n_ext, double* crowd);

/* ---- A12: SMPSO --------------------------------------------------------------------------
 * dmo_smpso_velocity: SMPSO.velocity_vector (dmosopt/SMPSO.py:316-348) for one swarm given its scalar
 *   draws: position (n,d) float32 state, velocity (n,d), the two leader rows (d,) -> out (n,d);
 *   f32_difference != 0 forms (leader - position) in float32 (both operands float32 in NumPy), else float64.
 * dmo_mutate_groups: per_group polynomial mutants per group (swarm), parents drawn uniformly inside each
 *   group of group_size rows of pop_x (SMPSO.py:167-182; MOEA.mutation, MOEA.py:191-212), Philox draws.
 *   children (n_groups*per_group, d); parent_rows (n_groups*per_group,) may be NULL. */
int dmo_smpso_velocity(dmo_ctx* ctx, const float* position, const double* velocity, const double* leader1,
                       const double* leader2, int f32_difference, int64_t n, int d, double w, double c1,
                       double r1, double c2, double r2, double chi, const double* xlb, const double* xub,
                       double* out);
int dmo_mutate_groups(dmo_ctx* ctx, const double* pop_x, int64_t group_size, int64_t n_groups,
                      int64_t per_group, int d, const double* di_mutation, const double* xlb,
                      const double* xub, double mutation_rate, uint64_t seed, uint64_t stream_id,
                      double* children, int64_t* parent_rows);
/* SMPSO with the swarm state resident in HBM: one call per generate / update instead of per-swarm host loops.
 * parm (swarms*pop, d), obj (swarms*pop, M), vel (swarms*pop, d): DEVICE float64 arrays owned by the caller; position and
 * objective values are float32-representable (the reference's state arrays are float32, SMPSO.py:107-113).
 * dmo_smpso_generate (SMPSO.py:143-185): x_gen (2*swarms*pop, d) float32, swarm-major, per swarm pop moved positions
 *   clip(x + v) then pop polynomial mutants of uniformly drawn particles of that swarm (Philox seed / stream_id);
 *   x_gen_f64 (optional, host or device) receives the same float32 values widened to float64 -- what MOEA.generate
 *   hands on after its np.clip (MOEA.py:155).  Either output may be NULL.
 * dmo_smpso_update (SMPSO.py:187-238): consumes rows [0, swarms*pop) of x_gen (float32 when x_is_f32, else float64) and
 *   y_gen (float64) exactly as the reference slices them; scalars (swarms, 8) HOST doubles per swarm = w, c1, r1, c2, r2,
 *   chi, ind1, ind2 drawn by the caller in the reference's order (velocity_vector, SMPSO.py:316-335; ind < 0 = no draw);
 *   the leader with the larger crowding distance of y_gen[swarm slice] goes first.  All velocities are updated against
 *   the old positions, then every swarm keeps the best pop of vstack(offspring slice, particles) (MOEA.remove_worst).
 *   ranks (swarms*pop,) int32 and perm (swarms*pop,) int64 (indices into the swarm's stacked 2*pop rows) are returned;
 *   parm_f32 / obj_f32 (optional) receive the new state as float32 host arrays. */
int dmo_smpso_generate(dmo_ctx* ctx, const double* parm, const double* vel, int swarms, int64_t pop, int d,
                       const double* di_mutation, const double* xlb, const double* xub, double mutation_rate,
                       uint64_t seed, uint64_t stream_id, float* x_gen, double* x_gen_f64);
int dmo_smpso_update(dmo_ctx* ctx, double* parm, double* obj, double* vel, const void* x_gen, int x_is_f32,
                     const double* y_gen, int swarms, int64_t pop, int d, int M, int metric, const double* scalars,
                     const double* xlb, const double* xub, int32_t* ranks, int64_t* perm, float* parm_f32,
                     float* obj_f32);

/* ---- A13 / A15: MO-CMA-ES ----------------------------------------------------------------
 * dmo_cmaes_sample: individuals[i] = x_p + sigma_p * (A_p @ z_i), p = p_idx[i] (dmosopt/CMAES.py:263-267);
 *   sigmas (n_parents, sigma_cols) with sigma_cols = 1 or d, A (n_parents,d,d), z (n,d).
 * dmo_cmaes_update_cholesky: CMAES.updateCholesky (dmosopt/CMAES.py:489-537) for n individuals at once,
 *   in place on A / Ainv (n,d,d) and pc (n,d); z (n,d), psucc (n,). */
int dmo_cmaes_sample(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols,
                     const double* A, int64_t n_parents, const int64_t* p_idx, const double* z, int64_t n,
                     int d, double* individuals);
int dmo_cmaes_update_cholesky(dmo_ctx* ctx, double* A, double* Ainv, double* pc, const double* z,
                              const double* psucc, int64_t n, int d, double cc, double ccov, double pthresh);
/* Device-resident MO-CMA-ES generation / update steps (parents_x, sigmas, factors stay in HBM between generations):
 * dmo_cmaes_generate: dmo_cmaes_sample followed by the reference's global rescale and MOEA.generate's clip,
 *   x = clip((individual / max|individuals|) * (xub - xlb) + xlb, xlb, xub)   (dmosopt/CMAES.py:265-270, MOEA.py:155);
 *   x_out (n, d) host or device.
 * dmo_cmaes_step_z: z[i] = ((x_gen[cand_idx[i]] - parents_x[par_idx[i]]) / (xub - xlb)) / steps[i]  (CMAES.py:359), the
 *   argument of updateCholesky for the chosen offspring; x_gen, parents_x, steps (n, d), z_out (n, d) are DEVICE arrays.
 * dmo_scale_rows: rows[seg_row[s], :] *= factors[e], e = seg_start[s] .. seg_start[s+1]-1, one rounded multiplication
 *   after the other (the per-parent step-size recurrences, CMAES.py:330-383, are sequential); seg_row NULL: row s,
 *   seg_start NULL: factors[s] only.  rows is a DEVICE array of row_elems doubles per row. */
int dmo_cmaes_generate(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols, const double* A,
                       int64_t n_parents, const int64_t* p_idx, const double* z, int64_t n, int d, const double* xlb,
                       const double* xub, double* x_out);
int dmo_cmaes_step_z(dmo_ctx* ctx, const double* x_gen, const int64_t* cand_idx, const double* parents_x,
                     const int64_t* par_idx, const double* xlb, const double* xub, const double* steps, int64_t n, int d,
                     double* z_out);
int dmo_scale_rows(dmo_ctx* ctx, double* rows, int64_t row_elems, int64_t n_seg, const int64_t* seg_row,
                   const int64_t* seg_start, const double* factors, int64_t n_factors);
/* Row gather between DEVICE-resident per-individual state arrays (the (n, d, d) Cholesky factors and (n, d) paths of
 * MO-CMA-ES stay in HBM across generations; CMAES.py:385-411 re-assembles the next parent set from old parents and
 * updated offspring): dst[i, :] = (sel && sel[i] ? alt : src)[idx[i], :], rows of row_elems doubles.  idx (n,) int64 and
 * sel (n,) uint8 (may be NULL, then alt is ignored) may be host arrays. */
int dmo_gather_rows(dmo_ctx* ctx, const double* src, const double* alt, const uint8_t* sel, const int64_t* idx,
                    int64_t n, int64_t row_elems, double* dst);

/* ---- N4: vectorised benchmark objective functions --------------------------------------------
 * replaces the row-at-a-time Python functions of dmosopt/benchmarks/moo_benchmarks.py (dtlz1 :21, dtlz2 :59,
 * dtlz3 :97, dtlz4 :136, dtlz5 :174, dtlz7 :218, wfg1 :286, wfg4 :335, maf1 :384, maf2 :422, maf4 :460) and the example
 * objectives ZDT1 / ZDT3 (examples/example_dmosopt_zdt1.py:9-20, examples/example_dmosopt_zdt3.py:9-21):
 * X (n, n_var) -> Y (n, n_obj), 2 <= n_obj <= 16, n_var >= n_obj except for ZDT (n_obj = 2).  X may be a device address.
 * alpha is DTLZ4's bias exponent (the reference's default is 100), ignored elsewhere.  WFG1 and WFG4 take the reference's
 * default position parameter k = n_obj - 1.  WFG1 refuses shapes whose last maximum window is empty,
 * (n_obj - 2) (n_var - n_obj + 1) >= n_var (np.max of an empty slice raises in the reference): at n_obj >= 4 only a few
 * variables are allowed.  WFG4 returns NaN for such a window (np.mean of an empty slice).  MaF4 multiplies objective i
 * by the correctly rounded double of 10^(2i). */
#define DMO_BM_ZDT1 0
#define DMO_BM_ZDT3 1
#define DMO_BM_DTLZ1 10
#define DMO_BM_DTLZ2 11
#define DMO_BM_DTLZ3 12
#define DMO_BM_DTLZ4 13
#define DMO_BM_DTLZ5 14
#define DMO_BM_DTLZ7 16
#define DMO_BM_WFG1 21
#define DMO_BM_WFG4 24
#define DMO_BM_MAF1 31
#define DMO_BM_MAF2 32
#define DMO_BM_MAF4 34
int dmo_benchmark_eval(dmo_ctx* ctx, int problem, const double* X, int64_t n, int n_var, int n_obj, double alpha,
                       double* Y);

/* ---- Sensitivity analysis: SA_DGSM / SA_FAST -------------------------------------------------
 * replaces SALib's finite_diff / fast_sampler samplers and dgsm.analyze behind dmosopt/sa.py:11-80 (SALib 1.5's
 * definitions, restated in oracle/sa.py).
 * dmo_sa_dgsm_design: base (N, d) points in the unit cube -> X (N (d+1), d): row i (d+1) is base_i, row i (d+1) + 1 + j
 *   is base_i + delta e_j, every row scaled to u (xub - xlb) + xlb with one rounding per operation in that order (no
 *   fused multiply-add), so X is bit-identical to the NumPy expression.
 * dmo_sa_fast_design: X (N d, d) of eFAST (interference factor 4): block i gives parameter i the frequency omega[0] and
 *   the others omega[1..d-1] in order; X[i N + k, j] = (0.5 + arcsin(sin(w_j s_k + phi[i])) / pi) (xub - xlb) + xlb with
 *   s_k = (2 pi / N) k.  arcsin(sin(.)) is evaluated as the triangle wave after an exact reduction modulo pi/2, which
 *   keeps it accurate next to the peaks.  64 < N <= 2^20; reads no input rows.
 * dmo_sa_dgsm_stats: X (N (d+1), d) the DGSM design, Y (N (d+1), M) its outputs, boot_idx (R, N) int32 base indices in
 *   [0, N) of R bootstrap replicates (R <= 4096), z the normal quantile of the confidence level -> vi, vi_std, dgsm,
 *   conf, each (M, d): with q_i = (Y[pert_ij, m] - Y[base_i, m]) / (X[pert_ij, j] - X[base_i, j]), vi = mean(q^2),
 *   vi_std = std(q^2), dgsm = vi (xub_j - xlb_j)^2 / (pi^2 var(Y[base, m])), conf = z std_ddof1(dgsm over the
 *   replicates).  One CTA per (m, j); sums in a fixed order, so the results do not depend on the launch. */
int dmo_sa_dgsm_design(dmo_ctx* ctx, const double* base, int64_t N, int d, const double* xlb, const double* xub,
                       double delta, double* X);
int dmo_sa_fast_design(dmo_ctx* ctx, int64_t N, int d, const double* omega, const double* phi, const double* xlb,
                       const double* xub, double* X);
int dmo_sa_dgsm_stats(dmo_ctx* ctx, const double* X, const double* Y, int64_t N, int d, int M, const double* xlb,
                      const double* xub, const int32_t* boot_idx, int R, double z, double* vi, double* vi_std,
                      double* dgsm, double* conf);

/* ---- Uniform designs: L2 discrepancies and the good-lattice-point search ----------------------
 * replaces the sums of dmosopt/discrepancy.py:38-129 and the candidate scoring of dmosopt/GLP.py:31-70.  A discrepancy
 * is D^2 = D1 + c2 D2 + c3 D3 with D2 = sum_k prod_i row(x_ki) and D3 = sum_{k,j} prod_i pair(x_ki, x_ji); these entry
 * points return D2 and D3 in float64, summed in a fixed order that differs from the reference's (results repeat bit
 * for bit from call to call).
 * dmo_l2_discrepancy_terms: X (n, s), metric DMO_L2_MD2 / CD2 / SD2 / WD2 -> d2[1], d3[1] (WD2 has no D2 sum: d2 = n).
 *   n <= 46340 * 64.
 * dmo_glp_cd2_terms: H (C, s) int64 multipliers in [0, lattice) -> CD2's d2[C], d3[C] of the C rank-1 lattices
 *   x_ki = (u - 0.5) / rows, u = ((k + 1) H[c, i] mod lattice) with 0 replaced by lattice, k < rows.  The designs are
 *   generated inside the kernel.  1 <= C <= 65535 (one grid row each), 2 <= lattice <= 2^31 - 1 (int64 products
 *   (k + 1) h), 1 <= rows <= lattice.
 * dmo_glp_cd2_pairs: the same lattices (L of them, same limits) -> P (L, rows^2): P[l, k rows + j] is the reference's
 *   CD2 pair product for rows (k, j), ((1 + 0.5 |x_ki - 0.5|) + 0.5 |x_ji - 0.5|) - 0.5 |x_ki - x_ji| multiplied over
 *   i = 0 .. s-1 from 1.0, each operation rounded on its own; summed sequentially in row-major order it is the
 *   reference's D3 bit for bit. */
#define DMO_L2_MD2 0
#define DMO_L2_CD2 1
#define DMO_L2_SD2 2
#define DMO_L2_WD2 3
int dmo_l2_discrepancy_terms(dmo_ctx* ctx, int metric, const double* X, int64_t n, int s, double* d2, double* d3);
int dmo_glp_cd2_terms(dmo_ctx* ctx, const int64_t* H, int64_t C, int s, int64_t lattice, int64_t rows, double* d2,
                      double* d3);
int dmo_glp_cd2_pairs(dmo_ctx* ctx, const int64_t* H, int64_t L, int s, int64_t lattice, int64_t rows, double* P);

/* ---- Logistic feasibility model ------------------------------------------------------------------------
 * replaces dmosopt/feasibility.py: per constraint, GridSearchCV over PCA(k) -> StandardScaler -> L1 logistic
 * regression, k in 1 .. d-1, C in Cs, 5 stratified folds, accuracy, refit on all rows.  2 <= d <= 90, 1 <= J <= 32.
 * dmo_feas_fit: X (N, d), 5 <= N <= 65536; labels (J, N) 0/1 and folds (J, N) test-fold ids 0..4 of the J two-class
 *   constraints; datasets s = 6 j + f (f < 5: the rows outside fold f, f = 5: all rows) with pca_mean (6 J, d) and
 *   pca_comps (6 J, d-1, d) the components of each dataset's training rows in descending eigenvalue order.  The
 *   scores are standardised with each dataset's training-row mean and population std -> scaler_mean, scaler_scale
 *   (6 J, d-1).  Problem p = (s nC + c)(d-1) + k-1 minimises C_c sum log(1 + exp(-s_i (z_i[:k] w + b))) + |w|_1 by
 *   proximal Newton (at most max_iter updates) until the minimum-norm subgradient is <= tol max(1, C n_train):
 *   coef (P, d) holds w in [0, k) and b in column d-1; iters (P) Newton updates (-1: the training rows hold one class,
 *   no fit), objective, kkt (P) at the returned w, converged (P) 0/1, correct (P) int64 held-out rows with
 *   (t > 0) == label (-1 without a fit, 0 for f = 5).  1 <= nC <= 16.
 * dmo_feas_create: a fitted model of J constraints from host arrays: k (J) components (0: single-class constraint,
 *   probability 1), mean (J, d), comps (J, d-1, d), smean, sscale, coef (J, d-1), intercept (J); rows past k unused.
 * dmo_feas_eval: X (n, d) -> rank (n) = sum_j p_j / J, proba (J, n) = p_j, decision (J, n) = t_j (+inf for a
 *   single-class constraint), each optional; per row and constraint in this order: centre, project, standardise,
 *   dot, + b, p = 1 / (1 + exp(-t)), all float64. */
int dmo_feas_fit(dmo_ctx* ctx, const double* X, int64_t N, int d, int J, const uint8_t* labels, const int8_t* folds,
                 const double* pca_mean, const double* pca_comps, int nC, const double* Cs, int max_iter, double tol,
                 double* scaler_mean, double* scaler_scale, double* coef, int32_t* iters, double* objective, double* kkt,
                 int8_t* converged, int64_t* correct);
int dmo_feas_create(dmo_ctx* ctx, int d, int J, const int32_t* k, const double* mean, const double* comps,
                    const double* smean, const double* sscale, const double* coef, const double* intercept,
                    dmo_feas** out);
int dmo_feas_destroy(dmo_ctx* ctx, dmo_feas* m);
int dmo_feas_eval(dmo_ctx* ctx, const dmo_feas* m, const double* X, int64_t n, int d, double* rank, double* proba,
                  double* decision);

#ifdef __cplusplus
}
#endif
#endif /* DMOSOPT_B200_H */
