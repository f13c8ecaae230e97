// Fused resident NSGA-II surrogate generation (SURVEY.md section 8b: "fused dmo_generation_step").
//
// One C call = one pass of MOASMO.optimize's loop body (dmosopt/MOASMO.py:105-116) for the NSGA-II plugin with a GP
// surrogate, population resident in HBM:
//   tournament (NSGA2.py:116-140) -> variation loop (NSGA2.py:142-178) -> GP posterior mean [+ variance]
//   (model.py:1254-1275) -> children stacked over parents, rank + stable truncation (NSGA2.py:205-214, MOEA.py:398-423)
//   -> float32 rounding of the stored objectives (NSGA2.py:228-230) -> optional hypervolume of the survivors.
// It is a composition of the device bodies of this library's entry points, without their trailing waits.  The host waits
// only for values it needs: the offspring count (it sizes the GP launch), one read-back after the GP (watchdog and rows to
// refine, read once the truncation is enqueued behind it), the rank's (the peel probe and one count per peeled front, mostly read while the next front is peeled; or the
// chain's watchdog) and the hypervolume's (its route and its value).  The truncation and the hypervolume run beside the
// GP's variance contraction, on a stream of its own (below).  bench.py's `value` leg is this call; scripts/step_phases.py times its
// phases (the step_* profile scopes) and counts the waits.
// dmo_nsga2_step_record runs the same body for MOASMO.optimize's resident epoch (dmosopt_b200/MOASMO.py): the mean only,
// optionally a feasibility rank as the truncation's last key, and the generation's offspring, their mean and operator
// counts copied out without a host wait.  dmo_nsga2_step_record_posterior runs it with the other posteriors the resident
// epoch serves: the exact GP (EGP_Matern's linear-mean model), the variational posterior and the deep GPs, each giving
// the mean its public predict writes when the variance is requested too (what those surrogates' evaluate returns),
// optionally rounded to float32 before the truncation.
#include <string.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "gp.cuh"

// counts[0..3] += children from crossover (kind < 2), mutants (kind == 2), and the same two among the survivors (the
// rows of perm below P): the values NSGA2.update_strategy derives its success counters from (NSGA2.py:216-222).  Sums of
// ones stay far below 2^53, so block_sum is exact; one integer atomic per CTA and counter.
constexpr int kCountWarps = 8;
__global__ void __launch_bounds__(kCountWarps * 32) step_counts_kernel(const int32_t* __restrict__ kind, int64_t P,
                                                                        const int64_t* __restrict__ perm, int64_t pop,
                                                                        unsigned long long* counts) {
  __shared__ double red[kCountWarps];
  double c[4] = {0.0, 0.0, 0.0, 0.0};
  const int64_t n = P > pop ? P : pop;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < P) {
      const int32_t k = kind[i];
      c[0] += k < 2 ? 1.0 : 0.0;
      c[1] += k == 2 ? 1.0 : 0.0;
    }
    if (i < pop) {
      const int64_t j = perm[i];
      if (j < P) {
        const int32_t k = kind[j];
        c[2] += k < 2 ? 1.0 : 0.0;
        c[3] += k == 2 ? 1.0 : 0.0;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double s = block_sum<kCountWarps>(c[k], red);
    if (threadIdx.x == 0 && s > 0.0) atomicAdd(&counts[k], (unsigned long long)s);
  }
}

int step_posterior(dmo_ctx* ctx, const char* who, int kind, void* posterior, uint64_t draw_seed, uint64_t draw_stream, bool var_route_mean,
                   bool mean_f32, int precision, int d, int M, StepPosterior* post) {
  DMO_REQUIRE(kind == DMO_POSTERIOR_GP || kind == DMO_POSTERIOR_SVGP || kind == DMO_POSTERIOR_DGP, "%s: unknown posterior kind %d", who,
              kind);
  DMO_REQUIRE(posterior, "%s: null posterior", who);
  // AUTO refines the rows its variance flags, so its mean cannot be had without the variance; the exact GP's surrogates
  // that evaluate on this route predict in float64 or on the tensor path
  if (var_route_mean)
    DMO_REQUIRE(precision == DMO_GP_FP64 || precision == DMO_GP_TENSOR, "%s: precision must be DMO_GP_FP64 or DMO_GP_TENSOR (got %d)", who,
                precision);
  post->kind = kind;
  post->var_route_mean = var_route_mean;
  post->mean_f32 = mean_f32;
  int md = 0, mM = 0;
  if (kind == DMO_POSTERIOR_GP) {
    post->gp = static_cast<dmo_gp*>(posterior);
    md = post->gp->d;
    mM = post->gp->M;
  } else if (kind == DMO_POSTERIOR_SVGP) {
    post->sv = static_cast<dmo_svgp*>(posterior);
    svgp_dims(post->sv, &md, &mM);
  } else {
    post->dg = static_cast<dmo_dgp*>(posterior);
    dgp_dims(post->dg, &md, &mM);
    DMO_REQUIRE(draw_stream < ((uint64_t)1 << 54), "%s: the draw stream must be below 2^54", who);
    post->draw_seed = draw_seed;
    post->draw_stream = draw_stream;
  }
  DMO_REQUIRE(md == d && mM == M, "%s: the posterior takes %d inputs and has %d outputs, the population has %d and %d", who, md, mM, d, M);
  if (kind != DMO_POSTERIOR_GP) {  // the exact GP's d fits every route (dmo_gp_create)
    GpUnitPredict up;
    DMO_TRY(up.check(ctx, who, precision, d));
  }
  return DMO_OK;
}

int step_predict(dmo_ctx* ctx, const char* who, const StepPosterior& post, const double* X, int64_t P, double* mean, double* var,
                 int precision, GpPending* gpp) {
  if (post.kind == DMO_POSTERIOR_GP) return gp_predict_device(ctx, post.gp, X, P, mean, var, precision, gpp, post.var_route_mean);
  GpUnitPredict up;
  if (post.kind == DMO_POSTERIOR_SVGP) {
    int dd = 0, mm = 0;
    svgp_dims(post.sv, &dd, &mm);
    DMO_TRY(up.check(ctx, who, precision, dd));
    DMO_TRY(svgp_predict_device(ctx, post.sv, up, X, P, mean, nullptr));
  } else {
    int dd = 0, tt = 0;
    dgp_dims(post.dg, &dd, &tt);
    DMO_TRY(up.check(ctx, who, precision, dd));
    DMO_TRY(dgp_predict_device(ctx, post.dg, up, X, P, post.draw_seed, post.draw_stream, nullptr, mean, nullptr));
  }
  return up.watchdog(ctx);
}

// The body of the entry points.  key (may be null): the feasibility rank of [children; parents] as the truncation's least
// significant descending key.  x_gen / y_gen / counts (all null, or all set): the offspring, their posterior mean and the
// operator counts of step_counts_kernel, copied out once the GP is final.
static int nsga2_step_body(dmo_ctx* ctx, const StepPosterior& post, const dmo_feas* key, double* pop_x, double* pop_y, int32_t* rank,
                           int64_t pop, int d, int M, double crossover_prob, double mutation_prob, double mutation_rate,
                           const double* di_crossover, const double* di_mutation, const double* xlb, const double* xub,
                           uint64_t seed, uint64_t stream_id, int precision, int distance_metric, int with_variance,
                           int round_to_f32, const double* hv_ref, int64_t* n_children, double* hv_out, double* x_gen,
                           double* y_gen, int64_t* counts) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE((post.gp || post.sv || post.dg) && pop_x && pop_y && rank && pop >= 2 && d >= 1 && M >= 1 && di_crossover && di_mutation && xlb && xub,
              "nsga2_step: bad arguments");
  DMO_REQUIRE(distance_metric == DMO_METRIC_NONE || distance_metric == DMO_METRIC_CROWDING || distance_metric == DMO_METRIC_EUCLIDEAN,
              "nsga2_step: unknown distance metric %d", distance_metric);
  DMO_REQUIRE(dmo_is_device_ptr(pop_x) && dmo_is_device_ptr(pop_y) && dmo_is_device_ptr(rank),
              "nsga2_step: the population (pop_x, pop_y, rank) must be resident on the device");
  int64_t poolsize = pop / 2;  // int(round(popsize / 2.0)), NSGA2.py:64: Python rounds halves to even
  if ((pop & 1) && (poolsize & 1)) poolsize += 1;
  const int64_t cap = pop + 1;             // the variation loop emits pop-1 .. pop+1 children (NSGA2.py:142)
  DevBuf<int64_t> pool, perm;
  DevBuf<double> Xs, Ys, var;
  DevBuf<int32_t> kind;
  DMO_TRY(pool.alloc(ctx, poolsize));
  DMO_TRY(perm.alloc(ctx, pop));
  DMO_TRY(Xs.alloc(ctx, (size_t)(cap + pop) * d));
  DMO_TRY(Ys.alloc(ctx, (size_t)(cap + pop) * M));
  DMO_TRY(kind.alloc(ctx, cap));
  if (with_variance) DMO_TRY(var.alloc(ctx, (size_t)cap * M));
  In<double> idc, idm, ilb, iub;
  DMO_TRY(idc.init(ctx, di_crossover, d));
  DMO_TRY(idm.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  {
    ProfileScope ps(ctx, "step_tournament");
    DMO_TRY(tournament_device(ctx, rank, nullptr, pop, poolsize, seed, stream_id, pool.p, nullptr));
  }
  int64_t P = 0;
  {
    ProfileScope ps(ctx, "step_generate");
    DMO_TRY(nsga2_generate_device(ctx, pop_x, d, pool.p, poolsize, pop, crossover_prob, mutation_prob, mutation_rate, idc.d, idm.d,
                                  ilb.d, iub.d, seed, stream_id + 1, Xs.p, kind.p, &P, nullptr));
  }
  if (n_children) *n_children = P;
  {
    ProfileScope ps(ctx, "step_truncate");
    // parents under the children (np.vstack((x_gen, population_parm)), NSGA2.py:205-206); the GP reads and writes the rows
    // above them only, so the copies are enqueued first and the host does not issue them after the GP's read-back
    DMO_CUDA(cudaMemcpyAsync(Xs.p + (size_t)P * d, pop_x, (size_t)pop * d * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(Ys.p + (size_t)P * M, pop_y, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  }
  // the feasibility rank of the merged rows (the key of dmo_remove_worst_pair_keys), on the main stream before the GP forks
  DevBuf<double> kx;
  const double* kp[1] = {nullptr};
  if (key) {
    ProfileScope ps(ctx, "step_truncate");
    DMO_TRY(kx.alloc(ctx, (size_t)(P + pop)));
    DMO_TRY(feas_rank_device(ctx, key, Xs.p, P + pop, kx.p));
    kp[0] = kx.p;
  }
  // The GP's read-back is left pending and the truncation is enqueued before the host waits for it.  The truncation and
  // the hypervolume of its survivors need the posterior mean only, which the tensor route writes before its variance
  // contraction: when the GP defers its read-back, both run on the context's lane stream from that point on, beside the
  // contraction, which runs on a higher-priority stream on the SMs its grid leaves free.  Otherwise (float64 or tensor
  // precision, a linear mean, a non-tensor AUTO route) the GP has finished inside the call and both follow it on the
  // main stream.  Either way the truncation's host waits (peel probe, peel counts) wait for its own stream only, and the
  // hypervolume's reads come after the GP's read-back.  If the GP then fails, the population is put back (the parents are
  // still in Xs / Ys) and hv_out is left alone; if AUTO refines rows, the truncation and the hypervolume run again on
  // them.  Every buffer the two streams share is allocated on the main stream before the fork and released after the join.
  // The hypervolume's reference point is staged before the fork, so that the lane can use it.
  const bool want_hv = hv_ref && hv_out;
  double h_ref[16] = {};
  if (want_hv && M <= 16) {
    if (dmo_is_device_ptr(hv_ref)) {
      ctx->waits++;  // a copy into pageable host memory returns once it has landed
      DMO_CUDA(cudaMemcpyAsync(h_ref, hv_ref, M * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    } else {
      memcpy(h_ref, hv_ref, M * sizeof(double));
    }
  }
  GpPending gpp;
  DevBuf<int32_t> rank_in;  // the ranks before the truncation, for the failure path
  if (P > 0) {
    DMO_TRY(rank_in.alloc(ctx, pop));
    DMO_TRY(dmo_lane_streams(ctx));
    gpp.ov.mean_ready = ctx->lane_ev[0];
    ProfileScope ps(ctx, "step_gp");
    DMO_TRY(step_predict(ctx, "nsga2_step", post, Xs.p, P, Ys.p, with_variance ? var.p : nullptr, precision, &gpp));
    // evaluate's float32 cast; the routes that round have finished their predict here (no pending read-back)
    if (post.mean_f32) DMO_TRY(prim_round_f32(ctx, Ys.p, P * M));
  }
  auto truncate = [&]() -> int {
    ProfileScope ps(ctx, "step_truncate");
    DMO_TRY(remove_worst_device(ctx, Xs.p, Ys.p, P + pop, d, M, distance_metric, key ? kp : nullptr, key ? 1 : 0, pop, pop_x, pop_y,
                                rank, perm.p));
    if (round_to_f32) DMO_TRY(prim_round_f32(ctx, pop_y, pop * M));
    return DMO_OK;
  };
  auto first_truncate = [&]() -> int {
    if (gpp.active) DMO_CUDA(cudaMemcpyAsync(rank_in.p, rank, (size_t)pop * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    return truncate();
  };
  // the survivors carry their ranks within the merged set: rows of rank > 0 cannot add volume (hv.cu)
  auto hypervolume = [&](double* h) -> int {
    ProfileScope ps(ctx, "step_hv");
    return hypervolume_device_ranked(ctx, pop_y, pop, M, h_ref, rank, h);
  };
  // With three objectives and a finite reference point the lane also enqueues the device work of the hypervolume, which
  // has no host read (hv3_ranked_enqueue); its reads and the volume follow gp_predict_finish, unless the GP fails (the
  // population is put back, hv_out is left alone) or refines rows (the lane's work is dropped unread, and the truncation
  // and the hypervolume run again).  So the step's host waits are the serial composition's whether or not AUTO refines.
  // The other routes read counts back from the device before their last kernels, and run after the join.
  Hv3Ranked hv_lane;
  const bool hv_on_lane = want_hv && M == 3 && std::isfinite(h_ref[0]) && std::isfinite(h_ref[1]) && std::isfinite(h_ref[2]);
  bool hv_enqueued = false;
  if (gpp.active && gpp.ov.mean_ready) {
    // The lane reads Xs, Ys (the mean rows and the parents) and writes pop_x, pop_y, rank, rank_in and its own scratch; the
    // GP's work after the fork point writes the variance and its own scratch only.  The lane may run on a few SMs while
    // the contraction holds the rest (it leaves GP_LANE_SMS free), so nothing in it may need all of its CTAs resident at
    // once.  Every kernel remove_worst_device reaches (metric none, crowding or euclidean) was checked for that: the
    // dense-id, lexicographic, cell and key radix sorts are CUB's (onesweep passes take their tile from an atomic counter
    // and look back only at tiles taken before; small sorts run as one tile, or as separate upsweep / scan / downsweep
    // kernels); CUB's scans look back only at lower block indices, which are dispatched first; the peel probe
    // is a grid-stride loop with atomicOr; the chain kernel (rank.cu) takes its blocks from an atomic ticket and waits
    // only for blocks taken before; everything else (keys, gathers, cell grid, prefix minima, peel marks, column min / max,
    // crowding, euclidean, round_f32) is one pass per element or per block, with atomics at most, and no grid-wide barrier.
    // So was every kernel hv3_ranked_enqueue reaches: the column sorts (prim_sort_by_column) and the compaction scan are
    // the CUB sorts and scans above; the inside / rank-0 flags, compaction, padding, inverse permutation and gathers, and
    // the tree's y_by_t, build_low, per-level build_high and carry kernels and its walks (hv3_tree.cu) are one pass per
    // element or per block, each block reading only what earlier launches wrote; final_sum_kernel is a single block.
    cudaStream_t main = ctx->stream;
    DMO_CUDA(cudaStreamWaitEvent(ctx->lane, gpp.ov.mean_ready, 0));
    ctx->stream = ctx->lane;
    int rc = first_truncate();
    if (rc == DMO_OK && hv_on_lane) {
      ProfileScope ps(ctx, "step_hv");
      rc = hv3_ranked_enqueue(ctx, pop_y, pop, h_ref, rank, hv_lane);
      hv_enqueued = rc == DMO_OK;
    }
    ctx->stream = main;
    // joined before gp_predict_finish: its refinement, the failure path and the second truncation come after the lane
    DMO_CUDA(cudaEventRecord(ctx->lane_ev[3], ctx->lane));
    DMO_CUDA(cudaStreamWaitEvent(main, ctx->lane_ev[3], 0));
    DMO_TRY(rc);
  } else {
    DMO_TRY(first_truncate());
  }
  bool refined = false;
  const int rc = gp_predict_finish(ctx, post.gp, gpp, &refined);
  if (rc != DMO_OK) {
    DMO_CUDA(cudaMemcpyAsync(pop_x, Xs.p + (size_t)P * d, (size_t)pop * d * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(pop_y, Ys.p + (size_t)P * M, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(rank, rank_in.p, (size_t)pop * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    return rc;
  }
  if (refined) {
    DMO_TRY(truncate());
    hv_enqueued = false;
  }
  if (x_gen) {
    ProfileScope ps(ctx, "step_record");
    DevBuf<unsigned long long> cnt;
    DMO_TRY(cnt.alloc(ctx, 4));
    DMO_CUDA(cudaMemsetAsync(cnt.p, 0, 4 * sizeof(unsigned long long), ctx->stream));
    const int64_t n = P > pop ? P : pop;
    const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n, kCountWarps * 32), 4 * (int64_t)ctx->sm_count);
    DMO_LAUNCH(step_counts_kernel, grid, kCountWarps * 32, 0, kind.p, P, perm.p, pop, cnt.p);
    DMO_CHECK_LAUNCH();
    DMO_TRY(copy_out(ctx, x_gen, Xs.p, (size_t)P * d * sizeof(double)));
    DMO_TRY(copy_out(ctx, y_gen, Ys.p, (size_t)P * M * sizeof(double)));
    DMO_TRY(copy_out(ctx, counts, cnt.p, 4 * sizeof(int64_t)));
  }
  if (want_hv) {
    if (hv_enqueued) {
      ProfileScope ps(ctx, "step_hv");
      double h = 0.0;
      DMO_TRY(hv3_ranked_finish(ctx, hv_lane, &h));
      *hv_out = h;
      return DMO_OK;
    }
    DMO_REQUIRE(M <= 16, "nsga2_step: too many objectives for the hypervolume");
    DMO_TRY(hypervolume(hv_out));
  }
  return DMO_OK;
}

extern "C" {
int dmo_nsga2_step(dmo_ctx* ctx, dmo_gp* gp, double* pop_x, double* pop_y, int32_t* rank, int64_t pop, int d, int M,
                   double crossover_prob, double mutation_prob, double mutation_rate, const double* di_crossover,
                   const double* di_mutation, const double* xlb, const double* xub, uint64_t seed, uint64_t stream_id,
                   int precision, int distance_metric, int with_variance, int round_to_f32, const double* hv_ref, int64_t* n_children,
                   double* hv_out) {
  StepPosterior post;
  post.gp = gp;
  return nsga2_step_body(ctx, post, nullptr, pop_x, pop_y, rank, pop, d, M, crossover_prob, mutation_prob, mutation_rate,
                         di_crossover, di_mutation, xlb, xub, seed, stream_id, precision, distance_metric, with_variance,
                         round_to_f32, hv_ref, n_children, hv_out, nullptr, nullptr, nullptr);
}

int dmo_nsga2_step_record(dmo_ctx* ctx, dmo_gp* gp, const dmo_feas* key, double* pop_x, double* pop_y, int32_t* rank,
                          int64_t pop, int d, int M, double crossover_prob, double mutation_prob, double mutation_rate,
                          const double* di_crossover, const double* di_mutation, const double* xlb, const double* xub,
                          uint64_t seed, uint64_t stream_id, int precision, int distance_metric, int round_to_f32,
                          double* x_gen, double* y_gen, int64_t* counts, int64_t* n_children) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_REQUIRE(x_gen && y_gen && counts, "nsga2_step_record: x_gen, y_gen and counts are required");
  DMO_REQUIRE(!key || feas_model_dim(key) == d, "nsga2_step_record: the key model takes %d columns, the population has %d",
              feas_model_dim(key), d);
  StepPosterior post;
  post.gp = gp;
  return nsga2_step_body(ctx, post, key, pop_x, pop_y, rank, pop, d, M, crossover_prob, mutation_prob, mutation_rate,
                         di_crossover, di_mutation, xlb, xub, seed, stream_id, precision, distance_metric, 0, round_to_f32,
                         nullptr, n_children, nullptr, x_gen, y_gen, counts);
}

int dmo_nsga2_step_record_posterior(dmo_ctx* ctx, int kind, void* posterior, uint64_t draw_seed, uint64_t draw_stream,
                                    const dmo_feas* key, double* pop_x, double* pop_y, int32_t* rank, int64_t pop, int d, int M,
                                    double crossover_prob, double mutation_prob, double mutation_rate, const double* di_crossover,
                                    const double* di_mutation, const double* xlb, const double* xub, uint64_t seed,
                                    uint64_t stream_id, int precision, int distance_metric, int mean_f32, int round_to_f32,
                                    double* x_gen, double* y_gen, int64_t* counts, int64_t* n_children) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  const char* who = "nsga2_step_record_posterior";
  DMO_REQUIRE(kind == DMO_POSTERIOR_GP || kind == DMO_POSTERIOR_SVGP || kind == DMO_POSTERIOR_DGP, "%s: unknown posterior kind %d", who,
              kind);
  DMO_REQUIRE(posterior, "%s: null posterior", who);
  DMO_REQUIRE(x_gen && y_gen && counts, "%s: x_gen, y_gen and counts are required", who);
  DMO_REQUIRE(pop >= 2, "%s: pop must be at least 2 (got %lld)", who, (long long)pop);
  StepPosterior post;
  DMO_TRY(step_posterior(ctx, who, kind, posterior, draw_seed, draw_stream, true, mean_f32 != 0, precision, d, M, &post));
  DMO_REQUIRE(!key || feas_model_dim(key) == d, "%s: the key model takes %d columns, the population has %d", who, feas_model_dim(key), d);
  return nsga2_step_body(ctx, post, key, pop_x, pop_y, rank, pop, d, M, crossover_prob, mutation_prob, mutation_rate,
                         di_crossover, di_mutation, xlb, xub, seed, stream_id, precision, distance_metric, 0, round_to_f32,
                         nullptr, n_children, nullptr, x_gen, y_gen, counts);
}
}
