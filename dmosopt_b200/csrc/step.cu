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
// chain's watchdog) and the hypervolume's (its route and its value).  bench.py's `value` leg is this call;
// scripts/step_phases.py times its phases (the step_* profile scopes) and counts the waits.
#include <string.h>

#include "common.cuh"
#include "gp.cuh"

extern "C" {
int dmo_nsga2_step(dmo_ctx* ctx, dmo_gp* gp, double* pop_x, double* pop_y, int32_t* rank, int64_t pop, int d, int M,
                   double crossover_prob, double mutation_prob, double mutation_rate, const double* di_crossover,
                   const double* di_mutation, const double* xlb, const double* xub, uint64_t seed, uint64_t stream_id,
                   int precision, int distance_metric, int with_variance, int round_to_f32, const double* hv_ref, int64_t* n_children,
                   double* hv_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(gp && pop_x && pop_y && rank && pop >= 2 && d >= 1 && M >= 1 && di_crossover && di_mutation && xlb && xub,
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
  // The GP's read-back is left pending and the truncation is enqueued behind it, so the host issues the truncation's first
  // launches while the GP runs; the truncation's own first wait comes after the GP anyway.  If the GP then fails, the
  // population is put back (the parents are still in Xs / Ys); if AUTO refines rows, the truncation runs again on them.
  GpPending gpp;
  DevBuf<int32_t> rank_in;
  if (P > 0) {
    ProfileScope ps(ctx, "step_gp");
    DMO_TRY(gp_predict_device(ctx, gp, Xs.p, P, Ys.p, with_variance ? var.p : nullptr, precision, &gpp));
  }
  if (gpp.active) {
    DMO_TRY(rank_in.alloc(ctx, pop));
    DMO_CUDA(cudaMemcpyAsync(rank_in.p, rank, (size_t)pop * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  }
  auto truncate = [&]() -> int {
    ProfileScope ps(ctx, "step_truncate");
    DMO_TRY(remove_worst_device(ctx, Xs.p, Ys.p, P + pop, d, M, distance_metric, nullptr, 0, pop, pop_x, pop_y, rank, perm.p));
    if (round_to_f32) DMO_TRY(prim_round_f32(ctx, pop_y, pop * M));
    return DMO_OK;
  };
  DMO_TRY(truncate());
  bool refined = false;
  const int rc = gp_predict_finish(ctx, gp, gpp, &refined);
  if (rc != DMO_OK) {
    DMO_CUDA(cudaMemcpyAsync(pop_x, Xs.p + (size_t)P * d, (size_t)pop * d * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(pop_y, Ys.p + (size_t)P * M, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(rank, rank_in.p, (size_t)pop * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    return rc;
  }
  if (refined) DMO_TRY(truncate());
  if (hv_ref && hv_out) {
    ProfileScope ps(ctx, "step_hv");
    // the survivors carry their ranks within the merged set: rows of rank > 0 cannot add volume (hv.cu)
    DMO_REQUIRE(M <= 16, "nsga2_step: too many objectives for the hypervolume");
    double h_ref[16];
    if (dmo_is_device_ptr(hv_ref)) {
      ctx->waits++;  // a copy into pageable host memory returns once it has landed: behind the truncation
      DMO_CUDA(cudaMemcpyAsync(h_ref, hv_ref, M * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    } else {
      memcpy(h_ref, hv_ref, M * sizeof(double));
    }
    DMO_TRY(hypervolume_device_ranked(ctx, pop_y, pop, M, h_ref, rank, hv_out));
  }
  return DMO_OK;
}
}
