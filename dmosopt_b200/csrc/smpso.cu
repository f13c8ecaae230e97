// SMPSO with the swarm state resident in HBM (SURVEY.md section 8a row A12).
//   SMPSO.generate_strategy   dmosopt/SMPSO.py:143-185   -> dmo_smpso_generate
//   SMPSO.update_strategy     dmosopt/SMPSO.py:187-238   -> dmo_smpso_update
//   velocity_vector           dmosopt/SMPSO.py:316-348   (scalar draws stay with the caller's NumPy generator)
// The reference keeps positions / objectives as float32 arrays and velocities as float64; here they are float64 device
// arrays whose position / objective values are float32-representable (rounded whenever the reference stores into its
// float32 state), so every comparison and every difference sees the values the reference sees.
// One call per generation replaces the per-swarm host loops (crowding, velocity, vstack + remove_worst per swarm).
// dmo_smpso_step_record runs one pass of MOASMO.optimize's loop body (dmosopt/MOASMO.py:105-122) for SMPSO: the body of
// dmo_smpso_generate, the surrogate's posterior mean of every offspring row (step_predict, step.cu), the body of
// dmo_smpso_update on the first swarms * pop rows, and the offspring and their mean copied out without a host wait.  The
// swarm state, the offspring and their mean never leave the device in between; the host waits only inside the predict
// (a tensor watchdog) and inside each swarm's truncation (the rank's peel reads).
#include "common.cuh"
#include "gp.cuh"

namespace {

enum : uint64_t { P_MUT_PARENT = 11, P_MUT_GENES = 12 };  // the Philox stream ids of mutate_groups_kernel (moea_ext.cu)

__device__ __forceinline__ double mutate_gene_sm(double parent, double u, double di, double lb, double ub, double rate) {
  double e = __ddiv_rn(1.0, __dadd_rn(di, 1.0));
  double delta;
  if (u < rate)
    delta = __dsub_rn(pow(__dmul_rn(2.0, u), e), 1.0);
  else
    delta = __dsub_rn(1.0, pow(__dmul_rn(2.0, __dsub_rn(1.0, u)), e));
  return np_clip(__dadd_rn(parent, __dmul_rn(__dsub_rn(ub, lb), delta)), lb, ub);
}

// x_gen rows, swarm-major: [swarm p][0 .. pop) = clip(x + v) of the swarm's particles, [pop .. 2 pop) = its mutants
// (SMPSO.py:163-184); values are rounded to float32 as the reference's final astype does.
__global__ void smpso_generate_kernel(const double* __restrict__ parm, const double* __restrict__ vel, int S, int64_t pop, int d,
                                      const double* __restrict__ di, const double* __restrict__ xlb,
                                      const double* __restrict__ xub, double rate, uint64_t seed, uint64_t stream_id,
                                      float* __restrict__ out32, double* __restrict__ out64) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * (int64_t)S * pop * d) return;
  const int64_t r = t / d;
  const int j = (int)(t - r * d);
  const int64_t p = r / (2 * pop), k = r - p * 2 * pop;
  double v;
  if (k < pop) {
    const int64_t row = p * pop + k;
    v = np_clip(parm[row * d + j] + vel[row * d + j], xlb[j], xub[j]);  // update_position, SMPSO.py:311-313
  } else {
    const int64_t c = p * pop + (k - pop);  // child index of mutate_groups: group p, child k - pop
    Philox ph(seed);
    const uint4 a = ph((uint64_t)c, (stream_id << 8) | P_MUT_PARENT);
    int64_t pi = (int64_t)(u01_53(a.x, a.y) * (double)pop);
    if (pi >= pop) pi = pop - 1;
    const int64_t prow = p * pop + pi;
    const uint4 b = ph((uint64_t)(c * d + j), (stream_id << 8) | P_MUT_GENES);
    v = mutate_gene_sm(parm[prow * d + j], u01_53(b.x, b.y), di[j], xlb[j], xub[j], rate);
  }
  if (out32) out32[t] = (float)v;
  if (out64) out64[t] = (double)(float)v;  // the same float32 values, widened (what np.clip(x_gen, xlb, xub) hands on, MOEA.py:155)
}

// velocity of one swarm, in place (SMPSO.py:316-348).  Leaders are rows ind1 / ind2 of the swarm's archive slice; the one
// with the larger crowding distance goes first (:332-335).  Differences are formed in float32 when the archive handed to
// update() is float32 (NumPy's promotion of archive[i] - position), in float64 otherwise.
__global__ void smpso_velocity_resident_kernel(const double* __restrict__ parm, double* __restrict__ vel,
                                               const double* __restrict__ arch, const double* __restrict__ crowd, int64_t ind1,
                                               int64_t ind2, int diff_f32, int64_t n, int d, double w, double c1r1, double c2r2,
                                               double chi, const double* __restrict__ xlb, const double* __restrict__ xub) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int j = (int)(t % d);
  if (crowd && crowd[ind1] < crowd[ind2]) {
    const int64_t s = ind1;
    ind1 = ind2;
    ind2 = s;
  }
  const double l1 = arch[ind1 * d + j], l2 = arch[ind2 * d + j];
  double d1, d2;
  if (diff_f32) {
    d1 = (double)((float)l1 - (float)parm[t]);
    d2 = (double)((float)l2 - (float)parm[t]);
  } else {
    d1 = l1 - parm[t];
    d2 = l2 - parm[t];
  }
  const double delta = (xub[j] - xlb[j]) / 2;
  const double v = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(w, vel[t]), __dmul_rn(c1r1, d1)), __dmul_rn(c2r2, d2)), chi);
  vel[t] = np_clip(v, -delta, delta);
}

__global__ void f32_to_f64_kernel(const float* __restrict__ a, int64_t n, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)a[i];
}
__global__ void f64_to_f32_kernel(const double* __restrict__ a, int64_t n, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)a[i];
}
}  // namespace

// the body of dmo_smpso_generate on device arrays, without its trailing wait
static int smpso_generate_device(dmo_ctx* ctx, const double* parm, const double* vel, int swarms, int64_t pop, int d, const double* d_di,
                          const double* d_xlb, const double* d_xub, double mutation_rate, uint64_t seed, uint64_t stream_id, float* d_out32,
                          double* d_out64) {
  const int64_t rows = 2 * (int64_t)swarms * pop;
  DMO_LAUNCH(smpso_generate_kernel, (unsigned)ceil_div(rows * d, 256), 256, 0, parm, vel, swarms, pop, d, d_di, d_xlb, d_xub, mutation_rate,
             seed, stream_id, d_out32, d_out64);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// the velocities of every swarm (first loop of update_strategy, SMPSO.py:211-221), against the positions before the
// truncation: xg / yg are the consumed rows [0, swarms * pop) of the offspring on the device, scalars the host array
static int smpso_velocities_device(dmo_ctx* ctx, const double* parm, double* vel, const double* xg, int diff_f32, const double* yg, int swarms,
                            int64_t pop, int d, int M, const double* scalars, const double* d_xlb, const double* d_xub) {
  DevBuf<double> crowd;
  DMO_TRY(crowd.alloc(ctx, (size_t)pop));
  for (int p = 0; p < swarms; ++p) {
    const double* sc = scalars + (size_t)p * 8;  // w, c1, r1, c2, r2, chi, ind1, ind2 (ind < 0: archive of <= 2 rows -> row 0 twice)
    const int64_t off = (int64_t)p * pop;
    int64_t i1 = (int64_t)sc[6], i2 = (int64_t)sc[7];
    const bool pick = i1 >= 0 && i2 >= 0;
    if (!pick) i1 = i2 = 0;
    DMO_REQUIRE(i1 < pop && i2 < pop, "smpso_update: leader index out of range");
    if (pick) DMO_TRY(crowding_device(ctx, yg + off * M, pop, M, crowd.p));  // crowding_distance_metric(y_gen[sl])
    DMO_LAUNCH(smpso_velocity_resident_kernel, (unsigned)ceil_div(pop * d, 256), 256, 0, parm + off * d, vel + off * d, xg + off * d,
               pick ? crowd.p : (const double*)nullptr, i1, i2, diff_f32, pop, d, sc[0], sc[1] * sc[2], sc[3] * sc[4], sc[5], d_xlb, d_xub);
  }
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// one swarm's remove_worst(vstack(x_gen[sl], particles), vstack(y_gen[sl], objectives)) (SMPSO.py:222-228), in place on
// its pop rows of parm / obj: dmo_remove_worst_pair on device arrays without its trailing wait
static int smpso_truncate_device(dmo_ctx* ctx, double* parm, double* obj, const double* xg, const double* yg, int64_t pop, int d, int M, int metric,
                          int32_t* d_rank, int64_t* d_perm) {
  DevBuf<double> x, y;
  DMO_TRY(x.alloc(ctx, (size_t)2 * pop * d));
  DMO_TRY(y.alloc(ctx, (size_t)2 * pop * M));
  DMO_CUDA(cudaMemcpyAsync(x.p, xg, (size_t)pop * d * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(x.p + (size_t)pop * d, parm, (size_t)pop * d * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(y.p, yg, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(y.p + (size_t)pop * M, obj, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  return remove_worst_device(ctx, x.p, y.p, 2 * pop, d, M, metric, nullptr, 0, pop, parm, obj, d_rank, d_perm);
}

extern "C" {

int dmo_smpso_generate(dmo_ctx* ctx, const double* parm, const double* vel, int swarms, int64_t pop, int d,
                       const double* di_mutation, const double* xlb, const double* xub, double mutation_rate, uint64_t seed,
                       uint64_t stream_id, float* x_gen, double* x_gen_f64) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(parm && vel && swarms >= 1 && pop >= 1 && d >= 1 && di_mutation && xlb && xub && (x_gen || x_gen_f64),
              "smpso_generate: bad arguments");
  DMO_REQUIRE(dmo_is_device_ptr(parm) && dmo_is_device_ptr(vel), "smpso_generate: the swarm state must be resident on the device");
  const int64_t rows = 2 * (int64_t)swarms * pop;
  In<double> idi, ilb, iub;
  Out<float> ox;
  Out<double> ox64;
  DMO_TRY(idi.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(ox.init(ctx, x_gen, (size_t)rows * d));
  DMO_TRY(ox64.init(ctx, x_gen_f64, (size_t)rows * d));
  DMO_TRY(smpso_generate_device(ctx, parm, vel, swarms, pop, d, idi.d, ilb.d, iub.d, mutation_rate, seed, stream_id, ox.d, ox64.d));
  DMO_TRY(ox.finish(ctx));
  DMO_TRY(ox64.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_smpso_update(dmo_ctx* ctx, double* parm, double* obj, double* vel, const void* x_gen, int x_is_f32, const double* y_gen,
                     int swarms, int64_t pop, int d, int M, int metric, const double* scalars, const double* xlb,
                     const double* xub, int32_t* ranks, int64_t* perm, float* parm_f32, float* obj_f32) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(parm && obj && vel && x_gen && y_gen && swarms >= 1 && pop >= 1 && d >= 1 && M >= 1 && scalars && xlb && xub && ranks && perm,
              "smpso_update: bad arguments");
  DMO_REQUIRE(dmo_is_device_ptr(parm) && dmo_is_device_ptr(obj) && dmo_is_device_ptr(vel),
              "smpso_update: the swarm state must be resident on the device");
  DMO_REQUIRE(!dmo_is_device_ptr(scalars), "smpso_update: the per-swarm scalars are a host array");
  const int64_t n = (int64_t)swarms * pop;  // rows of x_gen / y_gen that update_strategy consumes (SMPSO.py:211-221)
  // the consumed slices of the offspring, float64 on the device
  DevBuf<double> xg, yg;
  DMO_TRY(xg.alloc(ctx, (size_t)n * d));
  DMO_TRY(yg.alloc(ctx, (size_t)n * M));
  if (x_is_f32) {
    In<float> xf;
    DMO_TRY(xf.init(ctx, (const float*)x_gen, (size_t)n * d));
    DMO_LAUNCH(f32_to_f64_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, xf.d, n * d, xg.p);
    DMO_CUDA(dmo_wait(ctx));  // xf is released at the end of this scope
  } else {
    DMO_CUDA(cudaMemcpyAsync(xg.p, x_gen, (size_t)n * d * sizeof(double), cudaMemcpyDefault, ctx->stream));
    if (!dmo_is_device_ptr(x_gen)) ctx->h2d_bytes += (uint64_t)n * d * sizeof(double);
  }
  DMO_CUDA(cudaMemcpyAsync(yg.p, y_gen, (size_t)n * M * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (!dmo_is_device_ptr(y_gen)) ctx->h2d_bytes += (uint64_t)n * M * sizeof(double);
  In<double> ilb, iub;
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  // 1. velocities of every swarm, against the positions BEFORE the truncation (first loop of update_strategy)
  DMO_TRY(smpso_velocities_device(ctx, parm, vel, xg.p, x_is_f32, yg.p, swarms, pop, d, M, scalars, ilb.d, iub.d));
  // 2. per swarm: remove_worst(vstack(x_gen[sl], particles), vstack(y_gen[sl], objectives)) -> the swarm's new state
  Out<int32_t> orank;
  Out<int64_t> operm;
  DMO_TRY(orank.init(ctx, ranks, (size_t)n));
  DMO_TRY(operm.init(ctx, perm, (size_t)n));
  for (int p = 0; p < swarms; ++p) {
    const int64_t off = (int64_t)p * pop;
    DMO_TRY(smpso_truncate_device(ctx, parm + off * d, obj + off * M, xg.p + off * d, yg.p + off * M, pop, d, M, metric, orank.d + off,
                                  operm.d + off));
    DMO_CUDA(dmo_wait(ctx));  // each swarm's truncation ends in a wait, as dmo_remove_worst_pair's does
  }
  // the reference assigns the survivors into float32 state arrays
  DMO_TRY(prim_round_f32(ctx, parm, n * d));
  DMO_TRY(prim_round_f32(ctx, obj, n * M));
  DMO_TRY(orank.finish(ctx));
  DMO_TRY(operm.finish(ctx));
  if (parm_f32) {
    Out<float> o;
    DMO_TRY(o.init(ctx, parm_f32, (size_t)n * d));
    DMO_LAUNCH(f64_to_f32_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, parm, n * d, o.d);
    DMO_TRY(o.finish(ctx));
    DMO_CUDA(dmo_wait(ctx));
  }
  if (obj_f32) {
    Out<float> o;
    DMO_TRY(o.init(ctx, obj_f32, (size_t)n * M));
    DMO_LAUNCH(f64_to_f32_kernel, (unsigned)ceil_div(n * M, 256), 256, 0, obj, n * M, o.d);
    DMO_TRY(o.finish(ctx));
    DMO_CUDA(dmo_wait(ctx));
  }
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_smpso_step_record(dmo_ctx* ctx, int kind, void* posterior, uint64_t draw_seed, uint64_t draw_stream, int var_route_mean,
                          double* parm, double* obj, double* vel, int swarms, int64_t pop, int d, int M, const double* di_mutation,
                          const double* xlb, const double* xub, double mutation_rate, uint64_t seed, uint64_t stream_id, int precision,
                          int mean_f32, int metric, const double* scalars, int32_t* ranks, double* x_gen, double* y_gen) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  const char* who = "smpso_step_record";
  DMO_REQUIRE(parm && obj && vel && ranks && swarms >= 1 && pop >= 1 && d >= 1 && M >= 1 && di_mutation && xlb && xub && scalars,
              "%s: bad arguments", who);
  DMO_REQUIRE(x_gen && y_gen, "%s: x_gen and y_gen are required", who);
  DMO_REQUIRE(metric == DMO_METRIC_NONE || metric == DMO_METRIC_CROWDING || metric == DMO_METRIC_EUCLIDEAN, "%s: unknown distance metric %d",
              who, metric);
  DMO_REQUIRE(dmo_is_device_ptr(parm) && dmo_is_device_ptr(obj) && dmo_is_device_ptr(vel) && dmo_is_device_ptr(ranks),
              "%s: the swarm state (parm, obj, vel, ranks) must be resident on the device", who);
  DMO_REQUIRE(!dmo_is_device_ptr(scalars), "%s: the per-swarm scalars are a host array", who);
  // flag 0: the mean-only predict of the exact GP (GPR_Matern / GPR_RBF evaluate), any precision
  DMO_REQUIRE(var_route_mean || kind == DMO_POSTERIOR_GP, "%s: the mean-only predict is the exact GP's (kind %d)", who, kind);
  StepPosterior post;
  DMO_TRY(step_posterior(ctx, who, kind, posterior, draw_seed, draw_stream, var_route_mean != 0, mean_f32 != 0, precision, d, M, &post));
  for (int p = 0; p < swarms; ++p)
    for (int k = 6; k < 8; ++k)
      DMO_REQUIRE(scalars[(size_t)p * 8 + k] < (double)pop, "%s: leader index %g of swarm %d is not below pop = %lld", who,
                  scalars[(size_t)p * 8 + k], p, (long long)pop);
  const int64_t n = (int64_t)swarms * pop, P = 2 * n;
  DevBuf<double> xg, yg;
  DevBuf<int64_t> perm;
  DMO_TRY(xg.alloc(ctx, (size_t)P * d));
  DMO_TRY(yg.alloc(ctx, (size_t)P * M));
  DMO_TRY(perm.alloc(ctx, (size_t)n));
  In<double> idi, ilb, iub;
  DMO_TRY(idi.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  // 1. moved positions and mutants of every swarm, as float64 rows of float32 values (what the plugin's generate hands on)
  DMO_TRY(smpso_generate_device(ctx, parm, vel, swarms, pop, d, idi.d, ilb.d, iub.d, mutation_rate, seed, stream_id, nullptr, xg.p));
  // 2. the posterior mean of all P rows (evaluate(x_gen)); no variance is formed, so no read-back is left pending
  GpPending gpp;
  DMO_TRY(step_predict(ctx, who, post, xg.p, P, yg.p, nullptr, precision, &gpp));
  bool refined = false;
  DMO_TRY(gp_predict_finish(ctx, post.gp, gpp, &refined));
  if (post.mean_f32) DMO_TRY(prim_round_f32(ctx, yg.p, P * M));  // evaluate's float32 cast
  // 3. update_strategy on rows [0, n): velocities, one truncation per swarm, the float32 state
  DMO_TRY(smpso_velocities_device(ctx, parm, vel, xg.p, 0, yg.p, swarms, pop, d, M, scalars, ilb.d, iub.d));
  for (int p = 0; p < swarms; ++p) {
    const int64_t off = (int64_t)p * pop;
    DMO_TRY(smpso_truncate_device(ctx, parm + off * d, obj + off * M, xg.p + off * d, yg.p + off * M, pop, d, M, metric, ranks + off,
                                  perm.p + off));
  }
  DMO_TRY(prim_round_f32(ctx, parm, n * d));
  DMO_TRY(prim_round_f32(ctx, obj, n * M));
  // 4. the record, without a host wait into device or page-locked memory
  DMO_TRY(copy_out(ctx, x_gen, xg.p, (size_t)P * d * sizeof(double)));
  DMO_TRY(copy_out(ctx, y_gen, yg.p, (size_t)P * M * sizeof(double)));
  return DMO_OK;
}

}  // extern "C"
