// Tournament selection and the SBX / polynomial-mutation offspring generation
// (SURVEY.md section 8a rows A6, A7, A8, A9).
//   tournament_selection : dmosopt/MOEA.py:375-395
//   mutation             : dmosopt/MOEA.py:191-212
//   crossover_sbx        : dmosopt/MOEA.py:215-239
//   generate_strategy    : dmosopt/NSGA2.py:116-185 (same loop in dmosopt/AGEMOEA.py:121-183)
// Random numbers: Philox4x32-10 keyed by `seed`, counter = (index, stream_id << 8 | purpose), so every
// draw is a pure function of (seed, stream_id, purpose, index): reproducible, order-free, no state.
#include "common.cuh"

namespace {

enum Purpose : uint64_t { P_TOURNAMENT = 1, P_DECIDE = 2, P_PAIR = 3, P_SINGLE = 4, P_GENES = 5 };

__device__ __forceinline__ uint64_t ctr_hi(uint64_t stream_id, uint64_t purpose) { return (stream_id << 8) | purpose; }

// uniform in (0, 1]: never 0, so that -log(u) stays finite.  The top of the grid, (2^53 - 1) + 0.5, rounds to 2^53:
// once in 2^53 draws u == 1.0, and that candidate's key is +inf (it is drawn first)
__device__ __forceinline__ double u01_open(uint32_t hi, uint32_t lo) {
  return ((double)((((uint64_t)(hi >> 5)) << 26) | (uint64_t)(lo >> 6)) + 0.5) * (1.0 / 9007199254740992.0);
}

// ---- operators (float64, NumPy operation order, no FMA contraction) -----------------------------
__device__ __forceinline__ double clip(double x, double lo, double hi) { return np_clip(x, lo, hi); }

// MOEA.py:204-211
__device__ __forceinline__ double mutate_gene(double parent, double u, double di, double lb, double ub, double rate) {
  double e = __ddiv_rn(1.0, __dadd_rn(di, 1.0));
  double delta;
  if (u < rate)
    delta = __dsub_rn(pow(__dmul_rn(2.0, u), e), 1.0);
  else
    delta = __dsub_rn(1.0, pow(__dmul_rn(2.0, __dsub_rn(1.0, u)), e));
  return clip(__dadd_rn(parent, __dmul_rn(__dsub_rn(ub, lb), delta)), lb, ub);
}

// MOEA.py:228-238
__device__ __forceinline__ void sbx_gene(double p1, double p2, double u, double di, double lb, double ub, double& c1,
                                         double& c2) {
  double e = __ddiv_rn(1.0, __dadd_rn(di, 1.0));
  double beta;
  if (u <= 0.5)
    beta = pow(__dmul_rn(2.0, u), e);
  else
    beta = pow(__ddiv_rn(1.0, __dmul_rn(2.0, __dsub_rn(1.0, u))), e);
  double a = __dsub_rn(1.0, beta), b = __dadd_rn(1.0, beta);
  c1 = clip(__dmul_rn(0.5, __dadd_rn(__dmul_rn(a, p1), __dmul_rn(b, p2))), lb, ub);
  c2 = clip(__dmul_rn(0.5, __dadd_rn(__dmul_rn(b, p1), __dmul_rn(a, p2))), lb, ub);
}

__global__ void mutation_u_kernel(const double* __restrict__ parents, const double* __restrict__ u, int64_t n, int d,
                                  const double* __restrict__ di, const double* __restrict__ xlb,
                                  const double* __restrict__ xub, double rate, double* __restrict__ children) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  int j = (int)(t % d);
  children[t] = mutate_gene(parents[t], u[t], di[j], xlb[j], xub[j], rate);
}

__global__ void sbx_u_kernel(const double* __restrict__ p1, const double* __restrict__ p2, const double* __restrict__ u,
                             int64_t n, int d, const double* __restrict__ di, const double* __restrict__ xlb,
                             const double* __restrict__ xub, double* __restrict__ c1, double* __restrict__ c2) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  int j = (int)(t % d);
  double a, b;
  sbx_gene(p1[t], p2[t], u[t], di[j], xlb[j], xub[j], a, b);
  c1[t] = a;
  c2[t] = b;
}

// ---- tournament: Gumbel-top-k over log-weights i*log(1-p) in lexsort order ----------------------
__global__ void gumbel_keys_kernel(int64_t pop, uint64_t seed, uint64_t stream_id, double log1mp,
                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ idx, double* __restrict__ u_out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pop) return;
  Philox ph(seed);
  uint4 r = ph((uint64_t)p, ctr_hi(stream_id, P_TOURNAMENT));
  double u = u01_open(r.x, r.y);
  double key = (double)p * log1mp - log(-log(u));
  keys[p] = f64_to_ordered(-key);  // ascending sort of -key == descending key
  idx[p] = (uint32_t)p;
  if (u_out) u_out[p] = u;
}

__global__ void pool_gather_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ top, int64_t poolsize,
                                   int64_t* __restrict__ pool_idx) {
  int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < poolsize) pool_idx[q] = (int64_t)order[top[q]];
}

// ---- NSGA-II variation plan -----------------------------------------------------------------------
// iteration t: 2 children w.p. pc (SBX pair), then 1 child w.p. pm (mutant)  (NSGA2.py:143-177)
__global__ void plan_kernel(int64_t T, int64_t poolsize, double pc, double pm, uint64_t seed, uint64_t stream_id,
                            int32_t* __restrict__ count, int32_t* __restrict__ flags, int32_t* __restrict__ parents,
                            double* __restrict__ draws) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > T) return;
  if (t == T) {
    count[t] = 0;
    return;
  }
  Philox ph(seed);
  uint4 a = ph((uint64_t)t, ctr_hi(stream_id, P_DECIDE));
  uint4 b = ph((uint64_t)t, ctr_hi(stream_id, P_PAIR));
  uint4 c = ph((uint64_t)t, ctr_hi(stream_id, P_SINGLE));
  double uc = u01_53(a.x, a.y), um = u01_53(a.z, a.w);
  int cross = uc < pc ? 1 : 0, mut = um < pm ? 1 : 0;
  // ordered pair of distinct pool members == Generator.choice(poolsize, 2, replace=False)
  int64_t i1 = (int64_t)(u01_53(b.x, b.y) * (double)poolsize);
  if (i1 >= poolsize) i1 = poolsize - 1;
  int64_t i2 = poolsize > 1 ? (int64_t)(u01_53(b.z, b.w) * (double)(poolsize - 1)) : 0;
  if (poolsize > 1 && i2 >= poolsize - 1) i2 = poolsize - 2;
  if (poolsize > 1 && i2 >= i1) i2 += 1;
  int64_t i3 = (int64_t)(u01_53(c.x, c.y) * (double)poolsize);  // Generator.integers(0, poolsize)
  if (i3 >= poolsize) i3 = poolsize - 1;
  count[t] = 2 * cross + mut;
  flags[t] = cross | (mut << 1);
  parents[3 * t + 0] = (int32_t)i1;
  parents[3 * t + 1] = (int32_t)i2;
  parents[3 * t + 2] = (int32_t)i3;
  if (draws) {
    draws[t] = uc;
    draws[T + t] = um;
    draws[2 * T + 2 * t + 0] = (double)i1;
    draws[2 * T + 2 * t + 1] = (double)i2;
    draws[4 * T + t] = (double)i3;
  }
}

__global__ void children_kernel(int64_t T, int d, int64_t popsize, const int32_t* __restrict__ start,
                                const int32_t* __restrict__ flags, const int32_t* __restrict__ parents,
                                const double* __restrict__ pop_x, const int64_t* __restrict__ pool_idx,
                                const double* __restrict__ di_c, const double* __restrict__ di_m,
                                const double* __restrict__ xlb, const double* __restrict__ xub, double rate, uint64_t seed,
                                uint64_t stream_id, double* __restrict__ x_gen, int32_t* __restrict__ child_kind,
                                int64_t* __restrict__ n_children, double* __restrict__ draws) {
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= T * d) return;
  int64_t t = g / d;
  int j = (int)(g - t * d);
  const int64_t s = start[t];
  const bool active = s < popsize - 1;  // loop condition `while count < popsize - 1` (NSGA2.py:142)
  Philox ph(seed);
  uint4 r = ph((uint64_t)g, ctr_hi(stream_id, P_GENES));
  double ug_c = u01_53(r.x, r.y), ug_m = u01_53(r.z, r.w);
  if (draws) {
    draws[5 * T + (2 * t + 0) * d + j] = ug_c;
    draws[5 * T + (2 * t + 1) * d + j] = ug_m;
  }
  if (!active) return;
  const int f = flags[t];
  int64_t row = s;
  if (f & 1) {
    const double* p1 = pop_x + pool_idx[parents[3 * t + 0]] * d;
    const double* p2 = pop_x + pool_idx[parents[3 * t + 1]] * d;
    double c1, c2;
    sbx_gene(p1[j], p2[j], ug_c, di_c[j], xlb[j], xub[j], c1, c2);
    x_gen[row * d + j] = c1;
    x_gen[(row + 1) * d + j] = c2;
    if (j == 0) {
      child_kind[row] = 0;
      child_kind[row + 1] = 1;
    }
    row += 2;
  }
  if (f & 2) {
    const double* p = pop_x + pool_idx[parents[3 * t + 2]] * d;
    x_gen[row * d + j] = mutate_gene(p[j], ug_m, di_m[j], xlb[j], xub[j], rate);
    if (j == 0) child_kind[row] = 2;
    row += 1;
  }
  // the last active iteration defines the offspring count
  if (j == 0 && (int64_t)start[t + 1] >= popsize - 1) *n_children = (int64_t)start[t + 1];
}

}  // namespace

// dmo_tournament on device arrays, enqueued only (crowd and u_out may be null)
int tournament_device(dmo_ctx* ctx, const int32_t* d_rank, const double* d_crowd, int64_t pop, int64_t poolsize, uint64_t seed,
                      uint64_t stream_id, int64_t* d_pool, double* d_u) {
  // candidates in np.lexsort((-crowd, rank)) order (MOEA.py:388-389; AGEMOEA.py:140-142)
  DevBuf<uint32_t> order, i0, i1;
  DevBuf<uint64_t> k0, k1;
  DMO_TRY(order.alloc(ctx, pop));
  DMO_TRY(i0.alloc(ctx, pop));
  DMO_TRY(i1.alloc(ctx, pop));
  DMO_TRY(k0.alloc(ctx, pop));
  DMO_TRY(k1.alloc(ctx, pop));
  const double* keys[1] = {d_crowd};
  DMO_TRY(lexsort_device(ctx, d_rank, keys, d_crowd ? 1 : 0, pop, order.p, false));  // caller ranks: any int32
  DMO_LAUNCH(gumbel_keys_kernel, (unsigned)ceil_div(pop, 256), 256, 0, pop, seed, stream_id, log(0.5), k0.p, i0.p, d_u);
  DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, i1.p, pop, 0, 64));
  DMO_LAUNCH(pool_gather_kernel, (unsigned)ceil_div(poolsize, 256), 256, 0, order.p, i1.p, poolsize, d_pool);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// dmo_nsga2_generate on device arrays (d_draws may be null).  The one host wait is the read-back of the offspring count,
// *n_children: the caller sizes what follows by it.
int nsga2_generate_device(dmo_ctx* ctx, const double* d_pop_x, int d, const int64_t* d_pool, int64_t poolsize, int64_t popsize,
                          double crossover_prob, double mutation_prob, double mutation_rate, const double* d_dic,
                          const double* d_dim, const double* d_xlb, const double* d_xub, uint64_t seed, uint64_t stream_id,
                          double* d_x_gen, int32_t* d_kind, int64_t* n_children, double* d_draws) {
  DMO_REQUIRE(poolsize >= 2 || crossover_prob <= 0.0, "nsga2_generate: crossover needs a pool of at least 2");
  DMO_REQUIRE(crossover_prob > 0.0 || mutation_prob > 0.0, "nsga2_generate: both probabilities are zero");
  const int64_t T = dmo_nsga2_plan_length(popsize, crossover_prob, mutation_prob);
  DMO_REQUIRE(T > 0, "nsga2_generate: crossover_prob / mutation_prob too small for popsize %lld", (long long)popsize);
  const int64_t cap = popsize + 1;
  DevBuf<int32_t> count, start, flags, parents;
  DevBuf<int64_t> nch;
  DMO_TRY(count.alloc(ctx, T + 1));
  DMO_TRY(start.alloc(ctx, T + 1));
  DMO_TRY(flags.alloc(ctx, T));
  DMO_TRY(parents.alloc(ctx, 3 * T));
  DMO_TRY(nch.alloc(ctx, 1));
  // -1 = loop never finished; popsize 1: `while count < popsize - 1` never runs, no children
  DMO_CUDA(cudaMemsetAsync(nch.p, popsize > 1 ? 0xFF : 0, sizeof(int64_t), ctx->stream));
  DMO_CUDA(cudaMemsetAsync(d_kind, 0xFF, cap * sizeof(int32_t), ctx->stream));
  DMO_LAUNCH(plan_kernel, (unsigned)ceil_div(T + 1, 256), 256, 0, T, poolsize, crossover_prob, mutation_prob, seed,
             stream_id, count.p, flags.p, parents.p, d_draws);
  DMO_TRY(prim_exclusive_sum_i32(ctx, count.p, start.p, T + 1));
  DMO_LAUNCH(children_kernel, (unsigned)ceil_div(T * d, 256), 256, 0, T, d, popsize, start.p, flags.p, parents.p, d_pop_x,
             d_pool, d_dic, d_dim, d_xlb, d_xub, mutation_rate, seed, stream_id, d_x_gen, d_kind, nch.p, d_draws);
  DMO_CHECK_LAUNCH();
  int64_t h_n = -1;
  DMO_CUDA(cudaMemcpyAsync(&h_n, nch.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (h_n < 0 || h_n > cap)
    return dmo_fail(ctx, DMO_ERR_INTERNAL, "nsga2_generate: planned %lld iterations but produced %lld children",
                    (long long)T, (long long)h_n);
  *n_children = h_n;
  return DMO_OK;
}

extern "C" {

int dmo_mutation_u(dmo_ctx* ctx, const double* parents, const double* u, int64_t n, int d, const double* di_mutation,
                   const double* xlb, const double* xub, double mutation_rate, double* children) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && d >= 1 && parents && u && di_mutation && xlb && xub && children, "mutation_u: bad arguments");
  In<double> ip, iu, idi, ilb, iub;
  Out<double> oc;
  DMO_TRY(ip.init(ctx, parents, (size_t)n * d));
  DMO_TRY(iu.init(ctx, u, (size_t)n * d));
  DMO_TRY(idi.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(oc.init(ctx, children, (size_t)n * d));
  DMO_LAUNCH(mutation_u_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, ip.d, iu.d, n, d, idi.d, ilb.d, iub.d,
             mutation_rate, oc.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(oc.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_sbx_u(dmo_ctx* ctx, const double* parent1, const double* parent2, const double* u, int64_t n, int d,
              const double* di_crossover, const double* xlb, const double* xub, double* child1, double* child2) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && d >= 1 && parent1 && parent2 && u && di_crossover && xlb && xub && child1 && child2,
              "sbx_u: bad arguments");
  In<double> i1, i2, iu, idi, ilb, iub;
  Out<double> o1, o2;
  DMO_TRY(i1.init(ctx, parent1, (size_t)n * d));
  DMO_TRY(i2.init(ctx, parent2, (size_t)n * d));
  DMO_TRY(iu.init(ctx, u, (size_t)n * d));
  DMO_TRY(idi.init(ctx, di_crossover, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(o1.init(ctx, child1, (size_t)n * d));
  DMO_TRY(o2.init(ctx, child2, (size_t)n * d));
  DMO_LAUNCH(sbx_u_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, i1.d, i2.d, iu.d, n, d, idi.d, ilb.d, iub.d, o1.d,
             o2.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(o1.finish(ctx));
  DMO_TRY(o2.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_tournament(dmo_ctx* ctx, const int32_t* rank, const double* crowd, int64_t pop, int64_t poolsize, uint64_t seed,
                   uint64_t stream_id, int64_t* pool_idx, double* u_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(pop > 0 && poolsize > 0 && poolsize <= pop && rank && pool_idx, "tournament: bad arguments");
  In<int32_t> ir;
  In<double> icr;
  Out<int64_t> op;
  Out<double> ou;
  DMO_TRY(ir.init(ctx, rank, (size_t)pop));
  DMO_TRY(icr.init(ctx, crowd, (size_t)pop));
  DMO_TRY(op.init(ctx, pool_idx, (size_t)poolsize));
  DMO_TRY(ou.init(ctx, u_out, (size_t)pop));
  DMO_TRY(tournament_device(ctx, ir.d, icr.d, pop, poolsize, seed, stream_id, op.d, ou.d));
  DMO_TRY(op.finish(ctx));
  DMO_TRY(ou.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

// Iterations of the reference's variation loop (NSGA2.py:142-178) that are planned in parallel.  An iteration yields
// two children with probability pc and one more with probability pm, so the loop needs about popsize / (2 pc + pm)
// of them: the default rates (0.9 / 0.1) fit well inside 2 popsize + 64 (kept as the minimum, so recorded draw
// layouts do not move), a mutation-only or low-rate configuration gets the mean plus 12 standard deviations.
int64_t dmo_nsga2_plan_length(int64_t popsize, double crossover_prob, double mutation_prob) {
  const double pc = crossover_prob > 0.0 ? (crossover_prob < 1.0 ? crossover_prob : 1.0) : 0.0;
  const double pm = mutation_prob > 0.0 ? (mutation_prob < 1.0 ? mutation_prob : 1.0) : 0.0;
  const double e = 2.0 * pc + pm;
  const int64_t base = 2 * popsize + 64;
  if (!(e > 0.0)) return base;
  const double var = 4.0 * pc * (1.0 - pc) + pm * (1.0 - pm);  // variance of the children of one iteration
  const double n = (double)(popsize + 1);
  const double need = n / e + 12.0 * sqrt(var * n / e) / e + 64.0;
  if (need > 2.0e9) return -1;
  const int64_t t = (int64_t)ceil(need);
  return t > base ? t : base;
}

int dmo_nsga2_generate(dmo_ctx* ctx, const double* pop_x, int64_t npop, int d, const int64_t* pool_idx, int64_t poolsize,
                       int64_t popsize, double crossover_prob, double mutation_prob, double mutation_rate,
                       const double* di_crossover, const double* di_mutation, const double* xlb, const double* xub,
                       uint64_t seed, uint64_t stream_id, double* x_gen, int32_t* child_kind, int64_t* n_children,
                       double* draws) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(npop > 0 && d >= 1 && poolsize >= 1 && popsize >= 1 && pop_x && pool_idx && di_crossover && di_mutation &&
                  xlb && xub && x_gen && child_kind && n_children,
              "nsga2_generate: bad arguments");
  const int64_t T = dmo_nsga2_plan_length(popsize, crossover_prob, mutation_prob);
  const int64_t cap = popsize + 1;
  In<double> ipx, idc, idm, ilb, iub;
  In<int64_t> ipool;
  Out<double> ox, odraws;
  Out<int32_t> okind;
  DMO_TRY(ipx.init(ctx, pop_x, (size_t)npop * d));
  DMO_TRY(ipool.init(ctx, pool_idx, (size_t)poolsize));
  DMO_TRY(idc.init(ctx, di_crossover, d));
  DMO_TRY(idm.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(ox.init(ctx, x_gen, (size_t)cap * d));
  DMO_TRY(okind.init(ctx, child_kind, (size_t)cap));
  DMO_TRY(odraws.init(ctx, T > 0 ? draws : nullptr, (size_t)T * (5 + 2 * d)));
  DMO_TRY(nsga2_generate_device(ctx, ipx.d, d, ipool.d, poolsize, popsize, crossover_prob, mutation_prob, mutation_rate, idc.d,
                                idm.d, ilb.d, iub.d, seed, stream_id, ox.d, okind.d, n_children, odraws.d));
  DMO_TRY(ox.finish(ctx, (size_t)*n_children * d));
  DMO_TRY(okind.finish(ctx, (size_t)*n_children));
  DMO_TRY(odraws.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
