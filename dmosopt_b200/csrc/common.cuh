// Shared plumbing for the dmosopt_b200 CUDA library (sm_90a).
// Context, stream-ordered scratch buffers, host/device pointer staging,
// launch accounting, order-preserving float transforms and Philox4x32-10.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../include/dmosopt_b200.h"

struct dmo_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaMemPool_t pool = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int sm_count = 132;  // H100 SXM; replaced by the device's count in dmo_create
  int64_t launches = 0;
  int64_t waits = 0;  // times the host blocked on the stream (dmo_wait); dmo_wait_count() reports it
  std::string err;
  void* flush_buf = nullptr;
  size_t flush_bytes = 0;
  int* dev_flag = nullptr;  // device-side error / watchdog flag (int[4])
  uint64_t h2d_bytes = 0, d2h_bytes = 0;  // bytes staged for host buffers (In<> / Out<>)
  // pinned slots and their events for read-backs the host waits on later than it enqueues them: [0], [1] the front peel's
  // counts (rank.cu), [2] the fused step's GP read-back (gp.cu); created on first use (dmo_lag_slots), released by
  // dmo_destroy
  unsigned long long* lag_host = nullptr;
  cudaEvent_t lag_ev[3] = {nullptr, nullptr, nullptr};
  // side streams for independent work of one call (SideStreams below); created on first use, released by dmo_destroy
  static constexpr int kSide = 4;
  cudaStream_t side[kSide] = {};
  cudaEvent_t side_ev[kSide + 1] = {};  // [0]: fork point on the main stream, [1 + s]: end of side stream s
  // the fused step's concurrent lane (step.cu): `lane` runs the truncation beside the GP variance contraction, which runs on
  // `gp_hi`, a stream of the device's greatest priority, so that its CTAs take their SMs before the lane's kernels fill
  // the card.  lane_ev: [0] every mean written, [1] / [2] fork to / join from gp_hi, [3] end of the lane.  Created on
  // first use (dmo_lane_streams), released by dmo_destroy
  cudaStream_t lane = nullptr, gp_hi = nullptr;
  cudaEvent_t lane_ev[4] = {};
  // optional per-kernel CUDA-event timers (dmo_profile_enable); bench.py reads them for the roofline
  bool profiling = false;
  struct Timer {
    std::string name;
    cudaEvent_t a, b;
  };
  std::vector<Timer> timers;
};

// RAII: records a start/stop event pair around a kernel (or a group of launches) when profiling is on
struct ProfileScope {
  dmo_ctx* ctx;
  int idx = -1;
  ProfileScope(dmo_ctx* c, const char* name) : ctx(c) {
    if (!c->profiling) return;
    dmo_ctx::Timer t;
    t.name = name;
    if (cudaEventCreate(&t.a) != cudaSuccess || cudaEventCreate(&t.b) != cudaSuccess) return;
    cudaEventRecord(t.a, c->stream);
    c->timers.push_back(t);
    idx = (int)c->timers.size() - 1;
  }
  ~ProfileScope() {
    if (idx >= 0) cudaEventRecord(ctx->timers[idx].b, ctx->stream);
  }
};

int dmo_fail(dmo_ctx* ctx, int code, const char* fmt, ...);

#define DMO_CUDA(call)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return dmo_fail(ctx, DMO_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                      __FILE__, __LINE__);                                                    \
  } while (0)

#define DMO_TRY(expr)              \
  do {                             \
    int s__ = (expr);              \
    if (s__ != DMO_OK) return s__; \
  } while (0)

#define DMO_REQUIRE(cond, ...)                                 \
  do {                                                         \
    if (!(cond)) return dmo_fail(ctx, DMO_ERR_ARG, __VA_ARGS__); \
  } while (0)

// every kernel launch of the library goes through this macro so that
// dmo_launch_count() is the library's own count of launched kernels
#define DMO_LAUNCH(kernel, grid, block, smem, ...)                       \
  do {                                                                   \
    kernel<<<(grid), (block), (smem), ctx->stream>>>(__VA_ARGS__);       \
    ctx->launches++;                                                     \
  } while (0)

#define DMO_CHECK_LAUNCH() DMO_CUDA(cudaGetLastError())

// Independent work issued on side streams of the context: side s waits for everything enqueued on the main stream
// before the constructor, and the main stream waits for every side stream's work in the destructor.  Inside, on(s)
// points ctx->stream at side s, so any library function called there enqueues on it (and allocates and frees its own
// scratch there); back() returns to the main stream.  Scratch shared with the main stream is allocated before the
// constructor and released after the destructor.  The bits do not depend on the interleaving: the streams write
// disjoint buffers.
struct SideStreams {
  dmo_ctx* ctx;
  cudaStream_t main;
  int k = 0;
  int rc = DMO_OK;
  SideStreams(dmo_ctx* c, int nside);
  ~SideStreams();
  void on(int s) { ctx->stream = ctx->side[s]; }
  void back() { ctx->stream = main; }
};

int dmo_lag_slots(dmo_ctx* ctx);
int dmo_lane_streams(dmo_ctx* ctx);

// every host wait of the library on its stream goes through this, so that dmo_wait_count() counts them
static inline cudaError_t dmo_wait(dmo_ctx* ctx) {
  ctx->waits++;
  return cudaStreamSynchronize(ctx->stream);
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------
// Stream-ordered scratch buffer (cudaMallocAsync on the context's pool).
template <typename T>
struct DevBuf {
  dmo_ctx* ctx = nullptr;
  T* p = nullptr;
  size_t n = 0;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int alloc(dmo_ctx* c, size_t count) {
    release();
    ctx = c;
    n = count;
    if (count == 0) count = 1;
    cudaError_t e = cudaMallocAsync((void**)&p, count * sizeof(T), c->stream);
    if (e != cudaSuccess) {
      p = nullptr;
      return dmo_fail(c, DMO_ERR_CUDA, "cudaMallocAsync(%zu bytes) failed: %s", count * sizeof(T),
                      cudaGetErrorString(e));
    }
    return DMO_OK;
  }
  void release() {
    if (p) cudaFreeAsync(p, ctx->stream);
    p = nullptr;
  }
};

bool dmo_is_device_ptr(const void* p);

// Input array that may live on the host: gives a device pointer valid on ctx->stream.
template <typename T>
struct In {
  DevBuf<T> buf;
  const T* d = nullptr;
  int init(dmo_ctx* ctx, const T* src, size_t count) {
    if (src == nullptr || count == 0) {
      d = nullptr;
      return DMO_OK;
    }
    if (dmo_is_device_ptr(src)) {
      d = src;
      return DMO_OK;
    }
    DMO_TRY(buf.alloc(ctx, count));
    DMO_CUDA(cudaMemcpyAsync(buf.p, src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    ctx->h2d_bytes += count * sizeof(T);
    d = buf.p;
    return DMO_OK;
  }
};

// Output array that may live on the host: kernels write to .d, finish() copies back.
template <typename T>
struct Out {
  DevBuf<T> buf;
  T* d = nullptr;
  T* host = nullptr;
  size_t count = 0;
  int init(dmo_ctx* ctx, T* dst, size_t cnt) {
    count = cnt;
    if (dst == nullptr) {
      d = nullptr;
      return DMO_OK;
    }
    if (dmo_is_device_ptr(dst)) {
      d = dst;
      return DMO_OK;
    }
    host = dst;
    DMO_TRY(buf.alloc(ctx, cnt));
    d = buf.p;
    return DMO_OK;
  }
  int finish(dmo_ctx* ctx, size_t cnt = (size_t)-1) {
    if (host && d) {
      size_t c = (cnt == (size_t)-1) ? count : cnt;
      if (c) DMO_CUDA(cudaMemcpyAsync(host, d, c * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
      ctx->d2h_bytes += c * sizeof(T);
    }
    return DMO_OK;
  }
};

// An output the caller may hand in as device, page-locked or pageable host memory (ctx.cu).  The copy is enqueued on the
// stream; into pageable memory cudaMemcpyAsync returns only once it has landed, which is a host wait and counted as one.
int copy_out(dmo_ctx* ctx, void* dst, const void* src, size_t bytes);

// ---------------------------------------------------------------------------
// device helpers
#ifdef __CUDACC__

// IEEE-754 order-preserving maps (radix-sortable keys).  -0.0 is canonicalised to +0.0
// first so that it compares equal to +0.0 like numpy does.
__device__ __forceinline__ uint64_t f64_to_ordered(double x) {
  x = x + 0.0;
  uint64_t b = (uint64_t)__double_as_longlong(x);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
// the same, with every NaN (either sign bit, any payload) mapped to one key above +inf: the order of NumPy's sorts, which
// put NaN last and keep NaNs in input order.  The sort keys that mirror a NumPy sort use it; the key decodes to a NaN.
__device__ __forceinline__ uint64_t f64_to_ordered_nan_last(double x) {
  return isnan(x) ? 0xFFF8000000000000ull : f64_to_ordered(x);
}
__device__ __forceinline__ double ordered_to_f64(uint64_t k) {
  uint64_t b = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double((long long)b);
}
__device__ __forceinline__ uint32_t f32_to_ordered(float x) {
  x = x + 0.0f;
  uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// np.clip(x, lo, hi) == np.minimum(np.maximum(x, lo), hi): a NaN in any operand propagates (fmin / fmax would drop it),
// and between equal operands (+0.0 / -0.0) the first one is kept, as NumPy's maximum / minimum do
__device__ __forceinline__ double np_clip(double x, double lo, double hi) {
  const double m = (x >= lo || isnan(x)) ? x : lo;
  return (m <= hi || isnan(m)) ? m : hi;
}

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw 2011): counter-based, no state in memory.
struct Philox {
  uint32_t k0, k1;
  __device__ __forceinline__ Philox(uint64_t seed) : k0((uint32_t)seed), k1((uint32_t)(seed >> 32)) {}
  __device__ __forceinline__ uint4 operator()(uint64_t ctr_lo, uint64_t ctr_hi) const {
    uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32);
    uint32_t c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
    uint32_t a = k0, b = k1;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
      uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
      uint32_t n0 = h1 ^ c1 ^ a, n1 = l1, n2 = h0 ^ c3 ^ b, n3 = l0;
      c0 = n0;
      c1 = n1;
      c2 = n2;
      c3 = n3;
      a += 0x9E3779B9u;
      b += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
};
// 53-bit uniform in [0, 1) from two 32-bit words (same construction as numpy's Generator.random)
__device__ __forceinline__ double u01_53(uint32_t hi, uint32_t lo) {
  return (double)((((uint64_t)(hi >> 5)) << 26) | (uint64_t)(lo >> 6)) * (1.0 / 9007199254740992.0);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of one value per thread over a CTA of NW warps in a fixed order: warp_sum in each warp, then s = 0.0 + red[0] + ...
// + red[NW - 1] (red: NW doubles of shared memory), so repeated calls are bit-identical.  Every thread of the CTA must call
// it, and every thread gets the result.  The barriers before the slots are written and after they are read let a caller
// call it back to back or reuse red at once; the trailing one also completes the caller's earlier shared-memory writes.
// Reductions that combine the warps in another order (pairwise, or a shared-memory tree) keep their own code: folding them
// in here would change their bits.
template <int NW>
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll 8  // whole for CTAs of up to 256 threads; a whole 32-warp unroll spills in finish_fit_kernel (gp_fit.cu)
  for (int w = 0; w < NW; ++w) s += red[w];
  __syncthreads();
  return s;
}

#endif  // __CUDACC__

// ---------------------------------------------------------------------------
// primitives implemented in prims.cu (CUB is only included there)
int prim_sort_pairs_u64(dmo_ctx* ctx, const uint64_t* kin, uint64_t* kout, const uint32_t* vin,
                        uint32_t* vout, int64_t n, int begin_bit, int end_bit);
int prim_sort_pairs_u32(dmo_ctx* ctx, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                        uint32_t* vout, int64_t n, int begin_bit, int end_bit);
int prim_inclusive_sum_u32(dmo_ctx* ctx, const uint32_t* in, uint32_t* out, int64_t n);
int prim_exclusive_sum_i32(dmo_ctx* ctx, const int32_t* in, int32_t* out, int64_t n);
int prim_inclusive_min_f64(dmo_ctx* ctx, const double* in, double* out, int64_t n);
int prim_iota_u32(dmo_ctx* ctx, uint32_t* out, int64_t n);
// out[p] = src[idx[p]], p < n
int prim_gather_u32(dmo_ctx* ctx, const uint32_t* src, const uint32_t* idx, int64_t n, uint32_t* out);
// in place a[i] = (double)(float)a[i], i < n
int prim_round_f32(dmo_ctx* ctx, double* a, int64_t n);
// keys[i] = f64_to_ordered(F[i][j]) (-0.0 == +0.0) and idx[i] = i, i < n, of the row-major (n, M) F
int prim_col_keys(dmo_ctx* ctx, const double* dF, int64_t n, int M, int j, uint64_t* keys, uint32_t* idx);
// sidx (allocated here, n): the rows of F in ascending order of column j (prim_col_keys, then the radix sort), ties in row
// order.  dense_ids (rank.cu) runs the same two steps on scratch it keeps across the objectives, and also reads the keys.
int prim_sort_by_column(dmo_ctx* ctx, const double* dF, int64_t n, int M, int j, DevBuf<uint32_t>& sidx);

// internal device-pointer entry points shared between translation units
// (all pointers are device pointers; outputs in caller-provided device buffers)
int rank_nd_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, int32_t* d_rank);
int rank_nd_device_keep(dmo_ctx* ctx, const double* dY, int64_t n, int M, int64_t keep, int32_t* d_rank);
// 0 for non-dominated rows, non-zero otherwise (no ranks: no dependency chain)
int nondominated_flags_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, int32_t* d_flag01);
// flag[i] = 1 iff row i is non-dominated (identical rows do not dominate each other); flag holds n + 1 entries, flag[n] = 0
int nondominated_keep_flags(dmo_ctx* ctx, const double* dF, int64_t n, int M, DevBuf<int32_t>& flag);
// steps 1 and 2 of the rank (csrc/rank.cu): R[j * n + i] = dense id of Y[i, j] (order- and equality-preserving, -0.0 ==
// +0.0; 1 <= M <= 16), maxid[j] = its largest id; and the stable lexicographic order of the id vectors (sshift = 0), ties in
// ascending row order, *perm (position -> row) pointing into permA or permB
int dense_ids(dmo_ctx* ctx, const double* dY, int64_t n, int M, DevBuf<uint32_t>& R, DevBuf<uint32_t>& maxid);
int lex_order(dmo_ctx* ctx, const uint32_t* R, int64_t n, int M, int sshift, DevBuf<uint32_t>& permA, DevBuf<uint32_t>& permB,
              const uint32_t** perm);
int crowding_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, double* dD);
int euclidean_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, double* dD);
// perm (uint32, n) sorted by (rank asc, then each desc key descending, stable on index).  rank_below_n: the ranks are
// known to lie in [0, n) (ranks from rank_nd), so the radix sort needs only the bits of n; otherwise any int32 value
// (caller-supplied ranks, negative or >= n) sorts over all 32 bits
int lexsort_device(dmo_ctx* ctx, const int32_t* d_rank, const double* const* d_desc_keys, int nkeys,
                   int64_t n, uint32_t* d_perm, bool rank_below_n);
int hypervolume_device(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* h_ref, double* h_out);
// the same when the rows carry their non-dominated ranks within a superset (rank > 0 rows are skipped, no filter pass)
int hypervolume_device_ranked(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* h_ref, const int32_t* d_rank,
                              double* h_out);
// its M = 3 route in two halves (hv.cu): the device work, with no host read, then the route's reads and the volume.
// h_ref must be finite.  The buffers are released by the destructor, on the stream current at that point.
struct Hv3Ranked {
  int64_t n = 0;
  double ref[3] = {0.0, 0.0, 0.0};
  bool tree = false;
  DevBuf<int32_t> pos;
  DevBuf<double> xs, ys, zs, res;
  DevBuf<uint32_t> zo;
};
int hv3_ranked_enqueue(dmo_ctx* ctx, const double* dF, int64_t n, const double* h_ref, const int32_t* d_rank, Hv3Ranked& s);
int hv3_ranked_finish(dmo_ctx* ctx, Hv3Ranked& s, double* h_out);
// device bodies of dmo_tournament, dmo_nsga2_generate and dmo_remove_worst (variation.cu, sortmo.cu) for dmo_nsga2_step:
// device arrays only, enqueued on the context's stream without the public entry points' trailing wait.  The generate body
// waits once, for the offspring count it returns in *n_children.
int tournament_device(dmo_ctx* ctx, const int32_t* d_rank, const double* d_crowd, int64_t pop, int64_t poolsize, uint64_t seed,
                      uint64_t stream_id, int64_t* d_pool, double* d_u);
int nsga2_generate_device(dmo_ctx* ctx, const double* d_pop_x, int d, const int64_t* d_pool, int64_t poolsize, int64_t popsize,
                          double crossover_prob, double mutation_prob, double mutation_rate, const double* d_dic,
                          const double* d_dim, const double* d_xlb, const double* d_xub, uint64_t seed, uint64_t stream_id,
                          double* d_x_gen, int32_t* d_kind, int64_t* n_children, double* d_draws);
int remove_worst_device(dmo_ctx* ctx, const double* dX, const double* dY, int64_t n, int d, int M, int metric,
                        const double* const* d_extra, int n_extra, int64_t keep, double* dX_out, double* dY_out, int32_t* d_rank_out,
                        int64_t* d_perm_out);
// device bodies of dmo_gather_rows, dmo_cmaes_generate, dmo_cmaes_step_z, dmo_scale_rows, dmo_cmaes_update_cholesky
// (moea_ext.cu) and dmo_ehvi_select (hv.cu) for the resident CMA-ES step (cmaes_step.cu): device arrays only, without the
// entry points' trailing waits.  ehvi_select_device takes 1 <= k <= nc and waits once, for its box count.
int gather_rows_device(dmo_ctx* ctx, const double* src, const double* alt, const uint8_t* sel, const int64_t* idx, int64_t n,
                       int64_t row_elems, double* dst);
int cmaes_generate_device(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols, const double* A,
                          const int64_t* p_idx, const double* z, int64_t n, int d, const double* xlb, const double* xub, double* x_out);
int cmaes_step_z_device(dmo_ctx* ctx, const double* x_gen, const int64_t* cand_idx, const double* parents_x, const int64_t* par_idx,
                        const double* xlb, const double* xub, const double* steps, int64_t n, int d, double* z_out);
int scale_rows_device(dmo_ctx* ctx, double* rows, int64_t row_elems, int64_t n_seg, const int64_t* seg_row, const int64_t* seg_start,
                      const double* factors);
int cmaes_update_cholesky_device(dmo_ctx* ctx, double* A, double* Ainv, double* pc, const double* z, const double* psucc, int64_t n, int d,
                                 double cc, double ccov, double pthresh);
int ehvi_select_device(dmo_ctx* ctx, const double* F, int64_t nf, const double* means, const double* variances, int64_t nc, int M,
                       const double* ref, int nds, int64_t k, int64_t* sel, double* score);
// the feasibility model's rank (csrc/feasibility.cu) of n device rows into d_rank, enqueued on the context's stream
int feas_rank_device(dmo_ctx* ctx, const dmo_feas* m, const double* dX, int64_t n, double* d_rank);
int feas_model_dim(const dmo_feas* m);
