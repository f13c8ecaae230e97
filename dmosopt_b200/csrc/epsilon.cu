// Epsilon-nondominated archive (replaces dmosopt/MOEA.py:470-595 EpsilonSort, fed every row in order as
// dmosopt/MOASMO.py:743-748 epsilon_get_best does).
//
// Inserting the rows one by one gives the same archive as one batch, tie rule included:
//   * every row falls into its box, box_j = floor(y_j / eps_j);
//   * in each box the row of least dist = sum_j (y_j - box_j eps_j)^2 wins, the last row in input order on a tie (an
//     archived row only stays when its dist is strictly smaller); when some eps_j is infinite every dist is NaN
//     (corner 0 * inf) and the last row wins;
//   * the winners of the boxes that no other occupied box dominates are the archive, in ascending row order.
//
// Pipeline (the context's stream):
//   1. box_kernel: nan_to_num, the box (float64 floor values: exact at any magnitude, no integer overflow), the
//      overflow test and dist, in the reference's order of operations with explicit IEEE intrinsics (no FMA
//      contraction); key = -dist (0 for every row when an eps is infinite);
//   2. dense ids of the M box columns and of the key (rank.cu step 1), and the stable lexicographic order of
//      (box_1 .. box_M, key) (rank.cu step 2): inside a box the rows run by dist descending, ties in ascending row order,
//      so the last position of each box holds its winner;
//   3. the winners' boxes (one per occupied box) through the rank-0 filter of the hypervolume (hv.cu
//      nondominated_keep_flags);
//   4. the surviving winners flagged by row and compacted by a scan: ascending row indices.
//
// Work: (M + 1) radix sorts of n keys; the box filter costs up to k^2 / 2 id compares for k occupied boxes when most of
// them survive (M >= 4 at fine eps), the cell grid's linear pass for M <= 3 from 8192 boxes (DESIGN.md section 4.9).
#include <float.h>

#include "common.cuh"

namespace {

constexpr int EPS_MAXM = 16;

struct EpsArgs {
  double e[EPS_MAXM];  // eps with 0 / NaN replaced by 1e-8
};

__global__ void box_kernel(const double* __restrict__ Y, int64_t n, int M, EpsArgs ea, int inf_eps, double* __restrict__ box,
                           double* __restrict__ key, unsigned long long* __restrict__ first_overflow) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double dist = 0.0;
  bool ovf = false;
#pragma unroll
  for (int j = 0; j < EPS_MAXM; ++j) {  // unrolled: ea.e stays in the parameter bank
    if (j >= M) break;
    double y = Y[i * M + j];
    y = isnan(y) ? 0.0 : isinf(y) ? (y > 0.0 ? DBL_MAX : -DBL_MAX) : y;  // np.nan_to_num
    const double e = ea.e[j];
    const double q = __ddiv_rn(y, e);
    ovf |= isinf(q);
    const double b = floor(q);
    box[i * M + j] = b;
    const double d = __dsub_rn(y, __dmul_rn(b, e));
    const double s = __dmul_rn(d, d);
    dist = j == 0 ? s : __dadd_rn(dist, s);
  }
  key[i] = inf_eps ? 0.0 : -dist;
  if (ovf) atomicMin(first_overflow, (unsigned long long)i);
}

// win[p] = 1 iff position p is the last of its box in the lexicographic order (the box's winner); win[n] = 0
__global__ void winner_flag_kernel(const uint32_t* __restrict__ R, const uint32_t* __restrict__ perm, int64_t n, int M,
                                   int32_t* __restrict__ win) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p > n) return;
  if (p == n) {
    win[n] = 0;
    return;
  }
  int f = 1;
  if (p + 1 < n) {
    const uint32_t a = perm[p], b = perm[p + 1];
    f = 0;
    for (int j = 0; j < M; ++j) f |= R[(int64_t)j * n + a] != R[(int64_t)j * n + b];
  }
  win[p] = f;
}

// the winners' boxes, packed (k, M), and their rows
__global__ void gather_winners_kernel(const double* __restrict__ box, const uint32_t* __restrict__ perm, const int32_t* __restrict__ win,
                                      const int32_t* __restrict__ pos, int64_t n, int M, double* __restrict__ wbox,
                                      uint32_t* __restrict__ wrow) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || !win[p]) return;
  const uint32_t r = perm[p];
  const int64_t q = pos[p];
  for (int j = 0; j < M; ++j) wbox[q * M + j] = box[(int64_t)r * M + j];
  wrow[q] = r;
}

__global__ void mark_kept_kernel(const int32_t* __restrict__ flag, const uint32_t* __restrict__ wrow, int64_t k,
                                 int32_t* __restrict__ kept) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < k && flag[q]) kept[wrow[q]] = 1;
}

__global__ void write_rows_kernel(const int32_t* __restrict__ kept, const int32_t* __restrict__ pos, int64_t n,
                                  int64_t* __restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && kept[i]) idx[pos[i]] = i;
}

}  // namespace

extern "C" int dmo_epsilon_sort(dmo_ctx* ctx, const double* Y, int64_t n, int M, const double* eps, int64_t* idx, int64_t* count) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(count, "epsilon_sort: null count");
  *count = 0;
  DMO_REQUIRE(n >= 0 && M >= 1 && M <= EPS_MAXM, "epsilon_sort: bad shape n=%lld M=%d (1 <= M <= %d)", (long long)n, M, EPS_MAXM);
  DMO_REQUIRE(n < ((int64_t)1 << 31) - 4096, "epsilon_sort: n=%lld too large", (long long)n);
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(Y && eps && idx, "epsilon_sort: null pointer");

  EpsArgs ea;
  if (dmo_is_device_ptr(eps)) {
    DMO_CUDA(cudaMemcpyAsync(ea.e, eps, M * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
  } else {
    for (int j = 0; j < M; ++j) ea.e[j] = eps[j];
  }
  int inf_eps = 0;
  for (int j = 0; j < M; ++j) {
    if (ea.e[j] == 0.0 || isnan(ea.e[j])) ea.e[j] = 1e-8;  // MOEA.py:509
    inf_eps |= isinf(ea.e[j]) ? 1 : 0;
  }

  In<double> y;
  Out<int64_t> out;
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  DMO_TRY(out.init(ctx, idx, (size_t)n));
  const unsigned g = (unsigned)ceil_div(n, 256);
  const unsigned g1 = (unsigned)ceil_div(n + 1, 256);

  // 1. boxes, distances, overflow
  DevBuf<double> box, key;
  DevBuf<unsigned long long> ovf;
  DMO_TRY(box.alloc(ctx, (size_t)n * M));
  DMO_TRY(key.alloc(ctx, n));
  DMO_TRY(ovf.alloc(ctx, 1));
  DMO_CUDA(cudaMemsetAsync(ovf.p, 0xFF, sizeof(unsigned long long), ctx->stream));
  {
    ProfileScope ps(ctx, "epsilon_box");
    DMO_LAUNCH(box_kernel, g, 256, 0, y.d, n, M, ea, inf_eps, box.p, key.p, ovf.p);
  }
  DMO_CHECK_LAUNCH();
  unsigned long long first = 0;
  DMO_CUDA(cudaMemcpyAsync(&first, ovf.p, sizeof(first), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (first != ~0ull)
    return dmo_fail(ctx, DMO_ERR_OVERFLOW, "epsilon_sort: y / eps overflows to infinity in row %llu (the reference's math.floor raises OverflowError)", first);

  // 2. group by box, winner last in each box
  const uint32_t* perm = nullptr;
  DevBuf<uint32_t> permA, permB;
  DevBuf<int32_t> win, wpos;
  int32_t k = 0;
  {
    ProfileScope ps(ctx, "epsilon_group");
    DevBuf<uint32_t> Rb, Rk, R, maxb, maxk;
    DMO_TRY(dense_ids(ctx, box.p, n, M, Rb, maxb));
    DMO_TRY(dense_ids(ctx, key.p, n, 1, Rk, maxk));
    DMO_TRY(R.alloc(ctx, (size_t)(M + 1) * n));
    DMO_CUDA(cudaMemcpyAsync(R.p, Rb.p, (size_t)M * n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(R.p + (size_t)M * n, Rk.p, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_TRY(lex_order(ctx, R.p, n, M + 1, 0, permA, permB, &perm));
    DMO_TRY(win.alloc(ctx, n + 1));
    DMO_TRY(wpos.alloc(ctx, n + 1));
    DMO_LAUNCH(winner_flag_kernel, g1, 256, 0, R.p, perm, n, M, win.p);
    DMO_CHECK_LAUNCH();
    DMO_TRY(prim_exclusive_sum_i32(ctx, win.p, wpos.p, n + 1));
    DMO_CUDA(cudaMemcpyAsync(&k, wpos.p + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
  }

  // 3. the boxes no other occupied box dominates
  DevBuf<double> wbox;
  DevBuf<uint32_t> wrow;
  DevBuf<int32_t> flag;
  DMO_TRY(wbox.alloc(ctx, (size_t)k * M));
  DMO_TRY(wrow.alloc(ctx, k));
  DMO_LAUNCH(gather_winners_kernel, g, 256, 0, box.p, perm, win.p, wpos.p, n, M, wbox.p, wrow.p);
  DMO_CHECK_LAUNCH();
  DMO_TRY(nondominated_keep_flags(ctx, wbox.p, k, M, flag));

  // 4. their rows in ascending order
  DevBuf<int32_t> kept, kpos;
  DMO_TRY(kept.alloc(ctx, n + 1));
  DMO_TRY(kpos.alloc(ctx, n + 1));
  DMO_CUDA(cudaMemsetAsync(kept.p, 0, (size_t)(n + 1) * sizeof(int32_t), ctx->stream));
  DMO_LAUNCH(mark_kept_kernel, (unsigned)ceil_div(k, 256), 256, 0, flag.p, wrow.p, k, kept.p);
  DMO_CHECK_LAUNCH();
  DMO_TRY(prim_exclusive_sum_i32(ctx, kept.p, kpos.p, n + 1));
  int32_t h = 0;
  DMO_CUDA(cudaMemcpyAsync(&h, kpos.p + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_LAUNCH(write_rows_kernel, g, 256, 0, kept.p, kpos.p, n, out.d);
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  DMO_TRY(out.finish(ctx, (size_t)h));
  DMO_CUDA(dmo_wait(ctx));
  *count = h;
  return DMO_OK;
}
