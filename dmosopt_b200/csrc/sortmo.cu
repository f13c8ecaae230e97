// Distance metrics and the sortMO / remove_worst ordering
// (SURVEY.md section 8a rows A3, A4, A5, A21).
//   crowding  : dmosopt/indicators.py:12-51     euclidean : dmosopt/indicators.py:54-62
//   sortMO    : dmosopt/MOEA.py:242-297         remove_worst : dmosopt/MOEA.py:398-423
//   duplicates: dmosopt/MOEA.py:426-437
// All float64 arithmetic below uses explicit round-to-nearest intrinsics (no FMA contraction) in the
// order the reference performs it, so the distances are bit-identical to NumPy's.
#include "common.cuh"

namespace {

constexpr int MAX_OBJ = 16;  // objectives; the kernels below size their register arrays MAXM = 8 or 16

__global__ void minmax_init_kernel(uint64_t* mn, uint64_t* mx, int M) {
  int j = threadIdx.x;
  if (j < M) {
    mn[j] = 0xFFFFFFFFFFFFFFFFull;
    mx[j] = 0ull;
  }
}

// column-wise min / max of a row-major (n, M) matrix through order-preserving 64-bit keys
template <int MAXM>
__global__ void minmax_kernel(const double* __restrict__ Y, int64_t n, int M, uint64_t* mn, uint64_t* mx) {
  __shared__ uint64_t smn[MAXM], smx[MAXM];
  if (threadIdx.x < M) {
    smn[threadIdx.x] = 0xFFFFFFFFFFFFFFFFull;
    smx[threadIdx.x] = 0ull;
  }
  __syncthreads();
  uint64_t lmn[MAXM], lmx[MAXM];
#pragma unroll
  for (int j = 0; j < MAXM; ++j) {
    lmn[j] = 0xFFFFFFFFFFFFFFFFull;
    lmx[j] = 0ull;
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int j = 0; j < MAXM; ++j)
      if (j < M) {
        uint64_t k = f64_to_ordered(Y[i * M + j]);
        lmn[j] = k < lmn[j] ? k : lmn[j];
        lmx[j] = k > lmx[j] ? k : lmx[j];
      }
  }
#pragma unroll
  for (int j = 0; j < MAXM; ++j)
    if (j < M) {
      for (int o = 16; o > 0; o >>= 1) {
        uint64_t a = __shfl_xor_sync(0xffffffffu, lmn[j], o);
        uint64_t b = __shfl_xor_sync(0xffffffffu, lmx[j], o);
        lmn[j] = a < lmn[j] ? a : lmn[j];
        lmx[j] = b > lmx[j] ? b : lmx[j];
      }
      if ((threadIdx.x & 31) == 0) {
        atomicMin((unsigned long long*)&smn[j], (unsigned long long)lmn[j]);
        atomicMax((unsigned long long*)&smx[j], (unsigned long long)lmx[j]);
      }
    }
  __syncthreads();
  if (threadIdx.x < M) {
    atomicMin((unsigned long long*)&mn[threadIdx.x], (unsigned long long)smn[threadIdx.x]);
    atomicMax((unsigned long long*)&mx[threadIdx.x], (unsigned long long)smx[threadIdx.x]);
  }
}

// U = (Y - lb) / (ub - lb), zero range -> 1.0 (indicators.py:26-31)
__device__ __forceinline__ double normalise(double y, uint64_t kmn, uint64_t kmx) {
  double lb = ordered_to_f64(kmn), ub = ordered_to_f64(kmx);
  double rg = __dsub_rn(ub, lb);
  if (rg == 0.0) rg = 1.0;
  return __ddiv_rn(__dsub_rn(y, lb), rg);
}

__global__ void crowd_keys_kernel(const double* __restrict__ Y, int64_t n, int M, int j, const uint64_t* mn,
                                  const uint64_t* mx, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    keys[i] = f64_to_ordered_nan_last(normalise(Y[i * M + j], mn[j], mx[j]));
    idx[i] = (uint32_t)i;
  }
}

// contribution of sorted position p in objective j: ends 1.0, interior next - prev (indicators.py:39-44)
__global__ void crowd_contrib_kernel(const uint64_t* __restrict__ skeys, const uint32_t* __restrict__ sidx, int64_t n,
                                     int M, int j, double* __restrict__ contrib, uint32_t* __restrict__ pos) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  double ds;
  if (p == 0 || p == n - 1)
    ds = 1.0;
  else
    ds = __dsub_rn(ordered_to_f64(skeys[p + 1]), ordered_to_f64(skeys[p - 1]));
  uint32_t i = sidx[p];
  contrib[(int64_t)i * M + j] = ds;
  pos[(int64_t)i * M + j] = (uint32_t)p;
}

// D[i] = sum of the M contributions in (sorted position, objective) order (indicators.py:46-49)
template <int MAXM>
__global__ void crowd_sum_kernel(const double* __restrict__ contrib, const uint32_t* __restrict__ pos, int64_t n, int M,
                                 double* __restrict__ D) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t key[MAXM];
  double c[MAXM];
#pragma unroll
  for (int j = 0; j < MAXM; ++j)
    if (j < M) {
      key[j] = (uint64_t)pos[i * M + j] * (uint64_t)M + (uint64_t)j;
      c[j] = contrib[i * M + j];
    }
  // insertion sort of <= MAXM items by key
#pragma unroll
  for (int a = 1; a < MAXM; ++a)
    if (a < M) {
#pragma unroll
      for (int b = a; b > 0; --b) {
        if (key[b] < key[b - 1]) {
          uint64_t tk = key[b];
          key[b] = key[b - 1];
          key[b - 1] = tk;
          double tc = c[b];
          c[b] = c[b - 1];
          c[b - 1] = tc;
        }
      }
    }
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < MAXM; ++j)
    if (j < M) s = __dadd_rn(s, c[j]);
  if (isnan(s)) s = 0.0;
  D[i] = s;
}

__global__ void fill_f64_kernel(double* out, int64_t n, double v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

template <int MAXM>
__global__ void euclid_kernel(const double* __restrict__ Y, int64_t n, int M, const uint64_t* mn, const uint64_t* mx,
                              double* __restrict__ D) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double sq[MAXM];
#pragma unroll
  for (int j = 0; j < MAXM; ++j)
    if (j < M) {
      double u = normalise(Y[i * M + j], mn[j], mx[j]);
      sq[j] = __dmul_rn(u, u);
    }
  double s;
  if (MAXM > 8 && M > 8) {
    // numpy's pairwise sum from 8 elements on: 8 accumulators over the blocks of 8, combined as a tree, then the rest in order
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = (M == 16) ? __dadd_rn(sq[j], sq[8 + j]) : sq[j];
    s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
#pragma unroll
    for (int j = 8; j < MAXM; ++j)
      if (j < M && M < 16) s = __dadd_rn(s, sq[j]);
  } else if (M == 8) {  // numpy's pairwise sum switches to 8 accumulators at 8 elements
    s = __dadd_rn(__dadd_rn(__dadd_rn(sq[0], sq[1]), __dadd_rn(sq[2], sq[3])),
                  __dadd_rn(__dadd_rn(sq[4], sq[5]), __dadd_rn(sq[6], sq[7])));
  } else {
    s = 0.0;
#pragma unroll
    for (int j = 0; j < MAXM; ++j)
      if (j < M) s = __dadd_rn(s, sq[j]);
  }
  D[i] = __dsqrt_rn(s);
}

// ---- lexsort helpers
__global__ void desc_key_kernel(const double* __restrict__ key, const uint32_t* __restrict__ perm, int64_t n,
                                uint64_t* __restrict__ out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = f64_to_ordered_nan_last(-key[perm[p]]);
}
__global__ void rank_key_kernel(const int32_t* __restrict__ rank, const uint32_t* __restrict__ perm, int64_t n,
                                uint32_t* __restrict__ out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = (uint32_t)rank[perm[p]] ^ 0x80000000u;  // int32 order as unsigned order
}

__global__ void gather_rows_kernel(const double* __restrict__ src, const uint32_t* __restrict__ perm, int64_t keep, int w,
                                   double* __restrict__ out) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= keep * w) return;
  int64_t r = t / w;
  int c = (int)(t - r * w);
  out[t] = src[(int64_t)perm[r] * w + c];
}
__global__ void gather_sorted_kernel(const int32_t* __restrict__ rank, const double* __restrict__ dist,
                                     const uint32_t* __restrict__ perm, int64_t keep, int64_t* __restrict__ perm_out,
                                     int32_t* __restrict__ rank_out, double* __restrict__ dist_out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= keep) return;
  uint32_t i = perm[p];
  if (perm_out) perm_out[p] = (int64_t)i;
  if (rank_out) rank_out[p] = rank[i];
  if (dist_out && dist) dist_out[p] = dist[i];
}

// ---- duplicates: rows sorted by a fixed linear projection s = sum_c w_c x_c (w_c in [1, 2)); a row scans the window of
// rows whose projection can belong to a row within eps.  (A single coordinate is a poor key here: offspring are clipped to
// the bounds, so thousands of rows share x_0 == lower bound exactly and every one of them would scan all the others.)
// Rows within distance eps satisfy |s_i - s_j| <= ||w||_2 eps <= 2 sqrt(d) eps, plus the rounding of the two sums, which
// is bounded through the absolute projection t = sum_c w_c |x_c|; identical rows have identical projections.
__device__ __forceinline__ double dup_weight(int c) { return 1.0 + (double)(((uint32_t)c * 2654435761u >> 8) & 0xFFFFu) * (1.0 / 65536.0); }
__device__ __forceinline__ double dup_projection(const double* __restrict__ x, int d) {
  double s = 0.0;
  for (int c = 0; c < d; ++c) s = fma(dup_weight(c), x[c], s);
  return s;
}
__device__ __forceinline__ double dup_window(const double* __restrict__ x, int d, double eps) {
  double t = 0.0;
  for (int c = 0; c < d; ++c) t = fma(dup_weight(c), fabs(x[c]), t);
  const double reach = 2.0 * sqrt((double)d) * eps;
  return reach + 4.0 * d * 2.220446049250313e-16 * (t + reach);
}
__global__ void first_coord_keys_kernel(const double* __restrict__ X, int64_t n, int d, uint64_t* __restrict__ keys,
                                        uint32_t* __restrict__ idx) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    keys[i] = f64_to_ordered(dup_projection(X + i * d, d));
    idx[i] = (uint32_t)i;
  }
}
// two-set form, MOEA.get_duplicates(X, Y) (MOEA.py:426-437 as MOASMO.py:442 calls it): row i of X is a duplicate when
// some row j < i of Y lies within eps (cdist(X, Y) with the upper triangle INCLUDING the diagonal masked).  X and Y
// rows share one sorted order on the projection; ids >= n are rows of Y.
__global__ void pair_keys_kernel(const double* __restrict__ X, int64_t n, const double* __restrict__ Y, int64_t ny, int d,
                                 uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n + ny) return;
  keys[i] = f64_to_ordered(dup_projection(i < n ? X + i * d : Y + (i - n) * d, d));
  idx[i] = (uint32_t)i;
}

__global__ void duplicates_pair_kernel(const double* __restrict__ X, int64_t n, const double* __restrict__ Y, int64_t ny,
                                       const uint64_t* __restrict__ skeys, const uint32_t* __restrict__ sidx, int d,
                                       double eps, uint8_t* __restrict__ is_dup) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n + ny) return;
  const uint32_t i = sidx[p];
  if (i >= n) return;  // a row of Y: only probed, never flagged
  const double x0 = ordered_to_f64(skeys[p]);
  const double* xi = X + (int64_t)i * d;
  const double win = dup_window(xi, d, eps);
  bool dup = false;
  for (int dir = -1; dir <= 1 && !dup; dir += 2) {
    for (int64_t q = p + dir; q >= 0 && q < n + ny; q += dir) {
      if (fabs(ordered_to_f64(skeys[q]) - x0) > win) break;
      const uint32_t jx = sidx[q];
      if (jx < n) continue;              // another row of X
      const uint32_t j = jx - (uint32_t)n;
      if (j >= i) continue;              // np.triu_indices(len(X), m=len(Y)): only j < i is compared
      const double* yj = Y + (int64_t)j * d;
      double s = 0.0;
      for (int c = 0; c < d; ++c) {
        double t = xi[c] - yj[c];
        s += t * t;
      }
      if (sqrt(s) <= eps) {
        dup = true;
        break;
      }
    }
  }
  is_dup[i] = dup ? 1 : 0;
}

__global__ void duplicates_kernel(const double* __restrict__ X, const uint64_t* __restrict__ skeys,
                                  const uint32_t* __restrict__ sidx, int64_t n, int d, double eps,
                                  uint8_t* __restrict__ is_dup) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t i = sidx[p];
  const double x0 = ordered_to_f64(skeys[p]);
  const double* xi = X + (int64_t)i * d;
  const double win = dup_window(xi, d, eps);
  bool dup = false;
  for (int dir = -1; dir <= 1 && !dup; dir += 2) {
    for (int64_t q = p + dir; q >= 0 && q < n; q += dir) {
      double dx0 = ordered_to_f64(skeys[q]) - x0;
      if (fabs(dx0) > win) break;
      const uint32_t jx = sidx[q];
      if (jx >= i) continue;  // only earlier rows make a row a duplicate (lower triangle, MOEA.py:430)
      const double* xj = X + (int64_t)jx * d;
      double s = 0.0;
      for (int c = 0; c < d; ++c) {
        double t = xi[c] - xj[c];
        s += t * t;
      }
      if (sqrt(s) <= eps) {
        dup = true;
        break;
      }
    }
  }
  is_dup[i] = dup ? 1 : 0;
}

int column_minmax(dmo_ctx* ctx, const double* dY, int64_t n, int M, uint64_t* mn, uint64_t* mx) {
  DMO_LAUNCH(minmax_init_kernel, 1, 32, 0, mn, mx, M);
  int grid = (int)(ceil_div(n, 256) < ctx->sm_count * 4 ? ceil_div(n, 256) : ctx->sm_count * 4);
  if (M <= 8)
    DMO_LAUNCH(minmax_kernel<8>, grid, 256, 0, dY, n, M, mn, mx);
  else
    DMO_LAUNCH(minmax_kernel<16>, grid, 256, 0, dY, n, M, mn, mx);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

}  // namespace

int crowding_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, double* dD) {
  if (n <= 0) return DMO_OK;
  DMO_REQUIRE(M >= 1 && M <= MAX_OBJ, "crowding: M=%d out of range [1,%d]", M, MAX_OBJ);
  const unsigned g = (unsigned)ceil_div(n, 256);
  if (n == 1) {  // indicators.py:23-24
    DMO_LAUNCH(fill_f64_kernel, 1, 32, 0, dD, 1, 1.0);
    DMO_CHECK_LAUNCH();
    return DMO_OK;
  }
  DevBuf<uint64_t> mm, k0, k1;
  DevBuf<uint32_t> i0, i1, pos;
  DevBuf<double> contrib;
  DMO_TRY(mm.alloc(ctx, 2 * MAX_OBJ));
  DMO_TRY(k0.alloc(ctx, n));
  DMO_TRY(k1.alloc(ctx, n));
  DMO_TRY(i0.alloc(ctx, n));
  DMO_TRY(i1.alloc(ctx, n));
  DMO_TRY(pos.alloc(ctx, (size_t)n * M));
  DMO_TRY(contrib.alloc(ctx, (size_t)n * M));
  DMO_TRY(column_minmax(ctx, dY, n, M, mm.p, mm.p + MAX_OBJ));
  for (int j = 0; j < M; ++j) {
    DMO_LAUNCH(crowd_keys_kernel, g, 256, 0, dY, n, M, j, mm.p, mm.p + MAX_OBJ, k0.p, i0.p);
    DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, i1.p, n, 0, 64));
    DMO_LAUNCH(crowd_contrib_kernel, g, 256, 0, k1.p, i1.p, n, M, j, contrib.p, pos.p);
  }
  if (M <= 8)
    DMO_LAUNCH(crowd_sum_kernel<8>, g, 256, 0, contrib.p, pos.p, n, M, dD);
  else
    DMO_LAUNCH(crowd_sum_kernel<16>, g, 256, 0, contrib.p, pos.p, n, M, dD);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int euclidean_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, double* dD) {
  if (n <= 0) return DMO_OK;
  DMO_REQUIRE(M >= 1 && M <= MAX_OBJ, "euclidean: M=%d out of range [1,%d]", M, MAX_OBJ);
  DevBuf<uint64_t> mm;
  DMO_TRY(mm.alloc(ctx, 2 * MAX_OBJ));
  DMO_TRY(column_minmax(ctx, dY, n, M, mm.p, mm.p + MAX_OBJ));
  if (M <= 8)
    DMO_LAUNCH(euclid_kernel<8>, (unsigned)ceil_div(n, 256), 256, 0, dY, n, M, mm.p, mm.p + MAX_OBJ, dD);
  else
    DMO_LAUNCH(euclid_kernel<16>, (unsigned)ceil_div(n, 256), 256, 0, dY, n, M, mm.p, mm.p + MAX_OBJ, dD);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int lexsort_device(dmo_ctx* ctx, const int32_t* d_rank, const double* const* d_desc_keys, int nkeys, int64_t n,
                   uint32_t* d_perm, bool rank_below_n) {
  if (n <= 0) return DMO_OK;
  const unsigned g = (unsigned)ceil_div(n, 256);
  DevBuf<uint32_t> pa, pb, r0, r1;
  DevBuf<uint64_t> k0, k1;
  DMO_TRY(pa.alloc(ctx, n));
  DMO_TRY(pb.alloc(ctx, n));
  DMO_TRY(prim_iota_u32(ctx, pa.p, n));
  uint32_t* pin = pa.p;
  uint32_t* pout = pb.p;
  if (nkeys > 0) {
    DMO_TRY(k0.alloc(ctx, n));
    DMO_TRY(k1.alloc(ctx, n));
    for (int k = 0; k < nkeys; ++k) {  // least significant first, each stable
      DMO_LAUNCH(desc_key_kernel, g, 256, 0, d_desc_keys[k], pin, n, k0.p);
      DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, pin, pout, n, 0, 64));
      uint32_t* t = pin;
      pin = pout;
      pout = t;
    }
  }
  if (d_rank) {
    DMO_TRY(r0.alloc(ctx, n));
    DMO_TRY(r1.alloc(ctx, n));
    // keys in [0, n) share the flipped sign bit, so their low bits alone order them; other ranks need all 32
    int bits = 32;
    if (rank_below_n) {
      bits = 1;
      while (((int64_t)1 << bits) < n + 1) ++bits;
    }
    DMO_LAUNCH(rank_key_kernel, g, 256, 0, d_rank, pin, n, r0.p);
    DMO_TRY(prim_sort_pairs_u32(ctx, r0.p, r1.p, pin, pout, n, 0, bits));
    uint32_t* t = pin;
    pin = pout;
    pout = t;
  }
  DMO_CUDA(cudaMemcpyAsync(d_perm, pin, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// shared body of dmo_order_mo / dmo_remove_worst on device pointers
// keep > 0: only the first `keep` rows of the order are wanted (remove_worst), so the ranks of the rows behind them need not
// be told apart (rank_nd_device_keep)
static int order_mo_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, int metric, const double* const* d_extra,
                           int n_extra, DevBuf<int32_t>& rank, DevBuf<double>& dist, DevBuf<uint32_t>& perm, int64_t keep = 0) {
  DMO_TRY(rank.alloc(ctx, n));
  DMO_TRY(perm.alloc(ctx, n));
  if (keep > 0 && keep < n)
    DMO_TRY(rank_nd_device_keep(ctx, dY, n, M, keep, rank.p));
  else
    DMO_TRY(rank_nd_device(ctx, dY, n, M, rank.p));
  const double* keys[16];
  int nk = 0;
  for (int k = 0; k < n_extra && nk < 15; ++k) keys[nk++] = d_extra[k];
  if (metric == DMO_METRIC_CROWDING) {
    DMO_TRY(dist.alloc(ctx, n));
    DMO_TRY(crowding_device(ctx, dY, n, M, dist.p));
    keys[nk++] = dist.p;
  } else if (metric == DMO_METRIC_EUCLIDEAN) {
    DMO_TRY(dist.alloc(ctx, n));
    DMO_TRY(euclidean_device(ctx, dY, n, M, dist.p));
    keys[nk++] = dist.p;
  } else if (metric != DMO_METRIC_NONE) {
    return dmo_fail(ctx, DMO_ERR_ARG, "order_mo: unknown metric %d", metric);
  }
  DMO_TRY(lexsort_device(ctx, rank.p, keys, nk, n, perm.p, true));
  return DMO_OK;
}

// dmo_remove_worst on device arrays, keep <= n (any output may be null): no host wait of its own
int remove_worst_device(dmo_ctx* ctx, const double* dX, const double* dY, int64_t n, int d, int M, int metric,
                        const double* const* d_extra, int n_extra, int64_t keep, double* dX_out, double* dY_out, int32_t* d_rank_out,
                        int64_t* d_perm_out) {
  DevBuf<int32_t> rank;
  DevBuf<double> dist;
  DevBuf<uint32_t> p;
  DMO_TRY(order_mo_device(ctx, dY, n, M, metric, d_extra, n_extra, rank, dist, p, keep));
  if (dX_out) DMO_LAUNCH(gather_rows_kernel, (unsigned)ceil_div(keep * d, 256), 256, 0, dX, p.p, keep, d, dX_out);
  if (dY_out) DMO_LAUNCH(gather_rows_kernel, (unsigned)ceil_div(keep * M, 256), 256, 0, dY, p.p, keep, M, dY_out);
  DMO_LAUNCH(gather_sorted_kernel, (unsigned)ceil_div(keep, 256), 256, 0, rank.p, (const double*)nullptr, p.p, keep,
             d_perm_out, d_rank_out, (double*)nullptr);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

extern "C" {

int dmo_crowding_distance(dmo_ctx* ctx, const double* Y, int64_t n, int M, double* D) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && Y && D, "crowding_distance: bad arguments");
  In<double> y;
  Out<double> d;
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  DMO_TRY(d.init(ctx, D, (size_t)n));
  DMO_TRY(crowding_device(ctx, y.d, n, M, d.d));
  DMO_TRY(d.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_euclidean_distance(dmo_ctx* ctx, const double* Y, int64_t n, int M, double* D) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && Y && D, "euclidean_distance: bad arguments");
  In<double> y;
  Out<double> d;
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  DMO_TRY(d.init(ctx, D, (size_t)n));
  DMO_TRY(euclidean_device(ctx, y.d, n, M, d.d));
  DMO_TRY(d.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_order_mo(dmo_ctx* ctx, const double* Y, int64_t n, int M, int metric, const double* const* extra_desc_keys,
                 int n_extra, int64_t* perm, int32_t* rank_sorted, double* dist_sorted) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && Y && perm, "order_mo: bad arguments");
  DMO_REQUIRE(n_extra >= 0 && n_extra <= 8, "order_mo: at most 8 extra keys");
  In<double> y;
  In<double> ex[8];
  const double* dex[8];
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  for (int k = 0; k < n_extra; ++k) {
    DMO_TRY(ex[k].init(ctx, extra_desc_keys[k], (size_t)n));
    dex[k] = ex[k].d;
  }
  DevBuf<int32_t> rank;
  DevBuf<double> dist;
  DevBuf<uint32_t> p;
  DMO_TRY(order_mo_device(ctx, y.d, n, M, metric, dex, n_extra, rank, dist, p));
  Out<int64_t> op;
  Out<int32_t> orank;
  Out<double> odist;
  DMO_TRY(op.init(ctx, perm, (size_t)n));
  DMO_TRY(orank.init(ctx, rank_sorted, (size_t)n));
  DMO_TRY(odist.init(ctx, metric == DMO_METRIC_NONE ? nullptr : dist_sorted, (size_t)n));
  DMO_LAUNCH(gather_sorted_kernel, (unsigned)ceil_div(n, 256), 256, 0, rank.p, dist.p, p.p, n, op.d, orank.d, odist.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(op.finish(ctx));
  DMO_TRY(orank.finish(ctx));
  DMO_TRY(odist.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_remove_worst(dmo_ctx* ctx, const double* X, const double* Y, int64_t n, int d, int M, int metric,
                     const double* const* extra_desc_keys, int n_extra, int64_t keep, double* X_out, double* Y_out,
                     int32_t* rank_out, int64_t* perm_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && X && Y && d >= 1, "remove_worst: bad arguments");
  DMO_REQUIRE(n_extra >= 0 && n_extra <= 8, "remove_worst: at most 8 extra keys");
  if (keep > n) keep = n;
  In<double> x, y;
  In<double> ex[8];
  const double* dex[8];
  DMO_TRY(x.init(ctx, X, (size_t)n * d));
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  for (int k = 0; k < n_extra; ++k) {
    DMO_TRY(ex[k].init(ctx, extra_desc_keys[k], (size_t)n));
    dex[k] = ex[k].d;
  }
  Out<double> ox, oy;
  Out<int32_t> orank;
  Out<int64_t> op;
  DMO_TRY(ox.init(ctx, X_out, (size_t)keep * d));
  DMO_TRY(oy.init(ctx, Y_out, (size_t)keep * M));
  DMO_TRY(orank.init(ctx, rank_out, (size_t)keep));
  DMO_TRY(op.init(ctx, perm_out, (size_t)keep));
  DMO_TRY(remove_worst_device(ctx, x.d, y.d, n, d, M, metric, dex, n_extra, keep, ox.d, oy.d, orank.d, op.d));
  DMO_TRY(ox.finish(ctx));
  DMO_TRY(oy.finish(ctx));
  DMO_TRY(orank.finish(ctx));
  DMO_TRY(op.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

// dmo_remove_worst on the row-wise concatenation [A; B] without materialising it on the host: the two blocks are
// staged into adjacent regions of one device buffer (NSGA2.update_strategy stacks children over parents, NSGA2.py:205-206)
// key (optional): a feasibility model evaluated on the staged rows, the least significant descending key
static int remove_worst_pair_impl(dmo_ctx* ctx, const double* Xa, const double* Ya, int64_t na, const double* Xb,
                                  const double* Yb, int64_t nb, int d, int M, int metric, const dmo_feas* key, int64_t keep,
                                  double* X_out, double* Y_out, int32_t* rank_out, int64_t* perm_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = na + nb;
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(na >= 0 && nb >= 0 && d >= 1 && M >= 1 && (na == 0 || (Xa && Ya)) && (nb == 0 || (Xb && Yb)),
              "remove_worst_pair: bad arguments");
  if (keep > n) keep = n;
  DevBuf<double> x, y;
  DMO_TRY(x.alloc(ctx, (size_t)n * d));
  DMO_TRY(y.alloc(ctx, (size_t)n * M));
  auto stage = [&](double* dst, const double* src, size_t count) -> int {
    if (count == 0) return DMO_OK;
    DMO_CUDA(cudaMemcpyAsync(dst, src, count * sizeof(double), cudaMemcpyDefault, ctx->stream));
    if (!dmo_is_device_ptr(src)) ctx->h2d_bytes += count * sizeof(double);
    return DMO_OK;
  };
  DMO_TRY(stage(x.p, Xa, (size_t)na * d));
  DMO_TRY(stage(x.p + (size_t)na * d, Xb, (size_t)nb * d));
  DMO_TRY(stage(y.p, Ya, (size_t)na * M));
  DMO_TRY(stage(y.p + (size_t)na * M, Yb, (size_t)nb * M));
  DevBuf<double> kx;
  const double* kp[1] = {nullptr};
  if (key) {
    DMO_TRY(kx.alloc(ctx, (size_t)n));
    DMO_TRY(feas_rank_device(ctx, key, x.p, n, kx.p));
    kp[0] = kx.p;
  }
  DevBuf<int32_t> rank;
  DevBuf<double> dist;
  DevBuf<uint32_t> p;
  DMO_TRY(order_mo_device(ctx, y.p, n, M, metric, key ? kp : nullptr, key ? 1 : 0, rank, dist, p, keep));
  Out<double> ox, oy;
  Out<int32_t> orank;
  Out<int64_t> op;
  DMO_TRY(ox.init(ctx, X_out, (size_t)keep * d));
  DMO_TRY(oy.init(ctx, Y_out, (size_t)keep * M));
  DMO_TRY(orank.init(ctx, rank_out, (size_t)keep));
  DMO_TRY(op.init(ctx, perm_out, (size_t)keep));
  if (ox.d) DMO_LAUNCH(gather_rows_kernel, (unsigned)ceil_div(keep * d, 256), 256, 0, x.p, p.p, keep, d, ox.d);
  if (oy.d) DMO_LAUNCH(gather_rows_kernel, (unsigned)ceil_div(keep * M, 256), 256, 0, y.p, p.p, keep, M, oy.d);
  DMO_LAUNCH(gather_sorted_kernel, (unsigned)ceil_div(keep, 256), 256, 0, rank.p, (const double*)nullptr, p.p, keep,
             op.d, orank.d, (double*)nullptr);
  DMO_CHECK_LAUNCH();
  DMO_TRY(ox.finish(ctx));
  DMO_TRY(oy.finish(ctx));
  DMO_TRY(orank.finish(ctx));
  DMO_TRY(op.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_remove_worst_pair(dmo_ctx* ctx, const double* Xa, const double* Ya, int64_t na, const double* Xb, const double* Yb,
                          int64_t nb, int d, int M, int metric, int64_t keep, double* X_out, double* Y_out,
                          int32_t* rank_out, int64_t* perm_out) {
  return remove_worst_pair_impl(ctx, Xa, Ya, na, Xb, Yb, nb, d, M, metric, nullptr, keep, X_out, Y_out, rank_out, perm_out);
}

int dmo_remove_worst_pair_keys(dmo_ctx* ctx, const double* Xa, const double* Ya, int64_t na, const double* Xb,
                               const double* Yb, int64_t nb, int d, int M, int metric, const dmo_feas* key, int64_t keep,
                               double* X_out, double* Y_out, int32_t* rank_out, int64_t* perm_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_REQUIRE(key, "remove_worst_pair_keys: no key model");
  DMO_REQUIRE(feas_model_dim(key) == d, "remove_worst_pair_keys: the key model takes %d columns, X has %d", feas_model_dim(key), d);
  return remove_worst_pair_impl(ctx, Xa, Ya, na, Xb, Yb, nb, d, M, metric, key, keep, X_out, Y_out, rank_out, perm_out);
}

int dmo_get_duplicates(dmo_ctx* ctx, const double* X, int64_t n, int d, double eps, uint8_t* is_dup) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && X && is_dup && d >= 1, "get_duplicates: bad arguments");
  In<double> x;
  Out<uint8_t> o;
  DMO_TRY(x.init(ctx, X, (size_t)n * d));
  DMO_TRY(o.init(ctx, is_dup, (size_t)n));
  DevBuf<uint64_t> k0, k1;
  DevBuf<uint32_t> i0, i1;
  DMO_TRY(k0.alloc(ctx, n));
  DMO_TRY(k1.alloc(ctx, n));
  DMO_TRY(i0.alloc(ctx, n));
  DMO_TRY(i1.alloc(ctx, n));
  const unsigned g = (unsigned)ceil_div(n, 256);
  DMO_LAUNCH(first_coord_keys_kernel, g, 256, 0, x.d, n, d, k0.p, i0.p);
  DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, i1.p, n, 0, 64));
  DMO_LAUNCH(duplicates_kernel, g, 256, 0, x.d, k1.p, i1.p, n, d, eps, o.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(o.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_get_duplicates_pair(dmo_ctx* ctx, const double* X, int64_t n, const double* Y, int64_t ny, int d, double eps,
                            uint8_t* is_dup) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && ny >= 0 && X && is_dup && d >= 1 && (Y || ny == 0), "get_duplicates_pair: bad arguments");
  In<double> x, y;
  Out<uint8_t> o;
  DMO_TRY(x.init(ctx, X, (size_t)n * d));
  DMO_TRY(y.init(ctx, Y, (size_t)ny * d));
  DMO_TRY(o.init(ctx, is_dup, (size_t)n));
  const int64_t t = n + ny;
  DevBuf<uint64_t> k0, k1;
  DevBuf<uint32_t> i0, i1;
  DMO_TRY(k0.alloc(ctx, t));
  DMO_TRY(k1.alloc(ctx, t));
  DMO_TRY(i0.alloc(ctx, t));
  DMO_TRY(i1.alloc(ctx, t));
  const unsigned g = (unsigned)ceil_div(t, 256);
  DMO_LAUNCH(pair_keys_kernel, g, 256, 0, x.d, n, y.d, ny, d, k0.p, i0.p);
  DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, i1.p, t, 0, 64));
  DMO_LAUNCH(duplicates_pair_kernel, g, 256, 0, x.d, n, y.d, ny, k1.p, i1.p, d, eps, o.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(o.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
