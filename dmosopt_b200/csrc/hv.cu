// Exact hypervolume and HV-improvement (EHVI) candidate selection
// (SURVEY.md section 8a rows A16 / A17).
//   hv.AdaptiveHyperVolume.compute_hypervolume(.., 'box')      dmosopt/hv.py:123-189
//   HyperVolumeBoxDecomposition.compute_hypervolume            dmosopt/hv_box_decomposition.py:86-304
//   select_candidates / _compute_batch_ehvi / _decompose_...   dmosopt/hv_box_decomposition.py:306-437
//
// Hypervolume algorithm (not a transliteration of the reference's sequential local-upper-bound lists):
//   points outside ref are dropped (hv.py:159), then only the rank-0 subset is kept (the HV of a set is the HV of
//   its non-dominated subset).
//   M = 2: sort by f0, min-scan of f1 along that order; the staircase strips are independent -> one parallel reduction.
//   M = 3: HV = sum_k (r_z - z_k) * A_k, where A_k is the area of the xy-quadrant of k that is NOT covered by points
//          with smaller z.  Every A_k is an independent sweep over the x-sorted points (running min of y among the
//          points with smaller z), so the whole computation is n independent O(n) scans: thread-per-point, sources
//          streamed through shared memory in coalesced tiles, no dynamic data structures.
//   M = 4, 5: the same slicing identity applied recursively as chain sums (see hv_slice_kernel), O(n^(M-1)).
//   M = 6 .. 8: the identity with non-dominated limit sets at every level (hv_many.cu).
// All arithmetic is float64; block partial sums are combined in a fixed order (deterministic result).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

// hv3_tree.cu: O(n log^2 n) evaluation of the M = 3 slicing identity for large fronts
int hv_many_device(dmo_ctx* ctx, const double* Fnd, const uint32_t* sidx, int64_t n, int M, const double* dref, double* h_out);
int hv3_tree_device(dmo_ctx* ctx, const double* xs, const double* ys, const double* zs, const uint32_t* zo, int64_t n, double rx,
                    double ry, double rz, double* partial, int64_t* n_partial);

namespace {

constexpr int HV_T = 128;

// keep: optional (n,) array, rows with keep[i] != 0 are dropped up front (the caller knows they are dominated)
__global__ void inside_flag_kernel(const double* __restrict__ F, int64_t n, int M, const double* __restrict__ ref,
                                   const int32_t* __restrict__ drop, int32_t* __restrict__ flag) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) {
    flag[i] = 0;
    return;
  }
  bool in = drop == nullptr || drop[i] == 0;
  for (int j = 0; j < M; ++j) in = in && (ref[j] > F[i * M + j]);  // hv.py:159
  flag[i] = in ? 1 : 0;
}

__global__ void rank0_flag_kernel(const int32_t* __restrict__ rank, int64_t n, int32_t* __restrict__ flag) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  flag[i] = (i < n && rank[i] == 0) ? 1 : 0;
}

__global__ void compact_rows_kernel(const double* __restrict__ F, int64_t n, int M, const int32_t* __restrict__ flag,
                                    const int32_t* __restrict__ pos, double* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  for (int j = 0; j < M; ++j) out[(int64_t)pos[i] * M + j] = F[i * M + j];
}

__global__ void invert_perm_kernel(const uint32_t* __restrict__ sidx, int64_t n, uint32_t* __restrict__ inv) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) inv[sidx[p]] = (uint32_t)p;
}

// single block.  This kernel and final_sum_kernel reduce through a shared-memory tree, not block_sum's serial order over
// the warps: they keep the tree so that their results keep their bits.
__global__ void min_col_kernel(const double* __restrict__ F, int64_t n, double* out) {
  __shared__ double s[256];
  double m = INFINITY;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) m = fmin(m, F[i]);
  s[threadIdx.x] = m;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] = fmin(s[threadIdx.x], s[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = s[0];
}

// Non-dominated filter (rank-0 test only): points are sorted by objective 0; a target scans the sources whose
// objective 0 is <= its own and stops at the first dominator (warp-wide early exit).  For a scattered cloud almost
// every point finds a dominator within the first tile; for a true front it is the full n^2/2 scan.
constexpr int ND_T = 128;
// ND_MAXM: size of the target's register copy, 8 or 16 (two instances, so that the one for M <= 8 is unchanged)
template <int ND_MAXM>
__global__ void __launch_bounds__(ND_T) nondominated_flag_kernel(const double* __restrict__ F, const uint32_t* __restrict__ sidx,
                                                                 int64_t n, int M, int32_t* __restrict__ flag) {
  extern __shared__ double tile_nd[];  // [ND_T][M]
  const int64_t p = (int64_t)blockIdx.x * ND_T + threadIdx.x;
  const bool live = p < n;
  double v[ND_MAXM];
  const int64_t me = live ? (int64_t)sidx[p] : 0;
  for (int j = 0; j < ND_MAXM; ++j) v[j] = (j < M && live) ? F[me * M + j] : 0.0;
  bool dominated = !live;
  bool done = !live;
  for (int64_t t0 = 0; t0 < n; t0 += ND_T) {
    if (__syncthreads_and(done ? 1 : 0)) break;
    const int64_t q = t0 + threadIdx.x;
    if (q < n) {
      const int64_t src = sidx[q];
      for (int j = 0; j < M; ++j) tile_nd[threadIdx.x * M + j] = F[src * M + j];
    }
    __syncthreads();
    const int cnt = (int)((n - t0) < ND_T ? (n - t0) : ND_T);
    if (!done) {
      for (int s = 0; s < cnt; ++s) {
        const double* sp = tile_nd + s * M;
        if (sp[0] > v[0]) {  // sorted by objective 0: nothing further can dominate
          done = true;
          break;
        }
        bool le = true, lt = false;
        for (int j = 0; j < M; ++j) {
          le = le && (sp[j] <= v[j]);
          lt = lt || (sp[j] < v[j]);
        }
        if (le && lt) {
          dominated = true;
          done = true;
          break;
        }
      }
    }
  }
  if (live) flag[me] = dominated ? 0 : 1;
  if (blockIdx.x == 0 && threadIdx.x == 0) flag[n] = 0;
}

__global__ void final_sum_kernel(const double* __restrict__ partial, int64_t nb, double* out) {
  __shared__ double s[256];
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < nb; i += blockDim.x) a += partial[i];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = s[0];
}

// M = 2: sidx sorts the points by f0 ascending, ymin[p] = min of f1 over sorted positions 0 .. p.  The strip over
// [x_p, x_{p+1}) lies under the running minimum, so the sum holds for any set: f0 ties, duplicates and weakly or
// strictly dominated rows (the ranked entry keeps such rows after a float32 rounding) add no volume.
__global__ void hv2_kernel(const double* __restrict__ F, const uint32_t* __restrict__ sidx, const double* __restrict__ ymin,
                           int64_t n, double r0, double r1, double* __restrict__ partial) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (p < n) {
    const double x = F[(int64_t)sidx[p] * 2];
    const double xn = (p + 1 < n) ? F[(int64_t)sidx[p + 1] * 2] : r0;
    v = (xn - x) * (r1 - ymin[p]);
  }
  __shared__ double red[256 / 32];
  const double s = block_sum<256 / 32>(v, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// M = 3 (and the innermost level of the M >= 4 recursion).
// xs / ys: coordinates in x-sorted order; zo: total order id of each x-sorted point along z (ties by index).
// Thread k computes  (r_z - z_k) * [ (r_x - x_k)(r_y - y_k) - area covered by {j : zo_j < zo_k} inside k's quadrant ].
__global__ void __launch_bounds__(HV_T) hv3_kernel(const double* __restrict__ xs, const double* __restrict__ ys,
                                                   const double* __restrict__ zs, const uint32_t* __restrict__ zo,
                                                   int64_t n, double rx, double ry, double rz,
                                                   double* __restrict__ partial) {
  __shared__ double sx[HV_T], sy[HV_T];
  __shared__ uint32_t sz[HV_T];
  const int64_t k = (int64_t)blockIdx.x * HV_T + threadIdx.x;
  const bool live = k < n;
  const double xk = live ? xs[k] : 0.0, yk = live ? ys[k] : 0.0;
  const uint32_t zk = live ? zo[k] : 0u;
  double covered = 0.0, m = INFINITY, xcur = xk;
  for (int64_t t0 = 0; t0 < n; t0 += HV_T) {
    const int64_t j = t0 + threadIdx.x;
    __syncthreads();
    sx[threadIdx.x] = j < n ? xs[j] : INFINITY;
    sy[threadIdx.x] = j < n ? ys[j] : INFINITY;
    sz[threadIdx.x] = j < n ? zo[j] : 0xFFFFFFFFu;
    __syncthreads();
    // A point lowers the staircase only O(log n) times per sweep, but a data-dependent branch per point serialises the
    // loop.  Test eight points at a time against the current minimum without branching (a stale, larger minimum can
    // only produce false alarms, never a miss; the padding never fires) and fall into the exact loop only on a hit.
    for (int s0 = 0; s0 < HV_T; s0 += 8) {
      bool hit = false;
#pragma unroll
      for (int u = 0; u < 8; ++u) hit |= (sz[s0 + u] < zk) & (sy[s0 + u] < m);
      if (hit) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int s = s0 + u;
          const double yj = sy[s];
          if (sz[s] < zk && yj < m) {  // a point below k in z that lowers the staircase
            const double xj = fmax(sx[s], xk);
            const double h = ry - fmax(m, yk);  // m = inf -> negative -> no area yet
            covered += (xj - xcur) * fmax(h, 0.0);
            xcur = xj;
            m = yj;
          }
        }
      }
    }
  }
  double v = 0.0;
  if (live) {
    covered += (rx - xcur) * fmax(ry - fmax(m, yk), 0.0);
    const double excl = (rx - xk) * (ry - yk) - covered;
    v = excl * (rz - zs[k]);
  }
  __shared__ double red[HV_T / 32];
  const double s = block_sum<HV_T / 32>(v, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void gather_col_kernel(const double* __restrict__ F, const uint32_t* __restrict__ sidx, int64_t n, int M,
                                  int j, double* __restrict__ out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = F[(int64_t)sidx[p] * M + j];
}

// ---- M = 4, 5: the slicing identity applied recursively ----------------------------------------------------------
//   HV_d(S) = sum_k (r_d - p_k[d]) * [ vol_{d-1}(box of k) - HV_{d-1}( S_k clipped to the box of k ) ],  S_k = points before k
//   along axis d.  Unrolled to the 3-D base case this is an alternating sum over chains k1 > k2 (> k3):
//     HV_4 = sum_k1 h1 vol3(k1)                      - sum_{k1>k2} h1 h2 E2(k1,k2)
//     HV_5 = sum_k1 h1 vol4(k1) - sum_{k1>k2} h1 h2 vol3(k1,k2) + sum_{k1>k2>k3} h1 h2 h3 E2(k1,k2,k3)
//   with h_i = r - (clipped coordinate along the i-th slicing axis) and E2 the exclusive xy-area of the innermost point
//   inside the common box, against the points that precede it along every slicing axis (same sweep as hv3_kernel).
//   Clipping (component-wise max with the outer points) is monotone, so the original per-axis orders stay valid.
struct HvArrays {
  const double* x;  // coordinates in x-sorted order: x = obj0, y = obj1, s[0] = obj2 (innermost slicing axis), s[1], s[2]
  const double* y;
  const double* s[3];
  const uint32_t* o[3];  // total-order ids along the slicing axes
  double rx, ry, rs[3];
};

// D = 2 (M = 4): block = (k1, tile of k2).  D = 3 (M = 5): block = (k1, tile of k3), k2 looped inside the block.
template <int D>
__global__ void __launch_bounds__(HV_T) hv_slice_kernel(HvArrays A, int64_t n, double* __restrict__ partial) {
  __shared__ double sx[HV_T], sy[HV_T];
  __shared__ uint32_t so[3][HV_T];
  const int64_t k1 = blockIdx.x;
  const int64_t t = (int64_t)blockIdx.y * HV_T + threadIdx.x;  // innermost chain index
  const bool live = t < n;
  constexpr int TOP = D - 1;  // slicing axis of k1 (outermost)
  const double x1 = A.x[k1], y1 = A.y[k1];
  const uint32_t o1 = A.o[TOP][k1];
  const double h1 = A.rs[TOP] - A.s[TOP][k1];
  double c1[3];
  for (int a = 0; a < TOP; ++a) c1[a] = A.s[a][k1];
  const double xt = live ? A.x[t] : 0.0, yt = live ? A.y[t] : 0.0;
  double st[3];
  uint32_t ot[3];
  for (int a = 0; a < D; ++a) {
    st[a] = live ? A.s[a][t] : 0.0;
    ot[a] = live ? A.o[a][t] : 0u;
  }
  double total = 0.0;
  const int64_t n2 = (D == 3) ? n : 1;
  for (int64_t k2 = 0; k2 < n2; ++k2) {
    double X = fmax(xt, x1), Y = fmax(yt, y1), hprod = h1;
    double clipz = fmax(st[0], c1[0]);  // innermost slicing coordinate of t, clipped
    uint32_t lim_w = 0xFFFFFFFFu;       // D == 3: order limit along axis 1 given by k2
    bool valid = live && ot[TOP] < o1;
    if (D == 3) {
      const uint32_t o2v = A.o[2][k2];
      if (!(o2v < o1)) continue;  // k2 must precede k1 along the outermost axis (uniform over the block)
      const double x2 = A.x[k2], y2 = A.y[k2];
      lim_w = A.o[1][k2];
      valid = valid && ot[1] < lim_w;
      X = fmax(X, x2);
      Y = fmax(Y, y2);
      clipz = fmax(clipz, A.s[0][k2]);
      hprod *= A.rs[1] - fmax(A.s[1][k2], c1[1]);
    }
    double covered = 0.0, m = INFINITY, xcur = X;
    for (int64_t t0 = 0; t0 < n; t0 += HV_T) {
      const int64_t j = t0 + threadIdx.x;
      __syncthreads();
      sx[threadIdx.x] = j < n ? A.x[j] : INFINITY;
      sy[threadIdx.x] = j < n ? A.y[j] : INFINITY;
      for (int a = 0; a < D; ++a) so[a][threadIdx.x] = j < n ? A.o[a][j] : 0xFFFFFFFFu;
      __syncthreads();
      if (!valid) continue;
      const int cnt = (int)((n - t0) < HV_T ? (n - t0) : HV_T);
#pragma unroll 4
      for (int s = 0; s < cnt; ++s) {
        bool in = so[TOP][s] < o1 && so[0][s] < ot[0];
        if (D == 3) in = in && so[1][s] < lim_w;
        const double yj = sy[s];
        if (in && yj < m) {
          const double xj = fmax(sx[s], X);
          covered += (xj - xcur) * fmax(A.ry - fmax(m, Y), 0.0);
          xcur = xj;
          m = yj;
        }
      }
    }
    if (valid) {
      covered += (A.rx - xcur) * fmax(A.ry - fmax(m, Y), 0.0);
      const double excl = (A.rx - X) * (A.ry - Y) - covered;
      total += hprod * (A.rs[0] - clipz) * excl;
    }
  }
  __shared__ double red[HV_T / 32];
  const double acc = block_sum<HV_T / 32>(total, red);
  if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * gridDim.y + blockIdx.y] = acc;
}

// lower-order terms: sum_k1 h1 vol(k1)  [and for M = 5: sum_{k1>k2} h1 h2 vol3(k1,k2)]
template <int D>
__global__ void hv_volume_terms_kernel(HvArrays A, int64_t n, double* __restrict__ partial_a, double* __restrict__ partial_b) {
  const int64_t k1 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int TOP = D - 1;
  double ta = 0.0, tb = 0.0;
  if (k1 < n) {
    const double h1 = A.rs[TOP] - A.s[TOP][k1];
    double vol = (A.rx - A.x[k1]) * (A.ry - A.y[k1]);
    for (int a = 0; a < TOP; ++a) vol *= A.rs[a] - A.s[a][k1];
    ta = h1 * vol;
    if (D == 3) {
      const uint32_t o1 = A.o[2][k1];
      for (int64_t k2 = 0; k2 < n; ++k2) {
        if (!(A.o[2][k2] < o1)) continue;
        const double h2 = A.rs[1] - fmax(A.s[1][k2], A.s[1][k1]);
        const double v3 = (A.rx - fmax(A.x[k2], A.x[k1])) * (A.ry - fmax(A.y[k2], A.y[k1])) *
                          (A.rs[0] - fmax(A.s[0][k2], A.s[0][k1]));
        tb += h1 * h2 * v3;
      }
    }
  }
  __shared__ double red[256 / 32];
  const double sa = block_sum<256 / 32>(ta, red);
  if (threadIdx.x == 0) partial_a[blockIdx.x] = sa;
  if (D == 3) {
    const double sb = block_sum<256 / 32>(tb, red);
    if (threadIdx.x == 0) partial_b[blockIdx.x] = sb;
  }
}

// ---- EHVI -----------------------------------------------------------------------------------------------
constexpr int EH_MAX_OBJ = 16;

// boxes between consecutive f0-sorted front points (hv_box_decomposition.py:418-437)
__global__ void box_flag_kernel(const double* __restrict__ front, const uint32_t* __restrict__ sidx, int64_t nf, int M,
                                const double* __restrict__ ref, int32_t* __restrict__ flag) {
  int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nf + 1) return;
  if (b == nf + 1) {
    flag[b] = 0;
    return;
  }
  bool valid = true;
  for (int j = 0; j < M; ++j) {
    double lo = (b == 0) ? -INFINITY : front[(int64_t)sidx[b - 1] * M + j];
    double up = (b < nf) ? front[(int64_t)sidx[b] * M + j] : ref[j];
    valid = valid && (up > lo);
  }
  flag[b] = valid ? 1 : 0;
}
__global__ void box_write_kernel(const double* __restrict__ front, const uint32_t* __restrict__ sidx, int64_t nf, int M,
                                 const double* __restrict__ ref, const int32_t* __restrict__ flag,
                                 const int32_t* __restrict__ pos, double* __restrict__ lower, double* __restrict__ upper) {
  int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nf || !flag[b]) return;
  for (int j = 0; j < M; ++j) {
    lower[(int64_t)pos[b] * M + j] = (b == 0) ? -INFINITY : front[(int64_t)sidx[b - 1] * M + j];
    upper[(int64_t)pos[b] * M + j] = (b < nf) ? front[(int64_t)sidx[b] * M + j] : ref[j];
  }
}

// score_c = sum_b prod_j [ sd (phi(zl) - phi(zu)) + mu (Phi(zu) - Phi(zl)) ]   (hv_box_decomposition.py:353-416)
// EH_MAXM: size of the candidate's register copy, 8 or 16 (two instances, so that the one for M <= 8 is unchanged)
template <int EH_MAXM>
__global__ void ehvi_kernel(const double* __restrict__ lower, const double* __restrict__ upper, int64_t nb, int M,
                            const double* __restrict__ means, const double* __restrict__ variances, int64_t nc,
                            double* __restrict__ score) {
  extern __shared__ double sb[];  // [2][tile][M]
  const int TB = 64;
  double* sl = sb;
  double* su = sb + TB * M;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double mu[EH_MAXM], sd[EH_MAXM];
  for (int j = 0; j < M; ++j) {
    mu[j] = c < nc ? means[c * M + j] : 0.0;
    sd[j] = c < nc ? sqrt(variances[c * M + j]) : 1.0;
  }
  double total = 0.0;
  for (int64_t b0 = 0; b0 < nb; b0 += TB) {
    const int cnt = (int)((nb - b0) < TB ? (nb - b0) : TB);
    __syncthreads();
    for (int t = threadIdx.x; t < cnt * M; t += blockDim.x) {
      sl[t] = lower[b0 * M + t];
      su[t] = upper[b0 * M + t];
    }
    __syncthreads();
    for (int b = 0; b < cnt; ++b) {
      double prod = 1.0;
      for (int j = 0; j < M; ++j) {
        const double lo = sl[b * M + j], up = su[b * M + j];
        const double zl = (lo - mu[j]) / sd[j], zu = (up - mu[j]) / sd[j];
        const double pl = isinf(lo) ? 0.0 : normcdf(zl);
        const double pu = isinf(up) ? 1.0 : normcdf(zu);
        const double dl = 0.3989422804014326779 * exp(-0.5 * zl * zl);  // norm.pdf, 0 at +-inf
        const double du = 0.3989422804014326779 * exp(-0.5 * zu * zu);
        prod *= sd[j] * (dl - du) + mu[j] * (pu - pl);
      }
      total += prod;
    }
  }
  if (c < nc) score[c] = total;
}

__global__ void neg_key_kernel(const double* __restrict__ score, int64_t n, uint64_t* __restrict__ keys,
                               uint32_t* __restrict__ idx) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    keys[i] = f64_to_ordered_nan_last(-score[i]);
    idx[i] = (uint32_t)i;
  }
}
__global__ void widen_idx_kernel(const uint32_t* __restrict__ idx, int64_t k, int64_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) out[i] = (int64_t)idx[i];
}

// compaction: rows of F with flag set, in order.  Returns the count on the host.
int compact_rows(dmo_ctx* ctx, const double* dF, int64_t n, int M, DevBuf<int32_t>& flag, DevBuf<double>& out,
                 int64_t* count) {
  DevBuf<int32_t> pos;
  DMO_TRY(pos.alloc(ctx, n + 1));
  DMO_TRY(prim_exclusive_sum_i32(ctx, flag.p, pos.p, n + 1));
  int32_t h = 0;
  DMO_CUDA(cudaMemcpyAsync(&h, pos.p + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  *count = h;
  DMO_TRY(out.alloc(ctx, (size_t)(h > 0 ? h : 1) * M));
  if (h > 0) DMO_LAUNCH(compact_rows_kernel, (unsigned)ceil_div(n, 256), 256, 0, dF, n, M, flag.p, pos.p, out.p);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

}  // namespace

// flag[i] = 1 iff row i is rank 0 (identical vectors are mutually non-dominating), flag[n] = 0; flag holds n + 1 entries
int nondominated_keep_flags(dmo_ctx* ctx, const double* dF, int64_t n, int M, DevBuf<int32_t>& flag) {
  DevBuf<uint32_t> sidx;
  DMO_TRY(flag.alloc(ctx, n + 1));
  if (n >= 1024) {
    // large sets: the integer-id scan costs O(n^2 / 2) cheap id compares whatever the data looks like, while the
    // early-exit scan below degenerates to n^2 / 2 float64 tests as soon as every block holds a non-dominated point
    DevBuf<int32_t> rank;
    DMO_TRY(rank.alloc(ctx, n));
    DMO_TRY(nondominated_flags_device(ctx, dF, n, M, rank.p));
    DMO_LAUNCH(rank0_flag_kernel, (unsigned)ceil_div(n + 1, 256), 256, 0, rank.p, n, flag.p);
    return DMO_OK;
  }
  DMO_TRY(prim_sort_by_column(ctx, dF, n, M, 0, sidx));
  {
    ProfileScope ps(ctx, "nd_filter");
    if (M <= 8)
      DMO_LAUNCH(nondominated_flag_kernel<8>, (unsigned)ceil_div(n, ND_T), ND_T, (size_t)ND_T * M * sizeof(double), dF, sidx.p, n, M,
                 flag.p);
    else
      DMO_LAUNCH(nondominated_flag_kernel<16>, (unsigned)ceil_div(n, ND_T), ND_T, (size_t)ND_T * M * sizeof(double), dF, sidx.p, n, M,
                 flag.p);
  }
  return DMO_OK;
}

namespace {

// rank-0 subset of a device point set (identical vectors are mutually non-dominating and are all kept)
int nondominated_subset(dmo_ctx* ctx, const double* dF, int64_t n, int M, DevBuf<double>& out, int64_t* count) {
  DevBuf<int32_t> flag;
  DMO_TRY(nondominated_keep_flags(ctx, dF, n, M, flag));
  DMO_TRY(compact_rows(ctx, dF, n, M, flag, out, count));
  return DMO_OK;
}

__global__ void dominated_flag_kernel(const int32_t* __restrict__ keep, int64_t n, int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = keep[i] ? 0 : 1;
}

// M = 3, small fronts: one O(n) sweep per point (n^2 / 2 cheap tests, no set-up); large fronts: the merge-sort-tree walks
// of hv3_tree.cu (O(n log^2 n)).  DMO_HV3_TREE = 0 / 1 forces one or the other, any larger value moves the threshold.
int64_t hv3_tree_min() {
  if (const char* e = getenv("DMO_HV3_TREE")) {
    const long v = atol(e);
    return v == 0 ? INT64_MAX : (v == 1 ? 0 : v);
  }
  return 4096;
}

// rows [*count, n) of the row-major (n, M) F := ref
__global__ void pad_rows_kernel(double* __restrict__ F, int64_t n, int M, const int32_t* __restrict__ count,
                                const double* __restrict__ ref) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count && i < n)
    for (int j = 0; j < M; ++j) F[i * M + j] = ref[j];
}

int sum_partials(dmo_ctx* ctx, DevBuf<double>& partial, int64_t nb, double* h_out) {
  DevBuf<double> res;
  DMO_TRY(res.alloc(ctx, 1));
  DMO_LAUNCH(final_sum_kernel, 1, 256, 0, partial.p, nb, res.p);
  DMO_CHECK_LAUNCH();
  DMO_CUDA(cudaMemcpyAsync(h_out, res.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // namespace

// Rows strictly inside ref, then their non-dominated subset, in row order (the Monte-Carlo estimators' front, hv_mc.cu).
int hv_inside_nondominated(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* dref, DevBuf<double>& out,
                           int64_t* count) {
  *count = 0;
  DevBuf<int32_t> flag;
  DevBuf<double> Fin;
  int64_t n1 = 0;
  DMO_TRY(flag.alloc(ctx, n + 1));
  DMO_LAUNCH(inside_flag_kernel, (unsigned)ceil_div(n + 1, 256), 256, 0, dF, n, M, dref, (const int32_t*)nullptr, flag.p);
  DMO_TRY(compact_rows(ctx, dF, n, M, flag, Fin, &n1));
  if (n1 == 0) return DMO_OK;
  return nondominated_subset(ctx, Fin.p, n1, M, out, count);
}

// d_rank (optional, device, (n,)): non-dominated ranks of the rows within a SUPERSET they were selected from by rank
// (dmo_remove_worst).  Rows with rank > 0 are dominated by a rank-0 row of the same set, so they add no volume and are
// dropped without running the non-dominated filter again; this stays true after a monotone rounding of the
// coordinates (float64 -> float32 state).  The rank-0 rows kept are then not mutually non-dominated in general: the
// rounding can make two of them tie in a coordinate, or one Pareto-dominate the other (equal f0, smaller f1).  So every
// route behind this entry must be valid for any point set, and each is:
//   M = 1: the minimum.  M = 2: strips under the running minimum of f1 along the f0 order (hv2_kernel).
//   M = 3 (sweep and tree), M = 4, 5 (chain sums), M = 6 .. 8 (limit sets): the slicing identity
//   HV(S_<=k) - HV(S_<k) = (r - z_k) * [vol(k) - HV(S_<k clipped to k)] holds for any order that is non-decreasing
//   along the slicing axis, whatever the dominance among the points, and every lower level is evaluated by the same
//   identity or by a staircase under a running minimum.
// tests/test_gpu_hv_exact.py checks every route, ranked and unranked, for exact equality on dyadic inputs.
int hypervolume_device_ranked(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* h_ref, const int32_t* d_rank,
                              double* h_out);

int hypervolume_device(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* h_ref, double* h_out) {
  return hypervolume_device_ranked(ctx, dF, n, M, h_ref, nullptr, h_out);
}

int hypervolume_device_ranked(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* h_ref, const int32_t* d_rank,
                              double* h_out) {
  *h_out = 0.0;
  if (n <= 0) return DMO_OK;
  DMO_REQUIRE(M >= 1 && M <= 8, "hypervolume: M=%d not supported (1..8; >= 10 objectives use Monte-Carlo in the reference)", M);
  DevBuf<double> dref;
  DMO_TRY(dref.alloc(ctx, M));
  DMO_CUDA(cudaMemcpyAsync(dref.p, h_ref, M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  // 1. points strictly inside the reference box
  DevBuf<int32_t> flag;
  DevBuf<double> Fin;
  int64_t n1 = 0;
  DMO_TRY(flag.alloc(ctx, n + 1));
  DMO_LAUNCH(inside_flag_kernel, (unsigned)ceil_div(n + 1, 256), 256, 0, dF, n, M, dref.p, d_rank, flag.p);
  DMO_TRY(compact_rows(ctx, dF, n, M, flag, Fin, &n1));
  if (n1 == 0) return DMO_OK;
  if (M == 1) {
    DevBuf<double> mn;
    DMO_TRY(mn.alloc(ctx, 1));
    DMO_LAUNCH(min_col_kernel, 1, 256, 0, Fin.p, n1, mn.p);
    DMO_CHECK_LAUNCH();
    double h = 0.0;
    DMO_CUDA(cudaMemcpyAsync(&h, mn.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    *h_out = h_ref[0] - h;
    return DMO_OK;
  }
  // 2. non-dominated subset
  DevBuf<double> Fnd_own;
  int64_t n2 = 0;
  if (d_rank) {
    n2 = n1;  // already reduced to the rank-0 rows
  } else {
    DMO_TRY(nondominated_subset(ctx, Fin.p, n1, M, Fnd_own, &n2));
    if (n2 == 0) return DMO_OK;
  }
  DevBuf<double>& Fnd = d_rank ? Fin : Fnd_own;
  if (M >= 6 || (M >= 4 && getenv("DMO_HV_WFG") && atoi(getenv("DMO_HV_WFG")))) {
    // 6 .. 8 objectives: limit-set recursion (hv_many.cu); DMO_HV_WFG=1 sends M = 4, 5 there too (cross-check of the chain sums)
    DevBuf<uint32_t> sl;
    DMO_TRY(prim_sort_by_column(ctx, Fnd.p, n2, M, M - 1, sl));
    return hv_many_device(ctx, Fnd.p, sl.p, n2, M, dref.p, h_out);
  }
  DevBuf<uint32_t> sx;
  DMO_TRY(prim_sort_by_column(ctx, Fnd.p, n2, M, 0, sx));
  if (M == 2) {
    const int64_t nb = ceil_div(n2, 256);
    DevBuf<double> partial, ys, ymin;
    DMO_TRY(partial.alloc(ctx, nb));
    DMO_TRY(ys.alloc(ctx, n2));
    DMO_TRY(ymin.alloc(ctx, n2));
    DMO_LAUNCH(gather_col_kernel, (unsigned)nb, 256, 0, Fnd.p, sx.p, n2, M, 1, ys.p);
    DMO_TRY(prim_inclusive_min_f64(ctx, ys.p, ymin.p, n2));
    DMO_LAUNCH(hv2_kernel, (unsigned)nb, 256, 0, Fnd.p, sx.p, ymin.p, n2, h_ref[0], h_ref[1], partial.p);
    DMO_TRY(sum_partials(ctx, partial, nb, h_out));
    return DMO_OK;
  }
  if (M >= 4) {
    // x-sorted coordinate arrays and per-axis order ids for the slicing axes obj2 .. obj(M-1)
    const int D = M - 2;
    const unsigned g4 = (unsigned)ceil_div(n2, 256);
    DevBuf<double> xs4, ys4, sc[3];
    DevBuf<uint32_t> so_[3], sidx_a, inv_a;
    DMO_TRY(xs4.alloc(ctx, n2));
    DMO_TRY(ys4.alloc(ctx, n2));
    DMO_TRY(inv_a.alloc(ctx, n2));
    DMO_LAUNCH(gather_col_kernel, g4, 256, 0, Fnd.p, sx.p, n2, M, 0, xs4.p);
    DMO_LAUNCH(gather_col_kernel, g4, 256, 0, Fnd.p, sx.p, n2, M, 1, ys4.p);
    HvArrays A;
    A.x = xs4.p;
    A.y = ys4.p;
    A.rx = h_ref[0];
    A.ry = h_ref[1];
    for (int a = 0; a < 3; ++a) {
      A.s[a] = nullptr;
      A.o[a] = nullptr;
      A.rs[a] = 0.0;
    }
    for (int a = 0; a < D; ++a) {
      DMO_TRY(sc[a].alloc(ctx, n2));
      DMO_TRY(so_[a].alloc(ctx, n2));
      DMO_TRY(prim_sort_by_column(ctx, Fnd.p, n2, M, 2 + a, sidx_a));
      DMO_LAUNCH(invert_perm_kernel, g4, 256, 0, sidx_a.p, n2, inv_a.p);
      DMO_TRY(prim_gather_u32(ctx, inv_a.p, sx.p, n2, so_[a].p));
      DMO_LAUNCH(gather_col_kernel, g4, 256, 0, Fnd.p, sx.p, n2, M, 2 + a, sc[a].p);
      A.s[a] = sc[a].p;
      A.o[a] = so_[a].p;
      A.rs[a] = h_ref[2 + a];
    }
    const int64_t tiles = ceil_div(n2, HV_T);
    const int64_t nbv = ceil_div(n2, 256);
    DevBuf<double> part_main, part_a, part_b;
    DMO_TRY(part_main.alloc(ctx, (size_t)n2 * tiles));
    DMO_TRY(part_a.alloc(ctx, nbv));
    DMO_TRY(part_b.alloc(ctx, nbv));
    DMO_REQUIRE(tiles <= 65535, "hypervolume: front too large for M=%d (%lld non-dominated points)", M, (long long)n2);
    dim3 grid((unsigned)n2, (unsigned)tiles);
    double t_main = 0.0, t_a = 0.0, t_b = 0.0;
    {
      ProfileScope ps(ctx, M == 4 ? "hv4" : "hv5");
      if (M == 4) {
        DMO_LAUNCH(hv_slice_kernel<2>, grid, HV_T, 0, A, n2, part_main.p);
        DMO_LAUNCH(hv_volume_terms_kernel<2>, (unsigned)nbv, 256, 0, A, n2, part_a.p, part_b.p);
      } else {
        DMO_LAUNCH(hv_slice_kernel<3>, grid, HV_T, 0, A, n2, part_main.p);
        DMO_LAUNCH(hv_volume_terms_kernel<3>, (unsigned)nbv, 256, 0, A, n2, part_a.p, part_b.p);
      }
    }
    DMO_TRY(sum_partials(ctx, part_main, n2 * tiles, &t_main));
    DMO_TRY(sum_partials(ctx, part_a, nbv, &t_a));
    if (M == 5) DMO_TRY(sum_partials(ctx, part_b, nbv, &t_b));
    *h_out = (M == 4) ? (t_a - t_main) : (t_a - t_b + t_main);
    return DMO_OK;
  }
  // M == 3
  DevBuf<uint32_t> sz, zinv, zo;
  DevBuf<double> xs, ys, zs;
  DMO_TRY(prim_sort_by_column(ctx, Fnd.p, n2, M, 2, sz));
  DMO_TRY(zinv.alloc(ctx, n2));
  DMO_TRY(zo.alloc(ctx, n2));
  DMO_TRY(xs.alloc(ctx, n2));
  DMO_TRY(ys.alloc(ctx, n2));
  DMO_TRY(zs.alloc(ctx, n2));
  const unsigned g = (unsigned)ceil_div(n2, 256);
  DMO_LAUNCH(invert_perm_kernel, g, 256, 0, sz.p, n2, zinv.p);     // zinv[i] = position of point i along z
  DMO_TRY(prim_gather_u32(ctx, zinv.p, sx.p, n2, zo.p));            // ... re-indexed by x-sorted position
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fnd.p, sx.p, n2, M, 0, xs.p);
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fnd.p, sx.p, n2, M, 1, ys.p);
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fnd.p, sx.p, n2, M, 2, zs.p);
  int64_t nb = ceil_div(n2, HV_T);
  DevBuf<double> partial;
  DMO_TRY(partial.alloc(ctx, nb));
  if (n2 >= hv3_tree_min()) {
    DMO_TRY(hv3_tree_device(ctx, xs.p, ys.p, zs.p, zo.p, n2, h_ref[0], h_ref[1], h_ref[2], partial.p, &nb));
  } else {
    ProfileScope ps(ctx, "hv3");
    DMO_LAUNCH(hv3_kernel, (unsigned)nb, HV_T, 0, xs.p, ys.p, zs.p, zo.p, n2, h_ref[0], h_ref[1], h_ref[2], partial.p);
  }
  DMO_TRY(sum_partials(ctx, partial, nb, h_out));
  return DMO_OK;
}

// The M = 3 route of hypervolume_device_ranked for the fused step's lane (step.cu): hv3_ranked_enqueue issues no host
// read, so a caller can enqueue it beside other work and drop it unread.  The n1 rows it keeps (rank 0, strictly inside
// ref) are compacted into n rows and rows n1 .. n-1 are set to ref itself, which is greater than every kept row on every
// axis: the stable column sorts put those rows last, so the first n1 entries of the sorted orders, the z-order ids and
// the gathered coordinates are exactly those of the n1-row route.  A padding row adds no volume (its staircase is
// already below it and its z slab is empty), and in the tree it is never a drop for a kept row (its z-order id is >= n1);
// the walk over n rows therefore finds the same drops as the walk over n1, and blocks past n1 add exact zeros to the
// fixed-order final sum.  The tree is built and walked on the lane when n reaches the tree threshold; hv3_ranked_finish
// reads n1 (the route, as the n1-row route does) and then the tree's volume, or runs the sweep on the first n1 entries
// when n1 is below the threshold.  The volume has the bits of hypervolume_device_ranked's (tests/test_gpu_steps_hv_lane.py).
int hv3_ranked_enqueue(dmo_ctx* ctx, const double* dF, int64_t n, const double* h_ref, const int32_t* d_rank, Hv3Ranked& s) {
  s.n = n;
  memcpy(s.ref, h_ref, sizeof(s.ref));
  s.tree = n >= hv3_tree_min();
  DevBuf<double> dref, Fin;
  DevBuf<int32_t> flag;
  DevBuf<uint32_t> sx, sz, zinv;
  DMO_TRY(dref.alloc(ctx, 3));
  DMO_CUDA(cudaMemcpyAsync(dref.p, h_ref, 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_TRY(flag.alloc(ctx, n + 1));
  DMO_TRY(s.pos.alloc(ctx, n + 1));
  DMO_TRY(Fin.alloc(ctx, (size_t)n * 3));
  const unsigned g = (unsigned)ceil_div(n, 256);
  DMO_LAUNCH(inside_flag_kernel, (unsigned)ceil_div(n + 1, 256), 256, 0, dF, n, 3, dref.p, d_rank, flag.p);
  DMO_TRY(prim_exclusive_sum_i32(ctx, flag.p, s.pos.p, n + 1));
  DMO_LAUNCH(compact_rows_kernel, g, 256, 0, dF, n, 3, flag.p, s.pos.p, Fin.p);
  DMO_LAUNCH(pad_rows_kernel, g, 256, 0, Fin.p, n, 3, s.pos.p + n, dref.p);
  DMO_TRY(prim_sort_by_column(ctx, Fin.p, n, 3, 0, sx));
  DMO_TRY(prim_sort_by_column(ctx, Fin.p, n, 3, 2, sz));
  DMO_TRY(zinv.alloc(ctx, n));
  DMO_TRY(s.zo.alloc(ctx, n));
  DMO_TRY(s.xs.alloc(ctx, n));
  DMO_TRY(s.ys.alloc(ctx, n));
  DMO_TRY(s.zs.alloc(ctx, n));
  DMO_LAUNCH(invert_perm_kernel, g, 256, 0, sz.p, n, zinv.p);
  DMO_TRY(prim_gather_u32(ctx, zinv.p, sx.p, n, s.zo.p));
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fin.p, sx.p, n, 3, 0, s.xs.p);
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fin.p, sx.p, n, 3, 1, s.ys.p);
  DMO_LAUNCH(gather_col_kernel, g, 256, 0, Fin.p, sx.p, n, 3, 2, s.zs.p);
  if (s.tree) {
    DevBuf<double> partial;
    int64_t nb = ceil_div(n, HV_T);
    DMO_TRY(partial.alloc(ctx, nb));
    DMO_TRY(hv3_tree_device(ctx, s.xs.p, s.ys.p, s.zs.p, s.zo.p, n, h_ref[0], h_ref[1], h_ref[2], partial.p, &nb));
    DMO_TRY(s.res.alloc(ctx, 1));
    DMO_LAUNCH(final_sum_kernel, 1, 256, 0, partial.p, nb, s.res.p);
  }
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int hv3_ranked_finish(dmo_ctx* ctx, Hv3Ranked& s, double* h_out) {
  *h_out = 0.0;
  int32_t n1 = 0;
  DMO_CUDA(cudaMemcpyAsync(&n1, s.pos.p + s.n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (n1 == 0) return DMO_OK;
  if (s.tree && n1 >= hv3_tree_min()) {
    DMO_CUDA(cudaMemcpyAsync(h_out, s.res.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    return DMO_OK;
  }
  const int64_t nb = ceil_div(n1, HV_T);
  DevBuf<double> partial;
  DMO_TRY(partial.alloc(ctx, nb));
  {
    ProfileScope ps(ctx, "hv3");
    DMO_LAUNCH(hv3_kernel, (unsigned)nb, HV_T, 0, s.xs.p, s.ys.p, s.zs.p, s.zo.p, (int64_t)n1, s.ref[0], s.ref[1], s.ref[2],
               partial.p);
  }
  return sum_partials(ctx, partial, nb, h_out);
}

// The body of dmo_ehvi_select on device arrays (1 <= k <= nc), without its trailing wait: it waits once, for the box count
int ehvi_select_device(dmo_ctx* ctx, const double* F, int64_t nf, const double* means, const double* variances, int64_t nc, int M,
                       const double* ref, int nds, int64_t k, int64_t* sel, double* score) {
  // rank-0 subset of the chosen set (indicators.py:299-303)
  DevBuf<double> front_buf;
  const double* front = F;
  int64_t nfr = nf;
  if (nds) {
    DMO_TRY(nondominated_subset(ctx, F, nf, M, front_buf, &nfr));
    if (nfr > 0)
      front = front_buf.p;
    else
      nfr = nf;
  }
  DevBuf<uint32_t> sidx;
  DMO_TRY(prim_sort_by_column(ctx, front, nfr, M, 0, sidx));
  DevBuf<int32_t> flag, pos;
  DMO_TRY(flag.alloc(ctx, nfr + 2));
  DMO_TRY(pos.alloc(ctx, nfr + 2));
  DMO_LAUNCH(box_flag_kernel, (unsigned)ceil_div(nfr + 2, 256), 256, 0, front, sidx.p, nfr, M, ref, flag.p);
  DMO_TRY(prim_exclusive_sum_i32(ctx, flag.p, pos.p, nfr + 2));
  int32_t nb = 0;
  DMO_CUDA(cudaMemcpyAsync(&nb, pos.p + nfr + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  DevBuf<double> lower, upper, sc;
  DMO_TRY(lower.alloc(ctx, (size_t)(nb > 0 ? nb : 1) * M));
  DMO_TRY(upper.alloc(ctx, (size_t)(nb > 0 ? nb : 1) * M));
  DMO_TRY(sc.alloc(ctx, nc));
  if (nb > 0)
    DMO_LAUNCH(box_write_kernel, (unsigned)ceil_div(nfr + 1, 256), 256, 0, front, sidx.p, nfr, M, ref, flag.p, pos.p,
               lower.p, upper.p);
  if (M <= 8)
    DMO_LAUNCH(ehvi_kernel<8>, (unsigned)ceil_div(nc, 128), 128, 2 * 64 * M * sizeof(double), lower.p, upper.p, (int64_t)nb,
               M, means, variances, nc, sc.p);
  else
    DMO_LAUNCH(ehvi_kernel<16>, (unsigned)ceil_div(nc, 128), 128, 2 * 64 * M * sizeof(double), lower.p, upper.p, (int64_t)nb,
               M, means, variances, nc, sc.p);
  // k largest scores, ties by candidate index
  DevBuf<uint64_t> k0, k1;
  DevBuf<uint32_t> i0, i1;
  DMO_TRY(k0.alloc(ctx, nc));
  DMO_TRY(k1.alloc(ctx, nc));
  DMO_TRY(i0.alloc(ctx, nc));
  DMO_TRY(i1.alloc(ctx, nc));
  DMO_LAUNCH(neg_key_kernel, (unsigned)ceil_div(nc, 256), 256, 0, sc.p, nc, k0.p, i0.p);
  DMO_TRY(prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, i1.p, nc, 0, 64));
  DMO_LAUNCH(widen_idx_kernel, (unsigned)ceil_div(k, 256), 256, 0, i1.p, k, sel);
  if (score) DMO_CUDA(cudaMemcpyAsync(score, sc.p, nc * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}


extern "C" {

int dmo_hypervolume(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref, double* out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out && ref && n >= 0 && M >= 1 && M <= 16, "hypervolume: bad arguments");
  *out = 0.0;
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(F, "hypervolume: null points");
  double h_ref[16];
  DMO_CUDA(cudaMemcpy(h_ref, ref, M * sizeof(double), cudaMemcpyDefault));
  In<double> f;
  DMO_TRY(f.init(ctx, F, (size_t)n * M));
  DMO_TRY(hypervolume_device(ctx, f.d, n, M, h_ref, out));
  return DMO_OK;
}

int dmo_nondominated_flags(dmo_ctx* ctx, const double* Y, int64_t n, int M, int32_t* flags) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(n >= 0 && M >= 1 && M <= 16, "nondominated_flags: bad shape n=%lld M=%d", (long long)n, M);
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(Y && flags, "nondominated_flags: null pointer");
  In<double> y;
  Out<int32_t> f;
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  DMO_TRY(f.init(ctx, flags, (size_t)n));
  DevBuf<int32_t> keep;
  DMO_TRY(nondominated_keep_flags(ctx, y.d, n, M, keep));
  DMO_LAUNCH(dominated_flag_kernel, (unsigned)ceil_div(n, 256), 256, 0, keep.p, n, f.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(f.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_hypervolume_ranked(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref, const int32_t* rank,
                           double* out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out && ref && n >= 0 && M >= 1 && M <= 16, "hypervolume_ranked: bad arguments");
  *out = 0.0;
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(F && rank, "hypervolume_ranked: null points / ranks");
  double h_ref[16];
  DMO_CUDA(cudaMemcpy(h_ref, ref, M * sizeof(double), cudaMemcpyDefault));
  In<double> f;
  In<int32_t> r;
  DMO_TRY(f.init(ctx, F, (size_t)n * M));
  DMO_TRY(r.init(ctx, rank, (size_t)n));
  DMO_TRY(hypervolume_device_ranked(ctx, f.d, n, M, h_ref, r.d, out));
  return DMO_OK;
}

int dmo_ehvi_select(dmo_ctx* ctx, const double* F, int64_t nf, const double* means, const double* variances, int64_t nc,
                    int M, const double* ref, int nds, int64_t k, int64_t* sel, double* score) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(F && means && variances && ref && sel && nf > 0 && nc > 0 && k > 0 && M >= 1 && M <= EH_MAX_OBJ,
              "ehvi_select: bad arguments");
  if (k > nc) k = nc;
  In<double> f, mu, var, r;
  DMO_TRY(f.init(ctx, F, (size_t)nf * M));
  DMO_TRY(mu.init(ctx, means, (size_t)nc * M));
  DMO_TRY(var.init(ctx, variances, (size_t)nc * M));
  DMO_TRY(r.init(ctx, ref, (size_t)M));
  Out<int64_t> osel;
  Out<double> osc;
  DMO_TRY(osel.init(ctx, sel, (size_t)k));
  DMO_TRY(osc.init(ctx, score, (size_t)nc));
  DMO_TRY(ehvi_select_device(ctx, f.d, nf, mu.d, var.d, nc, M, r.d, nds, k, osel.d, osc.d));
  DMO_TRY(osel.finish(ctx));
  DMO_TRY(osc.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
