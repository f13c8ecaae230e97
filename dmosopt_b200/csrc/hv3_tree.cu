// Exact 3-D hypervolume in O(n log^2 n) for large fronts (SURVEY.md section 8a row A16; called from hv.cu).
//
//   HV_3 = sum_k (r_z - z_k) * E_k,   E_k = area of k's xy-quadrant [x_k, r_x] x [y_k, r_y] that is not covered by the
//   quadrants of the points that precede k along z
// (the slicing identity hv3_kernel in hv.cu evaluates with one O(n) sweep per point, O(n^2) in total: 5.9 ms for a
// 65 536-point front).  Here every E_k walks only the *steps* of the staircase it needs:
//
//   points in x-sorted position p, z-order id t (ties by index).  Q_k(p) = min{ y_q : q <= p, t_q < t_k } is the
//   staircase of the earlier points as a function of the position;
//       E_k = sum_{p >= p_k} (x_{p+1} - x_p) * max(0, min(r_y, Q_k(p)) - y_k),   x_n := r_x.
//   The walk starts with one prefix query Q_k(p_k) and then jumps from drop to drop ("next q > cur with t_q < t_k and
//   y_q < m") until the staircase falls below y_k.  A point is an interior drop for at most one k (the first later point
//   that dominates it in xy removes it from every later staircase), so all walks together take O(n) jumps.
//
//   Both queries run on a merge-sort tree over the positions: level l holds, for every aligned block of 2^l positions,
//   its points sorted by t together with the running minimum of y in that order, so "min y among the points of a block
//   with t < t_k" is one binary search.  A prefix query touches <= log n blocks, a jump climbs and descends <= 2 log n.
//   The tree is built bottom-up by rank-based merges: levels 1..10 inside shared memory (one CTA per 1024 positions),
//   the levels above with one output-centric merge-path kernel each (+ a carry pass for the running minimum).
//
// Every E_k is a sum of non-negative strip areas (no "full rectangle minus covered" cancellation), block partial sums are
// combined in a fixed order: deterministic, and valid for any point set (duplicates / weakly dominated points included).
#include <math_constants.h>

#include "common.cuh"

namespace {

constexpr int LOW = 10;            // levels built in shared memory
constexpr int CH = 1 << LOW;       // positions per CTA of the low build / chunk of the high levels
constexpr uint32_t T_PAD = 0xFFFFFFFFu;

struct Tree {
  const uint32_t* ts;  // [L + 1][NP] t values, sorted inside every aligned block of 2^l positions (level 0 = position order)
  const double* ym;    // [L + 1][NP] running minimum of y along that order
  int L;               // NP = 1 << L
  int64_t NP;
};

// level-l block (index b): min y among its points with t < tk
__device__ __forceinline__ double node_min(const Tree& T, int l, int64_t b, uint32_t tk) {
  const uint32_t* ts = T.ts + (int64_t)l * T.NP + (b << l);
  int lo = 0, hi = 1 << l;  // first index with ts >= tk
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(ts + mid) < tk) lo = mid + 1; else hi = mid;
  }
  return lo ? __ldg(T.ym + (int64_t)l * T.NP + (b << l) + lo - 1) : CUDART_INF;
}

// ---- build: levels 0 .. LOW for 1024 positions per CTA -------------------------------------------------------------
__global__ void __launch_bounds__(CH) build_low_kernel(const uint32_t* __restrict__ zo, const double* __restrict__ ys,
                                                       int64_t n, int64_t NP, int Ltop, uint32_t* __restrict__ ts,
                                                       double* __restrict__ ym) {
  __shared__ uint32_t st[2][CH];
  __shared__ double sy[2][CH];
  __shared__ double sm[CH];
  const int e = threadIdx.x;
  const int64_t g = (int64_t)blockIdx.x * CH + e;
  uint32_t t = g < n ? zo[g] : T_PAD;
  double y = g < n ? ys[g] : CUDART_INF;
  st[0][e] = t;
  sy[0][e] = y;
  ts[g] = t;  // level 0
  ym[g] = y;
  __syncthreads();
  int cur = 0;
  const int top = Ltop < LOW ? Ltop : LOW;
  for (int l = 1; l <= top; ++l) {
    const int half = 1 << (l - 1);
    const int run = e >> (l - 1);             // my sorted run at level l - 1
    const int sib = (run ^ 1) << (l - 1);     // start of the sibling run
    const uint32_t mt = st[cur][e];
    // rank of my t in the sibling run; equal keys only occur between padding entries: break the tie by run order
    int lo = 0, hi = half;
    const bool right = run & 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      const uint32_t v = st[cur][sib + mid];
      if (right ? (v <= mt) : (v < mt)) lo = mid + 1; else hi = mid;
    }
    const int dest = ((run >> 1) << l) + (e & (half - 1)) + lo;
    const double my = sy[cur][e];
    __syncthreads();
    st[cur ^ 1][dest] = mt;
    sy[cur ^ 1][dest] = my;
    __syncthreads();
    cur ^= 1;
    // running minimum of y inside every block of 2^l (Hillis-Steele with a block guard)
    sm[e] = sy[cur][e];
    __syncthreads();
    for (int off = 1; off < (1 << l); off <<= 1) {
      const double v = ((e & ((1 << l) - 1)) >= off) ? sm[e - off] : CUDART_INF;
      __syncthreads();
      sm[e] = fmin(sm[e], v);
      __syncthreads();
    }
    ts[(int64_t)l * NP + g] = st[cur][e];
    ym[(int64_t)l * NP + g] = sm[e];
  }
}

// ---- build: one level above LOW.  Output-centric merge path: thread o of a block of 2^l finds how many elements of the
// left run precede output o, writes the merged t and the chunk-local running minimum of y ----------------------------
__global__ void __launch_bounds__(CH) build_high_kernel(int l, int64_t NP, const double* __restrict__ y_by_t, uint32_t* __restrict__ ts,
                                                        double* __restrict__ ym, double* __restrict__ chunk_min) {
  __shared__ double sm[CH];
  const int e = threadIdx.x;
  const int64_t g = (int64_t)blockIdx.x * CH + e;
  const int64_t half = (int64_t)1 << (l - 1);
  const int64_t base = (g >> l) << l;
  const int64_t o = g - base;  // output index inside the block
  const uint32_t* A = ts + (int64_t)(l - 1) * NP + base;  // left run, sorted
  const uint32_t* B = A + half;                           // right run, sorted
  // a = number of elements taken from A among the first o outputs: largest a with A[a-1] <= B[o-a] (ties: A first)
  int64_t lo = o > half ? o - half : 0, hi = o < half ? o : half;
  while (lo < hi) {
    const int64_t a = (lo + hi + 1) >> 1;  // try to take a from A
    // valid iff A[a-1] <= B[o-a] (or o - a == half: B exhausted)
    const bool ok = (o - a >= half) || (__ldg(A + a - 1) <= __ldg(B + (o - a)));
    if (ok) lo = a; else hi = a - 1;
  }
  const int64_t a = lo, b = o - a;
  uint32_t t;
  if (a < half && (b >= half || __ldg(A + a) <= __ldg(B + b))) t = __ldg(A + a); else t = __ldg(B + b);
  const double y = (t == T_PAD) ? CUDART_INF : __ldg(y_by_t + t);
  ts[(int64_t)l * NP + g] = t;
  sm[e] = y;
  __syncthreads();
  for (int off = 1; off < CH; off <<= 1) {
    const double v = (e >= off) ? sm[e - off] : CUDART_INF;
    __syncthreads();
    sm[e] = fmin(sm[e], v);
    __syncthreads();
  }
  ym[(int64_t)l * NP + g] = sm[e];
  if (e == CH - 1) chunk_min[blockIdx.x] = sm[e];
}

// carry of the running minimum across the chunks of one block (2^(l - LOW) chunks per block)
__global__ void __launch_bounds__(CH) carry_kernel(int l, int64_t NP, const double* __restrict__ chunk_min, double* __restrict__ ym) {
  const int64_t c = blockIdx.x;
  const int64_t per = (int64_t)1 << (l - LOW);
  const int64_t first = (c / per) * per;
  double m = CUDART_INF;
  for (int64_t q = first; q < c; ++q) m = fmin(m, __ldg(chunk_min + q));
  if (c == first) return;
  const int64_t g = c * CH + threadIdx.x;
  ym[(int64_t)l * NP + g] = fmin(ym[(int64_t)l * NP + g], m);
}

__global__ void y_by_t_kernel(const uint32_t* __restrict__ zo, const double* __restrict__ ys, int64_t n, double* __restrict__ y_by_t) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) y_by_t[zo[p]] = ys[p];
}

// ---- the walks ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) hv3_tree_kernel(Tree T, const double* __restrict__ xs, const double* __restrict__ ys,
                                                       const double* __restrict__ zs, const uint32_t* __restrict__ zo,
                                                       int64_t n, double rx, double ry, double rz, double* __restrict__ partial) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (k < n) {
    const double xk = xs[k], yk = ys[k];
    const uint32_t tk = zo[k];
    // staircase height at k's own position: prefix query over the positions [0, k]
    double m = CUDART_INF;
    {
      const int64_t r = k + 1;
      int64_t base = 0;
      if (r == T.NP) {
        m = node_min(T, T.L, 0, tk);
      } else {
        for (int l = T.L - 1; l >= 0; --l)
          if (r & ((int64_t)1 << l)) {
            m = fmin(m, node_min(T, l, base >> l, tk));
            base += (int64_t)1 << l;
          }
      }
    }
    double area = 0.0, left = xk;
    int64_t pos = k + 1;  // next position to examine
    while (m > yk) {
      // smallest q >= pos with t_q < tk and y_q < m: skip aligned blocks that hold no such point, then descend
      int64_t q = n;
      while (pos < n) {
        int l = pos ? __ffsll((long long)pos) - 1 : T.L;
        if (l > T.L) l = T.L;
        if (node_min(T, l, pos >> l, tk) < m) {
          while (l > 0) {
            --l;
            if (!(node_min(T, l, pos >> l, tk) < m)) pos += (int64_t)1 << l;  // not in the left child: it is in the right one
          }
          q = pos;
          break;
        }
        pos += (int64_t)1 << l;
      }
      const double h = fmin(ry, m) - yk;  // > 0 here
      if (q >= n) {
        area += (rx - left) * h;
        left = rx;
        break;
      }
      const double xq = fmax(xs[q], xk);
      area += (xq - left) * h;
      left = xq;
      m = ys[q];
      pos = q + 1;
    }
    v = area * (rz - zs[k]);
  }
  // deterministic block partial: the four warps summed pairwise, not in block_sum's serial order (which would change the bits)
  __shared__ double ws[4];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) partial[blockIdx.x] = (ws[0] + ws[1]) + (ws[2] + ws[3]);
}

}  // namespace

// xs / ys / zs: coordinates in x-sorted order (ties in any order); zo: z-order id of each x-sorted point (a permutation of
// 0 .. n-1, ties by index).  partial must hold ceil(n / 128) doubles; returns the number of partial sums written.
int hv3_tree_device(dmo_ctx* ctx, const double* xs, const double* ys, const double* zs, const uint32_t* zo, int64_t n, double rx,
                    double ry, double rz, double* partial, int64_t* n_partial) {
  int L = LOW;
  while (((int64_t)1 << L) < n) ++L;
  const int64_t NP = (int64_t)1 << L;
  DevBuf<uint32_t> ts;
  DevBuf<double> ym, ybt, cmin;
  DMO_TRY(ts.alloc(ctx, (size_t)(L + 1) * NP));
  DMO_TRY(ym.alloc(ctx, (size_t)(L + 1) * NP));
  DMO_TRY(ybt.alloc(ctx, (size_t)n));
  DMO_TRY(cmin.alloc(ctx, (size_t)(NP / CH)));
  ProfileScope ps(ctx, "hv3_tree");
  DMO_LAUNCH(y_by_t_kernel, (unsigned)ceil_div(n, 256), 256, 0, zo, ys, n, ybt.p);
  DMO_LAUNCH(build_low_kernel, (unsigned)(NP / CH), CH, 0, zo, ys, n, NP, L, ts.p, ym.p);
  for (int l = LOW + 1; l <= L; ++l) {
    DMO_LAUNCH(build_high_kernel, (unsigned)(NP / CH), CH, 0, l, NP, ybt.p, ts.p, ym.p, cmin.p);
    DMO_LAUNCH(carry_kernel, (unsigned)(NP / CH), CH, 0, l, NP, cmin.p, ym.p);
  }
  Tree T;
  T.ts = ts.p;
  T.ym = ym.p;
  T.L = L;
  T.NP = NP;
  const int64_t nb = ceil_div(n, 128);
  DMO_LAUNCH(hv3_tree_kernel, (unsigned)nb, 128, 0, T, xs, ys, zs, zo, n, rx, ry, rz, partial);
  DMO_CHECK_LAUNCH();
  *n_partial = nb;
  return DMO_OK;
}
