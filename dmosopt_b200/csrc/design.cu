// Uniform-design scores (dmosopt/discrepancy.py, dmosopt/GLP.py): the L2 discrepancies MD2, CD2, SD2 and WD2 of a design,
// and the good-lattice-point generator search, which scores every candidate lattice by its centred L2 discrepancy.
//
// A discrepancy is D^2 = D1 + c2 D2 + c3 D3 with D2 = sum_k prod_i row(x_ki) and D3 = sum_{k,j} prod_i pair(x_ki, x_ji).
// D3 is n^2 s "pair-dims" and is the whole cost.  l2_pairs_kernel tiles it over 64 x 64 row pairs: each CTA stages a
// dimension chunk of both row tiles in shared memory (x plus the metric's per-row precomputed terms), each thread keeps
// a 4 x 4 block of running products in registers across the chunks, and the CTA's sum goes to one slot of a partials
// array.  pair() is symmetric, so only tiles with tk <= tj run and an off-diagonal tile counts twice.  l2_finish_kernel
// sums the partials and D2 of one design per CTA in a fixed order.  No atomics: results do not depend on the launch.
//
// The rows come from a Source: a given (n, s) matrix, or a rank-1 lattice generated in the tile loader from one row of
// per-column multipliers h (x_ki = (u - 0.5) / rows with u = ((k + 1) h_i mod lattice), 0 replaced by lattice), so the
// C candidate designs of a generator search are never materialised.
//
// These sums are in a different order from the reference's, so they rank candidates only up to a margin.
// glp_cd2_pairs_kernel recomputes the n^2 pair products of a few shortlisted lattices in the reference's own operation
// order (explicit roundings, no contraction); the host sums them sequentially (dmosopt_b200/sampling.py).
#include <algorithm>
#include <climits>

#include "common.cuh"

namespace {

constexpr int L2_THREADS = 256;
constexpr int L2_WARPS = L2_THREADS / 32;
constexpr int L2_TILE = 64;  // rows per side of a CTA's pair tile; each thread holds 4 x 4 pairs
constexpr int L2_CHUNK = 16; // dimensions staged per pass
constexpr int64_t L2_MAX_TILES = 46340;  // tiles per side: tiles^2 CTAs per design must stay below 2^31
constexpr int64_t GLP_MAX_CANDIDATES = 65535;  // one design per grid row (gridDim.y < 2^16)
constexpr int64_t GLP_MAX_LATTICE = INT_MAX;   // (k + 1) h < lattice^2 < 2^62 in int64

struct MatrixSrc {
  const double* X;
  int s;
  __device__ __forceinline__ double operator()(int64_t /*design*/, int64_t k, int i) const { return X[k * s + i]; }
};

struct LatticeSrc {
  const int64_t* H;
  int s;
  int64_t lattice;
  double rows;
  __device__ __forceinline__ double operator()(int64_t c, int64_t k, int i) const {
    int64_t u = ((k + 1) * H[c * s + i]) % lattice;
    if (u == 0) u = lattice;
    return __ddiv_rn(__dsub_rn((double)u, 0.5), rows);
  }
};

// Per-metric terms (Hickernell 1998).  left/right are precomputed per row and per dimension when a tile is staged; the
// k side of a pair reads left, the j side right.
struct MD2 {
  static __device__ __forceinline__ double row(double x) { return 3.0 - x * x; }
  static __device__ __forceinline__ double left(double x) { return x; }
  static __device__ __forceinline__ double right(double x) { return x; }
  static __device__ __forceinline__ double pair(double xk, double, double xj, double) { return 2.0 - fmax(xk, xj); }
};
struct CD2 {
  static __device__ __forceinline__ double row(double x) {
    const double a = fabs(x - 0.5);
    return 1.0 + 0.5 * a - 0.5 * a * a;
  }
  static __device__ __forceinline__ double left(double x) { return 1.0 + 0.5 * fabs(x - 0.5); }
  static __device__ __forceinline__ double right(double x) { return 0.5 * fabs(x - 0.5); }
  static __device__ __forceinline__ double pair(double xk, double lk, double xj, double rj) { return (lk + rj) - 0.5 * fabs(xk - xj); }
};
struct SD2 {
  static __device__ __forceinline__ double row(double x) { return 1.0 + 2.0 * x - 2.0 * x * x; }
  static __device__ __forceinline__ double left(double x) { return x; }
  static __device__ __forceinline__ double right(double x) { return x; }
  static __device__ __forceinline__ double pair(double xk, double, double xj, double) { return 1.0 - fabs(xk - xj); }
};
struct WD2 {
  static __device__ __forceinline__ double row(double) { return 1.0; }
  static __device__ __forceinline__ double left(double x) { return x; }
  static __device__ __forceinline__ double right(double x) { return x; }
  static __device__ __forceinline__ double pair(double xk, double, double xj, double) {
    const double d = fabs(xk - xj);
    return 1.5 - d * (1.0 - d);
  }
};

// CTA (tile pair blockIdx.x = tk T + tj, design blockIdx.y): partial[design T^2 + tk T + tj] = weight * sum of the
// 64 x 64 pair products; CTAs with tk > tj return at once (their slot is never read).
template <class Src, class Metric>
__global__ void __launch_bounds__(L2_THREADS) l2_pairs_kernel(Src src, int64_t n, int s, int64_t T, double* __restrict__ partial) {
  const int64_t tk = blockIdx.x / T, tj = blockIdx.x - tk * T;
  if (tk > tj) return;
  const int64_t c = blockIdx.y;
  __shared__ double xk[L2_CHUNK][L2_TILE], lk[L2_CHUNK][L2_TILE], xj[L2_CHUNK][L2_TILE], rj[L2_CHUNK][L2_TILE];
  __shared__ double part[L2_WARPS];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double p[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) p[a][b] = 1.0;
  const int64_t k0 = tk * L2_TILE, j0 = tj * L2_TILE;
  for (int i0 = 0; i0 < s; i0 += L2_CHUNK) {
    const int w = min(L2_CHUNK, s - i0);
    __syncthreads();
    for (int e = threadIdx.x; e < L2_CHUNK * L2_TILE; e += L2_THREADS) {
      const int r = e % L2_TILE, i = e / L2_TILE;
      const bool dim = i < w;
      const double a = dim && k0 + r < n ? src(c, k0 + r, i0 + i) : 0.5;
      const double b = dim && j0 + r < n ? src(c, j0 + r, i0 + i) : 0.5;
      xk[i][r] = a;
      lk[i][r] = Metric::left(a);
      xj[i][r] = b;
      rj[i][r] = Metric::right(b);
    }
    __syncthreads();
    for (int i = 0; i < w; ++i) {
      double ax[4], al[4], bx[4], br[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        ax[a] = xk[i][ty + 16 * a];
        al[a] = lk[i][ty + 16 * a];
        bx[a] = xj[i][tx + 16 * a];
        br[a] = rj[i][tx + 16 * a];
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) p[a][b] *= Metric::pair(ax[a], al[a], bx[b], br[b]);
    }
  }
  double acc = 0.0;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      if (k0 + ty + 16 * a < n && j0 + tx + 16 * b < n) acc += p[a][b];
  const double sum = block_sum<L2_WARPS>(acc, part);
  if (threadIdx.x == 0) partial[c * T * T + blockIdx.x] = tk == tj ? sum : 2.0 * sum;
}

// CTA per design: d3[c] = sum of its partials over tk <= tj, d2[c] = sum_k prod_i row(x_ki), both in a fixed order
template <class Src, class Metric>
__global__ void __launch_bounds__(L2_THREADS) l2_finish_kernel(Src src, int64_t n, int s, int64_t T, const double* __restrict__ partial,
                                                                double* __restrict__ d2, double* __restrict__ d3) {
  __shared__ double part[L2_WARPS];
  const int64_t c = blockIdx.x;
  double a = 0.0;
  for (int64_t t = threadIdx.x; t < T * T; t += L2_THREADS)
    if (t / T <= t % T) a += partial[c * T * T + t];
  const double s3 = block_sum<L2_WARPS>(a, part);
  double b = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += L2_THREADS) {
    double q = 1.0;
    for (int i = 0; i < s; ++i) q *= Metric::row(src(c, k, i));
    b += q;
  }
  const double s2 = block_sum<L2_WARPS>(b, part);
  if (threadIdx.x == 0) {
    d2[c] = s2;
    d3[c] = s3;
  }
}

// P[l, k rows + j] = prod_i (((1 + 0.5 |x_ki - 0.5|) + 0.5 |x_ji - 0.5|) - 0.5 |x_ki - x_ji|), the factors multiplied in
// order i = 0 .. s-1 from 1.0 and every operation rounded on its own: the reference's CD2 pair product bit for bit.
__global__ void __launch_bounds__(L2_THREADS) glp_cd2_pairs_kernel(LatticeSrc src, int64_t n, double* __restrict__ P) {
  const int64_t l = blockIdx.y;
  const int64_t e = blockIdx.x * (int64_t)L2_THREADS + threadIdx.x;
  if (e >= n * n) return;
  const int64_t k = e / n, j = e - k * n;
  double q = 1.0;
  for (int i = 0; i < src.s; ++i) {
    const double x = src(l, k, i), y = src(l, j, i);
    const double ax = fabs(__dsub_rn(x, 0.5)), ay = fabs(__dsub_rn(y, 0.5));
    const double t = __dsub_rn(__dadd_rn(__dadd_rn(1.0, __dmul_rn(0.5, ax)), __dmul_rn(0.5, ay)), __dmul_rn(0.5, fabs(__dsub_rn(x, y))));
    q = __dmul_rn(q, t);
  }
  P[l * n * n + e] = q;
}

template <class Src, class Metric>
int l2_terms(dmo_ctx* ctx, Src src, int64_t designs, int64_t n, int s, double* d2, double* d3) {
  const int64_t T = ceil_div(n, L2_TILE);
  DevBuf<double> partial;
  DMO_TRY(partial.alloc(ctx, (size_t)(designs * T * T)));
  {
    ProfileScope ps(ctx, "l2_pairs_kernel");
    DMO_LAUNCH((l2_pairs_kernel<Src, Metric>), dim3((unsigned)(T * T), (unsigned)designs), L2_THREADS, 0, src, n, s, T, partial.p);
  }
  DMO_CHECK_LAUNCH();
  {
    ProfileScope ps(ctx, "l2_finish_kernel");
    DMO_LAUNCH((l2_finish_kernel<Src, Metric>), (unsigned)designs, L2_THREADS, 0, src, n, s, T, partial.p, d2, d3);
  }
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// the multipliers index the lattice: check them on the host before any kernel forms (k + 1) h
int glp_check_multipliers(dmo_ctx* ctx, const int64_t* H, int64_t C, int s, int64_t lattice) {
  const int64_t* p = H;
  std::vector<int64_t> host;
  if (dmo_is_device_ptr(H)) {
    host.resize((size_t)(C * s));
    DMO_CUDA(cudaMemcpyAsync(host.data(), H, host.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    p = host.data();
  }
  int bad = 0;
  for (int64_t e = 0; e < C * s; ++e) bad |= (p[e] < 0) | (p[e] >= lattice);
  DMO_REQUIRE(!bad, "glp: multipliers outside [0, lattice=%lld)", (long long)lattice);
  return DMO_OK;
}

int glp_check(dmo_ctx* ctx, const char* what, const int64_t* H, int64_t C, int s, int64_t lattice, int64_t rows) {
  DMO_REQUIRE(H && C >= 1 && s >= 1, "%s: bad arguments (C=%lld s=%d)", what, (long long)C, s);
  DMO_REQUIRE(C <= GLP_MAX_CANDIDATES, "%s: C=%lld candidates above %lld (one grid row each)", what, (long long)C,
              (long long)GLP_MAX_CANDIDATES);
  DMO_REQUIRE(lattice >= 2 && lattice <= GLP_MAX_LATTICE, "%s: lattice=%lld outside [2, 2^31 - 1] (int64 products (k+1) h)", what,
              (long long)lattice);
  DMO_REQUIRE(rows >= 1 && rows <= lattice, "%s: rows=%lld outside [1, lattice=%lld]", what, (long long)rows, (long long)lattice);
  DMO_REQUIRE(ceil_div(rows, L2_TILE) <= L2_MAX_TILES, "%s: rows=%lld above %lld", what, (long long)rows,
              (long long)(L2_MAX_TILES * L2_TILE));
  return glp_check_multipliers(ctx, H, C, s, lattice);
}

}  // namespace

int dmo_glp_cd2_terms(dmo_ctx* ctx, const int64_t* H, int64_t C, int s, int64_t lattice, int64_t rows, double* d2, double* d3) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(d2 && d3, "glp_cd2_terms: null output");
  DMO_TRY(glp_check(ctx, "glp_cd2_terms", H, C, s, lattice, rows));
  In<int64_t> ih;
  Out<double> o2, o3;
  DMO_TRY(ih.init(ctx, H, (size_t)(C * s)));
  DMO_TRY(o2.init(ctx, d2, (size_t)C));
  DMO_TRY(o3.init(ctx, d3, (size_t)C));
  const LatticeSrc src{ih.d, s, lattice, (double)rows};
  DMO_TRY((l2_terms<LatticeSrc, CD2>(ctx, src, C, rows, s, o2.d, o3.d)));
  DMO_TRY(o2.finish(ctx));
  DMO_TRY(o3.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_glp_cd2_pairs(dmo_ctx* ctx, const int64_t* H, int64_t L, int s, int64_t lattice, int64_t rows, double* P) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(P, "glp_cd2_pairs: null output");
  DMO_TRY(glp_check(ctx, "glp_cd2_pairs", H, L, s, lattice, rows));
  const int64_t per = rows * rows;
  DMO_REQUIRE(ceil_div(per, L2_THREADS) <= INT_MAX, "glp_cd2_pairs: rows=%lld too large for one grid row", (long long)rows);
  In<int64_t> ih;
  Out<double> op;
  DMO_TRY(ih.init(ctx, H, (size_t)(L * s)));
  DMO_TRY(op.init(ctx, P, (size_t)(L * per)));
  const LatticeSrc src{ih.d, s, lattice, (double)rows};
  {
    ProfileScope ps(ctx, "glp_cd2_pairs_kernel");
    DMO_LAUNCH(glp_cd2_pairs_kernel, dim3((unsigned)ceil_div(per, L2_THREADS), (unsigned)L), L2_THREADS, 0, src, rows, op.d);
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(op.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_l2_discrepancy_terms(dmo_ctx* ctx, int metric, const double* X, int64_t n, int s, double* d2, double* d3) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(X && d2 && d3 && n >= 1 && s >= 1, "l2_discrepancy_terms: bad arguments (n=%lld s=%d)", (long long)n, s);
  DMO_REQUIRE(ceil_div(n, L2_TILE) <= L2_MAX_TILES, "l2_discrepancy_terms: n=%lld above %lld", (long long)n,
              (long long)(L2_MAX_TILES * L2_TILE));
  In<double> ix;
  Out<double> o2, o3;
  DMO_TRY(ix.init(ctx, X, (size_t)(n * s)));
  DMO_TRY(o2.init(ctx, d2, 1));
  DMO_TRY(o3.init(ctx, d3, 1));
  const MatrixSrc src{ix.d, s};
  switch (metric) {
    case DMO_L2_MD2: DMO_TRY((l2_terms<MatrixSrc, MD2>(ctx, src, 1, n, s, o2.d, o3.d))); break;
    case DMO_L2_CD2: DMO_TRY((l2_terms<MatrixSrc, CD2>(ctx, src, 1, n, s, o2.d, o3.d))); break;
    case DMO_L2_SD2: DMO_TRY((l2_terms<MatrixSrc, SD2>(ctx, src, 1, n, s, o2.d, o3.d))); break;
    case DMO_L2_WD2: DMO_TRY((l2_terms<MatrixSrc, WD2>(ctx, src, 1, n, s, o2.d, o3.d))); break;
    default: return dmo_fail(ctx, DMO_ERR_ARG, "l2_discrepancy_terms: unknown metric %d", metric);
  }
  DMO_TRY(o2.finish(ctx));
  DMO_TRY(o3.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}
