// Sensitivity analysis (dmosopt's default_sa_methods, dmosopt/sa.py): the DGSM forward-difference design and its
// statistics, and the eFAST design.  The designs are written elementwise with explicit IEEE roundings in NumPy's
// operation order (oracle/sa.py), so the DGSM design is bit-identical to the NumPy expression and the eFAST design
// follows its restatement operation for operation.  The statistics reduce in a fixed order: results do not depend on
// the launch.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int SA_THREADS = 256;
constexpr int SA_WARPS = SA_THREADS / 32;
constexpr int SA_DESIGN_BLOCKS_PER_SM = 16;  // the design kernels stride over their output beyond this grid
constexpr int SA_MAX_REPLICATES = 4096;
constexpr int64_t FAST_MAX_N = int64_t(1) << 20;  // keeps n = rint(theta 2/pi) < 2^20 in the eFAST range reduction

// Cody-Waite split of pi/2 (fdlibm's pio2_1, pio2_2, pio2_2t): n * P1 and n * P2 are exact for n < 2^20
constexpr double SA_PIO2_1 = 1.57079632673412561417e00;
constexpr double SA_PIO2_2 = 6.07710050630396597660e-11;
constexpr double SA_PIO2_3 = 2.02226624879595063154e-21;
constexpr double SA_TWO_OVER_PI = 6.36619772367581382433e-01;
constexpr double SA_PIO2 = 1.5707963267948966;   // fl(pi) / 2
constexpr double SA_INV_PI = 0.3183098861837907;  // fl(1 / fl(pi))
constexpr double SA_PI2 = 9.869604401089358;      // fl(fl(pi) * fl(pi)), numpy's np.pi**2

unsigned design_grid(dmo_ctx* ctx, int64_t total) {
  return (unsigned)std::min<int64_t>(ceil_div(total, SA_THREADS), (int64_t)ctx->sm_count * SA_DESIGN_BLOCKS_PER_SM);
}

// X[row, col] for row = i (d+1) + t: u = B[i, col] (+ delta when t == col + 1), x = u (ub - lb) + lb
__global__ void __launch_bounds__(SA_THREADS) dgsm_design_kernel(const double* __restrict__ B, int64_t N, int d,
                                                                 const double* __restrict__ lb, const double* __restrict__ ub,
                                                                 double delta, double* __restrict__ X) {
  const int64_t total = N * (d + 1) * d;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / d;
    const int col = (int)(e - row * d);
    const int64_t i = row / (d + 1);
    const int t = (int)(row - i * (d + 1));
    double u = B[i * d + col];
    if (t == col + 1) u = __dadd_rn(u, delta);
    __stcs(X + e, __dadd_rn(__dmul_rn(u, __dsub_rn(ub[col], lb[col])), lb[col]));
  }
}

// arcsin(sin(theta)) for 0 <= theta < 2^20 pi/2 (oracle/sa.py triangle): theta = n pi/2 + r, then r, pi/2 - |r|, -r,
// |r| - pi/2 for n = 0, 1, 2, 3 mod 4
__device__ __forceinline__ double sa_triangle(double th) {
  const double n = rint(__dmul_rn(th, SA_TWO_OVER_PI));
  double r = __dsub_rn(th, __dmul_rn(n, SA_PIO2_1));
  r = __dsub_rn(r, __dmul_rn(n, SA_PIO2_2));
  r = __dsub_rn(r, __dmul_rn(n, SA_PIO2_3));
  const int q = (int)(int64_t)n & 3;
  const double a = fabs(r);
  return q == 0 ? r : q == 1 ? __dsub_rn(SA_PIO2, a) : q == 2 ? -r : __dsub_rn(a, SA_PIO2);
}

// X[i N + k, j] = (0.5 + triangle(w_j s_k + phi_i) / pi) (ub - lb) + lb, s_k = (2 pi / N) k, w_i = omega[0] and the
// other columns take omega[1..] in order
__global__ void __launch_bounds__(SA_THREADS) fast_design_kernel(int64_t N, int d, const double* __restrict__ omega,
                                                                 const double* __restrict__ phi, const double* __restrict__ lb,
                                                                 const double* __restrict__ ub, double* __restrict__ X) {
  const int64_t total = N * d * d;
  const double c = __ddiv_rn(2.0 * M_PI, (double)N);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / d;
    const int col = (int)(e - row * d);
    const int i = (int)(row / N);
    const int64_t k = row - (int64_t)i * N;
    const double w = col == i ? omega[0] : omega[col < i ? col + 1 : col];
    const double th = __dadd_rn(__dmul_rn(w, __dmul_rn(c, (double)k)), phi[i]);
    const double x = __dadd_rn(0.5, __dmul_rn(SA_INV_PI, sa_triangle(th)));
    __stcs(X + e, __dadd_rn(__dmul_rn(x, __dsub_rn(ub[col], lb[col])), lb[col]));
  }
}

// One CTA per (output m, parameter j), blockIdx.x = m d + j.  Stages yb_i = Y[base_i, m] and q2_i = ((Y[pert_ij, m] -
// yb_i) / (X[pert_ij, j] - X[base_i, j]))^2 (shared memory when they fit, else this CTA's slice of scratch), reduces the
// full-sample statistics, then each warp runs replicates r = warp, warp + SA_WARPS, ... over the resampled indices.
__global__ void __launch_bounds__(SA_THREADS) dgsm_stats_kernel(const double* __restrict__ X, const double* __restrict__ Y, int64_t N,
                                                                int d, int M, const double* __restrict__ lb,
                                                                const double* __restrict__ ub, const int32_t* __restrict__ idx,
                                                                int R, double z, double* __restrict__ scratch, double* __restrict__ vi_o,
                                                                double* __restrict__ vis_o, double* __restrict__ dg_o,
                                                                double* __restrict__ conf_o) {
  extern __shared__ double sh[];
  __shared__ double part[SA_WARPS];
  const int j = blockIdx.x % d, m = blockIdx.x / d;
  double* rep = sh;
  double* yb = scratch ? scratch + (int64_t)blockIdx.x * 2 * N : sh + R;
  double* q2 = yb + N;
  const int64_t stride = d + 1;
  for (int64_t i = threadIdx.x; i < N; i += SA_THREADS) {
    const int64_t b = i * stride, p = b + 1 + j;
    const double y0 = Y[b * M + m];
    const double q = __ddiv_rn(__dsub_rn(Y[p * M + m], y0), __dsub_rn(X[p * d + j], X[b * d + j]));
    yb[i] = y0;
    q2[i] = __dmul_rn(q, q);
  }
  __syncthreads();
  const double rj = __dsub_rn(ub[j], lb[j]);
  const double r2 = __dmul_rn(rj, rj);
  const double dN = (double)N;
  double a = 0.0, c = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += SA_THREADS) {
    a += q2[i];
    c += yb[i];
  }
  const double vi = block_sum<SA_WARPS>(a, part) / dN;
  const double ym = block_sum<SA_WARPS>(c, part) / dN;
  a = 0.0;
  c = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += SA_THREADS) {
    const double e = q2[i] - vi, f = yb[i] - ym;
    a += e * e;
    c += f * f;
  }
  const double vs = sqrt(block_sum<SA_WARPS>(a, part) / dN);
  const double var = block_sum<SA_WARPS>(c, part) / dN;
  // replicates: one warp each, lane-strided sums then the butterfly
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < R; r += SA_WARPS) {
    const int32_t* ix = idx + (int64_t)r * N;
    double sq = 0.0, sy = 0.0;
    for (int64_t i = lane; i < N; i += 32) {
      const int32_t t = ix[i];
      sq += q2[t];
      sy += yb[t];
    }
    sq = warp_sum(sq);
    const double mr = warp_sum(sy) / dN;
    double sv = 0.0;
    for (int64_t i = lane; i < N; i += 32) {
      const double f = yb[ix[i]] - mr;
      sv += f * f;
    }
    sv = warp_sum(sv);
    if (lane == 0) rep[r] = (sq / dN) * r2 / ((sv / dN) * SA_PI2);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int r = 0; r < R; ++r) s += rep[r];
    const double mean = s / R;
    double v = 0.0;
    for (int r = 0; r < R; ++r) v += (rep[r] - mean) * (rep[r] - mean);
    const int o = m * d + j;
    vi_o[o] = vi;
    vis_o[o] = vs;
    dg_o[o] = vi * r2 / (var * SA_PI2);
    conf_o[o] = R > 1 ? z * sqrt(v / (R - 1)) : NAN;
  }
}

}  // namespace

int dmo_sa_dgsm_design(dmo_ctx* ctx, const double* base, int64_t N, int d, const double* xlb, const double* xub, double delta,
                       double* X) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(base && xlb && xub && X && N >= 1 && d >= 1, "sa_dgsm_design: bad arguments (N=%lld d=%d)", (long long)N, d);
  DMO_REQUIRE(isfinite(delta), "sa_dgsm_design: delta must be finite");
  In<double> ib, ilb, iub;
  Out<double> ox;
  DMO_TRY(ib.init(ctx, base, (size_t)N * d));
  DMO_TRY(ilb.init(ctx, xlb, (size_t)d));
  DMO_TRY(iub.init(ctx, xub, (size_t)d));
  const int64_t total = N * (d + 1) * d;
  DMO_TRY(ox.init(ctx, X, (size_t)total));
  {
    ProfileScope ps(ctx, "dgsm_design_kernel");
    DMO_LAUNCH(dgsm_design_kernel, design_grid(ctx, total), SA_THREADS, 0, ib.d, N, d, ilb.d, iub.d, delta, ox.d);
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(ox.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_sa_fast_design(dmo_ctx* ctx, int64_t N, int d, const double* omega, const double* phi, const double* xlb,
                       const double* xub, double* X) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(omega && phi && xlb && xub && X && d >= 1, "sa_fast_design: bad arguments");
  DMO_REQUIRE(N > 64 && N <= FAST_MAX_N, "sa_fast_design: N=%lld outside (4 M^2 = 64, 2^20]", (long long)N);
  In<double> iw, ip, ilb, iub;
  Out<double> ox;
  DMO_TRY(iw.init(ctx, omega, (size_t)d));
  DMO_TRY(ip.init(ctx, phi, (size_t)d));
  DMO_TRY(ilb.init(ctx, xlb, (size_t)d));
  DMO_TRY(iub.init(ctx, xub, (size_t)d));
  const int64_t total = N * d * d;
  DMO_TRY(ox.init(ctx, X, (size_t)total));
  {
    ProfileScope ps(ctx, "fast_design_kernel");
    DMO_LAUNCH(fast_design_kernel, design_grid(ctx, total), SA_THREADS, 0, N, d, iw.d, ip.d, ilb.d, iub.d, ox.d);
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(ox.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_sa_dgsm_stats(dmo_ctx* ctx, const double* X, const double* Y, int64_t N, int d, int M, const double* xlb,
                      const double* xub, const int32_t* boot_idx, int R, double z, double* vi, double* vi_std, double* dgsm,
                      double* conf) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(X && Y && xlb && xub && vi && vi_std && dgsm && conf && N >= 2 && N < INT32_MAX && d >= 1 && M >= 1,
              "sa_dgsm_stats: bad arguments (N=%lld d=%d M=%d)", (long long)N, d, M);
  DMO_REQUIRE(R >= 0 && R <= SA_MAX_REPLICATES && (R == 0 || boot_idx), "sa_dgsm_stats: R=%d outside [0, %d] or no indices", R,
              SA_MAX_REPLICATES);
  DMO_REQUIRE((int64_t)M * d < INT32_MAX, "sa_dgsm_stats: M d too large");
  const int64_t rows = N * (d + 1);
  In<double> ix, iy, ilb, iub;
  In<int32_t> ii;
  DMO_TRY(ix.init(ctx, X, (size_t)(rows * d)));
  DMO_TRY(iy.init(ctx, Y, (size_t)(rows * M)));
  DMO_TRY(ilb.init(ctx, xlb, (size_t)d));
  DMO_TRY(iub.init(ctx, xub, (size_t)d));
  DMO_TRY(ii.init(ctx, boot_idx, (size_t)R * N));
  if (R > 0) {
    // the bootstrap indices index the base rows: check them before any kernel gathers with them
    const int32_t* p = boot_idx;
    std::vector<int32_t> host;
    if (dmo_is_device_ptr(boot_idx)) {
      host.resize((size_t)R * N);
      DMO_CUDA(cudaMemcpyAsync(host.data(), boot_idx, host.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
      DMO_CUDA(dmo_wait(ctx));
      p = host.data();
    }
    int h = 0;
    for (int64_t k = 0; k < (int64_t)R * N; ++k) h |= (p[k] < 0) | (p[k] >= N);
    DMO_REQUIRE(!h, "sa_dgsm_stats: bootstrap indices outside [0, N=%lld)", (long long)N);
  }
  Out<double> o1, o2, o3, o4;
  const size_t nout = (size_t)M * d;
  DMO_TRY(o1.init(ctx, vi, nout));
  DMO_TRY(o2.init(ctx, vi_std, nout));
  DMO_TRY(o3.init(ctx, dgsm, nout));
  DMO_TRY(o4.init(ctx, conf, nout));
  int max_smem = 0;
  DMO_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
  size_t smem = (size_t)R * sizeof(double);
  DevBuf<double> scratch;
  if (smem + 2 * (size_t)N * sizeof(double) + SA_WARPS * sizeof(double) <= (size_t)max_smem) {
    smem += 2 * (size_t)N * sizeof(double);
  } else {  // the columns do not fit: stage them in global memory, one slice of 2 N per CTA
    DMO_TRY(scratch.alloc(ctx, nout * 2 * (size_t)N));
  }
  DMO_CUDA(cudaFuncSetAttribute(dgsm_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    ProfileScope ps(ctx, "dgsm_stats_kernel");
    DMO_LAUNCH(dgsm_stats_kernel, (unsigned)nout, SA_THREADS, smem, ix.d, iy.d, N, d, M, ilb.d, iub.d, ii.d, R, z, scratch.p, o1.d,
               o2.d, o3.d, o4.d);
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(o1.finish(ctx));
  DMO_TRY(o2.finish(ctx));
  DMO_TRY(o3.finish(ctx));
  DMO_TRY(o4.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}
