// Exact-GP fit on the GPU for given hyper-parameters (SURVEY.md section 8f row N1).
//   K = c k(X, X) + (noise + jitter) I ;  L = chol(K) ;  alpha = K^-1 y ;  log p(y | theta) = -y' alpha / 2 - sum log L_ii - N log(2 pi) / 2
// -- what scikit-learn's GaussianProcessRegressor.fit / log_marginal_likelihood compute per objective behind
// GPR_Matern.__init__ (dmosopt/model.py:1214-1251; sklearn/gaussian_process/_gpr.py, Rasmussen & Williams Alg. 2.1) and what
// every trial of the reference's SCE-UA hyper-parameter search evaluates (dmosopt/model.py:1419-1753): an N^3 / 3 float64
// Cholesky per trial and objective (0.3 .. 1 s on the host at N = 4096).
//
// Float64 throughout (this is the parity anchor of the posterior: alpha and L feed dmo_gp_create).  Right-looking blocked
// Cholesky with 64 x 64 blocks: per block column one diagonal factorisation (one CTA, shared memory), one panel solve
// X L_kk' = A_ik (one CTA per block row, forward substitution per row) and one trailing update A_ij -= A_ik A_jk' over
// the lower triangle (one CTA per 64 x 64 tile, 4 x 4 register blocking).  The targets ride along as one extra ROW of the
// matrix ([K y; y' big]): the factorisation then leaves z = L^-1 y in that row, so y' K^-1 y = z' z and the log marginal
// likelihood need no separate forward solve; alpha = L^-T z is one backward sweep (one CTA, only when alpha is wanted).
#include <math_constants.h>

#include "gp.cuh"

namespace {

constexpr int CB = 64;  // Cholesky block edge

// lower triangle (and diagonal) of K, row-major with leading dimension ld; the strict upper triangle is zeroed.
// One CTA per 32 x 32 tile of K: the 64 rows of X it needs are staged in shared memory once (scaled by 1 / l), tiles
// strictly above the diagonal only write zeros.  Batched over blockIdx.z: problem b has its own inv_ls (d), constant,
// diag_add, targets y (N) and matrix K + b * sK; X is shared.
__global__ void __launch_bounds__(256) kernel_matrix_kernel(const double* __restrict__ X, int64_t N, int d, int kind,
                                                            const double* __restrict__ inv_ls, const double* __restrict__ constant_b,
                                                            const double* __restrict__ diag_add_b, const double* __restrict__ y,
                                                            int64_t ld, double* __restrict__ K, int64_t sK) {
  extern __shared__ double xs[];  // [64][d + 1]: rows i0 .. i0+31 then j0 .. j0+31 of X, scaled
  const int bz = blockIdx.z;
  inv_ls += (size_t)bz * d;
  y += (size_t)bz * N;
  K += (size_t)bz * sK;
  const double constant = constant_b[bz], diag_add = diag_add_b[bz];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int64_t i0 = (int64_t)blockIdx.y * 32, j0 = (int64_t)blockIdx.x * 32;
  const int dp = d + 1;
  const bool upper = j0 > i0 + 31;
  if (!upper) {
    for (int t = threadIdx.x; t < 64 * d; t += 256) {
      const int r = t / d, c = t - r * d;
      const int64_t g = (r < 32 ? i0 + r : j0 + (r - 32));
      xs[r * dp + c] = g < N ? X[g * d + c] * inv_ls[c] : 0.0;
    }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int li = ty + 8 * u;
    const int64_t i = i0 + li, j = j0 + tx;
    if (i >= ld || j >= ld) continue;
    double v = 0.0;
    if (i < N && j < N) {
      if (j <= i) {
        const double* a = xs + li * dp;
        const double* b = xs + (32 + tx) * dp;
        double s = 0.0;
        for (int c = 0; c < d; ++c) {
          const double t = a[c] - b[c];
          s += t * t;
        }
        v = constant * stationary(s, kind);
        if (i == j) v += diag_add;
      }
    } else if (i == N && j < N) {
      v = y[j];  // the augmented row: the factorisation turns it into z = L^-1 y
    } else if (i == j) {
      v = i == N ? 1e300 : 1.0;  // its diagonal only has to stay positive; identity tail of the padded matrix
    }
    K[i * ld + j] = v;
  }
}

// ---- Cholesky steps (A: lower triangle, in place, leading dimension ld, ld % CB == 0) ----------------------------------
// Every step is batched over independent matrices A + b * sA (b: blockIdx.x of potrf_diag_kernel, blockIdx.y of the panel
// and trailing-update kernels); a CTA never mixes matrices, so each one's arithmetic is the same however many run.
__global__ void __launch_bounds__(256) potrf_diag_kernel(double* __restrict__ A, int64_t ld, int64_t sA, int64_t k0,
                                                         int* __restrict__ info) {
  A += (size_t)blockIdx.x * sA;
  info += blockIdx.x;
  // Thread (w, c) = (tid >> 6, tid & 63) keeps the 16 elements (r = w + 4 u, c) of the block in registers for the whole
  // factorisation.  Column j: its four owner threads publish the (unscaled) column to shared memory, one barrier, then every
  // thread scales what it needs itself (L_rj = a_rj / sqrt(a_jj)) and updates its own elements -- 16 independent FMAs per
  // thread and step, one barrier per column (the published column is double buffered).
  __shared__ double col[2][CB];
  const int tid = threadIdx.x, c = tid & 63, w = tid >> 6;
  double a[16];
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int r = w + 4 * u;
    a[u] = c <= r ? A[(k0 + r) * ld + k0 + c] : 0.0;
  }
  for (int j = 0; j < CB; ++j) {
    double* cb = col[j & 1];
    if (c == j) {
#pragma unroll
      for (int u = 0; u < 16; ++u) cb[w + 4 * u] = a[u];
    }
    __syncthreads();
    const double djj = cb[j];
    if (!(djj > 0.0)) {  // uniform over the block: not positive definite (numpy raises LinAlgError here)
      if (tid == 0) atomicExch(info, (int)(k0 + j) + 1);
      return;
    }
    const double s = sqrt(djj), rs = 1.0 / s;
    if (c == j) {
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const int r = w + 4 * u;
        a[u] = r == j ? s : (r > j ? a[u] * rs : a[u]);
      }
    } else if (c > j) {
      const double lc = cb[c] * rs;  // L_cj
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const int r = w + 4 * u;
        if (r >= c) a[u] = fma(-(cb[r] * rs), lc, a[u]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int r = w + 4 * u;
    if (c <= r) A[(k0 + r) * ld + k0 + c] = a[u];
  }
}

// A_ik <- A_ik L_kk^-T for the block rows below the diagonal block: thread r owns row r of the 64 x 64 block
constexpr size_t PAIR_SMEM = (size_t)2 * CB * (CB + 1) * sizeof(double);  // two padded 64 x 64 blocks: above the 48 KB static limit

__global__ void __launch_bounds__(CB) trsm_panel_kernel(double* __restrict__ A, int64_t ld, int64_t sA, int64_t k0) {
  extern __shared__ double dyn_sm[];
  A += (size_t)blockIdx.y * sA;
  double (*l)[CB + 1] = reinterpret_cast<double (*)[CB + 1]>(dyn_sm);
  double (*x)[CB + 1] = reinterpret_cast<double (*)[CB + 1]>(dyn_sm + CB * (CB + 1));
  __shared__ double linv[CB];
  const int r = threadIdx.x;
  const int64_t i0 = k0 + (int64_t)(blockIdx.x + 1) * CB;
  for (int c = 0; c < CB; ++c) {
    l[c][r] = r <= c ? A[(k0 + c) * ld + k0 + r] : 0.0;  // l[c][r] = L_kk[c][r]; coalesced over r
    x[c][r] = A[(i0 + c) * ld + k0 + r];                  // x[row c][col r]
  }
  __syncthreads();
  linv[r] = 1.0 / l[r][r];
  // row r in registers (fully unrolled: static indices): x_rj = (a_rj - sum_{t<j} x_rt L_jt) / L_jj, L_kk broadcast from
  // shared memory, two independent accumulation chains
  double xr[CB];
#pragma unroll
  for (int c = 0; c < CB; ++c) xr[c] = x[r][c];
  __syncthreads();
#pragma unroll
  for (int j = 0; j < CB; ++j) {
    double s0 = xr[j], s1 = 0.0;
#pragma unroll
    for (int t = 0; t + 1 < j; t += 2) {
      s0 = fma(-xr[t], l[j][t], s0);
      s1 = fma(-xr[t + 1], l[j][t + 1], s1);
    }
    if (j & 1) s0 = fma(-xr[j - 1], l[j][j - 1], s0);
    xr[j] = (s0 + s1) * linv[j];
  }
#pragma unroll
  for (int c = 0; c < CB; ++c) x[r][c] = xr[c];
  __syncthreads();
  for (int c = 0; c < CB; ++c) A[(i0 + c) * ld + k0 + r] = x[c][r];
}

// A_ij -= A_ik A_jk' for the tiles i >= j > k of the lower triangle; 256 threads, 4 x 4 outputs each
__global__ void __launch_bounds__(256) syrk_tile_kernel(double* __restrict__ A, int64_t ld, int64_t sA, int64_t k0, int nrem) {
  extern __shared__ double dyn_sm[];
  A += (size_t)blockIdx.y * sA;
  double (*sa)[CB + 1] = reinterpret_cast<double (*)[CB + 1]>(dyn_sm);                  // A_ik  [row][kk]
  double (*sb)[CB + 1] = reinterpret_cast<double (*)[CB + 1]>(dyn_sm + CB * (CB + 1));  // A_jk  [row][kk]
  // tile index -> (ti, tj) with ti >= tj, both in [0, nrem)
  const int t = blockIdx.x;
  int ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) / 2.0);
  while ((int64_t)(ti + 1) * (ti + 2) / 2 <= t) ++ti;
  while ((int64_t)ti * (ti + 1) / 2 > t) --ti;
  const int tj = t - ti * (ti + 1) / 2;
  const int64_t i0 = k0 + (int64_t)(ti + 1) * CB, j0 = k0 + (int64_t)(tj + 1) * CB;
  const int tid = threadIdx.x;
  for (int e = tid; e < CB * CB; e += 256) {
    const int r = e / CB, c = e % CB;
    sa[r][c] = A[(i0 + r) * ld + k0 + c];
    sb[r][c] = A[(j0 + r) * ld + k0 + c];
  }
  __syncthreads();
  const int ty = tid >> 4, tx = tid & 15;  // rows ty * 4 .., cols tx * 4 ..
  double acc[4][4] = {};
#pragma unroll 8
  for (int kk = 0; kk < CB; ++kk) {
    double a[4], b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      a[u] = sa[ty * 4 + u][kk];
      b[u] = sb[tx * 4 + u][kk];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int64_t gi = i0 + ty * 4 + u, gj = j0 + tx * 4 + v;
      if (gj <= gi) A[gi * ld + gj] -= acc[u][v];
    }
}

// ---- log marginal likelihood from the augmented row, alpha = L^-T z by one backward sweep: one CTA per factor ---------------
// (factor b: L + b * sL, work + b * ld, alpha + b * N, lml + b)
constexpr int SV_T = 1024;
__global__ void __launch_bounds__(SV_T) finish_fit_kernel(const double* __restrict__ L, int64_t ld, int64_t sL, int64_t N,
                                                          double* __restrict__ work, double* __restrict__ alpha, double* __restrict__ lml,
                                                          int want_alpha) {
  L += (size_t)blockIdx.x * sL;
  work += (size_t)blockIdx.x * ld;
  alpha += (size_t)blockIdx.x * N;
  lml += blockIdx.x;
  __shared__ double xs[CB];
  __shared__ double red[SV_T / 32];
  __shared__ double dl[CB][CB + 1];  // the current diagonal block of L
  const int tid = threadIdx.x;
  const int64_t nb = ld / CB;
  // z = row N of the factor; y' K^-1 y = z' z ; sum log L_ii over the N real rows
  double q = 0.0, ld_sum = 0.0;
  for (int64_t i = tid; i < N; i += SV_T) {
    const double z = L[N * ld + i];
    q += z * z;
    ld_sum += log(L[i * ld + i]);
  }
  const double quad = block_sum<SV_T / 32>(q, red);
  ld_sum = block_sum<SV_T / 32>(ld_sum, red);
  if (tid == 0) lml[0] = -0.5 * quad - ld_sum - 0.5 * (double)N * 1.8378770664093453;  // log(2 pi)
  if (!want_alpha) return;
  // backward: L' alpha = z over the whole padded matrix with right-hand side (z, 0, 0, ...): the augmented row and the identity
  // tail get alpha = 0 and drop out, the leading N x N block is solved exactly.  Block columns from the last to the first.
  for (int64_t i = tid; i < ld; i += SV_T) work[i] = i < N ? L[N * ld + i] : 0.0;
  __syncthreads();
  for (int64_t b = nb - 1; b >= 0; --b) {
    const int64_t k0 = b * CB;
    for (int e = tid; e < CB * CB; e += SV_T) dl[e / CB][e % CB] = L[(k0 + e / CB) * ld + k0 + e % CB];
    __syncthreads();
    if (tid < 32) {
      double a0 = work[k0 + tid], a1 = work[k0 + tid + 32];
      for (int j = CB - 1; j >= 0; --j) {
        const double ljj = dl[j][j];
        double aj = __shfl_sync(0xffffffffu, j < 32 ? a0 : a1, j & 31) / ljj;
        if (tid == (j & 31)) {
          if (j < 32) a0 = aj; else a1 = aj;
        }
        if (tid < j) a0 -= dl[j][tid] * aj;
        if (tid + 32 < j) a1 -= dl[j][tid + 32] * aj;
      }
      xs[tid] = a0;
      xs[tid + 32] = a1;
      work[k0 + tid] = a0;
      work[k0 + tid + 32] = a1;
    }
    __syncthreads();
    // rows above: work[i] -= sum_j L[k0 + j][i] * x_j   (column i of the block row k0..k0+63: coalesced over i)
    for (int64_t i = tid; i < k0; i += SV_T) {
      double s = 0.0;
#pragma unroll 8
      for (int j = 0; j < CB; ++j) s += L[(k0 + j) * ld + i] * xs[j];
      work[i] -= s;
    }
    __syncthreads();
  }
  for (int64_t i = tid; i < N; i += SV_T) alpha[i] = work[i];
}

__global__ void extract_lower_kernel(const double* __restrict__ A, int64_t ld, int64_t N, double* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N * N) return;
  const int64_t r = t / N, c = t - r * N;
  out[t] = c <= r ? A[r * ld + c] : 0.0;
}

}  // namespace

// nbat independent problems in one pass: problem b factors [K_b y_b; y_b' big] in A + b * ld^2 (ld = ceil((N + 1) / 64) * 64)
// with K_b = constant[b] k(X / l_b, X / l_b) + diag_add[b] I (inv_ls: (nbat, d)); info[b] (zeroed by the caller) receives a non-positive pivot + 1.
// lml (may be NULL: no finish) receives log p(y_b), alpha (may be NULL) K_b^-1 y_b, rows of N; work holds nbat * ld doubles.
// All pointers are device pointers; nothing is synchronised.
int gp_fit_batched(dmo_ctx* ctx, int64_t N, int d, int nbat, int kernel, const double* X, const double* inv_ls, const double* constant,
                   const double* diag_add, const double* y, double* A, int64_t ld, int* info, double* work, double* alpha, double* lml) {
  const int64_t sA = ld * ld;
  dim3 kg((unsigned)ceil_div(ld, 32), (unsigned)ceil_div(ld, 32), (unsigned)nbat);
  DMO_LAUNCH(kernel_matrix_kernel, kg, 256, (size_t)64 * (d + 1) * sizeof(double), X, N, d, kernel, inv_ls, constant, diag_add, y, ld,
             A, sA);
  DMO_TRY(gp_potrf_batched(ctx, A, ld, nbat, info));
  if (lml) DMO_LAUNCH(finish_fit_kernel, (unsigned)nbat, SV_T, 0, A, ld, sA, N, work, alpha, lml, alpha ? 1 : 0);
  return DMO_OK;
}

int gp_potrf_batched(dmo_ctx* ctx, double* A, int64_t ld, int nbat, int* info) {
  const int64_t nb = ld / CB, sA = ld * ld;
  DMO_REQUIRE(ld % CB == 0, "gp_potrf_batched: ld %lld is not a multiple of %d", (long long)ld, CB);
  DMO_CUDA(cudaFuncSetAttribute(trsm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PAIR_SMEM));
  DMO_CUDA(cudaFuncSetAttribute(syrk_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PAIR_SMEM));
  for (int64_t k = 0; k < nb; ++k) {
    const int64_t k0 = k * CB;
    DMO_LAUNCH(potrf_diag_kernel, (unsigned)nbat, 256, 0, A, ld, sA, k0, info);
    const int nrem = (int)(nb - k - 1);
    if (nrem > 0) {
      DMO_LAUNCH(trsm_panel_kernel, dim3((unsigned)nrem, (unsigned)nbat), CB, PAIR_SMEM, A, ld, sA, k0);
      DMO_LAUNCH(syrk_tile_kernel, dim3((unsigned)((int64_t)nrem * (nrem + 1) / 2), (unsigned)nbat), 256, PAIR_SMEM, A, ld, sA, k0, nrem);
    }
  }
  return DMO_OK;
}

extern "C" {

int dmo_gp_fit(dmo_ctx* ctx, int64_t N, int d, int M, int kernel, const double* X_train, const double* y, const double* constant,
               const double* length_scale, const double* noise, double jitter, double* L_out, double* alpha_out, double* lml_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(N >= 1 && d >= 1 && d <= 90 && M >= 1 && X_train && y && constant && length_scale && noise, "gp_fit: bad arguments");
  DMO_REQUIRE(kernel == DMO_KERNEL_MATERN52 || kernel == DMO_KERNEL_RBF, "gp_fit: unknown kernel %d", kernel);
  DMO_REQUIRE(alpha_out || lml_out || L_out, "gp_fit: nothing to compute");
  std::vector<double> h_c(M), h_n(M), h_ls((size_t)M * d), h_inv((size_t)M * d), h_dadd(M);
  DMO_CUDA(cudaMemcpy(h_c.data(), constant, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(h_n.data(), noise, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(h_ls.data(), length_scale, (size_t)M * d * sizeof(double), cudaMemcpyDefault));
  for (size_t t = 0; t < h_ls.size(); ++t) h_inv[t] = 1.0 / h_ls[t];
  for (int m = 0; m < M; ++m) h_dadd[m] = h_n[m] + jitter;
  const int64_t nb = ceil_div(N + 1, CB), ld = nb * CB;  // N rows of K + the row that carries the targets
  In<double> ix, iy;
  DMO_TRY(ix.init(ctx, X_train, (size_t)N * d));
  DMO_TRY(iy.init(ctx, y, (size_t)M * N));
  Out<double> oL, oa, ol;
  DMO_TRY(oL.init(ctx, L_out, L_out ? (size_t)M * N * N : 0));
  DMO_TRY(oa.init(ctx, alpha_out, alpha_out ? (size_t)M * N : 0));
  DMO_TRY(ol.init(ctx, lml_out, lml_out ? (size_t)M : 0));
  DevBuf<double> A, inv_ls, cd, work, alpha_d, lml_d;
  DevBuf<int> info;
  DMO_TRY(A.alloc(ctx, (size_t)ld * ld));
  DMO_TRY(inv_ls.alloc(ctx, (size_t)M * d));
  DMO_TRY(cd.alloc(ctx, (size_t)2 * M));
  DMO_TRY(work.alloc(ctx, (size_t)ld));
  DMO_TRY(alpha_d.alloc(ctx, (size_t)N));
  DMO_TRY(lml_d.alloc(ctx, 1));
  DMO_TRY(info.alloc(ctx, 1));
  DMO_CUDA(cudaMemcpyAsync(inv_ls.p, h_inv.data(), h_inv.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(cd.p, h_c.data(), M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(cd.p + M, h_dadd.data(), M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemsetAsync(info.p, 0, sizeof(int), ctx->stream));
  ProfileScope ps(ctx, "gp_fit");
  for (int m = 0; m < M; ++m) {
    // one objective at a time (a batch of one), sharing the scratch matrix
    DMO_TRY(gp_fit_batched(ctx, N, d, 1, kernel, ix.d, inv_ls.p + (size_t)m * d, cd.p + m, cd.p + M + m, iy.d + (size_t)m * N, A.p, ld,
                           info.p, work.p, oa.d ? alpha_d.p : nullptr, (oa.d || ol.d) ? lml_d.p : nullptr));
    if (oa.d || ol.d) {
      if (oa.d) DMO_CUDA(cudaMemcpyAsync(oa.d + (size_t)m * N, alpha_d.p, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
      if (ol.d) DMO_CUDA(cudaMemcpyAsync(ol.d + m, lml_d.p, sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (oL.d) DMO_LAUNCH(extract_lower_kernel, (unsigned)ceil_div(N * N, 256), 256, 0, A.p, ld, N, oL.d + (size_t)m * N * N);
  }
  DMO_CHECK_LAUNCH();
  int h_info = 0;
  DMO_CUDA(cudaMemcpyAsync(&h_info, info.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (h_info) return dmo_fail(ctx, DMO_ERR_ARG, "gp_fit: the kernel matrix is not positive definite (pivot %d)", h_info - 1);
  DMO_TRY(oL.finish(ctx));
  DMO_TRY(oa.finish(ctx));
  DMO_TRY(ol.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
