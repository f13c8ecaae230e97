// Exact log marginal likelihood of the multitask GP and its gradient (training of MEGP_Matern, SURVEY.md section 8f
// row N1; the reference trains with Adam on gpytorch's ExactMarginalLogLikelihood, dmosopt/model_gpytorch.py:1722-1829).
//
// With C = K_x (x) B + I (x) D, r = Y - m(X) and alpha = C^-1 r (N x M),
//     d lml / d theta = alpha' dC alpha / 2 - tr(C^-1 dC) / 2.
// The block decomposition of gp_multitask.cu gives C^-1 = (I (x) D^-1/2 Q) blockdiag(A_j^-1) (I (x) Q' D^-1/2) with
// A_j = lambda_j K_x + I, so with c_sj = Q_sj / sqrt(D_s) and a_j the block alphas:
//     alpha_.s     = sum_j c_sj a_j
//     d / d l_k    = 1/2 sum_{i,i'} W(i,i') dK_x(i,i') / d l_k,   W = alpha B alpha' - sum_j lambda_j A_j^-1
//     d / d B_st   = 1/2 [alpha_.s' K_x alpha_.t - sum_j c_sj c_tj tr(K_x A_j^-1)]
//     d / d D_s    = 1/2 [||alpha_.s||^2 - sum_j c_sj^2 tr(A_j^-1)]
//     d / d w_s    = X' alpha_.s,   d / d b_s = 1' alpha_.s
// GPU work per evaluation, after the block fit (dmo_gp_fit) and L_j^-1 (gp_linv_from_factor):
//   * mt_ainv_syrk_kernel: the lower triangle of S = sum_j lambda_j L_j^-T L_j^-1, skipping the rows of L_j^-1 that are
//     zero by triangularity.  The same tile also yields tr(K_x A_j^-1) and tr(A_j^-1) per block directly (K_x recomputed
//     for the tile), so no (N - tr A_j^-1) / lambda_j cancellation arises for a small lambda_j.
//   * mt_grad_pass_kernel: one pass over the lower triangle of training pairs; it recomputes the scaled distance, the
//     Matern value and its derivative factor from X, reads S, and sums the d length-scale terms and the M (M + 1) / 2
//     terms alpha_.s' K_x alpha_.t.
//   Both write one partial per tile and target; mt_fold_kernel adds them in tile order.  No atomics: deterministic.
// The rest (alpha from a_j, X' alpha, 1' alpha, the final combinations) is O(N M (M + d)) host arithmetic.
//
// Both kernels and the fold (their MODELS = true instances) also take a model index (blockIdx.y) over independent
// models with their own scaled inputs, L^-1 blocks, S, alpha, B alpha and partials; the MODELS = false instances, which
// dmo_mtgp_lml_grad launches, are the one-model kernels without those offsets.  dmo_gp_lml_grad uses the index for EGP_Matern's M independent GPs
// K_m = s_m K_x(X / l_m) + sigma2_m I, each a model with one block: lambda = s_m and "B" = s_m, with L^-1 the inverse
// factor of K_m itself, so S = s_m K_m^-1, W = s_m (alpha alpha' - K_m^-1), and the traces tr(K_x K_m^-1), tr(K_m^-1)
// come from the unscaled accumulators.  Every CTA works on one model and every sum runs in a fixed order, so a model's
// outputs do not depend on which other models share the launch.
#include <math.h>

#include <vector>

#include "gp.cuh"

namespace {

constexpr int GT = 64;  // tile edge of both kernels (256 threads, 4 x 4 outputs each, rows ty + 16 u, columns tx + 16 v)
constexpr int KC = 32;  // rows of L_j^-1 per shared-memory stage of the SYRK
constexpr int XP = 33;  // padded row of a 32-coordinate slice of the inputs

__device__ __forceinline__ void tile_of(int t, int& ti, int& tj) {
  ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) / 2.0);
  while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
  while (ti * (ti + 1) / 2 > t) --ti;
  tj = t - ti * (ti + 1) / 2;
}

// S = sum_j lambda_j L_j^-T L_j^-1 on the tiles ti >= tj (row-major, leading dimension ld = Npad), and per tile and block
// part[tile][j] = sum_{i,i'} K_x(i,i') A_j^-1(i,i') over the tile's lower triangle (twice off the diagonal) and
// part[tile][M + j] = its diagonal part of tr(A_j^-1).  Linv: (M, ld, ld), zero above the diagonal and in the padding;
// A_j^-1(i,i') = sum_{k >= max(i,i')} Linv_j(k,i) Linv_j(k,i'), so the k loop starts at the tile's first row.
template <bool MODELS>  // false: one model (MEGP), the kernel without the model offsets
__global__ void __launch_bounds__(256) mt_ainv_syrk_kernel(const double* __restrict__ Linv, int64_t ld, int64_t N, int M,
                                                           const double* __restrict__ lam, const double* __restrict__ xs, int d,
                                                           double* __restrict__ S, double* __restrict__ part) {
  __shared__ double sa[GT * XP], sb[GT * XP];  // [KC][GT] rows of L^-1, or [GT][XP] coordinate slices
  __shared__ double red[8];
  if constexpr (MODELS) {
    const size_t mdl = blockIdx.y;  // model index
    Linv += mdl * M * ld * ld;
    lam += mdl * M;
    xs += mdl * N * d;
    S += mdl * ld * ld;
    part += mdl * gridDim.x * 2 * M;
  }
  int ti, tj;
  tile_of(blockIdx.x, ti, tj);
  const int64_t i0 = (int64_t)ti * GT, j0 = (int64_t)tj * GT;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  // K_x on the tile from the scaled inputs, 32 coordinates per stage
  double kv[4][4] = {};
  for (int c0 = 0; c0 < d; c0 += 32) {
    const int nc = d - c0 < 32 ? d - c0 : 32;
    for (int e = tid; e < GT * 32; e += 256) {
      const int r = e >> 5, c = e & 31;
      const int64_t gi = i0 + r, gj = j0 + r;
      sa[r * XP + c] = (c < nc && gi < N) ? xs[gi * d + c0 + c] : 0.0;
      sb[r * XP + c] = (c < nc && gj < N) ? xs[gj * d + c0 + c] : 0.0;
    }
    __syncthreads();
    for (int c = 0; c < nc; ++c)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double a = sa[(ty + 16 * u) * XP + c];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const double t = a - sb[(tx + 16 * v) * XP + c];
          kv[u][v] = fma(t, t, kv[u][v]);
        }
      }
    __syncthreads();
  }
  double wk[4][4];  // symmetry weight times K_x: 2 below the diagonal, 1 on it, 0 above it and outside N
  bool dg[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int64_t i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
      const double r = sqrt(kv[u][v]) * 2.23606797749978969641;
      const double k = (1.0 + r + r * r / 3.0) * exp(-r);
      wk[u][v] = (i < N && j < N) ? (i > j ? 2.0 * k : (i == j ? 1.0 : 0.0)) : 0.0;
      dg[u][v] = i == j && i < N;
    }
  double s[4][4] = {};
  for (int jb = 0; jb < M; ++jb) {
    const double* L = Linv + (size_t)jb * ld * ld;
    double acc[4][4] = {};
    double pa[KC * GT / 256], pb[KC * GT / 256];  // the next stage, prefetched into registers
#pragma unroll
    for (int q = 0; q < KC * GT / 256; ++q) {
      const int e = tid + 256 * q, kk = e >> 6, c = e & 63;
      pa[q] = L[(i0 + kk) * ld + i0 + c];
      pb[q] = L[(i0 + kk) * ld + j0 + c];
    }
    for (int64_t k0 = i0; k0 < ld; k0 += KC) {
#pragma unroll
      for (int q = 0; q < KC * GT / 256; ++q) {
        const int e = tid + 256 * q;
        sa[e] = pa[q];
        sb[e] = pb[q];
      }
      __syncthreads();
      if (k0 + KC < ld) {
#pragma unroll
        for (int q = 0; q < KC * GT / 256; ++q) {
          const int e = tid + 256 * q, kk = e >> 6, c = e & 63;
          pa[q] = L[(k0 + KC + kk) * ld + i0 + c];
          pb[q] = L[(k0 + KC + kk) * ld + j0 + c];
        }
      }
#pragma unroll 4
      for (int kk = 0; kk < KC; ++kk) {
        double a[4], b[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          a[u] = sa[kk * GT + ty + 16 * u];
          b[u] = sb[kk * GT + tx + 16 * u];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
      }
      __syncthreads();
    }
    const double lj = lam[jb];
    double tka = 0.0, ta = 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        s[u][v] = fma(lj, acc[u][v], s[u][v]);
        tka = fma(wk[u][v], acc[u][v], tka);
        if (dg[u][v]) ta += acc[u][v];
      }
    tka = block_sum<8>(tka, red);
    ta = block_sum<8>(ta, red);
    if (tid == 0) {
      part[(size_t)blockIdx.x * 2 * M + jb] = tka;
      part[(size_t)blockIdx.x * 2 * M + M + jb] = ta;
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) S[(i0 + ty + 16 * u) * ld + j0 + tx + 16 * v] = s[u][v];
}

// One tile of training pairs (i in tile ti, i' in tile tj, ti >= tj), lower triangle only.  Phase 1 (4 x 4 pairs per
// thread): f(i,i') = (5/3) (1 + r) e^-r W(i,i') for i > i' (0 otherwise), with r = sqrt5 ||x_i / l - x_i' / l|| and
// W = sum_s alpha_is (B alpha)_i's - S(i,i'); kw(i,i') = K_x(i,i') for i > i', 1/2 for i = i'.  Phase 2 (one warp per
// target, lanes over i'): part[tile][k] = sum f (x_ik / l_k - x_i'k / l_k)^2 for k < d, and for the pairs s <= t
// part[tile][d + p(s,t)] = sum kw (alpha_is alpha_i't + alpha_it alpha_i's).  Summed over the tiles:
// d lml / d l_k = part_k / l_k, alpha_.s' K_x alpha_.t = part_{d + p(s,t)}.
template <bool MODELS>
__global__ void __launch_bounds__(256) mt_grad_pass_kernel(const double* __restrict__ xs, int64_t N, int d, int M,
                                                           const double* __restrict__ S, int64_t ld, const double* __restrict__ al,
                                                           const double* __restrict__ bal, double* __restrict__ part, int nq) {
  extern __shared__ double sm[];
  const int dp = d + 1;
  double* xi = sm;                  // [GT][dp]
  double* xj = xi + GT * dp;        // [GT][dp]
  double* f = xj + GT * dp;         // [GT][GT + 1]
  double* kw = f + GT * (GT + 1);   // [GT][GT + 1]
  double* ai = kw + GT * (GT + 1);  // [GT][M] alpha rows of tile ti
  double* aj = ai + GT * M;         // [GT][M] alpha rows of tile tj
  double* bj = aj + GT * M;         // [GT][M] (B alpha) rows of tile tj
  if constexpr (MODELS) {
    const size_t mdl = blockIdx.y;  // model index
    xs += mdl * N * d;
    S += mdl * ld * ld;
    al += mdl * N * M;
    bal += mdl * N * M;
    part += mdl * gridDim.x * nq;
  }
  int ti, tj;
  tile_of(blockIdx.x, ti, tj);
  const int64_t i0 = (int64_t)ti * GT, j0 = (int64_t)tj * GT;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < GT * d; e += 256) {
    const int r = e / d, c = e - r * d;
    xi[r * dp + c] = i0 + r < N ? xs[(i0 + r) * d + c] : 0.0;
    xj[r * dp + c] = j0 + r < N ? xs[(j0 + r) * d + c] : 0.0;
  }
  for (int e = tid; e < GT * M; e += 256) {
    const int r = e / M;
    ai[e] = i0 + r < N ? al[i0 * M + e] : 0.0;
    aj[e] = j0 + r < N ? al[j0 * M + e] : 0.0;
    bj[e] = j0 + r < N ? bal[j0 * M + e] : 0.0;
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int a = ty + 16 * u, b = tx + 16 * v;
      const int64_t i = i0 + a, j = j0 + b;
      double fv = 0.0, kwv = 0.0;
      if (i < N && j < N && i >= j) {
        if (i == j) {
          kwv = 0.5;
        } else {
          double s2 = 0.0;
          for (int c = 0; c < d; ++c) {
            const double t = xi[a * dp + c] - xj[b * dp + c];
            s2 = fma(t, t, s2);
          }
          const double r = sqrt(s2) * 2.23606797749978969641;
          const double e = exp(-r);
          kwv = (1.0 + r + r * r / 3.0) * e;
          double w = -S[i * ld + j];
          for (int s = 0; s < M; ++s) w = fma(ai[a * M + s], bj[b * M + s], w);
          fv = (5.0 / 3.0) * (1.0 + r) * e * w;
        }
      }
      f[a * (GT + 1) + b] = fv;
      kw[a * (GT + 1) + b] = kwv;
    }
  __syncthreads();
  const int npair = M * (M + 1) / 2;
  for (int q = warp; q < d + npair; q += 8) {
    double acc = 0.0;
    if (q < d) {
      const double x0 = xj[lane * dp + q], x1 = xj[(lane + 32) * dp + q];
      for (int a = 0; a < GT; ++a) {
        const double xa = xi[a * dp + q];
        const double u0 = xa - x0, u1 = xa - x1;
        acc = fma(f[a * (GT + 1) + lane] * u0, u0, acc);
        acc = fma(f[a * (GT + 1) + lane + 32] * u1, u1, acc);
      }
    } else {
      int p = q - d, s = 0;  // pair index -> (s, t), s <= t, row-major over the upper triangle
      while (p >= M - s) {
        p -= M - s;
        ++s;
      }
      const int t = s + p;
      const double as0 = aj[lane * M + s], at0 = aj[lane * M + t], as1 = aj[(lane + 32) * M + s], at1 = aj[(lane + 32) * M + t];
      for (int a = 0; a < GT; ++a) {
        const double xs_ = ai[a * M + s], xt_ = ai[a * M + t];
        acc = fma(kw[a * (GT + 1) + lane], fma(xs_, at0, xt_ * as0), acc);
        acc = fma(kw[a * (GT + 1) + lane + 32], fma(xs_, at1, xt_ * as1), acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) part[(size_t)blockIdx.x * nq + q] = acc;
  }
}

// out[q] = sum over tiles, in tile order, of part[tile][q]; with MODELS, model blockIdx.y: part + y * n_tiles * nq,
// out + y * nq
template <bool MODELS>
__global__ void mt_fold_kernel(const double* __restrict__ part, int n_tiles, int nq, double* __restrict__ out) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  if constexpr (MODELS) {
    part += (size_t)blockIdx.y * n_tiles * nq;
    out += (size_t)blockIdx.y * nq;
  }
  double s = 0.0;
  for (int t = 0; t < n_tiles; ++t) s += part[(size_t)t * nq + q];
  out[q] = s;
}

}  // namespace

extern "C" {

int dmo_mtgp_lml_grad(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* Y, const double* length_scale,
                      const double* B, const double* D, const double* weight, const double* bias, double* lml_out,
                      double* g_length_scale, double* g_B, double* g_D, double* g_weight, double* g_bias) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(lml_out && g_length_scale && g_B && g_D && g_weight && g_bias, "mtgp_lml_grad: null output");
  MtBlocks mb;
  std::vector<double> a((size_t)M * N > 0 ? (size_t)M * N : 1);  // block alphas a_j (M, N), filled by dmo_gp_fit
  {
    ProfileScope ps(ctx, "mtgp_lg_fit");
    DMO_TRY(mtgp_blocks_fit(ctx, "mtgp_lml_grad", N, d, M, X_train, Y, length_scale, B, D, weight, bias, mb, a.data()));
  }
  const int64_t Npad = ceil_div(N, GT) * GT;
  const int T = (int)(Npad / GT), n_tiles = T * (T + 1) / 2;
  DevBuf<double> Linv;
  {
    ProfileScope ps(ctx, "mtgp_lg_linv");
    DMO_TRY(Linv.alloc(ctx, (size_t)M * Npad * Npad));
    DMO_CUDA(cudaMemsetAsync(Linv.p, 0, (size_t)M * Npad * Npad * sizeof(double), ctx->stream));
    for (int j = 0; j < M; ++j)
      DMO_TRY(gp_linv_from_factor(ctx, mb.Lf.p + (size_t)j * N * N, N, Npad, Linv.p + (size_t)j * Npad * Npad));
  }
  mb.Lf.release();
  // alpha (N, M) = sum_j c_sj a_j and B alpha, row-major
  const std::vector<double>&hB = mb.hB, &Q = mb.Q, &sqD = mb.sqD, &hx = mb.hx;
  std::vector<double> al((size_t)N * M), bal((size_t)N * M);
  for (int64_t n = 0; n < N; ++n) {
    for (int s = 0; s < M; ++s) {
      double v = 0.0;
      for (int j = 0; j < M; ++j) v += Q[(size_t)s * M + j] * a[(size_t)j * N + n];
      al[(size_t)n * M + s] = v / sqD[s];
    }
    for (int s = 0; s < M; ++s) {
      double v = 0.0;
      for (int t = 0; t < M; ++t) v += hB[(size_t)s * M + t] * al[(size_t)n * M + t];
      bal[(size_t)n * M + s] = v;
    }
  }
  const int npair = M * (M + 1) / 2, nq = d + npair;
  DevBuf<double> xs_d, lam_d, al_d, bal_d, S, part_a, part_g, red;
  DMO_TRY(xs_d.alloc(ctx, (size_t)N * d));
  DMO_TRY(lam_d.alloc(ctx, M));
  DMO_TRY(al_d.alloc(ctx, (size_t)N * M));
  DMO_TRY(bal_d.alloc(ctx, (size_t)N * M));
  DMO_TRY(S.alloc(ctx, (size_t)Npad * Npad));
  DMO_TRY(part_a.alloc(ctx, (size_t)n_tiles * 2 * M));
  DMO_TRY(part_g.alloc(ctx, (size_t)n_tiles * nq));
  DMO_TRY(red.alloc(ctx, (size_t)2 * M + nq));
  DMO_CUDA(cudaMemcpyAsync(xs_d.p, mb.xs.data(), (size_t)N * d * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(lam_d.p, mb.lam.data(), M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(al_d.p, al.data(), (size_t)N * M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(bal_d.p, bal.data(), (size_t)N * M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  {
    ProfileScope ps(ctx, "mtgp_lg_ainv");
    DMO_LAUNCH(mt_ainv_syrk_kernel<false>, (unsigned)n_tiles, 256, 0, Linv.p, Npad, N, M, lam_d.p, xs_d.p, d, S.p, part_a.p);
    DMO_LAUNCH(mt_fold_kernel<false>, 1, 64, 0, part_a.p, n_tiles, 2 * M, red.p);
  }
  Linv.release();
  {
    ProfileScope ps(ctx, "mtgp_lg_grad");
    const size_t smem = ((size_t)2 * GT * (d + 1) + (size_t)2 * GT * (GT + 1) + (size_t)3 * GT * M) * sizeof(double);
    DMO_CUDA(cudaFuncSetAttribute(mt_grad_pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DMO_LAUNCH(mt_grad_pass_kernel<false>, (unsigned)n_tiles, 256, smem, xs_d.p, N, d, M, S.p, Npad, al_d.p, bal_d.p, part_g.p, nq);
    DMO_LAUNCH(mt_fold_kernel<false>, (unsigned)ceil_div(nq, 128), 128, 0, part_g.p, n_tiles, nq, red.p + 2 * M);
  }
  DMO_CHECK_LAUNCH();
  std::vector<double> hr((size_t)2 * M + nq);
  DMO_CUDA(cudaMemcpyAsync(hr.data(), red.p, hr.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  // host combination: trKA_j = tr(K_x A_j^-1), trA_j = tr(A_j^-1)
  const double* trKA = hr.data();
  const double* trA = hr.data() + M;
  const double* G = hr.data() + 2 * M;
  std::vector<double> gl(d), gB((size_t)M * M), gD(M), gw((size_t)M * d, 0.0), gb(M, 0.0);
  for (int k = 0; k < d; ++k) gl[k] = G[k] / mb.ls[k];
  std::vector<double> c((size_t)M * M);
  for (int s = 0; s < M; ++s)
    for (int j = 0; j < M; ++j) c[(size_t)s * M + j] = Q[(size_t)s * M + j] / sqD[s];
  for (int s = 0, p = 0; s < M; ++s)
    for (int t = s; t < M; ++t, ++p) {
      double tr = 0.0;
      for (int j = 0; j < M; ++j) tr += c[(size_t)s * M + j] * c[(size_t)t * M + j] * trKA[j];
      gB[(size_t)s * M + t] = gB[(size_t)t * M + s] = 0.5 * (G[d + p] - tr);
    }
  for (int64_t n = 0; n < N; ++n)
    for (int s = 0; s < M; ++s) {
      const double v = al[(size_t)n * M + s];
      for (int k = 0; k < d; ++k) gw[(size_t)s * d + k] += v * hx[(size_t)n * d + k];
      gb[s] += v;
    }
  for (int s = 0; s < M; ++s) {
    double q = 0.0, tr = 0.0;
    for (int64_t n = 0; n < N; ++n) q += al[(size_t)n * M + s] * al[(size_t)n * M + s];
    for (int j = 0; j < M; ++j) tr += c[(size_t)s * M + j] * c[(size_t)s * M + j] * trA[j];
    gD[s] = 0.5 * (q - tr);
  }
  DMO_CUDA(cudaMemcpy(lml_out, &mb.lml, sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_length_scale, gl.data(), d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_B, gB.data(), (size_t)M * M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_D, gD.data(), M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_weight, gw.data(), (size_t)M * d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_bias, gb.data(), M * sizeof(double), cudaMemcpyDefault));
  return DMO_OK;
}


int dmo_gp_lml_grad(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* y, const double* length_scale,
                    const double* outputscale, const double* noise, const double* weight, const double* bias, double* lml_out,
                    double* g_length_scale, double* g_outputscale, double* g_noise, double* g_weight, double* g_bias) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(N >= 1 && d >= 1 && d <= MT_FIT_DMAX && M >= 1 && M <= MT_MAX,
              "gp_lml_grad: unsupported shape N=%lld d=%d M=%d (1 <= M <= %d, d <= %d)", (long long)N, d, M, MT_MAX, MT_FIT_DMAX);
  DMO_REQUIRE(X_train && y && length_scale && outputscale && noise && weight && bias, "gp_lml_grad: null pointer");
  DMO_REQUIRE(lml_out && g_length_scale && g_outputscale && g_noise && g_weight && g_bias, "gp_lml_grad: null output");
  const size_t nd = (size_t)N * d, mn = (size_t)M * N, md = (size_t)M * d;
  std::vector<double> hx(nd), hy(mn), ls(md), hs(M), hn(M), hw(md), hb(M);
  DMO_CUDA(cudaMemcpy(hx.data(), X_train, nd * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hy.data(), y, mn * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ls.data(), length_scale, md * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hs.data(), outputscale, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hn.data(), noise, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hw.data(), weight, md * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hb.data(), bias, M * sizeof(double), cudaMemcpyDefault));
  for (int m = 0; m < M; ++m) {
    for (int k = 0; k < d; ++k) DMO_REQUIRE(ls[(size_t)m * d + k] > 0.0, "gp_lml_grad: objective %d: length scale %d must be > 0", m, k);
    DMO_REQUIRE(hs[m] > 0.0, "gp_lml_grad: objective %d: output scale %g must be > 0", m, hs[m]);
    DMO_REQUIRE(hn[m] > 0.0, "gp_lml_grad: objective %d: noise %g must be > 0", m, hn[m]);
  }
  // per objective: 1 / l_m, the scaled inputs x_n / l_m (the products kernel_matrix_kernel forms), the residuals y_m - m_m(X)
  std::vector<double> inv(md), xs((size_t)M * nd), res(mn), sd((size_t)2 * M);
  for (size_t t = 0; t < md; ++t) inv[t] = 1.0 / ls[t];
  for (int m = 0; m < M; ++m) {
    sd[m] = hs[m];
    sd[M + m] = hn[m];
    for (int64_t n = 0; n < N; ++n) {
      double mu = hb[m];
      for (int k = 0; k < d; ++k) {
        mu += hw[(size_t)m * d + k] * hx[(size_t)n * d + k];
        xs[((size_t)m * N + n) * d + k] = hx[(size_t)n * d + k] * inv[(size_t)m * d + k];
      }
      res[(size_t)m * N + n] = hy[(size_t)m * N + n] - mu;
    }
  }
  const int64_t ld = ceil_div(N + 1, GT) * GT;  // the fit's padded edge: N rows of K_m + the row that carries r_m
  const int64_t Npad = ceil_div(N, GT) * GT;
  const int T = (int)(Npad / GT), n_tiles = T * (T + 1) / 2;
  DevBuf<double> x_d, inv_d, sd_d, r_d, A, work, alpha_d, lml_d;
  DevBuf<int> info;
  DMO_TRY(x_d.alloc(ctx, nd));
  DMO_TRY(inv_d.alloc(ctx, md));
  DMO_TRY(sd_d.alloc(ctx, (size_t)2 * M));
  DMO_TRY(r_d.alloc(ctx, mn));
  DMO_TRY(A.alloc(ctx, (size_t)M * ld * ld));
  DMO_TRY(work.alloc(ctx, (size_t)M * ld));
  DMO_TRY(alpha_d.alloc(ctx, mn));
  DMO_TRY(lml_d.alloc(ctx, M));
  DMO_TRY(info.alloc(ctx, M));
  DMO_CUDA(cudaMemcpyAsync(x_d.p, hx.data(), nd * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(inv_d.p, inv.data(), md * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(sd_d.p, sd.data(), (size_t)2 * M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(r_d.p, res.data(), mn * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemsetAsync(info.p, 0, M * sizeof(int), ctx->stream));
  {
    // K_m = s_m K_x + sigma2_m I (no jitter): all M factorisations in one pass of the blocked Cholesky
    ProfileScope ps(ctx, "gp_lg_fit");
    DMO_TRY(gp_fit_batched(ctx, N, d, M, DMO_KERNEL_MATERN52, x_d.p, inv_d.p, sd_d.p, sd_d.p + M, r_d.p, A.p, ld, info.p, work.p, alpha_d.p,
                           lml_d.p));
  }
  DMO_CHECK_LAUNCH();
  std::vector<int> h_info(M);
  std::vector<double> h_lml(M), al(mn);
  DMO_CUDA(cudaMemcpyAsync(h_info.data(), info.p, M * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(h_lml.data(), lml_d.p, M * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(al.data(), alpha_d.p, mn * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  for (int m = 0; m < M; ++m)
    if (h_info[m])
      return dmo_fail(ctx, DMO_ERR_ARG, "gp_lml_grad: the kernel matrix of objective %d is not positive definite (pivot %d)", m,
                      h_info[m] - 1);
  work.release();
  r_d.release();
  DevBuf<double> Linv;
  {
    ProfileScope ps(ctx, "gp_lg_linv");
    DMO_TRY(Linv.alloc(ctx, (size_t)M * Npad * Npad));
    DMO_CUDA(cudaMemsetAsync(Linv.p, 0, (size_t)M * Npad * Npad * sizeof(double), ctx->stream));
    DMO_TRY(gp_linv_from_factor_batched(ctx, A.p, ld, ld * ld, N, M, Npad, Npad * Npad, Linv.p));
  }
  A.release();
  // "B alpha" of the one-block model: s_m alpha_m
  std::vector<double> bal(mn);
  for (int m = 0; m < M; ++m)
    for (int64_t n = 0; n < N; ++n) bal[(size_t)m * N + n] = hs[m] * al[(size_t)m * N + n];
  const int nq = d + 1;
  DevBuf<double> xs_d, bal_d, S, part_a, part_g, red;
  DMO_TRY(xs_d.alloc(ctx, (size_t)M * nd));
  DMO_TRY(bal_d.alloc(ctx, mn));
  DMO_TRY(S.alloc(ctx, (size_t)M * Npad * Npad));
  DMO_TRY(part_a.alloc(ctx, (size_t)M * n_tiles * 2));
  DMO_TRY(part_g.alloc(ctx, (size_t)M * n_tiles * nq));
  DMO_TRY(red.alloc(ctx, (size_t)M * (2 + nq)));
  DMO_CUDA(cudaMemcpyAsync(xs_d.p, xs.data(), (size_t)M * nd * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(bal_d.p, bal.data(), mn * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  {
    ProfileScope ps(ctx, "gp_lg_ainv");
    DMO_LAUNCH(mt_ainv_syrk_kernel<true>, dim3((unsigned)n_tiles, (unsigned)M), 256, 0, Linv.p, Npad, N, 1, sd_d.p, xs_d.p, d, S.p, part_a.p);
    DMO_LAUNCH(mt_fold_kernel<true>, dim3(1, (unsigned)M), 64, 0, part_a.p, n_tiles, 2, red.p);
  }
  Linv.release();
  {
    ProfileScope ps(ctx, "gp_lg_grad");
    const size_t smem = ((size_t)2 * GT * (d + 1) + (size_t)2 * GT * (GT + 1) + (size_t)3 * GT) * sizeof(double);
    DMO_CUDA(cudaFuncSetAttribute(mt_grad_pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DMO_LAUNCH(mt_grad_pass_kernel<true>, dim3((unsigned)n_tiles, (unsigned)M), 256, smem, xs_d.p, N, d, 1, S.p, Npad, alpha_d.p, bal_d.p,
               part_g.p, nq);
    DMO_LAUNCH(mt_fold_kernel<true>, dim3((unsigned)ceil_div(nq, 128), (unsigned)M), 128, 0, part_g.p, n_tiles, nq, red.p + 2 * M);
  }
  DMO_CHECK_LAUNCH();
  std::vector<double> hr((size_t)M * (2 + nq));
  DMO_CUDA(cudaMemcpyAsync(hr.data(), red.p, hr.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  // per objective: tr(K_x K_m^-1), tr(K_m^-1), then sum W dK_x / dl_k * l_k (k < d) and alpha' K_x alpha
  std::vector<double> gl(md), gs(M), gn(M), gw(md, 0.0), gb(M, 0.0);
  for (int m = 0; m < M; ++m) {
    const double trKA = hr[(size_t)2 * m], trA = hr[(size_t)2 * m + 1];
    const double* G = hr.data() + 2 * M + (size_t)m * nq;
    const double* a = al.data() + (size_t)m * N;
    for (int k = 0; k < d; ++k) gl[(size_t)m * d + k] = G[k] / ls[(size_t)m * d + k];
    gs[m] = 0.5 * (G[d] - trKA);
    double q = 0.0;
    for (int64_t n = 0; n < N; ++n) {
      q += a[n] * a[n];
      for (int k = 0; k < d; ++k) gw[(size_t)m * d + k] += a[n] * hx[(size_t)n * d + k];
      gb[m] += a[n];
    }
    gn[m] = 0.5 * (q - trA);
  }
  DMO_CUDA(cudaMemcpy(lml_out, h_lml.data(), M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_length_scale, gl.data(), md * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_outputscale, gs.data(), M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_noise, gn.data(), M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_weight, gw.data(), md * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(g_bias, gb.data(), M * sizeof(double), cudaMemcpyDefault));
  return DMO_OK;
}

}  // extern "C"
