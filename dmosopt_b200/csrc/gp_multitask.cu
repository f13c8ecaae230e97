// Multitask exact-GP posterior (SURVEY.md section 8a row A19: MEGP_Matern.predict, dmosopt/model_gpytorch.py:1872-1919).
//
// The gpytorch model (model_gpytorch.py:510-571) is one ExactGP over N points x M tasks with covariance
//     C = K_x (x) B + I_N (x) D,   K_x ARD Matern-5/2 (no output scale),  B = F F' + diag(v),  D_t = task noise + noise,
// and a linear prior mean per task.  The posterior splits exactly into M single-output GPs: with
//     D^-1/2 B D^-1/2 = Q diag(lambda) Q'   (M x M, host, cyclic Jacobi: deterministic)
// the whitened, rotated system is block diagonal with blocks lambda_j K_x + I.  Block j is an ordinary GP (constant
// lambda_j, noise 1) on the rotated residuals r_j = sum_s Q_sj (y_s - m_s(X)) / sqrt(D_s); dmo_gp_fit factors it and
// gives a_j = (lambda_j K_x + I)^-1 r_j.  With c_tj = lambda_j Q_tj sqrt(D_t) and k_* = K_x(x_*, X):
//     mean_t = m_t(x_*) + sum_j c_tj k_*' a_j
//     var_t  = B_tt + D_t - sum_j c_tj^2 ||L_j^-1 k_*||^2
//     log p(Y) = sum_j lml_j - (N / 2) sum_t log D_t
// Every block sees the same k_*: the inputs are pre-scaled by 1 / l, so the kernel is isotropic with unit length, and
// one K_* plane serves all M blocks.  Per predict this file's producer writes that plane once (fp16 hi / lo for the
// tensor path, float64 for the float64 path) and accumulates the M block means k_*' a_j from the same kernel values;
// the L_j^-1 are the M planes of one GpVarOps, contracted against that plane (K_* plane stride 0) by the exact GP's
// variance contractions (var_kernel, gp_var_wgmma_kernel); mt_mix_kernel adds their partial sums in a fixed order and
// mixes the blocks back into tasks.  GpUnitPredict, the chunking and scratch of that predict, is shared with the
// variational posterior (gp_variational.cu).
#include <math.h>

#include <memory>
#include <vector>

#include <cuda_fp16.h>

#include "gp.cuh"

struct dmo_mtgp {
  int64_t N = 0;
  int d = 0, M = 0;
  double lml = 0.0;
  GpVarOps blk;                    // (M, Npad, Npad) L_j^-1 of the blocks, zero padded
  DevBuf<double> XtT;              // (d, Npad) scaled training inputs x_n / l, transposed, zero padded
  DevBuf<double> A;                // (M, Npad) a_j, zero padded
  DevBuf<double> inv_ls, xlb, xrg; // (d,)
  DevBuf<double> mix;              // (M, M) c_tj
  DevBuf<double> prior;            // (M,) B_tt + D_t
  DevBuf<double> w, b;             // (M, d) linear-mean weights times l (they act on the scaled inputs), (M,)
  DevBuf<double> ymean, ystd;      // (M,)
};

namespace {

// xs = ((x - xlb) / xrg) / l: normalised as the reference does (model_gpytorch.py:1879-1886), then scaled
__global__ void mt_scale_inputs_kernel(const double* __restrict__ X, int64_t P, int d, const double* __restrict__ xlb,
                                       const double* __restrict__ xrg, const double* __restrict__ inv_ls,
                                       double* __restrict__ xs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P * d) return;
  const int j = (int)(t % d);
  xs[t] = ((X[t] - xlb[j]) / xrg[j]) * inv_ls[j];
}

// ---- float64 producer: one K_* plane Ks[p][n] and the block-mean partial sums --------------------------------------
// A thread owns one training point; a block covers 128 training points x 32 candidates.  The squared distances of the
// 32 candidates are accumulated in registers while the coordinates are walked once (any d); the block means are
// reduced over the warp and then over the four warps in a fixed order: mpart[blockIdx.x][j][p].
constexpr int PF_TN = 128, PF_TP = 32;

__global__ void __launch_bounds__(PF_TN)
    mt_kstar_f64_kernel(const double* __restrict__ xs, int64_t P, int64_t p_base, const double* __restrict__ XtT, int64_t N,
                        int64_t Npad, int d, int M, const double* __restrict__ A, double* __restrict__ Ks,
                        double* __restrict__ mpart, int64_t mp_ld) {
  extern __shared__ double sxd[];  // [PF_TP][d] candidate tile
  __shared__ double red[PF_TN / 32][PF_TP][MT_MAX];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t n = (int64_t)blockIdx.x * PF_TN + t;
  const int64_t pt0 = (int64_t)blockIdx.y * PF_TP;  // within the chunk
  for (int i = t; i < PF_TP * d; i += PF_TN) {
    const int64_t p = p_base + pt0 + i / d;
    sxd[i] = p < P ? xs[p * d + i % d] : 0.0;
  }
  __syncthreads();
  double s2[PF_TP];
#pragma unroll
  for (int q = 0; q < PF_TP; ++q) s2[q] = 0.0;
  for (int j = 0; j < d; ++j) {
    const double x = XtT[(int64_t)j * Npad + n];
#pragma unroll
    for (int q = 0; q < PF_TP; ++q) {
      const double u = sxd[q * d + j] - x;
      s2[q] = fma(u, u, s2[q]);
    }
  }
  double a[MT_MAX];
#pragma unroll
  for (int j = 0; j < MT_MAX; ++j) a[j] = j < M ? A[(int64_t)j * Npad + n] : 0.0;
  const bool live = n < N;
#pragma unroll
  for (int q = 0; q < PF_TP; ++q) {
    const double K = sqrt(s2[q]) * 2.23606797749978969641;  // sqrt(5) r
    const double k = live ? (1.0 + K + K * K / 3.0) * exp(-K) : 0.0;
    if (Ks) Ks[(pt0 + q) * Npad + n] = k;
#pragma unroll
    for (int j = 0; j < MT_MAX; ++j)
      if (j < M) {
        const double s = warp_sum(k * a[j]);
        if (lane == 0) red[warp][q][j] = s;
      }
  }
  __syncthreads();
  for (int i = t; i < PF_TP * M; i += PF_TN) {
    const int q = i / M, j = i - q * M;
    mpart[((int64_t)blockIdx.x * M + j) * mp_ld + pt0 + q] = (red[0][q][j] + red[1][q][j]) + (red[2][q][j] + red[3][q][j]);
  }
}

// ---- tensor producer: one fp16 hi / lo K_* plane and the block-mean partial sums -----------------------------------
// The layout of kstar_tensor_kernel (gp_tensor.cu): a thread owns two adjacent training points (coordinates in
// registers, results leave as packed half2), a block covers 256 training points x 32 candidates, the candidate tile is
// read from shared memory as 16-byte broadcasts.  Kernel values in fp32 (sqrt.approx / ex2.approx, ~2^-22 relative,
// inside the 22-bit budget of the hi + lo split), scaled by 2^kexp so that both halves stay normal; the block means use
// the unscaled fp32 values times float64 a_j, reduced in float64 in a fixed order.  4 bytes per (candidate, training
// point) are written, whatever M.
constexpr int PT_TN = 128, PT_TP = 32;

// flushes denormal results to zero, unlike gp_tensor.cu's stationary_f (see there); the two are not interchangeable
__device__ __forceinline__ float matern52_f(float s2) {
  float r, e;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s2));
  const float K = r * 2.2360679774997896f;
  const float t = K * -1.4426950408889634f;  // exp(-K) = 2^(-K log2 e)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  return fmaf(K, fmaf(K, 1.0f / 3.0f, 1.0f), 1.0f) * e;
}

template <int DMAX>
__global__ void __launch_bounds__(PT_TN, DMAX <= 32 ? 3 : 2)
    mt_kstar_tensor_kernel(const double* __restrict__ xs, int64_t P, int64_t p_base, const double* __restrict__ XtT,
                           int64_t N, int64_t Npad, int d, int M, const double* __restrict__ A, const int* __restrict__ k_exp,
                           uint16_t* __restrict__ Kh, uint16_t* __restrict__ Kl, double* __restrict__ mpart, int64_t mp_ld) {
  __shared__ __align__(16) float sx[PT_TP * DMAX];
  __shared__ double red[PT_TN / 32][PT_TP][MT_MAX];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t n0 = ((int64_t)blockIdx.x * PT_TN + t) * 2;
  const int64_t pt0 = (int64_t)blockIdx.y * PT_TP;
  for (int i = t; i < PT_TP * DMAX; i += PT_TN) {
    const int64_t p = p_base + pt0 + i / DMAX;
    const int j = i % DMAX;
    sx[i] = (p < P && j < d) ? (float)xs[p * d + j] : 0.f;
  }
  float xa[DMAX], xb[DMAX];
#pragma unroll
  for (int j = 0; j < DMAX; ++j) {
    xa[j] = j < d ? (float)XtT[(int64_t)j * Npad + n0] : 0.f;
    xb[j] = j < d ? (float)XtT[(int64_t)j * Npad + n0 + 1] : 0.f;
  }
  double aa[MT_MAX], ab[MT_MAX];
#pragma unroll
  for (int j = 0; j < MT_MAX; ++j) {
    aa[j] = j < M ? A[(int64_t)j * Npad + n0] : 0.0;
    ab[j] = j < M ? A[(int64_t)j * Npad + n0 + 1] : 0.0;
  }
  const float scale = Kh ? scalbnf(1.0f, k_exp[0]) : 1.0f;  // mean-only predicts write no K_*
  const bool live_a = n0 < N, live_b = n0 + 1 < N;
  uint32_t* Kh32 = reinterpret_cast<uint32_t*>(Kh);
  uint32_t* Kl32 = reinterpret_cast<uint32_t*>(Kl);
  __syncthreads();
  for (int q = 0; q < PT_TP; ++q) {
    const float4* xc = reinterpret_cast<const float4*>(sx + q * DMAX);
    float sa0 = 0.f, sa1 = 0.f, sb0 = 0.f, sb1 = 0.f;  // independent chains
#pragma unroll
    for (int j = 0; j < DMAX / 4; ++j) {
      const float4 c = xc[j];
      float u;
      u = c.x - xa[4 * j];
      sa0 = fmaf(u, u, sa0);
      u = c.y - xa[4 * j + 1];
      sa1 = fmaf(u, u, sa1);
      u = c.z - xa[4 * j + 2];
      sa0 = fmaf(u, u, sa0);
      u = c.w - xa[4 * j + 3];
      sa1 = fmaf(u, u, sa1);
      u = c.x - xb[4 * j];
      sb0 = fmaf(u, u, sb0);
      u = c.y - xb[4 * j + 1];
      sb1 = fmaf(u, u, sb1);
      u = c.z - xb[4 * j + 2];
      sb0 = fmaf(u, u, sb0);
      u = c.w - xb[4 * j + 3];
      sb1 = fmaf(u, u, sb1);
    }
    const float ka = live_a ? matern52_f(sa0 + sa1) : 0.f;
    const float kb = live_b ? matern52_f(sb0 + sb1) : 0.f;
    if (Kh) {
      const float va = ka * scale, vb = kb * scale;  // power-of-two scaling: exact
      const __half2 h = __floats2half2_rn(va, vb);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(va - hf.x, vb - hf.y);
      const int64_t o = ((pt0 + q) * Npad + n0) >> 1;
      Kh32[o] = *reinterpret_cast<const uint32_t*>(&h);
      Kl32[o] = *reinterpret_cast<const uint32_t*>(&l);
    }
#pragma unroll
    for (int j = 0; j < MT_MAX; ++j)
      if (j < M) {
        const double s = warp_sum(fma((double)ka, aa[j], (double)kb * ab[j]));
        if (lane == 0) red[warp][q][j] = s;
      }
  }
  __syncthreads();
  for (int i = t; i < PT_TP * M; i += PT_TN) {
    const int q = i / M, j = i - q * M;
    mpart[((int64_t)blockIdx.x * M + j) * mp_ld + pt0 + q] = (red[0][q][j] + red[1][q][j]) + (red[2][q][j] + red[3][q][j]);
  }
}

// ---- mixing epilogue: blocks -> tasks ------------------------------------------------------------------------------
// One thread per candidate: the block means and variance partial sums are added plane by plane in a fixed order (as
// var_finish_tc_kernel does), then per task mean_t = m_t + sum_j c_tj km_j, var_t = max(0, prior_t - sum_j c_tj^2 vn_j),
// un-normalised with y_std / y_mean (model_gpytorch.py:1915-1916).
__global__ void mt_mix_kernel(const double* __restrict__ xs, int64_t Pc, int d, int M, const double* __restrict__ mpart,
                              int n_mp, int64_t mp_ld, const double* __restrict__ vnorm, int n_vp, int64_t vn_ld,
                              const double* __restrict__ mix, const double* __restrict__ prior, const double* __restrict__ w,
                              const double* __restrict__ b, const double* __restrict__ ymean, const double* __restrict__ ystd,
                              int64_t p_base, double* __restrict__ mean, double* __restrict__ var) {
  const int64_t pl = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pl >= Pc) return;
  const int64_t p = p_base + pl;
  double km[MT_MAX], vn[MT_MAX];
#pragma unroll
  for (int j = 0; j < MT_MAX; ++j) {
    double s = 0.0, v = 0.0;
    if (j < M) {
      for (int z = 0; z < n_mp; ++z) s += mpart[((int64_t)z * M + j) * mp_ld + pl];
      if (var)
        for (int z = 0; z < n_vp; ++z) v += vnorm[((int64_t)z * M + j) * vn_ld + pl];
    }
    km[j] = s;
    vn[j] = v;
  }
  const double* x = xs + p * d;
  for (int t = 0; t < M; ++t) {
    double mu = b[t];
    for (int k = 0; k < d; ++k) mu = fma(w[(int64_t)t * d + k], x[k], mu);
    double red = 0.0;
#pragma unroll
    for (int j = 0; j < MT_MAX; ++j)
      if (j < M) {
        const double c = mix[t * M + j];
        mu = fma(c, km[j], mu);
        red = fma(c * c, vn[j], red);
      }
    mean[p * M + t] = ystd[t] * mu + ymean[t];
    if (var) {
      double v = prior[t] - red;
      if (v < 0.0) v = 0.0;
      var[p * M + t] = v * (ystd[t] * ystd[t]);
    }
  }
}

// ---- host: symmetric eigendecomposition A = Q diag(lam) Q' (cyclic Jacobi, fixed sweep order) ----------------------
void jacobi_eigh(int M, std::vector<double> A, std::vector<double>& lam, std::vector<double>& Q) {
  Q.assign((size_t)M * M, 0.0);
  for (int i = 0; i < M; ++i) Q[(size_t)i * M + i] = 1.0;
  double total = 0.0;
  for (double v : A) total += v * v;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < M; ++i)
      for (int j = i + 1; j < M; ++j) off += A[(size_t)i * M + j] * A[(size_t)i * M + j];
    if (!(off > 1e-36 * total)) break;
    for (int p = 0; p < M; ++p)
      for (int q = p + 1; q < M; ++q) {
        const double apq = A[(size_t)p * M + q];
        if (apq == 0.0) continue;
        // rotation that zeroes A[p][q] (Golub & Van Loan, Alg. 8.5.1)
        const double theta = (A[(size_t)q * M + q] - A[(size_t)p * M + p]) / (2.0 * apq);
        const double tn = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(tn * tn + 1.0), s = tn * c;
        for (int k = 0; k < M; ++k) {  // columns: A J
          const double akp = A[(size_t)k * M + p], akq = A[(size_t)k * M + q];
          A[(size_t)k * M + p] = c * akp - s * akq;
          A[(size_t)k * M + q] = s * akp + c * akq;
        }
        for (int k = 0; k < M; ++k) {  // rows: J' (A J)
          const double apk = A[(size_t)p * M + k], aqk = A[(size_t)q * M + k];
          A[(size_t)p * M + k] = c * apk - s * aqk;
          A[(size_t)q * M + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < M; ++k) {  // Q J
          const double qkp = Q[(size_t)k * M + p], qkq = Q[(size_t)k * M + q];
          Q[(size_t)k * M + p] = c * qkp - s * qkq;
          Q[(size_t)k * M + q] = s * qkp + c * qkq;
        }
      }
  }
  lam.resize(M);
  for (int i = 0; i < M; ++i) lam[i] = A[(size_t)i * M + i];
}

}  // namespace

int mt_scale_inputs(dmo_ctx* ctx, const double* X, int64_t P, int d, const double* xlb, const double* xrg, const double* inv_ls,
                    double* xs) {
  DMO_LAUNCH(mt_scale_inputs_kernel, (unsigned)ceil_div(P * d, 256), 256, 0, X, P, d, xlb, xrg, inv_ls, xs);
  return DMO_OK;
}

int64_t mt_kstar_span(bool tensor) { return tensor ? 2 * PT_TN : PF_TN; }

int mt_kstar_produce(dmo_ctx* ctx, bool tensor, const double* xs, int64_t P, int64_t p_base, int64_t Pcpad, const double* XtT, int64_t N,
                     int64_t Npad, int d, int M, const double* A, const int* k_exp, double* Ks, uint16_t* Kh, uint16_t* Kl,
                     double* mpart, int64_t mp_ld) {
  const unsigned n_mp = (unsigned)(Npad / mt_kstar_span(tensor));
  if (tensor) {
    dim3 g(n_mp, (unsigned)(Pcpad / PT_TP));
    if (d <= 32)
      DMO_LAUNCH(mt_kstar_tensor_kernel<32>, g, PT_TN, 0, xs, P, p_base, XtT, N, Npad, d, M, A, k_exp, Kh, Kl, mpart, mp_ld);
    else
      DMO_LAUNCH(mt_kstar_tensor_kernel<64>, g, PT_TN, 0, xs, P, p_base, XtT, N, Npad, d, M, A, k_exp, Kh, Kl, mpart, mp_ld);
  } else {
    dim3 g(n_mp, (unsigned)(Pcpad / PF_TP));
    DMO_LAUNCH(mt_kstar_f64_kernel, g, PF_TN, (size_t)PF_TP * d * sizeof(double), xs, P, p_base, XtT, N, Npad, d, M, A, Ks, mpart,
               mp_ld);
  }
  return DMO_OK;
}

int GpUnitPredict::check(dmo_ctx* ctx, const char* who_, int precision, int d) {
  who = who_;
  DMO_REQUIRE(precision == DMO_GP_FP64 || precision == DMO_GP_TENSOR, "%s: precision must be DMO_GP_FP64 or DMO_GP_TENSOR (got %d)",
              who, precision);
  tensor = precision == DMO_GP_TENSOR;
  DMO_REQUIRE(!tensor || d <= 64, "%s(tensor): at most 64 input dimensions (got %d); use DMO_GP_FP64", who, d);
  return DMO_OK;
}

int GpUnitPredict::alloc(dmo_ctx* ctx, int64_t P, int64_t Npad, int planes, bool want_var) {
  // candidate chunk: the one K_* plane (fp16 hi + lo, or float64) within ~6 GiB; the producer grid's y extent stays < 2^16
  tile = tensor ? GP_TC_TILE : GP_F64_TILE;
  int64_t Pc_max = ((int64_t)6 << 30) / (Npad * (tensor ? 4 : 8));
  if (Pc_max > GP_MAX_CHUNK) Pc_max = GP_MAX_CHUNK;
  Pc_max = (Pc_max / tile) * tile;
  if (Pc_max < tile) Pc_max = tile;
  Pc_alloc = P < Pc_max ? ceil_div(P, tile) * tile : Pc_max;
  if (!want_var) return DMO_OK;
  if (tensor) {
    n_vp = gp_tensor_var_planes(Npad);
  } else {  // the row blocks of the planes are split so that at least ~2 CTAs per SM exist for small candidate sets
    int64_t nsplit = ceil_div((int64_t)2 * ctx->sm_count, (Pc_alloc / GP_F64_TILE) * planes);
    const int64_t ntile = Npad / GP_F64_TILE;
    n_vp = (int)(nsplit > ntile ? ntile : (nsplit < 1 ? 1 : nsplit));
  }
  DMO_TRY(vnorm.alloc(ctx, (size_t)n_vp * planes * Pc_alloc));
  if (tensor) {
    DMO_TRY(Kh.alloc(ctx, (size_t)Pc_alloc * Npad));
    DMO_TRY(Kl.alloc(ctx, (size_t)Pc_alloc * Npad));
    DMO_TRY(abort_flag.alloc(ctx, 1));
    DMO_CUDA(cudaMemsetAsync(abort_flag.p, 0, sizeof(int), ctx->stream));
  } else {
    DMO_TRY(Ks.alloc(ctx, (size_t)Pc_alloc * Npad));
  }
  return DMO_OK;
}

int GpUnitPredict::contract(dmo_ctx* ctx, const GpVarOps& ops, int64_t Pcpad) {
  if (tensor) return gp_var_contract_tensor(ctx, ops, Kh.p, Kl.p, Pc_alloc, 0, Pcpad, vnorm.p, Pc_alloc, abort_flag.p);
  return gp_var_contract_fp64(ctx, ops, Ks.p, 0, Pcpad, n_vp, vnorm.p, Pc_alloc);
}

int GpUnitPredict::watchdog(dmo_ctx* ctx) {
  if (!abort_flag.p) return DMO_OK;  // no tensor-core contraction ran
  int h_abort = 0;
  DMO_CUDA(cudaMemcpyAsync(&h_abort, abort_flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (h_abort) return dmo_fail(ctx, DMO_ERR_INTERNAL, "%s(tensor): pipeline watchdog tripped", who);
  return DMO_OK;
}

int mtgp_blocks_fit(dmo_ctx* ctx, const char* who, int64_t N, int d, int M, const double* X_train, const double* Y,
                    const double* length_scale, const double* B, const double* D, const double* weight, const double* bias,
                    MtBlocks& mb, double* alpha_out) {
  DMO_REQUIRE(N >= 1 && d >= 1 && d <= MT_FIT_DMAX && M >= 1 && M <= MT_MAX,
              "%s: unsupported shape N=%lld d=%d M=%d (1 <= M <= %d, d <= %d)", who, (long long)N, d, M, MT_MAX, MT_FIT_DMAX);
  DMO_REQUIRE(X_train && Y && length_scale && B && D && weight && bias, "%s: null pointer", who);
  const size_t nd = (size_t)N * d, nm = (size_t)N * M, mm = (size_t)M * M;
  std::vector<double>& hx = mb.hx;
  std::vector<double>& ls = mb.ls;
  std::vector<double>& hB = mb.hB;
  std::vector<double>& hD = mb.hD;
  std::vector<double>& hw = mb.hw;
  std::vector<double>& hb = mb.hb;
  std::vector<double> hy(nm);
  hx.resize(nd);
  ls.resize(d);
  hB.resize(mm);
  hD.resize(M);
  hw.resize((size_t)M * d);
  hb.resize(M);
  DMO_CUDA(cudaMemcpy(hx.data(), X_train, nd * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hy.data(), Y, nm * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ls.data(), length_scale, d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hB.data(), B, mm * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hD.data(), D, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hw.data(), weight, (size_t)M * d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hb.data(), bias, M * sizeof(double), cudaMemcpyDefault));
  for (int j = 0; j < d; ++j) DMO_REQUIRE(ls[j] > 0.0, "%s: length scale %d must be > 0", who, j);
  double bmax = 0.0;
  for (double v : hB) bmax = fmax(bmax, fabs(v));
  for (int s = 0; s < M; ++s) {
    DMO_REQUIRE(hD[s] > 0.0, "%s: noise D[%d] = %g must be > 0", who, s, hD[s]);
    for (int t = 0; t < M; ++t)
      DMO_REQUIRE(fabs(hB[(size_t)s * M + t] - hB[(size_t)t * M + s]) <= 1e-12 * bmax, "%s: B is not symmetric", who);
  }
  // whitened task covariance D^-1/2 B D^-1/2 = Q diag(lam) Q'
  std::vector<double>& sqD = mb.sqD;
  std::vector<double>& lam = mb.lam;
  std::vector<double>& Q = mb.Q;
  std::vector<double> Bt(mm);
  sqD.resize(M);
  for (int s = 0; s < M; ++s) sqD[s] = sqrt(hD[s]);
  for (int s = 0; s < M; ++s)
    for (int t = 0; t < M; ++t)
      Bt[(size_t)s * M + t] = 0.5 * (hB[(size_t)s * M + t] + hB[(size_t)t * M + s]) / (sqD[s] * sqD[t]);
  jacobi_eigh(M, Bt, lam, Q);
  double lmax = 0.0;
  for (int j = 0; j < M; ++j) lmax = fmax(lmax, lam[j]);
  for (int j = 0; j < M; ++j) {
    DMO_REQUIRE(lam[j] >= -1e-12 * lmax, "%s: B is not positive semi-definite (eigenvalue %g)", who, lam[j]);
    if (lam[j] < 0.0) lam[j] = 0.0;
  }
  // rotated residuals r_j = sum_s Q_sj (y_s - w_s . x - b_s) / sqrt(D_s), (M, N)
  std::vector<double>& xs = mb.xs;
  std::vector<double> rhat(nm, 0.0), res(M);
  xs.resize(nd);
  for (int64_t n = 0; n < N; ++n) {
    for (int s = 0; s < M; ++s) {
      double m = hb[s];
      for (int k = 0; k < d; ++k) m += hw[(size_t)s * d + k] * hx[(size_t)n * d + k];
      res[s] = (hy[(size_t)n * M + s] - m) / sqD[s];
    }
    for (int j = 0; j < M; ++j) {
      double r = 0.0;
      for (int s = 0; s < M; ++s) r += Q[(size_t)s * M + j] * res[s];
      rhat[(size_t)j * N + n] = r;
    }
    for (int k = 0; k < d; ++k) xs[(size_t)n * d + k] = hx[(size_t)n * d + k] / ls[k];
  }
  // the M blocks: lambda_j K_x + I over the scaled inputs (unit length scale), factorised in float64
  std::vector<double> ones_d((size_t)M * d, 1.0), ones_m(M, 1.0);
  mb.blk_lml.assign(M, 0.0);
  DMO_TRY(mb.Lf.alloc(ctx, (size_t)M * N * N));
  DMO_TRY(dmo_gp_fit(ctx, N, d, M, DMO_KERNEL_MATERN52, xs.data(), rhat.data(), lam.data(), ones_d.data(), ones_m.data(), 0.0,
                     mb.Lf.p, alpha_out, mb.blk_lml.data()));
  double lml = 0.0;
  for (int j = 0; j < M; ++j) lml += mb.blk_lml[j];
  for (int t = 0; t < M; ++t) lml -= 0.5 * (double)N * log(hD[t]);
  mb.lml = lml;
  return DMO_OK;
}

extern "C" {

int dmo_mtgp_create(dmo_ctx* ctx, int64_t N, int d, int M, const double* X_train, const double* Y, const double* length_scale,
                    const double* B, const double* D, const double* weight, const double* bias, const double* y_mean,
                    const double* y_std, const double* xlb, const double* xub, double* lml_out, dmo_mtgp** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out, "mtgp_create: null output");
  *out = nullptr;
  DMO_REQUIRE(N >= 1 && d >= 1 && d <= MT_FIT_DMAX && M >= 1 && M <= MT_MAX,
              "mtgp_create: unsupported shape N=%lld d=%d M=%d (1 <= M <= %d, d <= %d)", (long long)N, d, M, MT_MAX, MT_FIT_DMAX);
  DMO_REQUIRE(y_mean && y_std && xlb && xub, "mtgp_create: null pointer");
  const size_t nm = (size_t)N * M, mm = (size_t)M * M;
  std::vector<double> ym(M), ys(M), lb(d), ub(d);
  DMO_CUDA(cudaMemcpy(ym.data(), y_mean, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ys.data(), y_std, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(lb.data(), xlb, d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ub.data(), xub, d * sizeof(double), cudaMemcpyDefault));
  for (int j = 0; j < d; ++j) DMO_REQUIRE(ub[j] != lb[j], "mtgp_create: the input range %d must be non-empty", j);
  MtBlocks mb;
  DevBuf<double> alpha;
  DMO_TRY(alpha.alloc(ctx, nm));
  DMO_TRY(mtgp_blocks_fit(ctx, "mtgp_create", N, d, M, X_train, Y, length_scale, B, D, weight, bias, mb, alpha.p));
  const std::vector<double>&ls = mb.ls, &hB = mb.hB, &hD = mb.hD, &hw = mb.hw, &hb = mb.hb, &sqD = mb.sqD, &lam = mb.lam,
                     &Q = mb.Q, &xs = mb.xs;
  DevBuf<double>& Lf = mb.Lf;
  std::unique_ptr<dmo_mtgp> mt(new dmo_mtgp());
  mt->N = N;
  mt->d = d;
  mt->M = M;
  mt->lml = mb.lml;
  const double lml = mb.lml;
  DMO_TRY(mt->blk.alloc(ctx, N, M));  // the blocks share K_* (unit scale) but not L_j^-1: one plane each
  const int64_t Npad = mt->blk.Npad;
  for (int j = 0; j < M; ++j)
    DMO_TRY(gp_linv_from_factor(ctx, Lf.p + (size_t)j * N * N, N, Npad, mt->blk.Linv.p + (size_t)j * Npad * Npad));
  DMO_TRY(mt->A.alloc(ctx, (size_t)M * Npad));
  DMO_CUDA(cudaMemsetAsync(mt->A.p, 0, (size_t)M * Npad * sizeof(double), ctx->stream));
  DMO_CUDA(cudaMemcpy2DAsync(mt->A.p, Npad * sizeof(double), alpha.p, N * sizeof(double), N * sizeof(double), M,
                             cudaMemcpyDeviceToDevice, ctx->stream));
  // small state
  const std::vector<double> xtT = mt_xt_transposed(N, d, Npad, [&](int64_t n, int k) { return xs[(size_t)n * d + k]; });
  std::vector<double> inv(d), rg(d), mix(mm), prior(M), ws((size_t)M * d);
  for (int k = 0; k < d; ++k) {
    inv[k] = 1.0 / ls[k];
    rg[k] = ub[k] - lb[k];
  }
  for (int t = 0; t < M; ++t) {
    for (int j = 0; j < M; ++j) mix[(size_t)t * M + j] = lam[j] * Q[(size_t)t * M + j] * sqD[t];
    prior[t] = hB[(size_t)t * M + t] + hD[t];
    for (int k = 0; k < d; ++k) ws[(size_t)t * d + k] = hw[(size_t)t * d + k] * ls[k];
  }
  DMO_TRY(upload(ctx, mt->XtT, xtT));
  DMO_TRY(upload(ctx, mt->inv_ls, inv));
  DMO_TRY(upload(ctx, mt->xlb, lb));
  DMO_TRY(upload(ctx, mt->xrg, rg));
  DMO_TRY(upload(ctx, mt->mix, mix));
  DMO_TRY(upload(ctx, mt->prior, prior));
  DMO_TRY(upload(ctx, mt->w, ws));
  DMO_TRY(upload(ctx, mt->b, hb));
  DMO_TRY(upload(ctx, mt->ymean, ym));
  DMO_TRY(upload(ctx, mt->ystd, ys));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));  // host vectors above are staged from the stack
  if (lml_out) DMO_CUDA(cudaMemcpy(lml_out, &lml, sizeof(double), cudaMemcpyDefault));
  *out = mt.release();
  return DMO_OK;
}

int dmo_mtgp_destroy(dmo_ctx* ctx, dmo_mtgp* mt) {
  if (!ctx) return DMO_ERR_ARG;
  if (!mt) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  delete mt;
  return DMO_OK;
}

int dmo_mtgp_predict(dmo_ctx* ctx, dmo_mtgp* mt, const double* X, int64_t P, double* mean, double* var, int precision) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(mt, "mtgp_predict: null model");
  const int M = mt->M, d = mt->d;
  const int64_t N = mt->N, Npad = mt->blk.Npad;
  GpUnitPredict up;
  DMO_TRY(up.check(ctx, "mtgp_predict", precision, d));
  const bool tensor = up.tensor;
  if (P == 0) return DMO_OK;
  DMO_REQUIRE(P > 0 && X && mean, "mtgp_predict: bad arguments");
  In<double> x;
  Out<double> om, ov;
  DMO_TRY(x.init(ctx, X, (size_t)P * d));
  DMO_TRY(om.init(ctx, mean, (size_t)P * M));
  DMO_TRY(ov.init(ctx, var, (size_t)P * M));
  const bool want_var = ov.d != nullptr;
  DevBuf<double> xs;
  DMO_TRY(xs.alloc(ctx, (size_t)P * d));
  DMO_TRY(mt_scale_inputs(ctx, x.d, P, d, mt->xlb.p, mt->xrg.p, mt->inv_ls.p, xs.p));
  if (tensor && want_var) DMO_TRY(gp_prepare_tensor(ctx, mt->blk));
  DMO_TRY(up.alloc(ctx, P, Npad, M, want_var));
  const int64_t Pc_alloc = up.Pc_alloc;
  const int n_mp = (int)(Npad / mt_kstar_span(tensor));
  DevBuf<double> mpart;
  DMO_TRY(mpart.alloc(ctx, (size_t)n_mp * M * Pc_alloc));
  for (int64_t p_base = 0; p_base < P; p_base += Pc_alloc) {
    const int64_t Pc = (P - p_base) < Pc_alloc ? (P - p_base) : Pc_alloc;
    const int64_t Pcpad = ceil_div(Pc, up.tile) * up.tile;
    {
      ProfileScope ps(ctx, "mtgp_kstar");
      DMO_TRY(mt_kstar_produce(ctx, tensor, xs.p, P, p_base, Pcpad, mt->XtT.p, N, Npad, d, M, mt->A.p,
                               tensor && want_var ? mt->blk.Kexp.p : nullptr, up.Ks.p, up.Kh.p, up.Kl.p, mpart.p, Pc_alloc));
    }
    if (want_var) {
      ProfileScope ps(ctx, "mtgp_var");
      DMO_TRY(up.contract(ctx, mt->blk, Pcpad));
    }
    {
      ProfileScope ps(ctx, "mtgp_mix");
      DMO_LAUNCH(mt_mix_kernel, (unsigned)ceil_div(Pc, 256), 256, 0, xs.p, Pc, d, M, mpart.p, n_mp, Pc_alloc, up.vnorm.p, up.n_vp,
                 Pc_alloc, mt->mix.p, mt->prior.p, mt->w.p, mt->b.p, mt->ymean.p, mt->ystd.p, p_base, om.d, ov.d);
    }
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(up.watchdog(ctx));
  DMO_TRY(om.finish(ctx));
  DMO_TRY(ov.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
