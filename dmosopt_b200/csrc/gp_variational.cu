// Variational GP posterior: the predict_f of GPflow's whitened SVGP / VGP with a Gaussian likelihood and an ARD
// Matern-5/2 kernel, behind dmosopt's SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern and CRV_Matern (dmosopt/model.py
// :290-318, 509-537, 730-757, 953-981, 1143-1172), and the closed-form optimum of q for fixed kernel hyper-parameters.
//
// Latent GP l has inducing points Z_l, kernel s_l k(x / ell_l, x' / ell_l), Lz = chol(K(Z, Z) + jitter I) and the
// whitened q(v) = N(q_mu, S), S = q_sqrt q_sqrt'.  With K_* = K(Z, x_*) = s_l k_u (k_u the unit-scale kernel values):
//     mean_l = K_*' Lz^-T q_mu = k_u' a_l,                           a_l = s_l Lz^-T q_mu
//     var_l  = s_l - ||Lz^-1 K_*||^2 + ||q_sqrt' Lz^-1 K_*||^2 = s_l - ||O0 k_u||^2 + ||O1 k_u||^2
// with O0 = s_l Lz^-1 and O1 = s_l T, T lower triangular with T'T = V'V, V = q_sqrt' Lz^-1 (dense).  T comes from a
// Householder QR of V J (J reverses the column order): V J = Q R gives V'V = J R'R J = (J R J)'(J R J), and J R J is lower
// triangular because R is upper triangular.  The QR exists for every q_sqrt, a singular S included.  So both variance terms
// are the column sums of squares of a lower-triangular operator applied to one K_* plane -- what the single-output
// contractions (var_kernel, gp_var_wgmma_kernel) compute -- and the predict needs no kernel of its own for them.
//
// Latents whose Z plane and length scales are bitwise equal share k_u (SIV, SPV with equal kernels, VGP, SVGP when Z is
// every training point): such a "K_* group" gets one producer pass (the multitask producer of gp_multitask.cu: one unit
// K_* plane plus the group's mean partial sums) and one contraction over its operator planes; latents of a group that also
// share s_l share O0 (SIV: one kernel for every output).  sv_gather_kernel forms each latent's mean and s_l - v0 + v1
// (gpflow does not clamp the variance, and neither path here does), sv_mix_kernel mixes the latents into outputs
// (mean = W g_mean, var = (W o W) g_var; W = I except for CRV) and un-normalises.
#include <math.h>
#include <string.h>

#include <memory>
#include <vector>

#include "gp.cuh"

namespace {

constexpr int SV_MAX = 8;        // latents and outputs per model
constexpr int64_t SV_ZMAX = 8192;  // inducing points per latent

// C[i][j] = alpha sum_k A(i, k) B(k, j) + (i == j ? diag : 0), i < m, j < n (rows of ldc), with A(i, k) = A[i sai + k sak]
// and B(k, j) = B[k sbk + j sbj] (any strides, negative ones included).  64 x 64 tiles, 4 x 4 per thread, k steps of 16;
// every output is one fixed-order chain.  Set-up work only (operators, the optimum of q), not the predict.
constexpr int GT = 64, GK = 16;
__global__ void __launch_bounds__(256)
    sv_gemm_kernel(int64_t m, int64_t n, int64_t K, double alpha, const double* __restrict__ A, int64_t sai, int64_t sak,
                   const double* __restrict__ B, int64_t sbk, int64_t sbj, double diag, double* __restrict__ C, int64_t ldc) {
  __shared__ double As[GK][GT + 1], Bs[GK][GT + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t i0 = (int64_t)blockIdx.y * GT, j0 = (int64_t)blockIdx.x * GT;
  double acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
  for (int64_t k0 = 0; k0 < K; k0 += GK) {
    for (int t = tid; t < GK * GT; t += 256) {
      const int kk = t / GT, r = t - kk * GT;
      const int64_t k = k0 + kk, i = i0 + r, j = j0 + r;
      As[kk][r] = (k < K && i < m) ? A[i * sai + k * sak] : 0.0;
      Bs[kk][r] = (k < K && j < n) ? B[k * sbk + j * sbj] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      double a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a[u] = As[kk][ty + 16 * u];
        b[u] = Bs[kk][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int64_t i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
      if (i < m && j < n) C[i * ldc + j] = alpha * acc[u][v] + (i == j ? diag : 0.0);
    }
}

// a shared-memory tree, not common.cuh's block_sum: the QR's results keep the bits of this order
__device__ double block_sum_256(double s, double* red) {
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  return red[0];
}

// ---- Householder QR of an n x n matrix C stored by columns (column c = C + c n), LAPACK's dlarfg / dlarf ---------------
// step j: the reflector H = I - tau v v' (v_j = 1) that zeroes C[j][j+1 ..); R_jj and v_{>j} overwrite column j
__global__ void __launch_bounds__(256) sv_house_kernel(double* __restrict__ C, int64_t n, int64_t j, double* __restrict__ tau) {
  __shared__ double red[256];
  double* x = C + j * n;
  const double a = x[j];  // read before the barrier: thread 0 overwrites it below
  double s = 0.0;
  for (int64_t i = j + 1 + threadIdx.x; i < n; i += 256) s = fma(x[i], x[i], s);
  const double sigma = block_sum_256(s, red);
  if (sigma == 0.0) {  // already upper triangular in this column: H = I
    if (threadIdx.x == 0) *tau = 0.0;
    return;
  }
  const double nrm = sqrt(fma(a, a, sigma));
  const double beta = a >= 0.0 ? -nrm : nrm;
  const double inv = 1.0 / (a - beta);
  for (int64_t i = j + 1 + threadIdx.x; i < n; i += 256) x[i] *= inv;
  if (threadIdx.x == 0) {
    x[j] = beta;
    *tau = (beta - a) / beta;
  }
}

// H applied to the trailing columns j + 1 + blockIdx.x
__global__ void __launch_bounds__(256) sv_house_apply_kernel(double* __restrict__ C, int64_t n, int64_t j, const double* __restrict__ tau) {
  __shared__ double red[256];
  const double t = *tau;
  if (t == 0.0) return;
  const double* v = C + j * n;
  double* y = C + (j + 1 + blockIdx.x) * n;
  double s = threadIdx.x == 0 ? y[j] : 0.0;
  for (int64_t i = j + 1 + threadIdx.x; i < n; i += 256) s = fma(v[i], y[i], s);
  const double w = t * block_sum_256(s, red);
  if (threadIdx.x == 0) y[j] -= w;
  for (int64_t i = j + 1 + threadIdx.x; i < n; i += 256) y[i] = fma(-w, v[i], y[i]);
}

// O[a][b] = s C[(n-1-b) n + (n-1-a)] for b <= a, else 0 (rows of ldo): with C the QR above, s J R J; with C a row-major
// lower-triangular matrix X, s J X' J.  Both are lower triangular.
__global__ void sv_flip_kernel(const double* __restrict__ C, int64_t n, double s, double* __restrict__ O, int64_t ldo) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * n) return;
  const int64_t a = t / n, b = t - a * n;
  O[a * ldo + b] = b <= a ? s * C[(n - 1 - b) * n + (n - 1 - a)] : 0.0;
}

__global__ void sv_scale_kernel(double* __restrict__ x, int64_t n, double s) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) x[t] *= s;
}

// A[a][b] = B[n-1-a][n-1-b] (rows of ld; the lower triangle is what the Cholesky reads), identity beyond n
__global__ void sv_reverse_pad_kernel(const double* __restrict__ B, int64_t n, int64_t ld, double* __restrict__ A) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ld * ld) return;
  const int64_t a = t / ld, b = t - a * ld;
  A[t] = (a < n && b < n) ? B[(n - 1 - a) * n + (n - 1 - b)] : (a == b ? 1.0 : 0.0);
}

// ---- predict epilogues ---------------------------------------------------------------------------------------------
struct SvGather {
  int nlat, n_o0, G;
  int lat[SV_MAX], o0[SV_MAX];
  double s[SV_MAX];
};

// latent means and variances of one K_* group: partial sums added plane by plane in a fixed order
__global__ void sv_gather_kernel(SvGather g, int64_t Pc, int64_t p_base, int64_t P, const double* __restrict__ mpart, int n_mp,
                                 int64_t mp_ld, const double* __restrict__ vnorm, int n_vp, int64_t vn_ld, double* __restrict__ fm,
                                 double* __restrict__ fv) {
  const int64_t pl = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pl >= Pc) return;
  const int64_t p = p_base + pl;
  for (int j = 0; j < g.nlat; ++j) {
    double s = 0.0;
    for (int z = 0; z < n_mp; ++z) s += mpart[((int64_t)z * g.nlat + j) * mp_ld + pl];
    fm[(int64_t)g.lat[j] * P + p] = s;
    if (fv) {
      double v0 = 0.0, v1 = 0.0;
      for (int z = 0; z < n_vp; ++z) {
        v0 += vnorm[((int64_t)z * g.G + g.o0[j]) * vn_ld + pl];
        v1 += vnorm[((int64_t)z * g.G + g.n_o0 + j) * vn_ld + pl];
      }
      fv[(int64_t)g.lat[j] * P + p] = (g.s[j] - v0) + v1;  // gpflow: Kss - sum(A^2), then + sum((L' A)^2); no clamp
    }
  }
}

// outputs: mean = y_std (W g_mean) + y_mean, var = ((W o W) g_var) y_var_scale
__global__ void sv_mix_kernel(int64_t P, int L, int M, const double* __restrict__ fm, const double* __restrict__ fv,
                              const double* __restrict__ W, const double* __restrict__ ymean, const double* __restrict__ ystd,
                              const double* __restrict__ vscale, double* __restrict__ mean, double* __restrict__ var) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P * M) return;
  const int64_t p = t / M;
  const int m = (int)(t - p * M);
  double mu = 0.0, v = 0.0;
  for (int l = 0; l < L; ++l) {
    const double w = W[m * L + l];
    mu = fma(w, fm[(int64_t)l * P + p], mu);
    if (var) v = fma(w * w, fv[(int64_t)l * P + p], v);
  }
  mean[t] = ystd[m] * mu + ymean[m];
  if (var) var[t] = v * vscale[m];
}

// Lz^-1 (rows of ldo, lower triangle; the rest untouched) of K(Z, Z) = s k(Z / ell) + jitter I, Z (n, d) on the host
int inducing_inverse_factor(dmo_ctx* ctx, const char* who, int l, int64_t n, int d, const double* Zl, double s, const double* ls,
                            double jitter, int64_t ldo, double* dst) {
  DevBuf<double> Lf;
  DMO_TRY(Lf.alloc(ctx, (size_t)n * n));
  std::vector<double> zero(n, 0.0);
  const double noise = 0.0;
  const int st = dmo_gp_fit(ctx, n, d, 1, DMO_KERNEL_MATERN52, Zl, zero.data(), &s, ls, &noise, jitter, Lf.p, nullptr, nullptr);
  if (st == DMO_ERR_ARG) return dmo_fail(ctx, DMO_ERR_ARG, "%s: K(Z, Z) + jitter I of latent %d is not positive definite", who, l);
  DMO_TRY(st);
  DMO_TRY(gp_linv_from_factor(ctx, Lf.p, n, ldo, dst));
  return DMO_OK;
}

// Householder QR of the n x n column-major matrix C in place (R in the upper triangle); tau: one device double
int householder_qr(dmo_ctx* ctx, double* C, int64_t n, double* tau) {
  for (int64_t j = 0; j + 1 < n; ++j) {
    DMO_LAUNCH(sv_house_kernel, 1, 256, 0, C, n, j, tau);
    DMO_LAUNCH(sv_house_apply_kernel, (unsigned)(n - 1 - j), 256, 0, C, n, j, tau);
  }
  return DMO_OK;
}

bool bits_equal(const double* a, const double* b, size_t n) { return memcmp(a, b, n * sizeof(double)) == 0; }

}  // namespace

int sv_gemm(dmo_ctx* ctx, int64_t m, int64_t n, int64_t K, double alpha, const double* A, int64_t sai, int64_t sak, const double* B,
            int64_t sbk, int64_t sbj, double diag, double* C, int64_t ldc) {
  dim3 g((unsigned)ceil_div(n, GT), (unsigned)ceil_div(m, GT));
  DMO_LAUNCH(sv_gemm_kernel, g, 256, 0, m, n, K, alpha, A, sai, sak, B, sbk, sbj, diag, C, ldc);
  return DMO_OK;
}

int sv_flip(dmo_ctx* ctx, const double* C, int64_t n, double s, double* O, int64_t ldo) {
  DMO_LAUNCH(sv_flip_kernel, (unsigned)ceil_div(n * n, 256), 256, 0, C, n, s, O, ldo);
  return DMO_OK;
}

struct SvGroup {
  std::vector<int> lat, o0;       // latents of the group; the O0 plane of each (its O1 plane is n_o0 + its index)
  int n_o0 = 0;
  GpVarOps ops;                   // (n_o0 + nlat, Npad, Npad) the O0 planes, then the O1 plane of each latent
  DevBuf<double> XtT;             // (d, Npad) Z / ell, transposed, zero padded
  DevBuf<double> A;               // (nlat, Npad) mean vectors a_l, zero padded
  DevBuf<double> inv_ls;          // (d,)
  SvGather gather;
};

struct dmo_svgp {
  int64_t Z = 0;
  int d = 0, L = 0, M = 0;
  std::vector<std::unique_ptr<SvGroup>> groups;
  DevBuf<double> xlb, xrg, W, ymean, ystd, vscale;
};

int svgp_latent_moments(dmo_ctx* ctx, dmo_svgp* sv, GpUnitPredict& up, const double* X, int64_t P, double* fm, double* fv) {
  const int d = sv->d;
  const int64_t Z = sv->Z, Npad = sv->groups[0]->ops.Npad;  // every group's planes have Z rows
  const bool tensor = up.tensor, want_var = fv != nullptr;
  int Gmax = 0;
  for (auto& g : sv->groups) Gmax = g->gather.G > Gmax ? g->gather.G : Gmax;
  DMO_TRY(up.alloc(ctx, P, Npad, Gmax, want_var));
  const int64_t Pc_alloc = up.Pc_alloc;
  const int n_mp = (int)(Npad / mt_kstar_span(false));  // the means always come from float64 kernel values
  DevBuf<double> xs, mpart;
  DMO_TRY(xs.alloc(ctx, (size_t)P * d));
  DMO_TRY(mpart.alloc(ctx, (size_t)n_mp * SV_MAX * Pc_alloc));
  for (auto& gp_ : sv->groups) {
    SvGroup& gr = *gp_;
    if (tensor && want_var) DMO_TRY(gp_prepare_tensor(ctx, gr.ops));
    DMO_TRY(mt_scale_inputs(ctx, X, P, d, sv->xlb.p, sv->xrg.p, gr.inv_ls.p, xs.p));
    for (int64_t p_base = 0; p_base < P; p_base += Pc_alloc) {
      const int64_t Pc = (P - p_base) < Pc_alloc ? (P - p_base) : Pc_alloc;
      const int64_t Pcpad = ceil_div(Pc, up.tile) * up.tile;
      {
        ProfileScope ps(ctx, "svgp_kstar");
        // The mean sums k_u' a_l in float64 kernel values on both paths: a_l = s Lz^-T q_mu alternates in sign near
        // interpolation, so sum |k_u a_l| can be ~100 times the mean and fp32 kernel values (~2^-22) would cost ~1e-5.
        // The tensor path adds a K_*-only pass for its fp16 hi / lo plane.
        if (tensor && want_var)
          DMO_TRY(mt_kstar_produce(ctx, true, xs.p, P, p_base, Pcpad, gr.XtT.p, Z, Npad, d, 0, nullptr, gr.ops.Kexp.p, nullptr,
                                   up.Kh.p, up.Kl.p, mpart.p, Pc_alloc));
        DMO_TRY(mt_kstar_produce(ctx, false, xs.p, P, p_base, Pcpad, gr.XtT.p, Z, Npad, d, gr.gather.nlat, gr.A.p, nullptr,
                                 tensor ? nullptr : up.Ks.p, nullptr, nullptr, mpart.p, Pc_alloc));
      }
      if (want_var) {
        ProfileScope ps(ctx, "svgp_var");
        DMO_TRY(up.contract(ctx, gr.ops, Pcpad));
      }
      DMO_LAUNCH(sv_gather_kernel, (unsigned)ceil_div(Pc, 256), 256, 0, gr.gather, Pc, p_base, P, mpart.p, n_mp, Pc_alloc, up.vnorm.p,
                 up.n_vp, Pc_alloc, fm, fv);
    }
  }
  return DMO_OK;
}

int svgp_predict_device(dmo_ctx* ctx, dmo_svgp* sv, GpUnitPredict& up, const double* X, int64_t P, double* mean, double* var) {
  const int M = sv->M, L = sv->L;
  DevBuf<double> fm, fv;
  DMO_TRY(fm.alloc(ctx, (size_t)L * P));
  if (var) DMO_TRY(fv.alloc(ctx, (size_t)L * P));
  DMO_TRY(svgp_latent_moments(ctx, sv, up, X, P, fm.p, var ? fv.p : nullptr));
  {
    ProfileScope ps(ctx, "svgp_mix");
    DMO_LAUNCH(sv_mix_kernel, (unsigned)ceil_div(P * M, 256), 256, 0, P, L, M, fm.p, fv.p, sv->W.p, sv->ymean.p, sv->ystd.p,
               sv->vscale.p, mean, var);
  }
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

void svgp_dims(const dmo_svgp* sv, int* d, int* M) {
  *d = sv->d;
  *M = sv->M;
}

int svgp_latent_view(const dmo_svgp* sv, int l, SvLatentView* v) {
  for (auto& gp_ : sv->groups) {
    const SvGroup& gr = *gp_;
    for (size_t j = 0; j < gr.lat.size(); ++j) {
      if (gr.lat[j] != l) continue;
      const int64_t Npad = gr.ops.Npad;
      const size_t plane = (size_t)Npad * Npad;
      v->O0 = gr.ops.Linv.p + gr.o0[j] * plane;
      v->O1 = gr.ops.Linv.p + (gr.n_o0 + j) * plane;
      v->A = gr.A.p + j * Npad;
      v->XtT = gr.XtT.p;
      v->inv_ls = gr.inv_ls.p;
      v->Npad = Npad;
      return DMO_OK;
    }
  }
  return DMO_ERR_ARG;
}

extern "C" {

int dmo_svgp_create(dmo_ctx* ctx, int L, int M, int64_t Z, int d, const double* Zpts, const double* variance,
                    const double* length_scale, const double* q_mu, const double* q_sqrt, const double* W, double jitter,
                    const double* y_mean, const double* y_std, const double* y_var_scale, const double* xlb, const double* xrng,
                    dmo_svgp** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out, "svgp_create: null output");
  *out = nullptr;
  DMO_REQUIRE(L >= 1 && L <= SV_MAX && M >= 1 && M <= SV_MAX, "svgp_create: 1 <= L, M <= %d (got L=%d M=%d)", SV_MAX, L, M);
  DMO_REQUIRE(Z >= 1 && Z <= SV_ZMAX && d >= 1 && d <= MT_FIT_DMAX, "svgp_create: unsupported shape Z=%lld d=%d (Z <= %lld, d <= %d)",
              (long long)Z, d, (long long)SV_ZMAX, MT_FIT_DMAX);
  DMO_REQUIRE(W || M == L, "svgp_create: without W the outputs are the latents (M=%d != L=%d)", M, L);
  DMO_REQUIRE(Zpts && variance && length_scale && q_mu && q_sqrt && y_mean && y_std && xlb && xrng, "svgp_create: null pointer");
  DMO_REQUIRE(jitter >= 0.0 && isfinite(jitter), "svgp_create: jitter must be finite and >= 0 (got %g)", jitter);
  const size_t zd = (size_t)Z * d, zz = (size_t)Z * Z;
  std::vector<double> hZ(L * zd), hs(L), hls((size_t)L * d), hqm((size_t)L * Z), hqs(L * zz), hW((size_t)M * L, 0.0), ym(M), ys(M),
      vs(M), lb(d), rg(d);
  DMO_CUDA(cudaMemcpy(hZ.data(), Zpts, hZ.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hs.data(), variance, L * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hls.data(), length_scale, hls.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hqm.data(), q_mu, hqm.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hqs.data(), q_sqrt, hqs.size() * sizeof(double), cudaMemcpyDefault));
  if (W)
    DMO_CUDA(cudaMemcpy(hW.data(), W, hW.size() * sizeof(double), cudaMemcpyDefault));
  else
    for (int m = 0; m < M; ++m) hW[(size_t)m * L + m] = 1.0;
  DMO_CUDA(cudaMemcpy(ym.data(), y_mean, M * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ys.data(), y_std, M * sizeof(double), cudaMemcpyDefault));
  if (y_var_scale)
    DMO_CUDA(cudaMemcpy(vs.data(), y_var_scale, M * sizeof(double), cudaMemcpyDefault));
  else
    for (int m = 0; m < M; ++m) vs[m] = ys[m] * ys[m];
  DMO_CUDA(cudaMemcpy(lb.data(), xlb, d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(rg.data(), xrng, d * sizeof(double), cudaMemcpyDefault));
  for (int k = 0; k < d; ++k) DMO_REQUIRE(rg[k] > 0.0, "svgp_create: xrng[%d] must be > 0", k);
  for (int l = 0; l < L; ++l) {
    DMO_REQUIRE(hs[l] > 0.0 && isfinite(hs[l]), "svgp_create: variance[%d] must be finite and > 0", l);
    for (int k = 0; k < d; ++k)
      DMO_REQUIRE(hls[(size_t)l * d + k] > 0.0 && isfinite(hls[(size_t)l * d + k]), "svgp_create: length_scale[%d][%d] must be > 0", l, k);
    const double* q = hqs.data() + l * zz;
    for (int64_t i = 0; i < Z; ++i)
      for (int64_t j = i + 1; j < Z; ++j)
        DMO_REQUIRE(q[i * Z + j] == 0.0, "svgp_create: q_sqrt[%d] is not lower triangular (entry %lld, %lld)", l, (long long)i,
                    (long long)j);
  }
  std::unique_ptr<dmo_svgp> sv(new dmo_svgp());
  sv->Z = Z;
  sv->d = d;
  sv->L = L;
  sv->M = M;
  // K_* groups: bitwise equal Z planes and length scales
  std::vector<int> grp_of(L, -1);
  std::vector<int> lead;
  for (int l = 0; l < L; ++l) {
    for (size_t g = 0; g < lead.size(); ++g) {
      const int f = lead[g];
      if (bits_equal(&hZ[l * zd], &hZ[f * zd], zd) && bits_equal(&hls[(size_t)l * d], &hls[(size_t)f * d], d)) {
        grp_of[l] = (int)g;
        break;
      }
    }
    if (grp_of[l] < 0) {
      grp_of[l] = (int)lead.size();
      lead.push_back(l);
    }
  }
  DevBuf<double> qm_d, qs_d, Ct, tau;
  DMO_TRY(upload(ctx, qm_d, hqm));
  DMO_TRY(upload(ctx, qs_d, hqs));
  DMO_TRY(Ct.alloc(ctx, zz));
  DMO_TRY(tau.alloc(ctx, 1));
  for (size_t g = 0; g < lead.size(); ++g) {
    std::unique_ptr<SvGroup> gr(new SvGroup());
    std::vector<int> o0_src;  // the latent whose s defines each O0 plane
    for (int l = 0; l < L; ++l) {
      if (grp_of[l] != (int)g) continue;
      int o = -1;
      for (size_t k = 0; k < o0_src.size(); ++k)
        if (bits_equal(&hs[l], &hs[o0_src[k]], 1)) o = (int)k;
      if (o < 0) {
        o = (int)o0_src.size();
        o0_src.push_back(l);
      }
      gr->lat.push_back(l);
      gr->o0.push_back(o);
    }
    const int nlat = (int)gr->lat.size(), n_o0 = gr->n_o0 = (int)o0_src.size(), G = n_o0 + nlat;
    GpVarOps& ops = gr->ops;
    DMO_TRY(ops.alloc(ctx, Z, G));  // K_* carries no output scale: unit K_* scales
    const int64_t Npad = ops.Npad;
    const size_t plane = (size_t)Npad * Npad;
    const int f = lead[g];
    for (int k = 0; k < n_o0; ++k) {
      const int l = o0_src[k];
      DMO_TRY(inducing_inverse_factor(ctx, "svgp_create", l, Z, d, &hZ[f * zd], hs[l], &hls[(size_t)f * d], jitter, Npad,
                                      ops.Linv.p + k * plane));
    }
    DMO_TRY(gr->A.alloc(ctx, (size_t)nlat * Npad));
    DMO_CUDA(cudaMemsetAsync(gr->A.p, 0, (size_t)nlat * Npad * sizeof(double), ctx->stream));
    for (int j = 0; j < nlat; ++j) {
      const int l = gr->lat[j];
      const double* Li = ops.Linv.p + gr->o0[j] * plane;  // unscaled Lz^-1 (the O0 planes are scaled below)
      // a_l = s_l Lz^-T q_mu:  a[i] = s sum_k Li[k][i] q_mu[k]
      DMO_TRY(sv_gemm(ctx,Z, 1, Z, hs[l], Li, 1, Npad, qm_d.p + (size_t)l * Z, 1, 0, 0.0, gr->A.p + (size_t)j * Npad, 1));
      // V J by columns: column c = row c of Ct, Ct[c][r] = V[r][Z-1-c] = sum_k Li[k][Z-1-c] q_sqrt[k][r]
      DMO_TRY(sv_gemm(ctx,Z, Z, Z, 1.0, Li + (Z - 1), -1, Npad, qs_d.p + (size_t)l * zz, Z, 1, 0.0, Ct.p, Z));
      DMO_TRY(householder_qr(ctx, Ct.p, Z, tau.p));
      DMO_LAUNCH(sv_flip_kernel, (unsigned)ceil_div((int64_t)zz, 256), 256, 0, Ct.p, Z, hs[l], ops.Linv.p + (n_o0 + j) * plane, Npad);
    }
    for (int k = 0; k < n_o0; ++k)
      DMO_LAUNCH(sv_scale_kernel, (unsigned)ceil_div((int64_t)plane, 256), 256, 0, ops.Linv.p + k * plane, (int64_t)plane, hs[o0_src[k]]);
    std::vector<double> inv(d);
    for (int k = 0; k < d; ++k) inv[k] = 1.0 / hls[(size_t)f * d + k];
    const std::vector<double> xtT =
        mt_xt_transposed(Z, d, Npad, [&](int64_t n, int k) { return hZ[f * zd + (size_t)n * d + k] * inv[k]; });
    DMO_TRY(upload(ctx, gr->XtT, xtT));
    DMO_TRY(upload(ctx, gr->inv_ls, inv));
    SvGather& ga = gr->gather;
    ga.nlat = nlat;
    ga.n_o0 = n_o0;
    ga.G = G;
    for (int j = 0; j < nlat; ++j) {
      ga.lat[j] = gr->lat[j];
      ga.o0[j] = gr->o0[j];
      ga.s[j] = hs[gr->lat[j]];
    }
    DMO_CHECK_LAUNCH();
    DMO_CUDA(dmo_wait(ctx));  // host vectors above are staged from the stack
    sv->groups.push_back(std::move(gr));
  }
  DMO_TRY(upload(ctx, sv->xlb, lb));
  DMO_TRY(upload(ctx, sv->xrg, rg));
  DMO_TRY(upload(ctx, sv->W, hW));
  DMO_TRY(upload(ctx, sv->ymean, ym));
  DMO_TRY(upload(ctx, sv->ystd, ys));
  DMO_TRY(upload(ctx, sv->vscale, vs));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  *out = sv.release();
  return DMO_OK;
}

int dmo_svgp_destroy(dmo_ctx* ctx, dmo_svgp* sv) {
  if (!ctx) return DMO_ERR_ARG;
  if (!sv) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  delete sv;
  return DMO_OK;
}

int dmo_svgp_groups(dmo_ctx* ctx, dmo_svgp* sv, int* n_groups, int* n_planes) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_REQUIRE(sv, "svgp_groups: null model");
  if (n_groups) *n_groups = (int)sv->groups.size();
  if (n_planes) {
    int t = 0;
    for (auto& g : sv->groups) t += g->gather.G;
    *n_planes = t;
  }
  return DMO_OK;
}

int dmo_svgp_predict(dmo_ctx* ctx, dmo_svgp* sv, const double* X, int64_t P, double* mean, double* var, int precision) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(sv, "svgp_predict: null model");
  const int M = sv->M, d = sv->d;
  GpUnitPredict up;
  DMO_TRY(up.check(ctx, "svgp_predict", precision, d));
  if (P == 0) return DMO_OK;
  DMO_REQUIRE(P > 0 && X && mean, "svgp_predict: bad arguments");
  In<double> x;
  Out<double> om, ov;
  DMO_TRY(x.init(ctx, X, (size_t)P * d));
  DMO_TRY(om.init(ctx, mean, (size_t)P * M));
  DMO_TRY(ov.init(ctx, var, (size_t)P * M));
  DMO_TRY(svgp_predict_device(ctx, sv, up, x.d, P, om.d, ov.d));
  DMO_TRY(up.watchdog(ctx));
  DMO_TRY(om.finish(ctx));
  DMO_TRY(ov.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_svgp_optimal_q(dmo_ctx* ctx, int64_t N, int64_t Z, int d, int L, const double* X, const double* y, const double* Zpts,
                       const double* variance, const double* length_scale, const double* noise, double jitter, int inducing_is_data,
                       double* q_mu_out, double* q_sqrt_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(L >= 1 && L <= SV_MAX, "svgp_optimal_q: 1 <= L <= %d (got %d)", SV_MAX, L);
  DMO_REQUIRE(N >= 1 && Z >= 1 && Z <= SV_ZMAX && d >= 1 && d <= MT_FIT_DMAX, "svgp_optimal_q: unsupported shape N=%lld Z=%lld d=%d",
              (long long)N, (long long)Z, d);
  DMO_REQUIRE(X && y && (Zpts || inducing_is_data) && variance && length_scale && noise && q_mu_out && q_sqrt_out,
              "svgp_optimal_q: null pointer");
  DMO_REQUIRE(!inducing_is_data || Z == N, "svgp_optimal_q: with inducing_is_data Z must equal N (got Z=%lld N=%lld)", (long long)Z,
              (long long)N);
  DMO_REQUIRE(jitter >= 0.0 && isfinite(jitter), "svgp_optimal_q: jitter must be finite and >= 0 (got %g)", jitter);
  const size_t zd = (size_t)Z * d, zz = (size_t)Z * Z;
  std::vector<double> hx((size_t)N * d), hZ(L * zd), hs(L), hls((size_t)L * d), hn(L);
  DMO_CUDA(cudaMemcpy(hx.data(), X, hx.size() * sizeof(double), cudaMemcpyDefault));
  if (inducing_is_data)
    for (int l = 0; l < L; ++l) memcpy(&hZ[l * zd], hx.data(), zd * sizeof(double));
  else
    DMO_CUDA(cudaMemcpy(hZ.data(), Zpts, hZ.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hs.data(), variance, L * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hls.data(), length_scale, hls.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hn.data(), noise, L * sizeof(double), cudaMemcpyDefault));
  for (int l = 0; l < L; ++l) {
    DMO_REQUIRE(hs[l] > 0.0 && isfinite(hs[l]), "svgp_optimal_q: variance[%d] must be finite and > 0", l);
    DMO_REQUIRE(hn[l] > 0.0 && isfinite(hn[l]), "svgp_optimal_q: noise[%d] must be finite and > 0", l);
    for (int k = 0; k < d; ++k)
      DMO_REQUIRE(hls[(size_t)l * d + k] > 0.0 && isfinite(hls[(size_t)l * d + k]), "svgp_optimal_q: length_scale[%d][%d] must be > 0", l, k);
  }
  In<double> iy;
  Out<double> oqm, oqs;
  DMO_TRY(iy.init(ctx, y, (size_t)L * N));
  DMO_TRY(oqm.init(ctx, q_mu_out, (size_t)L * Z));
  DMO_TRY(oqs.init(ctx, q_sqrt_out, (size_t)L * zz));
  const int64_t Npad = ceil_div(Z, 256) * 256, Pcpad = ceil_div(N, 32) * 32;
  const int64_t ld = ceil_div(Z, 64) * 64;  // the Cholesky block edge
  DevBuf<double> Li, Kxz, At, Bm, Lci, bvec, tvec, xs, XtT;
  DevBuf<int> info;
  if (!inducing_is_data) {
    DMO_TRY(Li.alloc(ctx, zz));
    DMO_TRY(Kxz.alloc(ctx, (size_t)Pcpad * Npad));
  }
  DMO_TRY(At.alloc(ctx, (size_t)N * Z));
  DMO_TRY(Bm.alloc(ctx, zz));
  DMO_TRY(Lci.alloc(ctx, (size_t)ld * ld));
  DMO_TRY(bvec.alloc(ctx, Z));
  DMO_TRY(tvec.alloc(ctx, Z));
  DMO_TRY(info.alloc(ctx, 1));
  const int n_mp = (int)(Npad / mt_kstar_span(false));
  for (int l = 0; l < L; ++l) {
    const double s = hs[l], s2 = hn[l];
    const double* ls = &hls[(size_t)l * d];
    if (inducing_is_data) {
      // VGP: f(X) = Lz v with Lz = chol(K(X, X) + jitter I), so A = Lz' and A' = Lz (the data term sees the jitter too)
      std::vector<double> zero(N, 0.0);
      const double nz0 = 0.0;
      const int st = dmo_gp_fit(ctx, N, d, 1, DMO_KERNEL_MATERN52, hx.data(), zero.data(), &s, ls, &nz0, jitter, At.p, nullptr, nullptr);
      if (st == DMO_ERR_ARG) return dmo_fail(ctx, DMO_ERR_ARG, "svgp_optimal_q: K(X, X) + jitter I of latent %d is not positive definite", l);
      DMO_TRY(st);
    } else {
    // Lz^-1 (Z x Z, rows of Z)
    DMO_CUDA(cudaMemsetAsync(Li.p, 0, zz * sizeof(double), ctx->stream));
    DMO_TRY(inducing_inverse_factor(ctx, "svgp_optimal_q", l, Z, d, &hZ[l * zd], s, ls, jitter, Z, Li.p));
    // unit K(X, Z) rows of Npad, from the multitask producer with the training inputs as candidates
    std::vector<double> xsh((size_t)N * d);
    for (int64_t n = 0; n < N; ++n)
      for (int k = 0; k < d; ++k) xsh[(size_t)n * d + k] = hx[(size_t)n * d + k] / ls[k];
    const std::vector<double> xtT =
        mt_xt_transposed(Z, d, Npad, [&](int64_t n, int k) { return hZ[l * zd + (size_t)n * d + k] / ls[k]; });
    DMO_TRY(upload(ctx, xs, xsh));
    DMO_TRY(upload(ctx, XtT, xtT));
    DevBuf<double> mpart;
    DMO_TRY(mpart.alloc(ctx, (size_t)n_mp));
    DMO_TRY(mt_kstar_produce(ctx, false, xs.p, N, 0, Pcpad, XtT.p, Z, Npad, d, 0, nullptr, nullptr, Kxz.p, nullptr, nullptr, mpart.p,
                             Pcpad));
    // A' = s K(X, Z) Lz^-T  (N x Z):  At[p][i] = s sum_k Kxz[p][k] Li[i][k]
    DMO_TRY(sv_gemm(ctx,N, Z, Z, s, Kxz.p, Npad, 1, Li.p, 1, Z, 0.0, At.p, Z));
    DMO_CHECK_LAUNCH();
    DMO_CUDA(dmo_wait(ctx));  // xsh / xtT are staged from the stack
    }
    // B = I + A A' / sigma^2 (Z x Z)
    DMO_TRY(sv_gemm(ctx,Z, Z, N, 1.0 / s2, At.p, 1, Z, At.p, Z, 1, 1.0, Bm.p, Z));
    // b = A y / sigma^2
    DMO_TRY(sv_gemm(ctx,Z, 1, N, 1.0 / s2, At.p, 1, Z, iy.d + (size_t)l * N, 1, 0, 0.0, bvec.p, 1));
    // S = B^-1 = U U' with U = J Lc^-T J lower triangular, Lc = chol(J B J):  B^-1 = J (Lc Lc')^-1 J = (J Lc^-T J)(J Lc^-1 J)
    DMO_LAUNCH(sv_reverse_pad_kernel, (unsigned)ceil_div(ld * ld, 256), 256, 0, Bm.p, Z, ld, Lci.p);
    DMO_CUDA(cudaMemsetAsync(info.p, 0, sizeof(int), ctx->stream));
    DMO_TRY(gp_potrf_batched(ctx, Lci.p, ld, 1, info.p));
    int h_info = 0;
    DMO_CUDA(cudaMemcpyAsync(&h_info, info.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    if (h_info) return dmo_fail(ctx, DMO_ERR_ARG, "svgp_optimal_q: I + A A' / noise of latent %d is not positive definite", l);
    DMO_CUDA(cudaMemsetAsync(Bm.p, 0, zz * sizeof(double), ctx->stream));
    DMO_TRY(gp_linv_from_factor_batched(ctx, Lci.p, ld, 0, Z, 1, Z, 0, Bm.p));  // Lc: the leading Z x Z block of Lci
    double* U = oqs.d + (size_t)l * zz;
    DMO_LAUNCH(sv_flip_kernel, (unsigned)ceil_div((int64_t)zz, 256), 256, 0, Bm.p, Z, 1.0, U, Z);
    // q_mu = U (U' b)
    DMO_TRY(sv_gemm(ctx,Z, 1, Z, 1.0, U, 1, Z, bvec.p, 1, 0, 0.0, tvec.p, 1));
    DMO_TRY(sv_gemm(ctx,Z, 1, Z, 1.0, U, Z, 1, tvec.p, 1, 0, 0.0, oqm.d + (size_t)l * Z, 1));
    DMO_CHECK_LAUNCH();
    DMO_CUDA(dmo_wait(ctx));  // xsh / xtT are staged from the stack
  }
  DMO_TRY(oqm.finish(ctx));
  DMO_TRY(oqs.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
