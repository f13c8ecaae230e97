// Training of the GPflow variational surrogates (SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern, CRV_Matern;
// dmosopt/model.py:98-1179): a device-resident state of one GPflow model -- L whitened latents over one set of inducing
// points, mixed into M outputs by W -- with the natural-gradient step on q and the minibatch ELBO with its gradient with
// respect to the kernel hyper-parameters, the likelihood variances and W at fixed q.
//
// Per latent l (unit kernel k_u, s_l the variance): Kzz = s k_u(Z, Z) + jitter I, Lz = chol(Kzz), and for a batch X_b
//   SVGP:  A = Lz^-1 s k_u(Z, X_b)  (Z x B),  mu = A' m,  v = s - colsum(A o A) + colsum(A o S A)
//   VGP:   Z = X, f(X) = Lz v, so A = Lz' restricted to the batch columns, and v = colsum(A o S A)
// q_l is kept in natural parameters: Lambda_l = S_l^-1 and theta1_l = Lambda_l m_l, with the factor kept current after
// every step: Lc = chol(J Lambda J) (J reverses the order), U = J Lc^-T J lower triangular, S = U U', m = U U' theta1.
// The output f = W g: mean_f = W mu, var_f = (W o W) v.
//
//   ELBO = (N / B) sum_b sum_m E_q log N(y_bm | f_bm, sigma2_m) - sum_l KL(q_l || N(0, I))
//
// Gradient at fixed q: the ELL gives mu_bar (B) and a constant v_bar per latent, A_bar = m mu_bar' + 2 v_bar (S A - A)
// (VGP: 2 v_bar S A); SVGP: K_zb_bar = Lz^-T A_bar and Lz_bar = -K_zb_bar A'; VGP: Lz_bar scattered from A_bar.  The
// Cholesky backward pass (Murray 2016, arXiv:1602.07527): Kzz_bar = sym(Lz^-T Phi(Lz' tril(Lz_bar)) Lz^-1) / 2, with
// Phi the lower triangle with a halved diagonal and sym(X) = X + X'.  svf_grad_pass_kernel then recomputes distances
// and Matern derivative factors from the inputs and contracts Kzz_bar and K_zb_bar into d / d s and d / d l.
//
// Natural-gradient step (GPflow's NaturalGradient with XiNat, Gaussian likelihood): a convex blend toward the minibatch
// optimum, Lambda <- (1 - g) Lambda + g (I + (N / B) c A A'), theta1 <- (1 - g) theta1 + g (N / B) A r~, with
// c_l = sum_m W_ml^2 / sigma2_m and r~_l = sum_m W_ml (y_m - sum_{l' != l} W_ml' mu_l') / sigma2_m (mu at the current q).
//
// Float64; every reduction runs in a fixed order and no kernel uses atomics, so repeated calls are bit-identical.  Dense
// products go through sv_gemm (gp_variational.cu), the factorisations through gp_fit_batched / gp_potrf_batched
// (gp_fit.cu) and gp_linv_from_factor_batched.
#include <math.h>
#include <string.h>

#include <memory>
#include <vector>

#include "gp.cuh"

namespace {

constexpr int SVF_MAX = 8;
constexpr int64_t SVF_ZMAX = 8192;
constexpr double SQRT5 = 2.23606797749978969641;
constexpr double LOG_2PI = 1.8378770664093453;

// xs[b][c] = X[idx[b]][c] inv_ls[c]  (idx NULL: row b)
__global__ void svf_scale_rows_kernel(const double* __restrict__ X, const int64_t* __restrict__ idx, int64_t n, int d,
                                      const double* __restrict__ inv_ls, double* __restrict__ xs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int64_t b = t / d;
  const int c = (int)(t - b * d);
  xs[t] = X[(idx ? idx[b] : b) * d + c] * inv_ls[c];
}

// K[i][b] = s k_u(zs_i, xs_b), rows of n
__global__ void svf_cross_kernel(const double* __restrict__ zs, int64_t Z, const double* __restrict__ xs, int64_t n, int d, double s,
                                 double* __restrict__ K) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Z * n) return;
  const int64_t i = t / n, b = t - i * n;
  double s2 = 0.0;
  for (int c = 0; c < d; ++c) {
    const double u = zs[i * d + c] - xs[b * d + c];
    s2 = fma(u, u, s2);
  }
  K[t] = s * stationary(s2, DMO_KERNEL_MATERN52);
}

// VGP: A[k][b] = Lz[batch[b]][k] (zero above the diagonal), Lz rows of ld
__global__ void svf_gather_cols_kernel(const double* __restrict__ Lf, int64_t ld, const int64_t* __restrict__ batch, int64_t Z, int64_t B,
                                       double* __restrict__ A) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Z * B) return;
  const int64_t k = t / B, b = t - k * B, p = batch[b];
  A[t] = k <= p ? Lf[p * ld + k] : 0.0;
}

// VGP: Lbar[batch[b]][k] = A_bar[k][b] for k <= batch[b], else 0 (batch is a permutation of [0, Z))
__global__ void svf_scatter_rows_kernel(const double* __restrict__ Abar, const int64_t* __restrict__ batch, int64_t Z,
                                        double* __restrict__ Lbar) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Z * Z) return;
  const int64_t k = t / Z, b = t - k * Z, p = batch[b];
  Lbar[p * Z + k] = k <= p ? Abar[t] : 0.0;
}

// per column b: mu[b] = sum_k A[k][b] m[k];  v[b] = (svgp ? s - sum_k A[k][b]^2 : 0) + sum_k T[k][b]^2, T = U' A
__global__ void svf_colstats_kernel(const double* __restrict__ A, const double* __restrict__ T, const double* __restrict__ m, int64_t Z,
                                    int64_t B, double s, int svgp, double* __restrict__ mu, double* __restrict__ v) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double sm = 0.0, a2 = 0.0, t2 = 0.0;
  for (int64_t k = 0; k < Z; ++k) {
    const double a = A[k * B + b], t = T[k * B + b];
    sm = fma(a, m[k], sm);
    a2 = fma(a, a, a2);
    t2 = fma(t, t, t2);
  }
  mu[b] = sm;
  v[b] = svgp ? (s - a2) + t2 : t2;
}

// KL(N(m, U U') || N(0, I)) = (||U||_F^2 + m'm - Z) / 2 - sum_k log U_kk, one block per latent
__global__ void __launch_bounds__(256) svf_kl_kernel(const double* __restrict__ U, const double* __restrict__ m, int64_t Z,
                                                     double* __restrict__ kl) {
  __shared__ double red[8];
  U += (size_t)blockIdx.x * Z * Z;
  m += (size_t)blockIdx.x * Z;
  double q = 0.0, ld = 0.0;
  for (int64_t t = threadIdx.x; t < Z * Z; t += 256) q = fma(U[t], U[t], q);
  for (int64_t k = threadIdx.x; k < Z; k += 256) {
    q = fma(m[k], m[k], q);
    ld += log(U[k * Z + k]);
  }
  q = block_sum<8>(q, red);
  ld = block_sum<8>(ld, red);
  if (threadIdx.x == 0) kl[blockIdx.x] = 0.5 * (q - (double)Z) - ld;
}

// one block per output m: ell[m] = scale sum_b E_q log N(y | f, sigma2_m), gnoise[m] its derivative by sigma2_m, and
// r[m][b] = (y - mean_f) / sigma2_m
__global__ void __launch_bounds__(256) svf_ell_kernel(const double* __restrict__ Y, int64_t N, const int64_t* __restrict__ batch, int64_t B,
                                                      int L, const double* __restrict__ W, const double* __restrict__ mu,
                                                      const double* __restrict__ v, const double* __restrict__ noise, double scale,
                                                      double* __restrict__ r, double* __restrict__ ell, double* __restrict__ gnoise) {
  __shared__ double red[8];
  const int m = blockIdx.x;
  const double s2 = noise[m], c0 = -0.5 * (LOG_2PI + log(s2));
  double e_acc = 0.0, g_acc = 0.0;
  for (int64_t b = threadIdx.x; b < B; b += 256) {
    double mf = 0.0, vf = 0.0;
    for (int l = 0; l < L; ++l) {
      const double w = W[m * L + l];
      mf = fma(w, mu[l * B + b], mf);
      vf = fma(w * w, v[l * B + b], vf);
    }
    const double e = Y[m * N + batch[b]] - mf;
    const double q = fma(e, e, vf);
    r[m * B + b] = e / s2;
    e_acc += c0 - q / (2.0 * s2);
    g_acc += -0.5 / s2 + q / (2.0 * s2 * s2);
  }
  e_acc = block_sum<8>(e_acc, red);
  g_acc = block_sum<8>(g_acc, red);
  if (threadIdx.x == 0) {
    ell[m] = scale * e_acc;
    gnoise[m] = scale * g_acc;
  }
}

// one block per latent l: mubar[l][b] = scale sum_m W_ml r[m][b]; the (constant) v_bar_l = -scale sum_m W_ml^2 / (2 sigma2_m)
// into vbar[l]; gW[m][l] = scale (sum_b r[m][b] mu_l[b] - W_ml / sigma2_m sum_b v_l[b]) when gW is not NULL
__global__ void __launch_bounds__(256) svf_latent_bar_kernel(int M, int L, int64_t B, const double* __restrict__ W,
                                                             const double* __restrict__ noise, const double* __restrict__ r,
                                                             const double* __restrict__ mu, const double* __restrict__ v, double scale,
                                                             double* __restrict__ mubar, double* __restrict__ vbar,
                                                             double* __restrict__ gW) {
  __shared__ double red[8];
  const int l = blockIdx.x;
  double cv = 0.0;
  for (int m = 0; m < M; ++m) cv += W[m * L + l] * W[m * L + l] / noise[m];
  for (int64_t b = threadIdx.x; b < B; b += 256) {
    double s = 0.0;
    for (int m = 0; m < M; ++m) s = fma(W[m * L + l], r[m * B + b], s);
    mubar[l * B + b] = scale * s;
  }
  if (threadIdx.x == 0) vbar[l] = -0.5 * scale * cv;
  if (!gW) return;
  double vs = 0.0;
  for (int64_t b = threadIdx.x; b < B; b += 256) vs += v[l * B + b];
  vs = block_sum<8>(vs, red);
  for (int m = 0; m < M; ++m) {
    double s = 0.0;
    for (int64_t b = threadIdx.x; b < B; b += 256) s = fma(r[m * B + b], mu[l * B + b], s);
    s = block_sum<8>(s, red);
    if (threadIdx.x == 0) gW[m * L + l] = scale * (s - W[m * L + l] / noise[m] * vs);
  }
}

// A_bar[k][b] = m[k] mubar[b] + 2 vbar (SA[k][b] - (svgp ? A[k][b] : 0))
__global__ void svf_abar_kernel(int64_t Z, int64_t B, const double* __restrict__ m, const double* __restrict__ mubar,
                                const double* __restrict__ vbar, const double* __restrict__ SA, const double* __restrict__ A, int svgp,
                                double* __restrict__ Abar) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Z * B) return;
  const int64_t k = t / B, b = t - k * B;
  const double d = svgp ? SA[t] - A[t] : SA[t];
  Abar[t] = fma(m[k], mubar[b], 2.0 * vbar[0] * d);
}

// in place on an n x n matrix: zero above the diagonal, the diagonal times dscale (1: tril, 1/2: Phi)
__global__ void svf_tril_kernel(double* __restrict__ X, int64_t n, double dscale) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * n) return;
  const int64_t i = t / n, j = t - i * n;
  if (j > i) X[t] = 0.0;
  else if (i == j) X[t] *= dscale;
}

// K_bar = (X + X') / 2
__global__ void svf_sym_kernel(const double* __restrict__ X, int64_t n, double* __restrict__ K) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * n) return;
  const int64_t i = t / n, j = t - i * n;
  K[t] = 0.5 * (X[t] + X[j * n + i]);
}

// One block per row i of Z: with w_ij = Kbar_ij s (5/3)(1 + r) e^-r over the columns j (Z points zs, then nb batch
// points xs with Kbar_zb), part[i][c] = sum_j w_ij (zs_ic - x_jc)^2 for c < d and part[i][d] = sum_j Kbar_ij k_u(r).
// Columns in chunks of 256: phase 1 one column per thread, phase 2 one coordinate per thread.
__global__ void __launch_bounds__(256) svf_grad_pass_kernel(const double* __restrict__ zs, int64_t Z, const double* __restrict__ xs,
                                                            int64_t nb, int d, double s, const double* __restrict__ Kzz,
                                                            const double* __restrict__ Kzb, double* __restrict__ part) {
  __shared__ double zi[MT_FIT_DMAX];
  __shared__ double w[256];
  __shared__ double red[8];
  const int64_t i = blockIdx.x;
  const int tid = threadIdx.x;
  for (int c = tid; c < d; c += 256) zi[c] = zs[i * d + c];
  __syncthreads();
  double acc = 0.0, ks = 0.0;  // acc: coordinate tid's sum; ks: this thread's share of sum Kbar k_u
  const int64_t ncol = Z + nb;
  for (int64_t j0 = 0; j0 < ncol; j0 += 256) {
    const int64_t j = j0 + tid;
    double wv = 0.0;
    if (j < ncol) {
      const double* xj = j < Z ? zs + j * d : xs + (j - Z) * d;
      const double kb = j < Z ? Kzz[i * Z + j] : Kzb[i * nb + (j - Z)];
      double s2 = 0.0;
      for (int c = 0; c < d; ++c) {
        const double u = zi[c] - xj[c];
        s2 = fma(u, u, s2);
      }
      const double r = sqrt(s2) * SQRT5, e = exp(-r);  // stationary()'s Matern, with exp(-r) kept for the derivative factor
      ks = fma(kb, (1.0 + r + r * r / 3.0) * e, ks);
      wv = kb * s * (5.0 / 3.0) * (1.0 + r) * e;
    }
    w[tid] = wv;
    __syncthreads();
    if (tid < d) {
      const int64_t n = ncol - j0 < 256 ? ncol - j0 : 256;
      for (int64_t t = 0; t < n; ++t) {
        const int64_t jj = j0 + t;
        const double u = zi[tid] - (jj < Z ? zs[jj * d + tid] : xs[(jj - Z) * d + tid]);
        acc = fma(w[t] * u, u, acc);
      }
    }
    __syncthreads();
  }
  ks = block_sum<8>(ks, red);
  if (tid < d) part[i * (d + 1) + tid] = acc;
  if (tid == 0) part[i * (d + 1) + d] = ks;
}

// g_ls[c] = sum_i part[i][c] / ls[c] (c < d), g_s = sum_i part[i][d] + B vbar (the direct term of v = s - ..., SVGP)
__global__ void svf_fold_kernel(const double* __restrict__ part, int64_t Z, int d, const double* __restrict__ ls, const double* __restrict__ vbar,
                                double direct, double* __restrict__ g_ls, double* __restrict__ g_s) {
  const int c = threadIdx.x;
  if (c > d) return;
  double s = 0.0;
  for (int64_t i = 0; i < Z; ++i) s += part[i * (d + 1) + c];
  if (c < d) g_ls[c] = s / ls[c];
  else g_s[0] = s + direct * vbar[0];
}

// r~[b] = sum_m W_ml (y_m[b] - sum_{l' != l} W_ml' mu_l'[b]) / sigma2_m
__global__ void svf_rtilde_kernel(const double* __restrict__ Y, int64_t N, const int64_t* __restrict__ batch, int64_t B, int M, int L, int l,
                                  const double* __restrict__ W, const double* __restrict__ noise, const double* __restrict__ mu,
                                  double* __restrict__ rt) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double s = 0.0;
  for (int m = 0; m < M; ++m) {
    double e = Y[m * N + batch[b]];
    for (int k = 0; k < L; ++k)
      if (k != l) e = fma(-W[m * L + k], mu[k * B + b], e);
    s = fma(W[m * L + l], e / noise[m], s);
  }
  rt[b] = s;
}

// Natural-gradient blend of one latent, one thread per element (a, b) of the lc x lc factor input:
//   Lambda_ij <- (1 - g) Lambda_ij + g (delta_ij + G_ij)  (i = Z-1-a, j = Z-1-b; G = (N / B) c A A')
//   LamJ[a][b] = the new Lambda_ij (J Lambda J), identity in the padding;  theta1_a <- (1 - g) theta1_a + g Ar_a (b == 0)
__global__ void svf_blend_kernel(double* __restrict__ Lam, const double* __restrict__ G, int64_t Z, int64_t lc, double gamma,
                                 double* __restrict__ th1, const double* __restrict__ Ar, double* __restrict__ LamJ) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= lc * lc) return;
  const int64_t a = t / lc, b = t - a * lc;
  if (a < Z && b < Z) {
    const int64_t i = Z - 1 - a, j = Z - 1 - b;
    const double nv = fma(1.0 - gamma, Lam[i * Z + j], gamma * ((i == j ? 1.0 : 0.0) + G[i * Z + j]));
    Lam[i * Z + j] = nv;
    LamJ[t] = nv;
    if (b == 0) th1[a] = fma(1.0 - gamma, th1[a], gamma * Ar[a]);
  } else {
    LamJ[t] = a == b ? 1.0 : 0.0;
  }
}

}  // namespace

struct dmo_svgp_fit {
  int64_t N = 0, Z = 0, ld = 0, lc = 0;  // ld: edge of the augmented K(Z, Z) factor; lc: edge of chol(J Lambda J)
  int d = 0, M = 0, L = 0;
  bool vgp = false;
  double jitter = 0.0;
  DevBuf<double> X, Y, Zp;       // (N,d), (M,N), (Z,d)
  DevBuf<double> Lam, U;         // (L,Z,Z)
  DevBuf<double> th1, m;         // (L,Z)
};

namespace {

// Hyper-parameters of one call, checked, on the host and on the device; the distinct kernels (bitwise equal variance
// and length scales) each get one factorisation
struct SvfParams {
  std::vector<double> s, ls, inv, noise, W, zero;
  std::vector<int> kof;  // latent -> distinct kernel
  std::vector<int> lead;  // distinct kernel -> its first latent
  DevBuf<double> d_inv, d_s, d_dadd, d_noise, d_W, d_zero;
  DevBuf<int64_t> d_batch;
  std::vector<int64_t> batch;
};

int svf_params(dmo_ctx* ctx, const char* who, dmo_svgp_fit* st, const int64_t* batch, int64_t B, const double* variance,
               const double* length_scale, const double* noise, const double* W, SvfParams& p) {
  const int L = st->L, M = st->M, d = st->d;
  DMO_REQUIRE(batch && variance && length_scale && noise, "%s: null pointer", who);
  DMO_REQUIRE(B >= 1 && B <= st->N, "%s: 1 <= B <= N (got B=%lld N=%lld)", who, (long long)B, (long long)st->N);
  DMO_REQUIRE(!st->vgp || B == st->N, "%s: the VGP form takes the full data (B=%lld N=%lld)", who, (long long)B, (long long)st->N);
  DMO_REQUIRE(W || M == L, "%s: without W the outputs are the latents (M=%d != L=%d)", who, M, L);
  p.s.resize(L);
  p.ls.resize((size_t)L * d);
  p.inv.resize((size_t)L * d);
  p.noise.resize(M);
  p.W.assign((size_t)M * L, 0.0);
  p.batch.resize(B);
  DMO_CUDA(cudaMemcpy(p.batch.data(), batch, B * sizeof(int64_t), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(p.s.data(), variance, L * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(p.ls.data(), length_scale, p.ls.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(p.noise.data(), noise, M * sizeof(double), cudaMemcpyDefault));
  if (W)
    DMO_CUDA(cudaMemcpy(p.W.data(), W, p.W.size() * sizeof(double), cudaMemcpyDefault));
  else
    for (int l = 0; l < L; ++l) p.W[(size_t)l * L + l] = 1.0;
  for (int64_t b = 0; b < B; ++b)
    DMO_REQUIRE(p.batch[b] >= 0 && p.batch[b] < st->N, "%s: batch[%lld] = %lld is outside [0, %lld)", who, (long long)b,
                (long long)p.batch[b], (long long)st->N);
  if (st->vgp) {  // a permutation: every row of the factor is scattered back exactly once
    std::vector<char> seen(st->N, 0);
    for (int64_t b = 0; b < B; ++b) {
      DMO_REQUIRE(!seen[p.batch[b]], "%s: the VGP batch repeats index %lld", who, (long long)p.batch[b]);
      seen[p.batch[b]] = 1;
    }
  }
  for (int l = 0; l < L; ++l) {
    DMO_REQUIRE(p.s[l] > 0.0 && isfinite(p.s[l]), "%s: variance[%d] must be finite and > 0", who, l);
    for (int k = 0; k < d; ++k) {
      const double v = p.ls[(size_t)l * d + k];
      DMO_REQUIRE(v > 0.0 && isfinite(v), "%s: length_scale[%d][%d] must be finite and > 0", who, l, k);
      p.inv[(size_t)l * d + k] = 1.0 / v;
    }
  }
  for (int m = 0; m < M; ++m) DMO_REQUIRE(p.noise[m] > 0.0 && isfinite(p.noise[m]), "%s: noise[%d] must be finite and > 0", who, m);
  for (size_t t = 0; t < p.W.size(); ++t) DMO_REQUIRE(isfinite(p.W[t]), "%s: W must be finite", who);
  p.kof.assign(L, -1);
  p.lead.clear();
  for (int l = 0; l < L; ++l) {
    for (size_t k = 0; k < p.lead.size(); ++k) {
      const int f = p.lead[k];
      if (memcmp(&p.s[l], &p.s[f], sizeof(double)) == 0 && memcmp(&p.ls[(size_t)l * d], &p.ls[(size_t)f * d], d * sizeof(double)) == 0) {
        p.kof[l] = (int)k;
        break;
      }
    }
    if (p.kof[l] < 0) {
      p.kof[l] = (int)p.lead.size();
      p.lead.push_back(l);
    }
  }
  const int K = (int)p.lead.size();
  std::vector<double> kinv((size_t)K * d), ks(K), dadd(K, st->jitter);
  for (int k = 0; k < K; ++k) {
    ks[k] = p.s[p.lead[k]];
    memcpy(&kinv[(size_t)k * d], &p.inv[(size_t)p.lead[k] * d], d * sizeof(double));
  }
  p.zero.assign((size_t)K * st->Z, 0.0);
  DMO_TRY(upload(ctx, p.d_inv, kinv));
  DMO_TRY(upload(ctx, p.d_s, ks));
  DMO_TRY(upload(ctx, p.d_dadd, dadd));
  DMO_TRY(upload(ctx, p.d_noise, p.noise));
  DMO_TRY(upload(ctx, p.d_W, p.W));
  DMO_TRY(upload(ctx, p.d_zero, p.zero));
  DMO_TRY(upload(ctx, p.d_batch, p.batch));
  return DMO_OK;
}

// Per distinct kernel k: the factor Lf_k (rows of ld) of K(Z, Z) + jitter I, Li_k = Lz^-1 (Z x Z), and A_k (Z x B); the
// scaled inducing points zs_k and batch points xs_k (SVGP).  Reads the Cholesky info back (synchronises).
struct SvfKernels {
  DevBuf<double> Lf, Li, A, zs, xs, work;
  DevBuf<int> info;
};

int svf_kernels(dmo_ctx* ctx, const char* who, dmo_svgp_fit* st, const SvfParams& p, int64_t B, SvfKernels& kk) {
  const int K = (int)p.lead.size(), d = st->d;
  const int64_t Z = st->Z, ld = st->ld, zz = Z * Z;
  DMO_TRY(kk.Lf.alloc(ctx, (size_t)K * ld * ld));
  DMO_TRY(kk.Li.alloc(ctx, (size_t)K * zz));
  DMO_TRY(kk.A.alloc(ctx, (size_t)K * Z * B));
  DMO_TRY(kk.zs.alloc(ctx, (size_t)K * Z * d));
  DMO_TRY(kk.xs.alloc(ctx, (size_t)K * B * d));
  DMO_TRY(kk.work.alloc(ctx, (size_t)K * ld));
  DMO_TRY(kk.info.alloc(ctx, K));
  DMO_CUDA(cudaMemsetAsync(kk.info.p, 0, K * sizeof(int), ctx->stream));
  DMO_CUDA(cudaMemsetAsync(kk.Li.p, 0, (size_t)K * zz * sizeof(double), ctx->stream));
  DMO_TRY(gp_fit_batched(ctx, Z, d, K, DMO_KERNEL_MATERN52, st->Zp.p, p.d_inv.p, p.d_s.p, p.d_dadd.p, p.d_zero.p, kk.Lf.p, ld, kk.info.p,
                         kk.work.p, nullptr, nullptr));
  std::vector<int> h_info(K);
  DMO_CUDA(cudaMemcpyAsync(h_info.data(), kk.info.p, K * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  for (int k = 0; k < K; ++k)
    if (h_info[k]) return dmo_fail(ctx, DMO_ERR_ARG, "%s: K(Z, Z) + jitter I of latent %d is not positive definite", who, p.lead[k]);
  DMO_TRY(gp_linv_from_factor_batched(ctx, kk.Lf.p, ld, ld * ld, Z, K, Z, zz, kk.Li.p));
  for (int k = 0; k < K; ++k) {
    const double* inv = p.d_inv.p + (size_t)k * d;
    double* zs = kk.zs.p + (size_t)k * Z * d;
    double* A = kk.A.p + (size_t)k * Z * B;
    DMO_LAUNCH(svf_scale_rows_kernel, (unsigned)ceil_div(Z * d, 256), 256, 0, st->Zp.p, nullptr, Z, d, inv, zs);
    if (st->vgp) {
      DMO_LAUNCH(svf_gather_cols_kernel, (unsigned)ceil_div(Z * B, 256), 256, 0, kk.Lf.p + (size_t)k * ld * ld, ld, p.d_batch.p, Z, B, A);
    } else {
      double* xs = kk.xs.p + (size_t)k * B * d;
      DevBuf<double> Kzb;
      DMO_TRY(Kzb.alloc(ctx, (size_t)Z * B));
      DMO_LAUNCH(svf_scale_rows_kernel, (unsigned)ceil_div(B * d, 256), 256, 0, st->X.p, p.d_batch.p, B, d, inv, xs);
      DMO_LAUNCH(svf_cross_kernel, (unsigned)ceil_div(Z * B, 256), 256, 0, zs, Z, xs, B, d, p.s[p.lead[k]], Kzb.p);
      DMO_TRY(sv_gemm(ctx, Z, B, Z, 1.0, kk.Li.p + (size_t)k * zz, Z, 1, Kzb.p, B, 1, 0.0, A, B));  // A = Lz^-1 K(Z, X_b)
    }
  }
  return DMO_OK;
}

// mu (L,B) at the current q; T = U' A and v (L,B) when T is not NULL
int svf_moments(dmo_ctx* ctx, dmo_svgp_fit* st, const SvfParams& p, const SvfKernels& kk, int64_t B, double* mu, double* T, double* v) {
  const int64_t Z = st->Z, zz = Z * Z;
  for (int l = 0; l < st->L; ++l) {
    const double* A = kk.A.p + (size_t)p.kof[l] * Z * B;
    const double* m = st->m.p + (size_t)l * Z;
    if (T) {
      double* Tl = T + (size_t)l * Z * B;
      DMO_TRY(sv_gemm(ctx, Z, B, Z, 1.0, st->U.p + (size_t)l * zz, 1, Z, A, B, 1, 0.0, Tl, B));  // U' A
      DMO_LAUNCH(svf_colstats_kernel, (unsigned)ceil_div(B, 128), 128, 0, A, Tl, m, Z, B, p.s[l], st->vgp ? 0 : 1, mu + (size_t)l * B,
                 v + (size_t)l * B);
    } else {
      DMO_TRY(sv_gemm(ctx, B, 1, Z, 1.0, A, 1, B, m, 1, 0, 0.0, mu + (size_t)l * B, 1));  // A' m
    }
  }
  return DMO_OK;
}

}  // namespace

extern "C" {

int dmo_svgp_fit_create(dmo_ctx* ctx, int64_t N, int d, int M, int L, int64_t Z, const double* X, const double* Y, const double* Zpts,
                        int inducing_is_data, double jitter, dmo_svgp_fit** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out, "svgp_fit_create: null output");
  *out = nullptr;
  DMO_REQUIRE(L >= 1 && L <= SVF_MAX && M >= 1 && M <= SVF_MAX, "svgp_fit_create: 1 <= L, M <= %d (got L=%d M=%d)", SVF_MAX, L, M);
  DMO_REQUIRE(N >= 1 && Z >= 1 && Z <= SVF_ZMAX && d >= 1 && d <= MT_FIT_DMAX,
              "svgp_fit_create: unsupported shape N=%lld Z=%lld d=%d (Z <= %lld, d <= %d)", (long long)N, (long long)Z, d,
              (long long)SVF_ZMAX, MT_FIT_DMAX);
  DMO_REQUIRE(X && Y && (Zpts || inducing_is_data), "svgp_fit_create: null pointer");
  DMO_REQUIRE(!inducing_is_data || Z == N, "svgp_fit_create: with inducing_is_data Z must equal N (got Z=%lld N=%lld)", (long long)Z,
              (long long)N);
  DMO_REQUIRE(jitter >= 0.0 && isfinite(jitter), "svgp_fit_create: jitter must be finite and >= 0 (got %g)", jitter);
  std::unique_ptr<dmo_svgp_fit> st(new dmo_svgp_fit());
  st->N = N;
  st->Z = Z;
  st->d = d;
  st->M = M;
  st->L = L;
  st->vgp = inducing_is_data != 0;
  st->jitter = jitter;
  st->ld = ceil_div(Z + 1, 64) * 64;
  st->lc = ceil_div(Z, 64) * 64;
  std::vector<double> hx((size_t)N * d), hy((size_t)M * N), hz((size_t)Z * d);
  DMO_CUDA(cudaMemcpy(hx.data(), X, hx.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hy.data(), Y, hy.size() * sizeof(double), cudaMemcpyDefault));
  if (st->vgp)
    hz = hx;
  else
    DMO_CUDA(cudaMemcpy(hz.data(), Zpts, hz.size() * sizeof(double), cudaMemcpyDefault));
  DMO_TRY(upload(ctx, st->X, hx));
  DMO_TRY(upload(ctx, st->Y, hy));
  DMO_TRY(upload(ctx, st->Zp, hz));
  // q = N(0, I): Lambda = I, theta1 = 0, U = I, m = 0
  std::vector<double> eye((size_t)L * Z * Z, 0.0), zero((size_t)L * Z, 0.0);
  for (int l = 0; l < L; ++l)
    for (int64_t i = 0; i < Z; ++i) eye[((size_t)l * Z + i) * Z + i] = 1.0;
  DMO_TRY(upload(ctx, st->Lam, eye));
  DMO_TRY(upload(ctx, st->U, eye));
  DMO_TRY(upload(ctx, st->th1, zero));
  DMO_TRY(upload(ctx, st->m, zero));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  *out = st.release();
  return DMO_OK;
}

int dmo_svgp_fit_destroy(dmo_ctx* ctx, dmo_svgp_fit* st) {
  if (!ctx) return DMO_ERR_ARG;
  if (!st) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  delete st;
  return DMO_OK;
}

int dmo_svgp_fit_natgrad(dmo_ctx* ctx, dmo_svgp_fit* st, const int64_t* batch, int64_t B, const double* variance,
                         const double* length_scale, const double* noise, const double* W, double gamma) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st, "svgp_fit_natgrad: null state");
  DMO_REQUIRE(gamma > 0.0 && gamma <= 1.0, "svgp_fit_natgrad: gamma must be in (0, 1] (got %g)", gamma);
  SvfParams p;
  DMO_TRY(svf_params(ctx, "svgp_fit_natgrad", st, batch, B, variance, length_scale, noise, W, p));
  SvfKernels kk;
  DMO_TRY(svf_kernels(ctx, "svgp_fit_natgrad", st, p, B, kk));
  const int L = st->L, M = st->M;
  const int64_t Z = st->Z, zz = Z * Z, lc = st->lc;
  const double scale = (double)st->N / (double)B;
  DevBuf<double> mu, rt, Ar, G, LamJ, Lci;
  DevBuf<int> info;
  DMO_TRY(mu.alloc(ctx, (size_t)L * B));
  DMO_TRY(rt.alloc(ctx, (size_t)B));
  DMO_TRY(Ar.alloc(ctx, (size_t)Z));
  DMO_TRY(G.alloc(ctx, zz));
  DMO_TRY(LamJ.alloc(ctx, (size_t)L * lc * lc));
  DMO_TRY(Lci.alloc(ctx, (size_t)L * zz));
  DMO_TRY(info.alloc(ctx, L));
  DMO_TRY(svf_moments(ctx, st, p, kk, B, mu.p, nullptr, nullptr));  // every latent's mean at the current q
  for (int l = 0; l < L; ++l) {
    const double* A = kk.A.p + (size_t)p.kof[l] * Z * B;
    double c = 0.0;
    for (int m = 0; m < M; ++m) c += p.W[(size_t)m * L + l] * p.W[(size_t)m * L + l] / p.noise[m];
    DMO_LAUNCH(svf_rtilde_kernel, (unsigned)ceil_div(B, 128), 128, 0, st->Y.p, st->N, p.d_batch.p, B, M, L, l, p.d_W.p, p.d_noise.p, mu.p,
               rt.p);
    DMO_TRY(sv_gemm(ctx, Z, Z, B, scale * c, A, B, 1, A, 1, B, 0.0, G.p, Z));         // G = (N / B) c A A'
    DMO_TRY(sv_gemm(ctx, Z, 1, B, scale, A, B, 1, rt.p, 1, 0, 0.0, Ar.p, 1));          // (N / B) A r~
    DMO_LAUNCH(svf_blend_kernel, (unsigned)ceil_div(lc * lc, 256), 256, 0, st->Lam.p + (size_t)l * zz, G.p, Z, lc, gamma,
               st->th1.p + (size_t)l * Z, Ar.p, LamJ.p + (size_t)l * lc * lc);
  }
  DMO_CUDA(cudaMemsetAsync(info.p, 0, L * sizeof(int), ctx->stream));
  DMO_TRY(gp_potrf_batched(ctx, LamJ.p, lc, L, info.p));
  std::vector<int> h_info(L);
  DMO_CUDA(cudaMemcpyAsync(h_info.data(), info.p, L * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  for (int l = 0; l < L; ++l)
    if (h_info[l]) return dmo_fail(ctx, DMO_ERR_ARG, "svgp_fit_natgrad: the precision Lambda of latent %d is not positive definite", l);
  DMO_CUDA(cudaMemsetAsync(Lci.p, 0, (size_t)L * zz * sizeof(double), ctx->stream));
  DMO_TRY(gp_linv_from_factor_batched(ctx, LamJ.p, lc, lc * lc, Z, L, Z, zz, Lci.p));
  for (int l = 0; l < L; ++l) {
    double* U = st->U.p + (size_t)l * zz;
    DMO_TRY(sv_flip(ctx, Lci.p + (size_t)l * zz, Z, 1.0, U, Z));  // U = J Lc^-T J, S = U U' = Lambda^-1
    // m = U (U' theta1)
    DMO_TRY(sv_gemm(ctx, Z, 1, Z, 1.0, U, 1, Z, st->th1.p + (size_t)l * Z, 1, 0, 0.0, Ar.p, 1));
    DMO_TRY(sv_gemm(ctx, Z, 1, Z, 1.0, U, Z, 1, Ar.p, 1, 0, 0.0, st->m.p + (size_t)l * Z, 1));
  }
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_svgp_fit_elbo_grad(dmo_ctx* ctx, dmo_svgp_fit* st, const int64_t* batch, int64_t B, const double* variance,
                           const double* length_scale, const double* noise, const double* W, double* ell_out, double* kl_out,
                           double* g_variance, double* g_length_scale, double* g_noise, double* g_W) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st, "svgp_fit_elbo_grad: null state");
  DMO_REQUIRE(ell_out && kl_out, "svgp_fit_elbo_grad: null output");
  const bool grad = g_variance || g_length_scale || g_noise || g_W;
  DMO_REQUIRE(!grad || (g_variance && g_length_scale && g_noise), "svgp_fit_elbo_grad: g_variance, g_length_scale and g_noise go together");
  DMO_REQUIRE(!g_W || W, "svgp_fit_elbo_grad: g_W needs W");
  SvfParams p;
  DMO_TRY(svf_params(ctx, "svgp_fit_elbo_grad", st, batch, B, variance, length_scale, noise, W, p));
  SvfKernels kk;
  DMO_TRY(svf_kernels(ctx, "svgp_fit_elbo_grad", st, p, B, kk));
  const int L = st->L, M = st->M, d = st->d;
  const int64_t Z = st->Z, zz = Z * Z, ld = st->ld;
  const double scale = (double)st->N / (double)B;
  Out<double> o_ell, o_kl, o_gs, o_gl, o_gn, o_gw;
  DMO_TRY(o_ell.init(ctx, ell_out, M));
  DMO_TRY(o_kl.init(ctx, kl_out, L));
  DMO_TRY(o_gs.init(ctx, g_variance, L));
  DMO_TRY(o_gl.init(ctx, g_length_scale, (size_t)L * d));
  DMO_TRY(o_gn.init(ctx, g_noise, M));
  DMO_TRY(o_gw.init(ctx, g_W, (size_t)M * L));
  DevBuf<double> mu, v, T, r, mubar, vbar, gn;
  DMO_TRY(mu.alloc(ctx, (size_t)L * B));
  DMO_TRY(v.alloc(ctx, (size_t)L * B));
  DMO_TRY(T.alloc(ctx, (size_t)L * Z * B));
  DMO_TRY(r.alloc(ctx, (size_t)M * B));
  DMO_TRY(mubar.alloc(ctx, (size_t)L * B));
  DMO_TRY(vbar.alloc(ctx, L));
  DMO_TRY(gn.alloc(ctx, M));
  DMO_TRY(svf_moments(ctx, st, p, kk, B, mu.p, T.p, v.p));
  DMO_LAUNCH(svf_kl_kernel, (unsigned)L, 256, 0, st->U.p, st->m.p, Z, o_kl.d);
  DMO_LAUNCH(svf_ell_kernel, (unsigned)M, 256, 0, st->Y.p, st->N, p.d_batch.p, B, L, p.d_W.p, mu.p, v.p, p.d_noise.p, scale, r.p, o_ell.d,
             gn.p);
  if (grad) {
    DMO_CUDA(cudaMemcpyAsync(o_gn.d, gn.p, M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    DMO_LAUNCH(svf_latent_bar_kernel, (unsigned)L, 256, 0, M, L, B, p.d_W.p, p.d_noise.p, r.p, mu.p, v.p, scale, mubar.p, vbar.p, o_gw.d);
    DevBuf<double> SA, Abar, Kzb_bar, Lbar, Pm, T1, Xm, Kzz_bar, part, d_ls;
    DMO_TRY(SA.alloc(ctx, (size_t)Z * B));
    DMO_TRY(Abar.alloc(ctx, (size_t)Z * B));
    if (!st->vgp) DMO_TRY(Kzb_bar.alloc(ctx, (size_t)Z * B));
    DMO_TRY(Lbar.alloc(ctx, zz));
    DMO_TRY(Pm.alloc(ctx, zz));
    DMO_TRY(T1.alloc(ctx, zz));
    DMO_TRY(Xm.alloc(ctx, zz));
    DMO_TRY(Kzz_bar.alloc(ctx, zz));
    DMO_TRY(part.alloc(ctx, (size_t)Z * (d + 1)));
    DMO_TRY(upload(ctx, d_ls, p.ls));
    for (int l = 0; l < L; ++l) {
      const int k = p.kof[l];
      const double* A = kk.A.p + (size_t)k * Z * B;
      const double* Li = kk.Li.p + (size_t)k * zz;
      const double* Lf = kk.Lf.p + (size_t)k * ld * ld;
      // S A = U (U' A)
      DMO_TRY(sv_gemm(ctx, Z, B, Z, 1.0, st->U.p + (size_t)l * zz, Z, 1, T.p + (size_t)l * Z * B, B, 1, 0.0, SA.p, B));
      DMO_LAUNCH(svf_abar_kernel, (unsigned)ceil_div(Z * B, 256), 256, 0, Z, B, st->m.p + (size_t)l * Z, mubar.p + (size_t)l * B, vbar.p + l,
                 SA.p, A, st->vgp ? 0 : 1, Abar.p);
      if (st->vgp) {
        DMO_LAUNCH(svf_scatter_rows_kernel, (unsigned)ceil_div(zz, 256), 256, 0, Abar.p, p.d_batch.p, Z, Lbar.p);
      } else {
        DMO_TRY(sv_gemm(ctx, Z, B, Z, 1.0, Li, 1, Z, Abar.p, B, 1, 0.0, Kzb_bar.p, B));   // Lz^-T A_bar
        DMO_TRY(sv_gemm(ctx, Z, Z, B, -1.0, Kzb_bar.p, B, 1, A, 1, B, 0.0, Lbar.p, Z));   // -K_zb_bar A'
        DMO_LAUNCH(svf_tril_kernel, (unsigned)ceil_div(zz, 256), 256, 0, Lbar.p, Z, 1.0);
      }
      // Cholesky backward: P = Phi(Lz' Lbar), X = Lz^-T P Lz^-1, Kzz_bar = (X + X') / 2
      DMO_TRY(sv_gemm(ctx, Z, Z, Z, 1.0, Lf, 1, ld, Lbar.p, Z, 1, 0.0, Pm.p, Z));
      DMO_LAUNCH(svf_tril_kernel, (unsigned)ceil_div(zz, 256), 256, 0, Pm.p, Z, 0.5);
      DMO_TRY(sv_gemm(ctx, Z, Z, Z, 1.0, Pm.p, Z, 1, Li, Z, 1, 0.0, T1.p, Z));
      DMO_TRY(sv_gemm(ctx, Z, Z, Z, 1.0, Li, 1, Z, T1.p, Z, 1, 0.0, Xm.p, Z));
      DMO_LAUNCH(svf_sym_kernel, (unsigned)ceil_div(zz, 256), 256, 0, Xm.p, Z, Kzz_bar.p);
      DMO_LAUNCH(svf_grad_pass_kernel, (unsigned)Z, 256, 0, kk.zs.p + (size_t)k * Z * d, Z, kk.xs.p + (size_t)k * B * d, st->vgp ? 0 : B, d,
                 p.s[l], Kzz_bar.p, st->vgp ? nullptr : Kzb_bar.p, part.p);
      DMO_LAUNCH(svf_fold_kernel, 1, 128, 0, part.p, Z, d, d_ls.p + (size_t)l * d, vbar.p + l, st->vgp ? 0.0 : (double)B,
                 o_gl.d + (size_t)l * d, o_gs.d + l);
    }
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(o_ell.finish(ctx));
  DMO_TRY(o_kl.finish(ctx));
  DMO_TRY(o_gs.finish(ctx));
  DMO_TRY(o_gl.finish(ctx));
  DMO_TRY(o_gn.finish(ctx));
  DMO_TRY(o_gw.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_svgp_fit_q(dmo_ctx* ctx, dmo_svgp_fit* st, double* q_mu_out, double* q_sqrt_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st && q_mu_out && q_sqrt_out, "svgp_fit_q: null argument");
  const size_t zz = (size_t)st->Z * st->Z;
  DMO_CUDA(cudaMemcpyAsync(q_mu_out, st->m.p, (size_t)st->L * st->Z * sizeof(double), cudaMemcpyDefault, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(q_sqrt_out, st->U.p, st->L * zz * sizeof(double), cudaMemcpyDefault, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
