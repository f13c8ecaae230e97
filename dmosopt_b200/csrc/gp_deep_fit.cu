// Training of the two-layer deep GPs behind dmosopt's MDSPP_Matern and MDGP_Matern (gpytorch's DSPP and DeepGP,
// dmosopt/model_gpytorch.py:185-247, 359-416, 991-1585): a device-resident state holding the data, a flat float64 vector
// of raw parameters, its gradient and the Adam moments, and the minibatch loss with its full gradient.
//
// Units u < U = H + T: the H hidden units (over the normalised x, d dims, one (Z1, d) inducing matrix shared by all
// units) and the T last-layer units (over the layer-2 inputs, H dims, (Z2, H) inducing points per task).  Per unit
// (s the output scale, ell the isotropic length scale, k_u the unit Matern-5/2 kernel, jitter 1e-4 in the models):
//   Kzz = s k_u(Z, Z) + jitter I = Lz Lz',  a = Lz^-1 s k_u(Z, x),  m = prior(x) + a' mu,  v = s + jitter - a'a + ||Lq' a||^2
// with Lq = tril(chol_variational_covar).  Hidden: sd1 = sqrt(max(v1, min_var)), u_ij = m1_i + e_ij o sd1_i (e the
// quadrature sites, or N(0, I) draws from Philox4x32-10 keyed by (seed, step, row)).  Rows r = j B + i of the last layer.
//   loss = (1 / (J B)) sum_r sum_t 1/2 [((y - m)^2 + max(v, min_var)) / sigma2_t + log sigma2_t + log 2 pi] + sum_u KL_u / N
//   KL_u = 1/2 (||Lq||_F^2 + mu'mu - Z - sum log Lq_ii^2)
//
// Backward per unit, with m_bar, v_bar per row: a_bar = m_bar mu + 2 v_bar (Lq Lq' a - a), K_bar = Lz^-T a_bar (d loss /
// d s k_u(Z, x)), mu_bar = sum_r m_bar a, Lq_bar = tril(2 sum_r v_bar a (Lq' a)'), Lz_bar = -tril(sum_r K_bar a'), and the
// Cholesky backward pass (Murray 2016, arXiv:1602.07527): Kzz_bar = (X + X') / 2, X = Lz^-T Phi(Lz' Lz_bar) Lz^-1.  The
// kernel derivatives: with q = sqrt(5) r and w = K_bar s (5/3)(1 + q) e^-q, d/dz_i = -w (z_i - x) / ell^2,
// d/dx = +w (z_i - x) / ell^2, d/d ell = w r^2 / ell, d/ds = K_bar k_u.
//
// Kernels of one step (11 launches; Adam is a 12th): dgf_factor_kernel (one CTA per unit: Kzz and its Cholesky factor
// in shared memory, KL), dgf_rows_fwd_kernel (one CTA per unit and 32 rows: K* tile in shared memory, a by a
// triangular solve against Lz in shared memory, Lq' a; hidden layer, then last layer), dgf_hidden_out_kernel (sd1,
// draws, layer-2 inputs), dgf_ell_kernel, dgf_rows_bwd_kernel (last layer, then hidden), dgf_hidden_bar_kernel,
// dgf_gram_kernel (Lq_bar and Lz_bar partial sums over row chunks), dgf_unit_bwd_kernel (one CTA per unit: the
// Cholesky backward in shared memory and every per-unit gradient block), dgf_assemble_kernel (the loss and the shared
// blocks).  Float64; every sum runs in a fixed order and no kernel uses atomics, so repeated calls are bit-identical.
#include <math.h>
#include <string.h>

#include <memory>
#include <vector>

#include "gp.cuh"

namespace {

constexpr int DF_MAX_HT = 8;
constexpr int DF_ZMAX = 128;
constexpr int DF_RT = 32;    // rows per CTA of the row kernels
constexpr int DF_RC = 512;   // rows per chunk of the Gram partial sums
constexpr int64_t DF_MAX_ROWS = (int64_t)1 << 16;  // J * batch_max
constexpr double DF_LOG_2PI = 1.8378770664093453;

struct DfLayout {
  int d, H, T, J, Z1, Z2, ZS;
  int quadrature, bounded;
  double lo, hi, jitter, min_var;
  int64_t N;
  // offsets of the blocks of the flat raw-parameter vector (see dmosopt_b200.h) and its length
  int64_t oZ1, ols1, oos1, omu1, och1, ow, ob, oZ2, ols2, oos2, omu2, och2, oc, otn, on, osite, P;
};

struct DfUnit {
  int Z, D;
  int64_t ozp, ols, oos, omu, och;
};

__host__ __device__ inline DfUnit df_unit(const DfLayout& L, int u) {
  DfUnit v;
  if (u < L.H) {
    v.Z = L.Z1;
    v.D = L.d;
    v.ozp = L.oZ1;
    v.ols = L.ols1 + u;
    v.oos = L.oos1 + u;
    v.omu = L.omu1 + (int64_t)u * L.Z1;
    v.och = L.och1 + (int64_t)u * L.Z1 * L.Z1;
  } else {
    const int t = u - L.H;
    v.Z = L.Z2;
    v.D = L.H;
    v.ozp = L.oZ2 + (int64_t)t * L.Z2 * L.H;
    v.ols = L.ols2 + t;
    v.oos = L.oos2 + t;
    v.omu = L.omu2 + (int64_t)t * L.Z2;
    v.och = L.och2 + (int64_t)t * L.Z2 * L.Z2;
  }
  return v;
}

// torch.nn.functional.softplus (threshold 20) and its derivative
__device__ __forceinline__ double df_softplus(double x) { return x > 20.0 ? x : log1p(exp(x)); }
__device__ __forceinline__ double df_softplus_grad(double x) {
  if (x > 20.0) return 1.0;
  const double z = exp(x);
  return z / (z + 1.0);
}
__device__ __forceinline__ double df_sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }
__device__ __forceinline__ double df_lscale(const DfLayout& L, double x) {
  return L.bounded ? L.lo + (L.hi - L.lo) * df_sigmoid(x) : df_softplus(x);
}
__device__ __forceinline__ double df_lscale_grad(const DfLayout& L, double x) {
  if (!L.bounded) return df_softplus_grad(x);
  const double s = df_sigmoid(x);
  return (L.hi - L.lo) * (s * (1.0 - s));
}

// scaled squared distance ||(a - b) / ell||^2
__device__ __forceinline__ double df_d2(const double* a, const double* b, int D, double il) {
  double s = 0.0;
  for (int c = 0; c < D; ++c) {
    const double t = (a[c] - b[c]) * il;
    s = fma(t, t, s);
  }
  return s;
}

// One CTA per unit: Kzz and its Cholesky factor in shared memory (a non-positive pivot is recorded in info[u] and
// replaced by 1 so that the step stays finite), Lz to global (rows of ZS), and KL_u
__global__ void __launch_bounds__(256) dgf_factor_kernel(DfLayout L, const double* __restrict__ p, double* __restrict__ Lzg,
                                                         int* __restrict__ info, double* __restrict__ kl) {
  extern __shared__ double S[];
  __shared__ double red[8];
  __shared__ int bad;
  const int u = blockIdx.x, tid = threadIdx.x;
  const DfUnit v = df_unit(L, u);
  const int Z = v.Z, D = v.D;
  const double s = df_softplus(p[v.oos]), il = 1.0 / df_lscale(L, p[v.ols]);
  const double* zp = p + v.ozp;
  if (tid == 0) bad = 0;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, j = e - i * Z;
    double val = 0.0;
    if (j <= i) {
      // sqrt(5 d2) rounds differently from gp.cuh's stationary (sqrt(d2) sqrt(5)): the deep GP keeps its own Matern
      const double q = sqrt(5.0 * df_d2(zp + (size_t)i * D, zp + (size_t)j * D, D, il));
      val = s * ((1.0 + q + q * q / 3.0) * exp(-q));
      if (i == j) val += L.jitter;
    }
    S[e] = val;
  }
  __syncthreads();
  for (int k = 0; k < Z; ++k) {
    if (tid == 0) {
      double piv = S[k * Z + k];
      if (!(piv > 0.0) || !isfinite(piv)) {
        if (!bad) bad = k + 1;
        piv = 1.0;
      }
      S[k * Z + k] = sqrt(piv);
    }
    __syncthreads();
    const double dk = S[k * Z + k];
    for (int i = k + 1 + tid; i < Z; i += 256) S[i * Z + k] /= dk;
    __syncthreads();
    const int n = Z - k - 1;
    for (int e = tid; e < n * n; e += 256) {
      const int i = k + 1 + e / n, j = k + 1 + e % n;
      if (j <= i) S[i * Z + j] = fma(-S[i * Z + k], S[j * Z + k], S[i * Z + j]);
    }
    __syncthreads();
  }
  double* Lz = Lzg + (size_t)u * L.ZS * L.ZS;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, j = e - i * Z;
    Lz[(size_t)i * L.ZS + j] = j <= i ? S[e] : 0.0;
  }
  const double* ch = p + v.och;
  const double* mu = p + v.omu;
  double q = 0.0, ld = 0.0;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, j = e - i * Z;
    if (j <= i) q = fma(ch[e], ch[e], q);
  }
  for (int k = tid; k < Z; k += 256) {
    q = fma(mu[k], mu[k], q);
    ld += log(ch[k * Z + k] * ch[k * Z + k]);
  }
  q = block_sum<8>(q, red);
  ld = block_sum<8>(ld, red);
  if (tid == 0) {
    kl[u] = 0.5 * ((q - (double)Z) - ld);
    if (bad) info[u] = bad;
  }
}

// K* tile Xt[k][rr] = s k_u(z_k, x_r) of rows r0 + rr < R (zero beyond)
__device__ void df_kstar_tile(const double* zp, int Z, int D, double s, double il, const double* xr, const int64_t* idx, int64_t r0,
                              int nr, double* Xt) {
  for (int e = threadIdx.x; e < Z * DF_RT; e += 256) {
    const int k = e / DF_RT, rr = e - k * DF_RT;
    double val = 0.0;
    if (rr < nr) {
      const int64_t r = r0 + rr;
      const double* x = xr + (size_t)(idx ? idx[r] : r) * D;
      const double q = sqrt(5.0 * df_d2(zp + (size_t)k * D, x, D, il));
      val = s * ((1.0 + q + q * q / 3.0) * exp(-q));
    }
    Xt[e] = val;
  }
}

// Ls <- the lower triangle of a unit matrix (rows of ld)
__device__ void df_load_lower(const double* src, int64_t ld, int Z, double* Ls) {
  for (int e = threadIdx.x; e < Z * Z; e += 256) {
    const int i = e / Z, j = e - i * Z;
    Ls[e] = j <= i ? src[(size_t)i * ld + j] : 0.0;
  }
}

// One CTA per (unit u0 + blockIdx.y, 32 rows): A = Lz^-1 K* and G = Lq' A (Z x rows, to global with rows of RS), and
// per row mb = a' mu, vb = s + jitter - a'a + g'g
__global__ void __launch_bounds__(256, 1)
    dgf_rows_fwd_kernel(DfLayout L, const double* __restrict__ p, int u0, const double* __restrict__ xr, const int64_t* __restrict__ idx,
                        int64_t R, int64_t RS, const double* __restrict__ Lzg, double* __restrict__ A, double* __restrict__ G,
                        double* __restrict__ mb, double* __restrict__ vb) {
  extern __shared__ double sm[];
  const int u = u0 + blockIdx.y, tid = threadIdx.x;
  const DfUnit v = df_unit(L, u);
  const int Z = v.Z, D = v.D;
  double* Ls = sm;
  double* Xt = sm + L.ZS * L.ZS;
  double* Gt = Xt + L.ZS * DF_RT;
  const int64_t r0 = (int64_t)blockIdx.x * DF_RT;
  const int nr = (int)(R - r0 < DF_RT ? R - r0 : DF_RT);
  const double s = df_softplus(p[v.oos]), il = 1.0 / df_lscale(L, p[v.ols]);
  df_load_lower(Lzg + (size_t)u * L.ZS * L.ZS, L.ZS, Z, Ls);
  df_kstar_tile(p + v.ozp, Z, D, s, il, xr, idx, r0, nr, Xt);
  __syncthreads();
  for (int i = 0; i < Z; ++i) {  // forward substitution, all columns at once
    if (tid < DF_RT) Xt[i * DF_RT + tid] /= Ls[i * Z + i];
    __syncthreads();
    for (int e = tid; e < (Z - i - 1) * DF_RT; e += 256) {
      const int k = i + 1 + e / DF_RT, rr = e % DF_RT;
      Xt[k * DF_RT + rr] = fma(-Ls[k * Z + i], Xt[i * DF_RT + rr], Xt[k * DF_RT + rr]);
    }
    __syncthreads();
  }
  df_load_lower(p + v.och, Z, Z, Ls);
  __syncthreads();
  for (int e = tid; e < Z * DF_RT; e += 256) {
    const int k = e / DF_RT, rr = e - k * DF_RT;
    double g = 0.0;
    for (int i = k; i < Z; ++i) g = fma(Ls[i * Z + k], Xt[i * DF_RT + rr], g);
    Gt[e] = g;
  }
  __syncthreads();
  const size_t ub = (size_t)u * L.ZS * RS;
  for (int e = tid; e < Z * DF_RT; e += 256) {
    const int k = e / DF_RT, rr = e - k * DF_RT;
    if (rr < nr) {
      A[ub + (size_t)k * RS + r0 + rr] = Xt[e];
      G[ub + (size_t)k * RS + r0 + rr] = Gt[e];
    }
  }
  if (tid < nr) {
    const double* mu = p + v.omu;
    double m = 0.0, aa = 0.0, gg = 0.0;
    for (int k = 0; k < Z; ++k) {
      const double a = Xt[k * DF_RT + tid], g = Gt[k * DF_RT + tid];
      m = fma(a, mu[k], m);
      aa = fma(a, a, aa);
      gg = fma(g, g, gg);
    }
    mb[(size_t)u * RS + r0 + tid] = m;
    vb[(size_t)u * RS + r0 + tid] = ((s + L.jitter) - aa) + gg;
  }
}

// per (batch row i, hidden unit h): m1 = w . x + b + mb, sd1 = sqrt(max(v1, min_var)); for every site j the draw or
// site e (into eps, (J, B, H)) and the layer-2 input U[j B + i][h] = m1 + e sd1
__global__ void dgf_hidden_out_kernel(DfLayout L, const double* __restrict__ p, const double* __restrict__ X, const int64_t* __restrict__ batch,
                                      int64_t B, int64_t RS, const double* __restrict__ mb, const double* __restrict__ vb,
                                      const double* __restrict__ eps_in, uint64_t seed, uint64_t step, double* __restrict__ eps,
                                      double* __restrict__ U) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = L.H, d = L.d;
  if (t >= B * H) return;
  const int64_t i = t / H;
  const int h = (int)(t - i * H);
  const double* x = X + (size_t)batch[i] * d;
  double m = 0.0;
  for (int c = 0; c < d; ++c) m = fma(x[c], p[L.ow + c], m);
  m = (m + p[L.ob]) + mb[(size_t)h * RS + i];
  const double sd = sqrt(fmax(vb[(size_t)h * RS + i], L.min_var));
  for (int j = 0; j < L.J; ++j) {
    const size_t o = ((size_t)j * B + i) * H + h;
    double e;
    if (L.quadrature) {
      e = p[L.osite + j * H + h];
    } else if (eps_in) {
      e = eps_in[o];
    } else {
      const uint4 q = Philox(seed)(step, ((uint64_t)i << 32) | (uint64_t)(j * H + h));
      const double u1 = u01_53(q.x, q.y), u2 = u01_53(q.z, q.w);
      e = sqrt(-2.0 * log1p(-u1)) * cospi(2.0 * u2);  // Box-Muller; 1 - u1 lies in (0, 1]
    }
    eps[o] = e;
    U[o] = fma(e, sd, m);
  }
}

// per (row r, task t): the loss term, m_bar, v_bar of the last-layer unit, and d loss / d sigma2_t
__global__ void dgf_ell_kernel(DfLayout L, const double* __restrict__ p, const double* __restrict__ Y, const int64_t* __restrict__ batch,
                               int64_t B, int64_t RS, const double* __restrict__ mb, const double* __restrict__ vb, double* __restrict__ lterm,
                               double* __restrict__ sterm, double* __restrict__ mbar, double* __restrict__ vbar) {
  const int64_t R = (int64_t)L.J * B;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= R * L.T) return;
  const int t = (int)(e / R);
  const int64_t r = e - (int64_t)t * R, i = r % B;
  const size_t o = (size_t)(L.H + t) * RS + r;
  const double y = Y[(size_t)batch[i] * L.T + t];
  const double m = p[L.oc] + mb[o], v = vb[o], vc = fmax(v, L.min_var);
  const double s2 = (1e-4 + df_softplus(p[L.otn + t])) + (1e-4 + df_softplus(p[L.on]));
  const double sc = 1.0 / (double)R;
  const double dy = y - m, q = fma(dy, dy, vc);
  lterm[(size_t)t * RS + r] = 0.5 * ((q / s2 + log(s2)) + DF_LOG_2PI) * sc;
  sterm[(size_t)t * RS + r] = 0.5 * (1.0 / s2 - q / (s2 * s2)) * sc;
  mbar[o] = -(dy / s2) * sc;
  vbar[o] = v >= L.min_var ? 0.5 / s2 * sc : 0.0;
}

// One CTA per (unit, 32 rows): a_bar, K_bar = Lz^-T a_bar (to global), and the CTA's partial sums of the K(Z, x) terms:
// pz (Z, D) of d / dz, pmu (Z) of mu_bar, psc = {d / d ell, d / d s (with the direct sum of v_bar)}; ubar (rows, D) the
// input gradient when not NULL (last layer)
__global__ void __launch_bounds__(256, 1)
    dgf_rows_bwd_kernel(DfLayout L, const double* __restrict__ p, int u0, const double* __restrict__ xr, const int64_t* __restrict__ idx,
                        int64_t R, int64_t RS, const double* __restrict__ Lzg, const double* __restrict__ A, const double* __restrict__ G,
                        const double* __restrict__ mbar, const double* __restrict__ vbar, double* __restrict__ Kb, double* __restrict__ pz,
                        int64_t pz_unit, int64_t pz_base, int ctamax, double* __restrict__ pmu, double* __restrict__ psc,
                        double* __restrict__ ubar) {
  extern __shared__ double sm[];
  __shared__ double red[8];
  __shared__ double mbs[DF_RT], vbs[DF_RT];
  const int u = u0 + blockIdx.y, tid = threadIdx.x, cta = blockIdx.x;
  const DfUnit v = df_unit(L, u);
  const int Z = v.Z, D = v.D;
  double* Ls = sm;
  double* At = sm + L.ZS * L.ZS;
  double* Bt = At + L.ZS * DF_RT;
  const int64_t r0 = (int64_t)cta * DF_RT;
  const int nr = (int)(R - r0 < DF_RT ? R - r0 : DF_RT);
  const double s = df_softplus(p[v.oos]), ell = df_lscale(L, p[v.ols]), il = 1.0 / ell;
  const double* zp = p + v.ozp;
  const double* mu = p + v.omu;
  const size_t ub = (size_t)u * L.ZS * RS;
  for (int e = tid; e < Z * DF_RT; e += 256) {
    const int k = e / DF_RT, rr = e - k * DF_RT;
    const bool in = rr < nr;
    At[e] = in ? A[ub + (size_t)k * RS + r0 + rr] : 0.0;
    Bt[e] = in ? G[ub + (size_t)k * RS + r0 + rr] : 0.0;
  }
  if (tid < DF_RT) {
    mbs[tid] = tid < nr ? mbar[(size_t)u * RS + r0 + tid] : 0.0;
    vbs[tid] = tid < nr ? vbar[(size_t)u * RS + r0 + tid] : 0.0;
  }
  df_load_lower(p + v.och, Z, Z, Ls);
  __syncthreads();
  double reg[DF_ZMAX * DF_RT / 256];
  for (int qq = 0; qq < DF_ZMAX * DF_RT / 256; ++qq) {  // a_bar = m_bar mu + 2 v_bar (Lq g - a)
    const int e = tid + 256 * qq;
    reg[qq] = 0.0;
    if (e < Z * DF_RT) {
      const int i = e / DF_RT, rr = e - i * DF_RT;
      double lg = 0.0;
      for (int k = 0; k <= i; ++k) lg = fma(Ls[i * Z + k], Bt[k * DF_RT + rr], lg);
      reg[qq] = fma(mbs[rr], mu[i], 2.0 * vbs[rr] * (lg - At[e]));
    }
  }
  __syncthreads();
  for (int qq = 0; qq < DF_ZMAX * DF_RT / 256; ++qq) {
    const int e = tid + 256 * qq;
    if (e < Z * DF_RT) Bt[e] = reg[qq];
  }
  df_load_lower(Lzg + (size_t)u * L.ZS * L.ZS, L.ZS, Z, Ls);
  __syncthreads();
  for (int i = Z - 1; i >= 0; --i) {  // back substitution Lz' X = a_bar, all columns at once
    if (tid < DF_RT) Bt[i * DF_RT + tid] /= Ls[i * Z + i];
    __syncthreads();
    for (int e = tid; e < i * DF_RT; e += 256) {
      const int k = e / DF_RT, rr = e % DF_RT;
      Bt[k * DF_RT + rr] = fma(-Ls[i * Z + k], Bt[i * DF_RT + rr], Bt[k * DF_RT + rr]);
    }
    __syncthreads();
  }
  double ks = 0.0, dl = 0.0;
  for (int e = tid; e < Z * DF_RT; e += 256) {  // K_bar out, then the W tile in its place
    const int k = e / DF_RT, rr = e - k * DF_RT;
    double w = 0.0;
    if (rr < nr) {
      Kb[ub + (size_t)k * RS + r0 + rr] = Bt[e];
      const int64_t r = r0 + rr;
      const double* x = xr + (size_t)(idx ? idx[r] : r) * D;
      const double r2 = df_d2(zp + (size_t)k * D, x, D, il), q = sqrt(5.0 * r2), ex = exp(-q);
      ks = fma(Bt[e], (1.0 + q + q * q / 3.0) * ex, ks);
      w = Bt[e] * s * (5.0 / 3.0) * (1.0 + q) * ex;
      dl = fma(w, r2, dl);
    }
    Bt[e] = w;
  }
  ks = block_sum<8>(ks, red);  // synchronises: the W tile is complete
  dl = block_sum<8>(dl, red);
  const double il2 = il * il;
  double* pzc = pz + pz_base + (size_t)(u - u0) * pz_unit + (size_t)cta * Z * D;
  for (int e = tid; e < Z * D; e += 256) {
    const int k = e / D, c = e - k * D;
    double acc = 0.0;
    for (int rr = 0; rr < nr; ++rr) {
      const int64_t r = r0 + rr;
      acc = fma(Bt[k * DF_RT + rr], zp[(size_t)k * D + c] - xr[(size_t)(idx ? idx[r] : r) * D + c], acc);
    }
    pzc[e] = -il2 * acc;
  }
  if (ubar)
    for (int e = tid; e < nr * D; e += 256) {
      const int rr = e / D, c = e - rr * D;
      const int64_t r = r0 + rr;
      const double xc = xr[(size_t)r * D + c];
      double acc = 0.0;
      for (int k = 0; k < Z; ++k) acc = fma(Bt[k * DF_RT + rr], zp[(size_t)k * D + c] - xc, acc);
      ubar[(size_t)(u - u0) * RS * D + (size_t)r * D + c] = il2 * acc;
    }
  const size_t pc = (size_t)u * ctamax + cta;
  for (int k = tid; k < Z; k += 256) {
    double acc = 0.0;
    for (int rr = 0; rr < DF_RT; ++rr) acc = fma(mbs[rr], At[k * DF_RT + rr], acc);
    pmu[pc * L.ZS + k] = acc;
  }
  if (tid == 0) {
    double sv = 0.0;
    for (int rr = 0; rr < nr; ++rr) sv += vbs[rr];
    psc[pc * 2] = dl / ell;
    psc[pc * 2 + 1] = ks + sv;
  }
}

// per (batch row i, hidden unit h): usum[j B + i][h] = sum_t ubar_t, m_bar1 = sum_j usum, v_bar1 through the clamped sqrt
__global__ void dgf_hidden_bar_kernel(DfLayout L, int64_t B, int64_t RS, const double* __restrict__ ubar, const double* __restrict__ eps,
                                      const double* __restrict__ vb, double* __restrict__ usum, double* __restrict__ mbar,
                                      double* __restrict__ vbar) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = L.H;
  if (t >= B * H) return;
  const int64_t i = t / H;
  const int h = (int)(t - i * H);
  double mbs = 0.0, sdb = 0.0;
  for (int j = 0; j < L.J; ++j) {
    const size_t o = ((size_t)j * B + i) * H + h;
    double ub = 0.0;
    for (int k = 0; k < L.T; ++k) ub += ubar[(size_t)k * RS * H + o];
    usum[o] = ub;
    mbs += ub;
    sdb = fma(ub, eps[o], sdb);
  }
  const double v = vb[(size_t)h * RS + i];
  mbar[(size_t)h * RS + i] = mbs;
  vbar[(size_t)h * RS + i] = v >= L.min_var ? sdb / (2.0 * sqrt(v)) : 0.0;
}

// grid (32 x 32 output tiles, row chunks, units): pq = 2 sum_r v_bar a_i g_k, pzz = -sum_r K_bar_i a_k over the chunk
__global__ void __launch_bounds__(256) dgf_gram_kernel(DfLayout L, int64_t B, int64_t R2, int64_t RS, const double* __restrict__ A,
                                                       const double* __restrict__ G, const double* __restrict__ Kb,
                                                       const double* __restrict__ vbar, int nchunk, double* __restrict__ pq,
                                                       double* __restrict__ pzz) {
  __shared__ double sAi[32][33], sGk[32][33], sKi[32][33], sAk[32][33], sv[32];
  const int u = blockIdx.z, c = blockIdx.y, nt = (L.ZS + 31) / 32;
  const int ti = blockIdx.x / nt, tk = blockIdx.x % nt;
  const int Z = u < L.H ? L.Z1 : L.Z2;
  const int i0 = ti * 32, k0 = tk * 32;
  if (tk > ti || i0 >= Z) return;  // only the lower triangle is read
  const int64_t Ru = u < L.H ? B : R2;
  const int tid = threadIdx.x, oi = tid >> 3, ok = (tid & 7) * 4;
  double aq[4] = {0.0, 0.0, 0.0, 0.0}, az[4] = {0.0, 0.0, 0.0, 0.0};
  const int64_t rb = (int64_t)c * DF_RC, re = Ru < rb + DF_RC ? Ru : rb + DF_RC;
  const size_t ub = (size_t)u * L.ZS * RS;
  for (int64_t r0 = rb; r0 < re; r0 += 32) {
    for (int e = tid; e < 32 * 32; e += 256) {
      const int ii = e >> 5, rr = e & 31;
      const int64_t r = r0 + rr;
      const bool okr = r < re;
      const bool oki = okr && i0 + ii < Z, okk = okr && k0 + ii < Z;
      sAi[ii][rr] = oki ? A[ub + (size_t)(i0 + ii) * RS + r] : 0.0;
      sKi[ii][rr] = oki ? Kb[ub + (size_t)(i0 + ii) * RS + r] : 0.0;
      sGk[ii][rr] = okk ? G[ub + (size_t)(k0 + ii) * RS + r] : 0.0;
      sAk[ii][rr] = okk ? A[ub + (size_t)(k0 + ii) * RS + r] : 0.0;
    }
    if (tid < 32) sv[tid] = r0 + tid < re ? vbar[(size_t)u * RS + r0 + tid] : 0.0;
    __syncthreads();
    for (int rr = 0; rr < 32; ++rr) {
      const double ai = sAi[oi][rr] * sv[rr], ki = sKi[oi][rr];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        aq[q] = fma(ai, sGk[ok + q][rr], aq[q]);
        az[q] = fma(ki, sAk[ok + q][rr], az[q]);
      }
    }
    __syncthreads();
  }
  const int i = i0 + oi;
  const size_t zz = (size_t)L.ZS * L.ZS, base = ((size_t)u * nchunk + c) * zz;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + ok + q;
    if (i < Z && k < Z) {
      pq[base + (size_t)i * L.ZS + k] = 2.0 * aq[q];
      pzz[base + (size_t)i * L.ZS + k] = -az[q];
    }
  }
}

// One CTA per unit: Lz_bar, the Cholesky backward pass in shared memory, the K(Z, Z) terms, and the unit's gradient
// blocks (raw length scale and output scale, mu, chol, and its inducing points: into g for a last-layer unit, into
// gz1[h] for a hidden unit, whose inducing points are shared)
__global__ void __launch_bounds__(256) dgf_unit_bwd_kernel(DfLayout L, const double* __restrict__ p, int nchunk, int nc1, int nc2,
                                                           int ctamax, int64_t pz_unit1, int64_t pz_unit2, int64_t pz_base2,
                                                           const double* __restrict__ Lzg, const double* __restrict__ pq,
                                                           const double* __restrict__ pzz, double* __restrict__ Pg,
                                                           const double* __restrict__ pz, const double* __restrict__ pmu,
                                                           const double* __restrict__ psc, double* __restrict__ gz1, double* __restrict__ g) {
  extern __shared__ double S[];
  __shared__ double red[8];
  const int u = blockIdx.x, tid = threadIdx.x;
  const DfUnit v = df_unit(L, u);
  const int Z = v.Z, D = v.D, ZS = L.ZS;
  const size_t zz = (size_t)ZS * ZS;
  const double* Lz = Lzg + (size_t)u * zz;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, k = e - i * Z;
    double a = 0.0;
    if (k <= i)
      for (int c = 0; c < nchunk; ++c) a += pzz[((size_t)u * nchunk + c) * zz + (size_t)i * ZS + k];
    S[e] = a;
  }
  __syncthreads();
  double* P = Pg + (size_t)u * zz;
  for (int e = tid; e < Z * Z; e += 256) {  // P = Phi(Lz' Lz_bar)
    const int i = e / Z, j = e - i * Z;
    double a = 0.0;
    if (j <= i) {
      for (int k = i; k < Z; ++k) a = fma(Lz[(size_t)k * ZS + i], S[k * Z + j], a);
      if (i == j) a *= 0.5;
    }
    P[(size_t)i * ZS + j] = a;
  }
  __syncthreads();
  for (int e = tid; e < Z * Z; e += 256) S[e] = P[(size_t)(e / Z) * ZS + e % Z];
  __syncthreads();
  for (int j = Z - 1; j >= 0; --j) {  // Y Lz = P
    const double ljj = Lz[(size_t)j * ZS + j];
    for (int i = tid; i < Z; i += 256) S[i * Z + j] /= ljj;
    __syncthreads();
    for (int e = tid; e < Z * j; e += 256) {
      const int i = e / j, k = e - i * j;
      S[i * Z + k] = fma(-S[i * Z + j], Lz[(size_t)j * ZS + k], S[i * Z + k]);
    }
    __syncthreads();
  }
  for (int i = Z - 1; i >= 0; --i) {  // Lz' X = Y
    const double lii = Lz[(size_t)i * ZS + i];
    for (int c = tid; c < Z; c += 256) S[i * Z + c] /= lii;
    __syncthreads();
    for (int e = tid; e < i * Z; e += 256) {
      const int k = e / Z, c = e - k * Z;
      S[k * Z + c] = fma(-Lz[(size_t)i * ZS + k], S[i * Z + c], S[k * Z + c]);
    }
    __syncthreads();
  }
  for (int e = tid; e < Z * Z; e += 256) {  // Kzz_bar = (X + X') / 2
    const int i = e / Z, j = e - i * Z;
    if (j < i) {
      const double a = 0.5 * (S[e] + S[j * Z + i]);
      S[e] = a;
      S[j * Z + i] = a;
    }
  }
  __syncthreads();
  const double xs = p[v.oos], xl = p[v.ols];
  const double s = df_softplus(xs), ell = df_lscale(L, xl), il = 1.0 / ell;
  const double* zp = p + v.ozp;
  double ks = 0.0, dl = 0.0;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, j = e - i * Z;
    const double r2 = df_d2(zp + (size_t)i * D, zp + (size_t)j * D, D, il), q = sqrt(5.0 * r2), ex = exp(-q);
    const double kb = S[e];
    ks = fma(kb, (1.0 + q + q * q / 3.0) * ex, ks);
    const double w = kb * s * (5.0 / 3.0) * (1.0 + q) * ex;
    dl = fma(w, r2, dl);
    S[e] = w;
  }
  ks = block_sum<8>(ks, red);
  dl = block_sum<8>(dl, red);
  const bool hid = u < L.H;
  const int nc = hid ? nc1 : nc2;
  const double* pzu = hid ? pz + (size_t)u * pz_unit1 : pz + pz_base2 + (size_t)(u - L.H) * pz_unit2;
  const double il2 = il * il;
  for (int e = tid; e < Z * D; e += 256) {
    const int i = e / D, c = e - i * D;
    double acc = 0.0;
    for (int j = 0; j < Z; ++j) acc = fma(S[i * Z + j], zp[(size_t)i * D + c] - zp[(size_t)j * D + c], acc);
    double gzv = -2.0 * il2 * acc;
    for (int k = 0; k < nc; ++k) gzv += pzu[(size_t)k * Z * D + e];
    if (hid)
      gz1[(size_t)u * Z * D + e] = gzv;
    else
      g[v.ozp + e] = gzv;
  }
  const double inv_n = 1.0 / (double)L.N;
  const double* mu = p + v.omu;
  for (int k = tid; k < Z; k += 256) {
    double a = 0.0;
    for (int c = 0; c < nc; ++c) a += pmu[((size_t)u * ctamax + c) * ZS + k];
    g[v.omu + k] = a + mu[k] * inv_n;
  }
  const double* ch = p + v.och;
  for (int e = tid; e < Z * Z; e += 256) {
    const int i = e / Z, k = e - i * Z;
    double a = 0.0;
    if (k <= i) {
      for (int c = 0; c < nchunk; ++c) a += pq[((size_t)u * nchunk + c) * zz + (size_t)i * ZS + k];
      a += (ch[e] - (i == k ? 1.0 / ch[e] : 0.0)) * inv_n;
    }
    g[v.och + e] = a;
  }
  if (tid == 0) {
    double gl = dl / ell, gs = ks;
    for (int c = 0; c < nc; ++c) {
      gl += psc[((size_t)u * ctamax + c) * 2];
      gs += psc[((size_t)u * ctamax + c) * 2 + 1];
    }
    g[v.ols] = gl * df_lscale_grad(L, xl);
    g[v.oos] = gs * df_softplus_grad(xs);
  }
}

// one CTA: the loss (into loss_out[0]) and the shared gradient blocks: c, the noises, w, b, the hidden inducing
// points (sum over the units) and the quadrature sites
__global__ void __launch_bounds__(256) dgf_assemble_kernel(DfLayout L, const double* __restrict__ p, const double* __restrict__ X,
                                                           const int64_t* __restrict__ batch, int64_t B, int64_t RS,
                                                           const double* __restrict__ lterm, const double* __restrict__ sterm,
                                                           const double* __restrict__ kl, const double* __restrict__ mbar,
                                                           const double* __restrict__ vb, const double* __restrict__ usum,
                                                           const double* __restrict__ gz1, double* __restrict__ g, double* __restrict__ loss_out) {
  __shared__ double red[8];
  const int tid = threadIdx.x, H = L.H, T = L.T, d = L.d;
  const int64_t R2 = (int64_t)L.J * B;
  double a = 0.0, cb = 0.0;
  for (int64_t e = tid; e < (int64_t)T * R2; e += 256) {
    const int t = (int)(e / R2);
    const int64_t r = e - (int64_t)t * R2;
    a += lterm[(size_t)t * RS + r];
    cb += mbar[(size_t)(H + t) * RS + r];
  }
  a = block_sum<8>(a, red);
  cb = block_sum<8>(cb, red);
  if (tid == 0) {
    double k = 0.0;
    for (int u = 0; u < H + T; ++u) k += kl[u];
    loss_out[0] = a + k / (double)L.N;
    g[L.oc] = cb;
  }
  double gsum = 0.0;
  for (int t = 0; t < T; ++t) {
    double st = 0.0;
    for (int64_t r = tid; r < R2; r += 256) st += sterm[(size_t)t * RS + r];
    st = block_sum<8>(st, red);
    if (tid == 0) g[L.otn + t] = st * df_softplus_grad(p[L.otn + t]);
    gsum += st;
  }
  if (tid == 0) g[L.on] = gsum * df_softplus_grad(p[L.on]);
  double bb = 0.0;
  for (int64_t e = tid; e < B * H; e += 256) bb += mbar[(size_t)(e % H) * RS + e / H];
  bb = block_sum<8>(bb, red);
  if (tid == 0) g[L.ob] = bb;
  for (int c = tid; c < d; c += 256) {
    double acc = 0.0;
    for (int64_t i = 0; i < B; ++i) {
      double mi = 0.0;
      for (int h = 0; h < H; ++h) mi += mbar[(size_t)h * RS + i];
      acc = fma(mi, X[(size_t)batch[i] * d + c], acc);
    }
    g[L.ow + c] = acc;
  }
  const int64_t nz = (int64_t)L.Z1 * d;
  for (int64_t e = tid; e < nz; e += 256) {
    double acc = 0.0;
    for (int h = 0; h < H; ++h) acc += gz1[(size_t)h * nz + e];
    g[L.oZ1 + e] = acc;
  }
  if (L.quadrature)
    for (int e = tid; e < L.J * H; e += 256) {
      const int j = e / H, h = e - j * H;
      double acc = 0.0;
      for (int64_t i = 0; i < B; ++i)
        acc = fma(usum[((size_t)j * B + i) * H + h], sqrt(fmax(vb[(size_t)h * RS + i], L.min_var)), acc);
      g[L.osite + e] = acc;
    }
}

// torch.optim.Adam's step (betas 0.9 / 0.999, eps 1e-8) in its order of operations, every rounding explicit:
// m <- fma(1 - b1, g - m, m); v <- fma((1 - b2) g, g, v b2); p <- p + (-step_size m) / (sqrt(v) / bc2_sqrt + eps)
__global__ void dgf_adam_kernel(int64_t P, double* __restrict__ p, const double* __restrict__ g, double* __restrict__ m,
                                double* __restrict__ v, double omb1, double omb2, double b2, double neg_step, double bc2s, double eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const double gi = g[i];
  const double mi = __fma_rn(omb1, __dsub_rn(gi, m[i]), m[i]);
  const double vi = __fma_rn(__dmul_rn(omb2, gi), gi, __dmul_rn(v[i], b2));
  m[i] = mi;
  v[i] = vi;
  const double den = __dadd_rn(__ddiv_rn(__dsqrt_rn(vi), bc2s), eps);
  p[i] = __dadd_rn(p[i], __ddiv_rn(__dmul_rn(neg_step, mi), den));
}

constexpr size_t df_rows_smem(int ZS) { return (size_t)(ZS * ZS + 2 * ZS * DF_RT) * sizeof(double); }

}  // namespace

struct dmo_dgp_fit {
  DfLayout L;
  int64_t Bmax = 0, RS = 0;  // batch rows at most, and row stride J * Bmax
  int nct1 = 0, nct2 = 0, ctamax = 0, nchunk = 0;
  int64_t adam_t = 0;
  DevBuf<double> X, Y, p, g, am, av;
  DevBuf<double> Lz, Pg, kl, A, G, Kb, mb, vb, mbar, vbar, lterm, sterm, U, eps, ubar, usum;
  DevBuf<double> pz, pmu, psc, pq, pzz, gz1, losses;
  DevBuf<int64_t> bidx, perm;
  DevBuf<int> info;
};

namespace {

// one step's loss and gradient at the current parameters: batch (B rows, device), eps_in (J, B, H, device) or NULL;
// the loss into *d_loss (device).  Not synchronised.
int dgf_loss_grad(dmo_ctx* ctx, dmo_dgp_fit* st, const int64_t* batch, int64_t B, uint64_t seed, uint64_t step, const double* eps_in,
                  double* d_loss) {
  const DfLayout& L = st->L;
  const int H = L.H, T = L.T, U = H + T, ZS = L.ZS;
  const int64_t RS = st->RS, R2 = (int64_t)L.J * B;
  const int nc1 = (int)ceil_div(B, DF_RT), nc2 = (int)ceil_div(R2, DF_RT), nchunk = (int)ceil_div(R2, DF_RC), nt = (ZS + 31) / 32;
  const size_t rsm = df_rows_smem(ZS), usm = (size_t)ZS * ZS * sizeof(double);
  const int64_t pz_unit1 = (int64_t)st->nct1 * L.Z1 * L.d, pz_unit2 = (int64_t)st->nct2 * L.Z2 * H, pz_base2 = (int64_t)H * pz_unit1;
  DMO_LAUNCH(dgf_factor_kernel, U, 256, usm, L, st->p.p, st->Lz.p, st->info.p, st->kl.p);
  DMO_LAUNCH(dgf_rows_fwd_kernel, dim3(nc1, H), 256, rsm, L, st->p.p, 0, st->X.p, batch, B, RS, st->Lz.p, st->A.p, st->G.p, st->mb.p,
             st->vb.p);
  DMO_LAUNCH(dgf_hidden_out_kernel, (unsigned)ceil_div(B * H, 128), 128, 0, L, st->p.p, st->X.p, batch, B, RS, st->mb.p, st->vb.p, eps_in,
             seed, step, st->eps.p, st->U.p);
  {
    ProfileScope pl(ctx, "dgp_fit_last_fwd");
    DMO_LAUNCH(dgf_rows_fwd_kernel, dim3(nc2, T), 256, rsm, L, st->p.p, H, st->U.p, nullptr, R2, RS, st->Lz.p, st->A.p, st->G.p, st->mb.p,
               st->vb.p);
  }
  DMO_LAUNCH(dgf_ell_kernel, (unsigned)ceil_div(R2 * T, 128), 128, 0, L, st->p.p, st->Y.p, batch, B, RS, st->mb.p, st->vb.p, st->lterm.p,
             st->sterm.p, st->mbar.p, st->vbar.p);
  {
    ProfileScope pl(ctx, "dgp_fit_last_bwd");
    DMO_LAUNCH(dgf_rows_bwd_kernel, dim3(nc2, T), 256, rsm, L, st->p.p, H, st->U.p, nullptr, R2, RS, st->Lz.p, st->A.p, st->G.p,
               st->mbar.p, st->vbar.p, st->Kb.p, st->pz.p, pz_unit2, pz_base2, st->ctamax, st->pmu.p, st->psc.p, st->ubar.p);
  }
  DMO_LAUNCH(dgf_hidden_bar_kernel, (unsigned)ceil_div(B * H, 128), 128, 0, L, B, RS, st->ubar.p, st->eps.p, st->vb.p, st->usum.p,
             st->mbar.p, st->vbar.p);
  DMO_LAUNCH(dgf_rows_bwd_kernel, dim3(nc1, H), 256, rsm, L, st->p.p, 0, st->X.p, batch, B, RS, st->Lz.p, st->A.p, st->G.p, st->mbar.p,
             st->vbar.p, st->Kb.p, st->pz.p, pz_unit1, (int64_t)0, st->ctamax, st->pmu.p, st->psc.p, nullptr);
  {
    ProfileScope pl(ctx, "dgp_fit_gram");
    DMO_LAUNCH(dgf_gram_kernel, dim3(nt * nt, nchunk, U), 256, 0, L, B, R2, RS, st->A.p, st->G.p, st->Kb.p, st->vbar.p, nchunk, st->pq.p,
               st->pzz.p);
  }
  DMO_LAUNCH(dgf_unit_bwd_kernel, U, 256, usm, L, st->p.p, nchunk, nc1, nc2, st->ctamax, pz_unit1, pz_unit2, pz_base2, st->Lz.p, st->pq.p,
             st->pzz.p, st->Pg.p, st->pz.p, st->pmu.p, st->psc.p, st->gz1.p, st->g.p);
  DMO_LAUNCH(dgf_assemble_kernel, 1, 256, 0, L, st->p.p, st->X.p, batch, B, RS, st->lterm.p, st->sterm.p, st->kl.p, st->mbar.p, st->vb.p,
             st->usum.p, st->gz1.p, st->g.p, d_loss);
  return DMO_OK;
}

int dgf_adam(dmo_ctx* ctx, dmo_dgp_fit* st, double lr) {
  st->adam_t += 1;
  const double t = (double)st->adam_t, b1 = 0.9, b2 = 0.999;
  const double bc1 = 1.0 - pow(b1, t);
  const double bc2s = pow(1.0 - pow(b2, t), 0.5);
  const double step_size = lr / bc1;
  DMO_LAUNCH(dgf_adam_kernel, (unsigned)ceil_div(st->L.P, 256), 256, 0, st->L.P, st->p.p, st->g.p, st->am.p, st->av.p, 1.0 - b1, 1.0 - b2, b2,
             -step_size, bc2s, 1e-8);
  return DMO_OK;
}

// fails with the first unit whose K(Z, Z) + jitter I was not positive definite since info was last cleared (synchronises)
int dgf_check_info(dmo_ctx* ctx, dmo_dgp_fit* st, const char* who) {
  const int U = st->L.H + st->L.T;
  std::vector<int> h(U);
  DMO_CUDA(cudaMemcpyAsync(h.data(), st->info.p, U * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  for (int u = 0; u < U; ++u)
    if (h[u])
      return dmo_fail(ctx, DMO_ERR_ARG, "%s: K(Z, Z) + jitter I of %s unit %d is not positive definite (pivot %d)", who,
                      u < st->L.H ? "hidden layer" : "last layer", u < st->L.H ? u : u - st->L.H, h[u] - 1);
  return DMO_OK;
}

int dgf_batch(dmo_ctx* ctx, dmo_dgp_fit* st, const char* who, const int64_t* batch, int64_t B, std::vector<int64_t>& hb) {
  DMO_REQUIRE(batch, "%s: null batch", who);
  DMO_REQUIRE(B >= 1 && B <= st->Bmax, "%s: 1 <= B <= batch_max (got B=%lld, batch_max=%lld)", who, (long long)B, (long long)st->Bmax);
  hb.resize(B);
  DMO_CUDA(cudaMemcpy(hb.data(), batch, B * sizeof(int64_t), cudaMemcpyDefault));
  for (int64_t b = 0; b < B; ++b)
    DMO_REQUIRE(hb[b] >= 0 && hb[b] < st->L.N, "%s: batch[%lld] = %lld is outside [0, %lld)", who, (long long)b, (long long)hb[b],
                (long long)st->L.N);
  return DMO_OK;
}

}  // namespace

extern "C" {

int dmo_dgp_fit_create(dmo_ctx* ctx, int64_t N, int d, int H, int T, int64_t Z1, int64_t Z2, int n_sites, int quadrature,
                       int64_t batch_max, const double* X, const double* Y, const double* lengthscale_bounds, double jitter,
                       double min_variance, dmo_dgp_fit** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out, "dgp_fit_create: null output");
  *out = nullptr;
  DMO_REQUIRE(H >= 1 && H <= DF_MAX_HT && T >= 1 && T <= DF_MAX_HT, "dgp_fit_create: 1 <= H, T <= %d (got H=%d T=%d)", DF_MAX_HT, H, T);
  DMO_REQUIRE(Z1 >= 1 && Z1 <= DF_ZMAX && Z2 >= 1 && Z2 <= DF_ZMAX, "dgp_fit_create: 1 <= Z1, Z2 <= %d (got Z1=%lld Z2=%lld)", DF_ZMAX,
              (long long)Z1, (long long)Z2);
  DMO_REQUIRE(d >= 1 && d <= MT_FIT_DMAX, "dgp_fit_create: 1 <= d <= %d (got %d)", MT_FIT_DMAX, d);
  DMO_REQUIRE(N >= 1 && batch_max >= 1 && batch_max <= N, "dgp_fit_create: N >= 1 and 1 <= batch_max <= N (got N=%lld batch_max=%lld)",
              (long long)N, (long long)batch_max);
  DMO_REQUIRE(n_sites >= 1 && (int64_t)n_sites * batch_max <= DF_MAX_ROWS, "dgp_fit_create: 1 <= n_sites and n_sites * batch_max <= %lld (got %d * %lld)",
              (long long)DF_MAX_ROWS, n_sites, (long long)batch_max);
  DMO_REQUIRE(X && Y, "dgp_fit_create: null pointer");
  DMO_REQUIRE(jitter >= 0.0 && isfinite(jitter), "dgp_fit_create: jitter must be finite and >= 0 (got %g)", jitter);
  DMO_REQUIRE(min_variance >= 0.0 && isfinite(min_variance), "dgp_fit_create: min_variance must be finite and >= 0 (got %g)", min_variance);
  std::vector<double> hx((size_t)N * d), hy((size_t)N * T);
  DMO_CUDA(cudaMemcpy(hx.data(), X, hx.size() * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hy.data(), Y, hy.size() * sizeof(double), cudaMemcpyDefault));
  for (double v : hx) DMO_REQUIRE(isfinite(v), "dgp_fit_create: X must be finite");
  for (double v : hy) DMO_REQUIRE(isfinite(v), "dgp_fit_create: Y must be finite");
  std::unique_ptr<dmo_dgp_fit> st(new dmo_dgp_fit());
  DfLayout& L = st->L;
  memset(&L, 0, sizeof(L));
  if (lengthscale_bounds) {
    double lb[2];
    DMO_CUDA(cudaMemcpy(lb, lengthscale_bounds, sizeof(lb), cudaMemcpyDefault));
    DMO_REQUIRE(isfinite(lb[0]) && isfinite(lb[1]) && lb[0] > 0.0 && lb[1] > lb[0],
                "dgp_fit_create: lengthscale_bounds must be finite with 0 < lo < hi (got %g, %g)", lb[0], lb[1]);
    L.bounded = 1;
    L.lo = lb[0];
    L.hi = lb[1];
  }
  L.d = d;
  L.H = H;
  L.T = T;
  L.J = n_sites;
  L.Z1 = (int)Z1;
  L.Z2 = (int)Z2;
  L.ZS = (int)(Z1 > Z2 ? Z1 : Z2);
  L.quadrature = quadrature ? 1 : 0;
  L.jitter = jitter;
  L.min_var = min_variance;
  L.N = N;
  int64_t o = 0;
  auto take = [&](int64_t n) {
    const int64_t at = o;
    o += n;
    return at;
  };
  L.oZ1 = take(Z1 * d);
  L.ols1 = take(H);
  L.oos1 = take(H);
  L.omu1 = take(H * Z1);
  L.och1 = take(H * Z1 * Z1);
  L.ow = take(d);
  L.ob = take(1);
  L.oZ2 = take(T * Z2 * H);
  L.ols2 = take(T);
  L.oos2 = take(T);
  L.omu2 = take(T * Z2);
  L.och2 = take(T * Z2 * Z2);
  L.oc = take(1);
  L.otn = take(T);
  L.on = take(1);
  L.osite = take(quadrature ? (int64_t)n_sites * H : 0);
  L.P = o;
  const int U = H + T, ZS = L.ZS;
  st->Bmax = batch_max;
  st->RS = (int64_t)n_sites * batch_max;
  const int64_t RS = st->RS;
  st->nct1 = (int)ceil_div(batch_max, DF_RT);
  st->nct2 = (int)ceil_div(RS, DF_RT);
  st->ctamax = st->nct1 > st->nct2 ? st->nct1 : st->nct2;
  st->nchunk = (int)ceil_div(RS, DF_RC);
  const size_t zz = (size_t)ZS * ZS;
  DMO_TRY(upload(ctx, st->X, hx));
  DMO_TRY(upload(ctx, st->Y, hy));
  const std::vector<double> zeros(L.P, 0.0);
  DMO_TRY(upload(ctx, st->p, zeros));
  DMO_TRY(upload(ctx, st->g, zeros));
  DMO_TRY(upload(ctx, st->am, zeros));
  DMO_TRY(upload(ctx, st->av, zeros));
  DMO_TRY(st->Lz.alloc(ctx, U * zz));
  DMO_TRY(st->Pg.alloc(ctx, U * zz));
  DMO_TRY(st->kl.alloc(ctx, U));
  DMO_TRY(st->A.alloc(ctx, U * (size_t)ZS * RS));
  DMO_TRY(st->G.alloc(ctx, U * (size_t)ZS * RS));
  DMO_TRY(st->Kb.alloc(ctx, U * (size_t)ZS * RS));
  DMO_TRY(st->mb.alloc(ctx, U * (size_t)RS));
  DMO_TRY(st->vb.alloc(ctx, U * (size_t)RS));
  DMO_TRY(st->mbar.alloc(ctx, U * (size_t)RS));
  DMO_TRY(st->vbar.alloc(ctx, U * (size_t)RS));
  DMO_TRY(st->lterm.alloc(ctx, T * (size_t)RS));
  DMO_TRY(st->sterm.alloc(ctx, T * (size_t)RS));
  DMO_TRY(st->U.alloc(ctx, (size_t)RS * H));
  DMO_TRY(st->eps.alloc(ctx, (size_t)RS * H));
  DMO_TRY(st->usum.alloc(ctx, (size_t)RS * H));
  DMO_TRY(st->ubar.alloc(ctx, (size_t)T * RS * H));
  DMO_TRY(st->pz.alloc(ctx, (size_t)H * st->nct1 * Z1 * d + (size_t)T * st->nct2 * Z2 * H));
  DMO_TRY(st->pmu.alloc(ctx, (size_t)U * st->ctamax * ZS));
  DMO_TRY(st->psc.alloc(ctx, (size_t)U * st->ctamax * 2));
  DMO_TRY(st->pq.alloc(ctx, (size_t)U * st->nchunk * zz));
  DMO_TRY(st->pzz.alloc(ctx, (size_t)U * st->nchunk * zz));
  DMO_TRY(st->gz1.alloc(ctx, (size_t)H * Z1 * d));
  DMO_TRY(st->losses.alloc(ctx, (size_t)N));
  DMO_TRY(st->bidx.alloc(ctx, batch_max));
  DMO_TRY(st->perm.alloc(ctx, N));
  DMO_TRY(st->info.alloc(ctx, U));
  DMO_CUDA(cudaMemsetAsync(st->info.p, 0, U * sizeof(int), ctx->stream));
  DMO_CUDA(cudaFuncSetAttribute(dgf_rows_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)df_rows_smem(DF_ZMAX)));
  DMO_CUDA(cudaFuncSetAttribute(dgf_rows_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)df_rows_smem(DF_ZMAX)));
  DMO_CUDA(cudaFuncSetAttribute(dgf_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(DF_ZMAX * DF_ZMAX * sizeof(double))));
  DMO_CUDA(cudaFuncSetAttribute(dgf_unit_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(DF_ZMAX * DF_ZMAX * sizeof(double))));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  *out = st.release();
  return DMO_OK;
}

int dmo_dgp_fit_destroy(dmo_ctx* ctx, dmo_dgp_fit* st) {
  if (!ctx) return DMO_ERR_ARG;
  if (!st) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  delete st;
  return DMO_OK;
}

int dmo_dgp_fit_set_params(dmo_ctx* ctx, dmo_dgp_fit* st, const double* raw, int64_t n) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st && raw, "dgp_fit_set_params: null argument");
  DMO_REQUIRE(n == st->L.P, "dgp_fit_set_params: the raw vector has %lld entries (got %lld)", (long long)st->L.P, (long long)n);
  std::vector<double> h(n);
  DMO_CUDA(cudaMemcpy(h.data(), raw, n * sizeof(double), cudaMemcpyDefault));
  for (int64_t i = 0; i < n; ++i) DMO_REQUIRE(isfinite(h[i]), "dgp_fit_set_params: raw[%lld] must be finite", (long long)i);
  DMO_CUDA(cudaMemcpyAsync(st->p.p, h.data(), n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_dgp_fit_get_params(dmo_ctx* ctx, dmo_dgp_fit* st, double* raw, int64_t n) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st && raw, "dgp_fit_get_params: null argument");
  DMO_REQUIRE(n == st->L.P, "dgp_fit_get_params: the raw vector has %lld entries (got %lld)", (long long)st->L.P, (long long)n);
  DMO_CUDA(cudaMemcpyAsync(raw, st->p.p, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_dgp_fit_loss_grad(dmo_ctx* ctx, dmo_dgp_fit* st, const int64_t* batch, int64_t B, uint64_t seed, uint64_t step, const double* eps_in,
                          double* eps_out, double* loss_out, double* grad_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st && loss_out, "dgp_fit_loss_grad: null argument");
  std::vector<int64_t> hb;
  DMO_TRY(dgf_batch(ctx, st, "dgp_fit_loss_grad", batch, B, hb));
  const size_t ne = (size_t)st->L.J * B * st->L.H;
  In<double> ein;
  DMO_TRY(ein.init(ctx, st->L.quadrature ? nullptr : eps_in, ne));
  if (ein.d) {
    std::vector<double> he(ne);
    DMO_CUDA(cudaMemcpy(he.data(), eps_in, ne * sizeof(double), cudaMemcpyDefault));
    for (double v : he) DMO_REQUIRE(isfinite(v), "dgp_fit_loss_grad: eps must be finite");
  }
  DMO_CUDA(cudaMemcpyAsync(st->bidx.p, hb.data(), B * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemsetAsync(st->info.p, 0, (st->L.H + st->L.T) * sizeof(int), ctx->stream));
  DMO_TRY(dgf_loss_grad(ctx, st, st->bidx.p, B, seed, step, ein.d, st->losses.p));
  DMO_CHECK_LAUNCH();
  DMO_TRY(dgf_check_info(ctx, st, "dgp_fit_loss_grad"));
  DMO_CUDA(cudaMemcpyAsync(loss_out, st->losses.p, sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (grad_out) DMO_CUDA(cudaMemcpyAsync(grad_out, st->g.p, st->L.P * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (eps_out) DMO_CUDA(cudaMemcpyAsync(eps_out, st->eps.p, ne * sizeof(double), cudaMemcpyDefault, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_dgp_fit_adam_step(dmo_ctx* ctx, dmo_dgp_fit* st, double lr) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st, "dgp_fit_adam_step: null state");
  DMO_REQUIRE(lr > 0.0 && isfinite(lr), "dgp_fit_adam_step: lr must be finite and > 0 (got %g)", lr);
  DMO_TRY(dgf_adam(ctx, st, lr));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_dgp_fit_epoch(dmo_ctx* ctx, dmo_dgp_fit* st, const int64_t* perm, int64_t B, double lr, uint64_t seed, uint64_t step0,
                      double* losses_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(st && perm && losses_out, "dgp_fit_epoch: null argument");
  DMO_REQUIRE(B >= 1 && B <= st->Bmax, "dgp_fit_epoch: 1 <= B <= batch_max (got B=%lld, batch_max=%lld)", (long long)B, (long long)st->Bmax);
  DMO_REQUIRE(lr > 0.0 && isfinite(lr), "dgp_fit_epoch: lr must be finite and > 0 (got %g)", lr);
  const int64_t N = st->L.N;
  std::vector<int64_t> hp(N);
  DMO_CUDA(cudaMemcpy(hp.data(), perm, N * sizeof(int64_t), cudaMemcpyDefault));
  std::vector<char> seen(N, 0);
  for (int64_t i = 0; i < N; ++i) {
    DMO_REQUIRE(hp[i] >= 0 && hp[i] < N && !seen[hp[i]], "dgp_fit_epoch: perm must be a permutation of range(%lld)", (long long)N);
    seen[hp[i]] = 1;
  }
  DMO_CUDA(cudaMemcpyAsync(st->perm.p, hp.data(), N * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemsetAsync(st->info.p, 0, (st->L.H + st->L.T) * sizeof(int), ctx->stream));
  const int64_t nb = ceil_div(N, B);
  for (int64_t b = 0; b < nb; ++b) {
    const int64_t Bb = N - b * B < B ? N - b * B : B;
    DMO_TRY(dgf_loss_grad(ctx, st, st->perm.p + b * B, Bb, seed, step0 + (uint64_t)b, nullptr, st->losses.p + b));
    DMO_TRY(dgf_adam(ctx, st, lr));
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(dgf_check_info(ctx, st, "dgp_fit_epoch"));
  DMO_CUDA(cudaMemcpyAsync(losses_out, st->losses.p, nb * sizeof(double), cudaMemcpyDefault, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
