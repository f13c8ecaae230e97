// Two-layer deep GP posterior: the predict of gpytorch's DSPP and DeepGP behind dmosopt's MDSPP_Matern and MDGP_Matern
// (dmosopt/model_gpytorch.py:991-1306, 1308-1620).  Both are two whitened variational GP layers with a Matern-5/2 kernel.
//
// Hidden layer, unit h < H: a whitened variational GP over the normalised input x_n (the posterior of gp_variational.cu,
// built by dmo_svgp_create with L = H latents, W = I and unit output statistics), plus the prior mean w . x_n + b that
// every unit shares, plus gpytorch's jitter on k(x, x); its variance is clamped at min_variance and kept as sd1 = sqrt(var1).
// Layer-2 inputs, site j < J: u_j = mean1 + e_j o sd1, the same u_j for every task; e_j the quadrature sites (DSPP) or
// N(0, I) draws (DeepGP, Philox4x32-10 keyed by seed, counter (candidate, j H + h, stream_id)).
// Last layer, task t < T: the same whitened posterior at u_j (its operator planes again built by dmo_svgp_create, with
// L = T latents over H input dimensions), plus the constant c and the jitter:
//     m_tj = c + k' a_t,   v_tj = s_t + jitter - ||O0_t k||^2 + ||O1_t k||^2,   k = k_u(u_j, Z2_t)
//     mean_t = y_std_t (1/J) sum_j m_tj + y_mean_t,   var_t = y_std_t^2 (1/J) sum_j max(v_tj + noise_t, min_variance)
// (gpytorch's batch_preds.mean.mean(0) / .variance.mean(0): unweighted, no between-site spread).
//
// dgp_layer2_kernel is the hot path: J P T small-input variational predicts, each a K_* row of Z2 Matern values and two
// triangular mat-vecs.  A CTA takes the J sites of PT = 64 / J candidates for one task (rows r = j PT + p), forms their
// K_* rows chunk by chunk in shared memory (never in HBM) and runs the two mat-vecs as one register-blocked float64 FMA
// product Y = Ks O' over 128-row blocks of the operator planes, staged through shared memory 16 columns at a time; a warp
// skips the column steps that lie wholly above the diagonal of its 16 operator rows.
#include <math.h>

#include <memory>
#include <string>
#include <vector>

#include "gp.cuh"

namespace {

constexpr int DG_MAX_HT = 8;       // hidden units and tasks
constexpr int DG_MAX_SITES = 64;   // sites per candidate
constexpr int64_t DG_ZMAX = 8192;  // inducing points per layer
constexpr int DG_ROWS = 64;        // (site, candidate) rows per CTA
constexpr int DG_IB = 128;         // operator rows per block (the outputs of one pass of the product)
constexpr int DG_KC = 128;         // K_* columns per shared-memory chunk
constexpr int DG_KS = 16;          // operator columns staged per step
constexpr int DG_OLD = DG_IB + 1;  // row length of a staged operator tile (padded against bank conflicts)
constexpr size_t DG_SMEM = (size_t)(DG_KC * DG_ROWS + 2 * DG_KS * DG_OLD) * sizeof(double);

struct DgTask {
  const double *O0, *O1, *A, *XtT, *inv_ls;
  double s_jit;  // s_t + jitter
  double noise;  // task + global likelihood noise
  double ystd, ymean;
};
struct DgTasks {
  DgTask t[DG_MAX_HT];
};

// mean1 = fm + w . x_n + b, sd1 = sqrt(max(fv + jitter, min_variance)), (H, P) planes, in place over fm / fv
__global__ void dgp_hidden_epilogue_kernel(const double* __restrict__ X, int64_t P, int d, int H, const double* __restrict__ xlb,
                                           const double* __restrict__ xrg, const double* __restrict__ w, double b, double jitter,
                                           double min_var, double* __restrict__ fm, double* __restrict__ fv) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double mu = 0.0;
  for (int k = 0; k < d; ++k) mu = fma((X[p * d + k] - xlb[k]) / xrg[k], w[k], mu);
  mu += b;
  for (int h = 0; h < H; ++h) {
    fm[(int64_t)h * P + p] += mu;
    fv[(int64_t)h * P + p] = sqrt(fmax(fv[(int64_t)h * P + p] + jitter, min_var));
  }
}

template <bool VAR>
__global__ void __launch_bounds__(256, 1)
    dgp_layer2_kernel(DgTasks tasks, int T, int64_t P, int H, int J, int PT, int64_t Z, int64_t Npad, const double* __restrict__ mean1,
                      const double* __restrict__ sd1, const double* __restrict__ sites, uint64_t seed, uint64_t stream_id, double c,
                      double min_var, double* __restrict__ eps_out, double* __restrict__ mean, double* __restrict__ var) {
  extern __shared__ double dg_smem[];
  double* Ks = dg_smem;                  // [DG_KC][DG_ROWS] unit K_* values of the chunk
  double* Os = Ks + DG_KC * DG_ROWS;     // [2][DG_KS][DG_OLD] operator tiles, O0 then O1
  __shared__ double us[DG_ROWS][DG_MAX_HT + 1];  // u / ell of each row
  __shared__ double red[2][16][DG_ROWS];
  __shared__ double rm[DG_ROWS], rv[DG_ROWS];
  const int t = blockIdx.y;
  const DgTask tk = tasks.t[t];
  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * PT;
  const int nrow = PT * J;
  for (int e = tid; e < DG_ROWS * H; e += 256) {
    const int r = e / H, h = e - r * H;
    double v = 0.0;
    const int j = r / PT;
    const int64_t p = p0 + (r - j * PT);
    if (r < nrow && p < P) {
      double eps;
      if (sites) {
        eps = sites[j * H + h];
      } else {
        const uint4 q = Philox(seed)((uint64_t)p, (stream_id << 10) | (uint64_t)(j * H + h));
        const double u1 = u01_53(q.x, q.y), u2 = u01_53(q.z, q.w);
        eps = sqrt(-2.0 * log1p(-u1)) * cospi(2.0 * u2);  // Box-Muller; 1 - u1 lies in (0, 1]
      }
      if (eps_out && t == 0) eps_out[((int64_t)j * P + p) * H + h] = eps;
      v = (mean1[(int64_t)h * P + p] + eps * sd1[(int64_t)h * P + p]) * tk.inv_ls[h];
    }
    us[r][h] = v;
  }
  const int ty = tid & 15, tx = tid >> 4;  // rows ty + 16 u (u < 4); operator rows ib + 8 tx + v (v < 8)
  const int64_t warp_last = 16 * (tid >> 5) + 15;  // the last operator row of this warp within a block
  double msum = 0.0, q0[4] = {0.0, 0.0, 0.0, 0.0}, q1[4] = {0.0, 0.0, 0.0, 0.0};
  const int64_t nib = VAR ? (Z + DG_IB - 1) / DG_IB : 1;
  for (int64_t bi = 0; bi < nib; ++bi) {
    const int64_t ib = bi * DG_IB;
    const int64_t kend = VAR ? (Z < ib + DG_IB ? Z : ib + DG_IB) : Z;
    double acc0[4][8], acc1[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 8; ++v) acc0[u][v] = acc1[u][v] = 0.0;
    for (int64_t kc = 0; kc < kend; kc += DG_KC) {
      __syncthreads();  // us written; the previous chunk's readers are done
      for (int e = tid; e < DG_KC * DG_ROWS; e += 256) {
        const int kk = e / DG_ROWS, r = e - kk * DG_ROWS;
        const int64_t z = kc + kk;
        double k = 0.0;
        if (z < Z && r < nrow) {
          double s = 0.0;
          for (int h = 0; h < H; ++h) {
            const double dl = us[r][h] - tk.XtT[(int64_t)h * Npad + z];
            s = fma(dl, dl, s);
          }
          const double rr = sqrt(5.0 * s);
          k = (1.0 + rr + rr * rr / 3.0) * exp(-rr);
        }
        Ks[kk * DG_ROWS + r] = k;
      }
      __syncthreads();
      if ((!VAR || kc == ib) && tid < DG_ROWS)  // each chunk's first visit
        for (int kk = 0; kk < DG_KC; ++kk) msum = fma(Ks[kk * DG_ROWS + tid], tk.A[kc + kk], msum);  // a_t is zero padded to Npad
      if constexpr (VAR) {
        for (int k0 = 0; k0 < DG_KC && kc + k0 < kend; k0 += DG_KS) {
          for (int e = tid; e < DG_KS * DG_IB; e += 256) {
            const int i = e / DG_KS, kk = e - i * DG_KS;
            const int64_t g = (ib + i) * Npad + kc + k0 + kk;  // inside the zero-padded Npad x Npad plane
            Os[kk * DG_OLD + i] = tk.O0[g];
            Os[(DG_KS + kk) * DG_OLD + i] = tk.O1[g];
          }
          __syncthreads();
          if (kc + k0 <= ib + warp_last) {  // O is lower triangular: columns past the warp's last row add nothing
  #pragma unroll
            for (int kk = 0; kk < DG_KS; ++kk) {
              double a[4], b[8];
  #pragma unroll
              for (int u = 0; u < 4; ++u) a[u] = Ks[(k0 + kk) * DG_ROWS + ty + 16 * u];
  #pragma unroll
              for (int v = 0; v < 8; ++v) b[v] = Os[kk * DG_OLD + 8 * tx + v];
  #pragma unroll
              for (int u = 0; u < 4; ++u)
  #pragma unroll
                for (int v = 0; v < 8; ++v) acc0[u][v] = fma(a[u], b[v], acc0[u][v]);
  #pragma unroll
              for (int v = 0; v < 8; ++v) b[v] = Os[(DG_KS + kk) * DG_OLD + 8 * tx + v];
  #pragma unroll
              for (int u = 0; u < 4; ++u)
  #pragma unroll
                for (int v = 0; v < 8; ++v) acc1[u][v] = fma(a[u], b[v], acc1[u][v]);
            }
          }
          __syncthreads();
        }
      }
    }
    if (VAR) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 8; ++v) {
          q0[u] = fma(acc0[u][v], acc0[u][v], q0[u]);
          q1[u] = fma(acc1[u][v], acc1[u][v], q1[u]);
        }
    }
  }
  if (VAR)
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      red[0][tx][ty + 16 * u] = q0[u];
      red[1][tx][ty + 16 * u] = q1[u];
    }
  if (tid < DG_ROWS) rm[tid] = msum;
  __syncthreads();
  if (VAR && tid < DG_ROWS) {
    double v0 = 0.0, v1 = 0.0;
    for (int x = 0; x < 16; ++x) {
      v0 += red[0][x][tid];
      v1 += red[1][x][tid];
    }
    rv[tid] = (tk.s_jit - v0) + v1;
  }
  __syncthreads();
  if (tid < PT) {
    const int64_t p = p0 + tid;
    if (p < P) {
      double ms = 0.0, vs = 0.0;
      for (int j = 0; j < J; ++j) {
        const int r = j * PT + tid;
        ms += c + rm[r];
        if (VAR) vs += fmax(rv[r] + tk.noise, min_var);
      }
      mean[p * T + t] = tk.ystd * (ms / J) + tk.ymean;
      if (VAR) var[p * T + t] = (tk.ystd * tk.ystd) * (vs / J);
    }
  }
}

// DMO_ERR_ARG from dmo_svgp_create, re-reported with the layer it came from
int layer_error(dmo_ctx* ctx, int st, const char* layer) {
  if (st != DMO_ERR_ARG) return st;
  const std::string inner = ctx->err;
  return dmo_fail(ctx, DMO_ERR_ARG, "dgp_create: %s layer: %s", layer, inner.c_str());
}

}  // namespace

struct dmo_dgp {
  int d = 0, H = 0, T = 0, J = 0;
  int64_t Z2 = 0;
  dmo_svgp* hidden = nullptr;  // unit statistics, W = I: its latents are the hidden units
  dmo_svgp* last = nullptr;    // only its operator planes, mean vectors and scaled inducing points are used
  DgTasks tasks;
  int64_t Npad2 = 0;
  double b1 = 0.0, c2 = 0.0, jitter = 0.0, min_var = 0.0;
  bool quadrature = false;
  DevBuf<double> w1, xlb, xrg, sites;
};

void dgp_dims(const dmo_dgp* g, int* d, int* T) {
  *d = g->d;
  *T = g->T;
}

int dgp_predict_device(dmo_ctx* ctx, dmo_dgp* g, GpUnitPredict& up, const double* X, int64_t P, uint64_t seed, uint64_t stream_id,
                       double* eps, double* mean, double* var) {
  const int d = g->d, H = g->H, T = g->T, J = g->J;
  DevBuf<double> m1, s1;
  DMO_TRY(m1.alloc(ctx, (size_t)H * P));
  DMO_TRY(s1.alloc(ctx, (size_t)H * P));
  {
    // the hidden layer's variance is not optional: its standard deviation places the last layer's inputs
    ProfileScope ps(ctx, "dgp_hidden");
    DMO_TRY(svgp_latent_moments(ctx, g->hidden, up, X, P, m1.p, s1.p));
    DMO_LAUNCH(dgp_hidden_epilogue_kernel, (unsigned)ceil_div(P, 256), 256, 0, X, P, d, H, g->xlb.p, g->xrg.p, g->w1.p, g->b1,
               g->jitter, g->min_var, m1.p, s1.p);
  }
  {
    ProfileScope ps(ctx, "dgp_layer2");
    const int PT = DG_ROWS / J;
    dim3 grid((unsigned)ceil_div(P, PT), (unsigned)T);
    const double* sites = g->quadrature ? g->sites.p : nullptr;
    if (var) {
      DMO_CUDA(cudaFuncSetAttribute(dgp_layer2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DG_SMEM));
      DMO_LAUNCH(dgp_layer2_kernel<true>, grid, 256, DG_SMEM, g->tasks, T, P, H, J, PT, g->Z2, g->Npad2, m1.p, s1.p, sites, seed,
                 stream_id, g->c2, g->min_var, eps, mean, var);
    } else {
      DMO_CUDA(cudaFuncSetAttribute(dgp_layer2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DG_SMEM));
      DMO_LAUNCH(dgp_layer2_kernel<false>, grid, 256, DG_SMEM, g->tasks, T, P, H, J, PT, g->Z2, g->Npad2, m1.p, s1.p, sites, seed,
                 stream_id, g->c2, g->min_var, eps, mean, nullptr);
    }
  }
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

extern "C" {

int dmo_dgp_destroy(dmo_ctx* ctx, dmo_dgp* g) {
  if (!ctx) return DMO_ERR_ARG;
  if (!g) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  if (g->hidden) dmo_svgp_destroy(ctx, g->hidden);
  if (g->last) dmo_svgp_destroy(ctx, g->last);
  delete g;
  return DMO_OK;
}

int dmo_dgp_create(dmo_ctx* ctx, int d, int H, int T, int64_t Z1, int64_t Z2, const double* Z1pts, const double* s1, const double* ls1,
                   const double* q_mu1, const double* q_sqrt1, const double* w1, double b1, const double* Z2pts, const double* s2,
                   const double* ls2, const double* q_mu2, const double* q_sqrt2, double c2, const double* noise, double jitter,
                   double min_variance, int n_sites, const double* quad_sites, const double* y_mean, const double* y_std,
                   const double* xlb, const double* xrng, dmo_dgp** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out, "dgp_create: null output");
  *out = nullptr;
  DMO_REQUIRE(H >= 1 && H <= DG_MAX_HT && T >= 1 && T <= DG_MAX_HT, "dgp_create: 1 <= H, T <= %d (got H=%d T=%d)", DG_MAX_HT, H, T);
  DMO_REQUIRE(n_sites >= 1 && n_sites <= DG_MAX_SITES, "dgp_create: 1 <= n_sites <= %d (got %d)", DG_MAX_SITES, n_sites);
  DMO_REQUIRE(Z1 >= 1 && Z1 <= DG_ZMAX && Z2 >= 1 && Z2 <= DG_ZMAX && d >= 1 && d <= MT_FIT_DMAX,
              "dgp_create: unsupported shape d=%d Z1=%lld Z2=%lld (d <= %d, Z <= %lld)", d, (long long)Z1, (long long)Z2, MT_FIT_DMAX,
              (long long)DG_ZMAX);
  DMO_REQUIRE(Z1pts && s1 && ls1 && q_mu1 && q_sqrt1 && w1 && Z2pts && s2 && ls2 && q_mu2 && q_sqrt2 && noise && y_mean && y_std && xlb &&
                  xrng,
              "dgp_create: null pointer");
  DMO_REQUIRE(jitter >= 0.0 && isfinite(jitter), "dgp_create: jitter must be finite and >= 0 (got %g)", jitter);
  DMO_REQUIRE(min_variance >= 0.0 && isfinite(min_variance), "dgp_create: min_variance must be finite and >= 0 (got %g)", min_variance);
  DMO_REQUIRE(isfinite(b1) && isfinite(c2), "dgp_create: the prior means must be finite");
  std::vector<double> hn(T), hw(d), ym(T), ys(T), hq;
  DMO_CUDA(cudaMemcpy(hn.data(), noise, T * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(hw.data(), w1, d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ym.data(), y_mean, T * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(ys.data(), y_std, T * sizeof(double), cudaMemcpyDefault));
  for (int t = 0; t < T; ++t) {
    DMO_REQUIRE(hn[t] > 0.0 && isfinite(hn[t]), "dgp_create: noise[%d] must be finite and > 0 (got %g)", t, hn[t]);
    DMO_REQUIRE(isfinite(ym[t]) && isfinite(ys[t]), "dgp_create: y_mean / y_std[%d] must be finite", t);
  }
  for (int k = 0; k < d; ++k) DMO_REQUIRE(isfinite(hw[k]), "dgp_create: w1[%d] must be finite", k);
  if (quad_sites) {
    hq.resize((size_t)n_sites * H);
    DMO_CUDA(cudaMemcpy(hq.data(), quad_sites, hq.size() * sizeof(double), cudaMemcpyDefault));
    for (double q : hq) DMO_REQUIRE(isfinite(q), "dgp_create: quad_sites must be finite");
  }
  struct Del {
    dmo_ctx* c;
    void operator()(dmo_dgp* g) const { dmo_dgp_destroy(c, g); }
  };
  std::unique_ptr<dmo_dgp, Del> g(new dmo_dgp(), Del{ctx});
  g->d = d;
  g->H = H;
  g->T = T;
  g->J = n_sites;
  g->Z2 = Z2;
  g->b1 = b1;
  g->c2 = c2;
  g->jitter = jitter;
  g->min_var = min_variance;
  g->quadrature = quad_sites != nullptr;
  // the svgp checks s > 0, ell > 0, xrng > 0, a lower-triangular q_sqrt and a positive-definite K(Z, Z) + jitter I
  const std::vector<double> zeros((size_t)DG_MAX_HT, 0.0), ones((size_t)DG_MAX_HT, 1.0);
  DMO_TRY(layer_error(ctx, dmo_svgp_create(ctx, H, H, Z1, d, Z1pts, s1, ls1, q_mu1, q_sqrt1, nullptr, jitter, zeros.data(), ones.data(),
                                           nullptr, xlb, xrng, &g->hidden),
                      "hidden"));
  DMO_TRY(layer_error(ctx, dmo_svgp_create(ctx, T, T, Z2, H, Z2pts, s2, ls2, q_mu2, q_sqrt2, nullptr, jitter, zeros.data(), ones.data(),
                                           nullptr, zeros.data(), ones.data(), &g->last),
                      "last"));
  std::vector<double> hs2(T), lb(d), rg(d);
  DMO_CUDA(cudaMemcpy(hs2.data(), s2, T * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(lb.data(), xlb, d * sizeof(double), cudaMemcpyDefault));
  DMO_CUDA(cudaMemcpy(rg.data(), xrng, d * sizeof(double), cudaMemcpyDefault));
  for (int t = 0; t < T; ++t) {
    SvLatentView v;
    if (svgp_latent_view(g->last, t, &v) != DMO_OK) return dmo_fail(ctx, DMO_ERR_INTERNAL, "dgp_create: task %d has no operator planes", t);
    DgTask& tk = g->tasks.t[t];
    tk.O0 = v.O0;
    tk.O1 = v.O1;
    tk.A = v.A;
    tk.XtT = v.XtT;
    tk.inv_ls = v.inv_ls;
    tk.s_jit = hs2[t] + jitter;
    tk.noise = hn[t];
    tk.ystd = ys[t];
    tk.ymean = ym[t];
    g->Npad2 = v.Npad;
  }
  DMO_TRY(upload(ctx, g->w1, hw));
  DMO_TRY(upload(ctx, g->xlb, lb));
  DMO_TRY(upload(ctx, g->xrg, rg));
  if (quad_sites) DMO_TRY(upload(ctx, g->sites, hq));
  DMO_CHECK_LAUNCH();
  DMO_CUDA(dmo_wait(ctx));  // host vectors above are staged from the stack
  *out = g.release();
  return DMO_OK;
}

int dmo_dgp_predict(dmo_ctx* ctx, dmo_dgp* g, const double* X, int64_t P, uint64_t seed, uint64_t stream_id, double* eps_out,
                    double* mean, double* var, int precision) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(g, "dgp_predict: null model");
  GpUnitPredict up;
  DMO_TRY(up.check(ctx, "dgp_predict", precision, g->d));
  if (P == 0) return DMO_OK;
  DMO_REQUIRE(P > 0 && X && mean, "dgp_predict: bad arguments");
  DMO_REQUIRE(stream_id < ((uint64_t)1 << 54), "dgp_predict: stream_id must be below 2^54");
  const int d = g->d, H = g->H, T = g->T, J = g->J;
  In<double> x;
  Out<double> om, ov, oe;
  DMO_TRY(x.init(ctx, X, (size_t)P * d));
  DMO_TRY(om.init(ctx, mean, (size_t)P * T));
  DMO_TRY(ov.init(ctx, var, (size_t)P * T));
  DMO_TRY(oe.init(ctx, eps_out, (size_t)J * P * H));
  DMO_TRY(dgp_predict_device(ctx, g, up, x.d, P, seed, stream_id, oe.d, om.d, ov.d));
  DMO_TRY(up.watchdog(ctx));
  DMO_TRY(om.finish(ctx));
  DMO_TRY(ov.finish(ctx));
  DMO_TRY(oe.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
