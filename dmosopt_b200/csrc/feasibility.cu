// Logistic feasibility model (dmosopt/feasibility.py): the cross-validated L1-logistic grid search of
// LogisticFeasibilityModel and its rank.  The host (dmosopt_b200/feasibility.py) assigns the stratified folds and
// eigendecomposes each dataset's d x d covariance; everything that touches the N rows runs here:
//   feas_scores_kernel     centred rows projected on the d - 1 principal components of every dataset (5 folds + all)
//   feas_scaler_kernel     mean / population std of each score column over the dataset's training rows
//   feas_solve_kernel      one CTA per (dataset, C, k) problem: proximal Newton on C sum log(1 + exp(-s t)) + |w|_1,
//                          its weighted Gram H = C [Z_k 1]^T diag(p(1 - p)) [Z_k 1] in 4 x 4 register blocks, the L1
//                          quadratic subproblem by coordinate descent in shared memory, a backtracking line search,
//                          then the held-out count of its fold.  A problem leaves the GPU when its CTA converges.
//   feas_eval_kernel       rank / probabilities of fitted models: centre, project, standardise, dot, expit, mean.
// Every sum runs in a fixed order, so a fit and an evaluation repeat bit for bit.
#include <algorithm>

#include "common.cuh"

struct dmo_feas {
  int d = 0, J = 0;
  int64_t stride = 0;    // doubles per constraint in par
  DevBuf<int32_t> k;     // (J,) components of each constraint, 0 = single-class constraint (p = 1)
  DevBuf<double> par;    // (J, stride): mean[d], comps[(d-1) d], smean[d-1], sscale[d-1], coef[d-1], intercept
};

namespace {

constexpr int FEAS_MAX_D = 90;
constexpr int FEAS_MAX_J = 32;
constexpr int64_t FEAS_MAX_N = 65536;
constexpr int FEAS_MAX_C = 16;
constexpr int FEAS_SETS = 6;                 // the five cross-validation folds, then all rows
constexpr int FS_THREADS = 256;
constexpr int FS_WARPS = FS_THREADS / 32;
constexpr int FS_ROWS = 32;                  // rows per Gram tile (a multiple of FS_WARPS)
constexpr int FS_MAXBLK = 2;                 // 4 x 4 blocks of H per thread: 23 * 24 / 2 = 276 <= 2 * 256
constexpr int ROW_TILE = 128;                // rows per CTA of the projection kernels
constexpr int CD_MAX_SWEEPS = 500;
constexpr double FS_F_SLACK = 1e-15;  // rounding allowance per training row of the line search's comparison of F
constexpr int LS_MAX = 60;
constexpr size_t FEAS_SCORE_BYTES = size_t(1) << 31;  // score matrices of one batch of constraints

int64_t feas_stride(int d) { return (int64_t)d + (int64_t)(d - 1) * d + 3 * (int64_t)(d - 1) + 1; }

// log(1 + exp(-m)) without overflow
__device__ __forceinline__ double log1pexp_neg(double m) { return m > 0.0 ? log1p(exp(-m)) : -m + log1p(exp(m)); }

// Z[s, i, c] = sum_l V_s[c, l] (x_il - mean_s[l]) for every row i and component c < d - 1 of dataset s = blockIdx.y
__global__ void __launch_bounds__(ROW_TILE) feas_scores_kernel(const double* __restrict__ X, int64_t N, int d,
                                                               const double* __restrict__ mean, const double* __restrict__ comps,
                                                               double* __restrict__ Z) {
  extern __shared__ double xs[];
  const int ld = d | 1, km = d - 1, s = blockIdx.y;
  const int64_t r0 = (int64_t)blockIdx.x * ROW_TILE;
  const int rows = (int)(N - r0 < ROW_TILE ? N - r0 : ROW_TILE);
  for (int e = threadIdx.x; e < rows * d; e += blockDim.x) {
    const int r = e / d, l = e - r * d;
    xs[r * ld + l] = X[(r0 + r) * d + l];
  }
  __syncthreads();
  if ((int)threadIdx.x >= rows) return;
  const double* mu = mean + (int64_t)s * d;
  const double* V = comps + (int64_t)s * km * d;
  const double* x = xs + threadIdx.x * ld;
  double* z = Z + ((int64_t)s * N + r0 + threadIdx.x) * km;
  for (int c = 0; c < km; ++c) {
    double u = 0.0;
    for (int l = 0; l < d; ++l) u = fma(V[c * d + l], x[l] - mu[l], u);
    z[c] = u;
  }
}

// mean and scale of score column c = blockIdx.x of dataset s = blockIdx.y over its training rows (StandardScaler: the
// population std; a column whose variance is within rounding of zero keeps scale 1)
__global__ void __launch_bounds__(FS_THREADS) feas_scaler_kernel(const double* __restrict__ Z, int64_t N, int d,
                                                                 const int8_t* __restrict__ fold, double* __restrict__ smean,
                                                                 double* __restrict__ sscale) {
  __shared__ double part[FS_WARPS];
  const int km = d - 1, c = blockIdx.x, s = blockIdx.y, f = s % FEAS_SETS;
  const int8_t* fo = fold + (int64_t)(s / FEAS_SETS) * N;
  const double* z = Z + (int64_t)s * N * km + c;
  double a = 0.0, n = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += FS_THREADS)
    if (f == FEAS_SETS - 1 || fo[i] != f) {
      a += z[i * km];
      n += 1.0;
    }
  const double cnt = block_sum<FS_WARPS>(n, part);
  const double mean = block_sum<FS_WARPS>(a, part) / cnt;
  a = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += FS_THREADS)
    if (f == FEAS_SETS - 1 || fo[i] != f) {
      const double e = z[i * km] - mean;
      a += e * e;
    }
  const double var = block_sum<FS_WARPS>(a, part) / cnt;
  if (threadIdx.x == 0) {
    const double eps = 2.220446049250313e-16, nm = cnt * mean * eps;
    const bool constant = var <= cnt * eps * var + nm * nm;
    smean[(int64_t)s * km + c] = mean;
    sscale[(int64_t)s * km + c] = constant || var == 0.0 ? 1.0 : sqrt(var);
  }
}

__global__ void feas_standardise_kernel(double* __restrict__ Z, int64_t N, int d, int S, const double* __restrict__ smean,
                                        const double* __restrict__ sscale) {
  const int km = d - 1;
  const int64_t total = (int64_t)S * N * km;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / km;
    const int c = (int)(e - row * km);
    const int s = (int)(row / N);
    Z[e] = (Z[e] - smean[(int64_t)s * km + c]) / sscale[(int64_t)s * km + c];
  }
}

// t = z_i[:k] . w[:k] (lanes stride the columns, then the butterfly) + w[k]; every lane gets t
__device__ __forceinline__ double feas_margin(const double* z, const double* w, int k, int lane) {
  double t = 0.0;
  for (int c = lane; c < k; c += 32) t = fma(z[c], w[c], t);
  return warp_sum(t) + w[k];
}

// One CTA per problem p = (s nC + ci) (d - 1) + k - 1 of the batch: dataset s (constraint s / 6, fold s % 6, fold 5 =
// all rows), C = Cs[ci], the first k standardised scores.  Minimises F(w, b) = C sum_train log(1 + exp(-s_i t_i)) +
// |w|_1 by proximal Newton until the minimum-norm subgradient is below tol max(1, C n_train).
__global__ void __launch_bounds__(FS_THREADS) feas_solve_kernel(const double* __restrict__ Z, int64_t N, int d,
                                                                const uint8_t* __restrict__ lab, const int8_t* __restrict__ fold,
                                                                const double* __restrict__ Cs, int nC, int max_iter, double tol,
                                                                double* __restrict__ coef, int32_t* __restrict__ iters,
                                                                double* __restrict__ fobj, double* __restrict__ kkt_o,
                                                                int8_t* __restrict__ conv_o, int64_t* __restrict__ correct) {
  extern __shared__ double sm[];
  __shared__ double part[FS_WARPS];
  __shared__ double s_F, s_kkt, s_D, s_Fn, s_mu;
  __shared__ int s_stop, s_acc;
  const int km = d - 1, p = blockIdx.x;
  const int k = p % km + 1, ci = (p / km) % nC, s = p / (km * nC);
  const int j = s / FEAS_SETS, f = s % FEAS_SETS;
  const double C = Cs[ci];
  const double* Zs = Z + (int64_t)s * N * km;
  const uint8_t* y = lab + (int64_t)j * N;
  const int8_t* fo = fold + (int64_t)j * N;
  const int K1 = k + 1, KP = (K1 + 3) & ~3, nb = KP / 4;
  const int KPmax = (d + 3) & ~3;
  const int R0 = max(KPmax * KPmax, FS_ROWS * KPmax);
  double* H = sm;   // KP x KP, aliases the tile
  double* zt = sm;  // FS_ROWS x KP
  double* w = sm + R0;
  double* dl = w + KPmax;
  double* g = dl + KPmax;
  double* hd = g + KPmax;
  double* wt = hd + KPmax;
  double* tv = wt + KPmax;
  double* tr = tv + FS_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  auto train = [&](int64_t i) { return f == FEAS_SETS - 1 || fo[i] != f; };

  // training rows and positives: a training set of one class has no classifier (the fold scores NaN)
  double a0 = 0.0, a1 = 0.0;
  for (int64_t i = tid; i < N; i += FS_THREADS)
    if (train(i)) {
      a0 += 1.0;
      a1 += y[i];
    }
  const double ntr = block_sum<FS_WARPS>(a0, part), npos = block_sum<FS_WARPS>(a1, part);
  const int64_t out = (int64_t)p * d;
  if (npos == 0.0 || npos == ntr) {
    for (int c = tid; c < d; c += FS_THREADS) coef[out + c] = 0.0;
    if (tid == 0) {
      iters[p] = -1;
      fobj[p] = kkt_o[p] = NAN;
      conv_o[p] = 0;
      correct[p] = -1;
    }
    return;
  }
  for (int c = tid; c < KPmax; c += FS_THREADS) w[c] = 0.0;
  // this thread's 4 x 4 blocks (A, B), A <= B < nb, of the upper triangle of H
  int blkA[FS_MAXBLK], blkB[FS_MAXBLK];
  const int nblk = nb * (nb + 1) / 2;
#pragma unroll
  for (int q = 0; q < FS_MAXBLK; ++q) {
    int b = tid + q * FS_THREADS, A = 0;
    if (b < nblk) {
      while (b >= nb - A) {
        b -= nb - A;
        ++A;
      }
      blkA[q] = A;
      blkB[q] = A + b;
    } else {
      blkA[q] = blkB[q] = -1;
    }
  }
  const double gtol = tol * fmax(1.0, C * ntr);
  int it = 0;
  __syncthreads();
  for (;; ++it) {
    // ---- margins, loss, gradient and weighted Gram at w
    double acc[FS_MAXBLK][16];
#pragma unroll
    for (int q = 0; q < FS_MAXBLK; ++q)
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[q][e] = 0.0;
    double gacc = 0.0, lpart = 0.0;
    for (int64_t base = 0; base < N; base += FS_ROWS) {
      const int rows = (int)(N - base < FS_ROWS ? N - base : FS_ROWS);
      for (int e = tid; e < FS_ROWS * KP; e += FS_THREADS) {
        const int r = e / KP, c = e - r * KP;
        zt[e] = r < rows ? (c < k ? Zs[(base + r) * km + c] : c == k ? 1.0 : 0.0) : 0.0;
      }
      __syncthreads();
      for (int r = warp; r < FS_ROWS; r += FS_WARPS) {
        const double t = feas_margin(zt + r * KP, w, k, lane);
        if (lane == 0) {
          double v = 0.0, res = 0.0;
          if (r < rows && train(base + r)) {
            const int yi = y[base + r];
            lpart += log1pexp_neg(yi ? t : -t);
            const double pr = 1.0 / (1.0 + exp(-t));
            v = C * (pr * (1.0 - pr));
            res = C * (pr - yi);
          }
          tv[r] = v;
          tr[r] = res;
        }
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < FS_MAXBLK; ++q) {
        if (blkA[q] < 0) continue;
        const int ca = 4 * blkA[q], cb = 4 * blkB[q];
        for (int r = 0; r < rows; ++r) {
          const double v = tv[r];
          const double2 a01 = *reinterpret_cast<const double2*>(zt + r * KP + ca);
          const double2 a23 = *reinterpret_cast<const double2*>(zt + r * KP + ca + 2);
          const double2 b01 = *reinterpret_cast<const double2*>(zt + r * KP + cb);
          const double2 b23 = *reinterpret_cast<const double2*>(zt + r * KP + cb + 2);
          const double za[4] = {a01.x, a01.y, a23.x, a23.y};
          const double vb[4] = {v * b01.x, v * b01.y, v * b23.x, v * b23.y};
#pragma unroll
          for (int x = 0; x < 4; ++x)
#pragma unroll
            for (int z = 0; z < 4; ++z) acc[q][x * 4 + z] = fma(za[x], vb[z], acc[q][x * 4 + z]);
        }
      }
      if (tid < K1)
        for (int r = 0; r < rows; ++r) gacc = fma(tr[r], zt[r * KP + tid], gacc);
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < FS_MAXBLK; ++q) {
      if (blkA[q] < 0) continue;
      for (int x = 0; x < 4; ++x)
        for (int z = 0; z < 4; ++z) {
          const int ia = 4 * blkA[q] + x, ib = 4 * blkB[q] + z;
          if (ia < K1 && ib < K1 && (blkA[q] < blkB[q] || x <= z)) {
            H[ia * KP + ib] = acc[q][x * 4 + z];
            H[ib * KP + ia] = acc[q][x * 4 + z];
          }
        }
    }
    if (tid < K1) g[tid] = gacc;
    if (lane == 0) part[warp] = lpart;
    __syncthreads();
    if (tid == 0) {
      double L = 0.0;
      for (int q = 0; q < FS_WARPS; ++q) L += part[q];
      double l1 = 0.0, kkt = fabs(g[k]), hmax = 0.0;
      for (int c = 0; c < k; ++c) {
        l1 += fabs(w[c]);
        const double e = w[c] != 0.0 ? fabs(g[c] + copysign(1.0, w[c])) : fmax(0.0, fabs(g[c]) - 1.0);
        kkt = fmax(kkt, e);
      }
      for (int c = 0; c < K1; ++c) hmax = fmax(hmax, H[c * KP + c]);
      s_F = C * L + l1;
      s_kkt = kkt;
      s_mu = 1e-12 * hmax + 1e-300;
      s_stop = kkt <= gtol || it >= max_iter;
    }
    __syncthreads();
    if (s_stop) break;
    // ---- L1 quadratic subproblem: min_D g.D + D^T H D / 2 + |w + D|_1 by cyclic coordinate descent (warp 0)
    if (warp == 0) {
      for (int c = lane; c < K1; c += 32) dl[c] = hd[c] = 0.0;
      __syncwarp();
      const double mu = s_mu;
      double maxdl = 0.0;  // largest |D| coordinate so far: the sweeps stop once they move D by 1e-7 of it
      for (int sweep = 0; sweep < CD_MAX_SWEEPS; ++sweep) {
        double maxd = 0.0, maxu = 0.0;
        for (int a = 0; a < K1; ++a) {
          const double haa = H[a * KP + a] + mu;
          const double gq = g[a] + hd[a];
          double delta, un;
          if (a < k) {
            const double u = w[a] + dl[a];
            const double zz = u - gq / haa, th = 1.0 / haa;
            un = zz > th ? zz - th : zz < -th ? zz + th : 0.0;
            delta = un - u;
          } else {
            delta = -gq / haa;
            un = w[a] + dl[a] + delta;
          }
          __syncwarp();
          if (delta != 0.0) {
            for (int l = lane; l < K1; l += 32) hd[l] = fma(H[l * KP + a], delta, hd[l]);
            if (lane == 0) dl[a] += delta;
          }
          __syncwarp();
          maxd = fmax(maxd, fabs(delta));
          maxu = fmax(maxu, fabs(un));
          maxdl = fmax(maxdl, fabs(dl[a]));
        }
        if (maxd <= 1e-7 * maxdl + 1e-15 * fmax(1.0, maxu)) break;
      }
      double D = 0.0;
      for (int c = lane; c < K1; c += 32) {
        D += g[c] * dl[c];
        if (c < k) D += fabs(w[c] + dl[c]) - fabs(w[c]);
      }
      D = warp_sum(D);
      if (lane == 0) s_D = D;
    }
    __syncthreads();
    if (!(s_D < 0.0)) break;  // no descent direction left at this precision
    // ---- backtracking line search on F(w + alpha D) (Armijo, sigma = 1e-4).  Near the optimum the predicted decrease
    // falls below the rounding of F (a sum of n terms of size up to C), so a step that raises F by no more than
    // FS_F_SLACK n_train |F| passes: it keeps the Newton iteration going until the KKT measure, not F, says it has converged.
    double alpha = 1.0;
    int ls = 0;
    for (; ls < LS_MAX; ++ls, alpha *= 0.5) {
      for (int c = tid; c < K1; c += FS_THREADS) wt[c] = w[c] + alpha * dl[c];
      __syncthreads();
      double lp = 0.0;
      for (int64_t i = warp; i < N; i += FS_WARPS) {
        const double t = feas_margin(Zs + i * km, wt, k, lane);
        if (lane == 0 && train(i)) lp += log1pexp_neg(y[i] ? t : -t);
      }
      if (lane == 0) part[warp] = lp;
      __syncthreads();
      if (tid == 0) {
        double L = 0.0, l1 = 0.0;
        for (int q = 0; q < FS_WARPS; ++q) L += part[q];
        for (int c = 0; c < k; ++c) l1 += fabs(wt[c]);
        s_Fn = C * L + l1;
        s_acc = s_Fn <= s_F + 1e-4 * alpha * s_D + FS_F_SLACK * ntr * fabs(s_F);
      }
      __syncthreads();
      if (s_acc) break;
    }
    if (ls == LS_MAX) break;  // w stays; F and the KKT measure above describe it
    for (int c = tid; c < K1; c += FS_THREADS) w[c] = wt[c];
    __syncthreads();
  }
  for (int c = tid; c < d; c += FS_THREADS) coef[out + c] = c < k ? w[c] : c == d - 1 ? w[k] : 0.0;
  // held-out rows of this fold: correct when (t > 0) == label
  int64_t hit = 0;
  if (f < FEAS_SETS - 1)
    for (int64_t i = warp; i < N; i += FS_WARPS) {
      if (fo[i] != f) continue;
      const double t = feas_margin(Zs + i * km, w, k, lane);
      if (lane == 0) hit += (t > 0.0) == (y[i] != 0);
    }
  if (lane == 0) part[warp] = (double)hit;
  __syncthreads();
  if (tid == 0) {
    int64_t h = 0;
    for (int q = 0; q < FS_WARPS; ++q) h += (int64_t)part[q];
    iters[p] = it;
    fobj[p] = s_F;
    kkt_o[p] = s_kkt;
    conv_o[p] = s_kkt <= gtol;
    correct[p] = h;
  }
}

// rank[i] = sum_j p_j(x_i) / J, proba[j, i] = p_j, dec[j, i] = t_j (+inf for a single-class constraint)
__global__ void __launch_bounds__(ROW_TILE) feas_eval_kernel(const double* __restrict__ X, int64_t n, int d, int J,
                                                             const int32_t* __restrict__ kk, const double* __restrict__ par,
                                                             int64_t stride, double* __restrict__ rank, double* __restrict__ proba,
                                                             double* __restrict__ dec) {
  extern __shared__ double xs[];
  const int ld = d | 1, km = d - 1;
  const int64_t r0 = (int64_t)blockIdx.x * ROW_TILE;
  const int rows = (int)(n - r0 < ROW_TILE ? n - r0 : ROW_TILE);
  for (int e = threadIdx.x; e < rows * d; e += blockDim.x) {
    const int r = e / d, l = e - r * d;
    xs[r * ld + l] = X[(r0 + r) * d + l];
  }
  __syncthreads();
  if ((int)threadIdx.x >= rows) return;
  const double* x = xs + threadIdx.x * ld;
  const int64_t i = r0 + threadIdx.x;
  double acc = 0.0;
  for (int j = 0; j < J; ++j) {
    const int k = kk[j];
    double t = INFINITY, pr = 1.0;
    if (k > 0) {
      const double* mu = par + (int64_t)j * stride;
      const double* V = mu + d;
      const double* smu = V + (int64_t)km * d;
      const double* ssc = smu + km;
      const double* wc = ssc + km;
      t = 0.0;
      for (int c = 0; c < k; ++c) {
        double u = 0.0;
        for (int l = 0; l < d; ++l) u = fma(V[c * d + l], x[l] - mu[l], u);
        t = fma((u - smu[c]) / ssc[c], wc[c], t);
      }
      t = t + wc[km];
      pr = 1.0 / (1.0 + exp(-t));
    }
    acc += pr;
    if (proba) proba[(int64_t)j * n + i] = pr;
    if (dec) dec[(int64_t)j * n + i] = t;
  }
  if (rank) rank[i] = acc / J;
}

int eval_launch(dmo_ctx* ctx, const dmo_feas* m, const double* dX, int64_t n, double* rank, double* proba, double* dec) {
  if (n == 0) return DMO_OK;
  const size_t smem = (size_t)ROW_TILE * (m->d | 1) * sizeof(double);
  DMO_CUDA(cudaFuncSetAttribute(feas_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfileScope ps(ctx, "feas_eval_kernel");
  DMO_LAUNCH(feas_eval_kernel, (unsigned)ceil_div(n, ROW_TILE), ROW_TILE, smem, dX, n, m->d, m->J, m->k.p, m->par.p, m->stride,
             rank, proba, dec);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

}  // namespace

int feas_rank_device(dmo_ctx* ctx, const dmo_feas* m, const double* dX, int64_t n, double* d_rank) {
  return eval_launch(ctx, m, dX, n, d_rank, nullptr, nullptr);
}

int feas_model_dim(const dmo_feas* m) { return m->d; }

extern "C" {

int dmo_feas_fit(dmo_ctx* ctx, const double* X, int64_t N, int d, int J, const uint8_t* labels, const int8_t* folds,
                 const double* pca_mean, const double* pca_comps, int nC, const double* Cs, int max_iter, double tol,
                 double* scaler_mean, double* scaler_scale, double* coef, int32_t* iters, double* objective, double* kkt,
                 int8_t* converged, int64_t* correct) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(X && labels && folds && pca_mean && pca_comps && Cs && scaler_mean && scaler_scale && coef && iters && objective &&
                  kkt && converged && correct,
              "feas_fit: null argument");
  DMO_REQUIRE(d >= 2 && d <= FEAS_MAX_D, "feas_fit: d=%d outside [2, %d]", d, FEAS_MAX_D);
  DMO_REQUIRE(J >= 1 && J <= FEAS_MAX_J, "feas_fit: J=%d outside [1, %d]", J, FEAS_MAX_J);
  DMO_REQUIRE(N >= 5 && N <= FEAS_MAX_N, "feas_fit: N=%lld outside [5, %lld]", (long long)N, (long long)FEAS_MAX_N);
  DMO_REQUIRE(nC >= 1 && nC <= FEAS_MAX_C, "feas_fit: %d values of C outside [1, %d]", nC, FEAS_MAX_C);
  DMO_REQUIRE(max_iter >= 0 && tol >= 0.0, "feas_fit: bad max_iter / tol");
  for (int c = 0; c < nC; ++c) DMO_REQUIRE(Cs[c] > 0.0 && isfinite(Cs[c]), "feas_fit: C must be positive and finite");
  const int km = d - 1, S = J * FEAS_SETS;
  const int64_t per_set = (int64_t)nC * km;  // problems per dataset
  In<double> ix, imean, icomps, iC;
  In<uint8_t> ilab;
  In<int8_t> ifold;
  DMO_TRY(ix.init(ctx, X, (size_t)N * d));
  DMO_TRY(ilab.init(ctx, labels, (size_t)J * N));
  DMO_TRY(ifold.init(ctx, folds, (size_t)J * N));
  DMO_TRY(imean.init(ctx, pca_mean, (size_t)S * d));
  DMO_TRY(icomps.init(ctx, pca_comps, (size_t)S * km * d));
  DMO_TRY(iC.init(ctx, Cs, (size_t)nC));
  const int64_t P = (int64_t)S * per_set;
  Out<double> osm, oss, ocoef, oobj, okkt;
  Out<int32_t> oit;
  Out<int8_t> oconv;
  Out<int64_t> ocor;
  DMO_TRY(osm.init(ctx, scaler_mean, (size_t)S * km));
  DMO_TRY(oss.init(ctx, scaler_scale, (size_t)S * km));
  DMO_TRY(ocoef.init(ctx, coef, (size_t)P * d));
  DMO_TRY(oit.init(ctx, iters, (size_t)P));
  DMO_TRY(oobj.init(ctx, objective, (size_t)P));
  DMO_TRY(okkt.init(ctx, kkt, (size_t)P));
  DMO_TRY(oconv.init(ctx, converged, (size_t)P));
  DMO_TRY(ocor.init(ctx, correct, (size_t)P));
  // constraints in batches whose score matrices fit FEAS_SCORE_BYTES
  const size_t set_bytes = (size_t)N * km * sizeof(double);
  const int jb = (int)std::max<size_t>(1, std::min<size_t>(J, FEAS_SCORE_BYTES / (FEAS_SETS * set_bytes)));
  DevBuf<double> Z;
  DMO_TRY(Z.alloc(ctx, (size_t)std::min(J, jb) * FEAS_SETS * N * km));
  const int KPmax = (d + 3) & ~3;
  const size_t solve_smem = ((size_t)std::max(KPmax * KPmax, FS_ROWS * KPmax) + 5 * KPmax + 2 * FS_ROWS) * sizeof(double);
  const size_t score_smem = (size_t)ROW_TILE * (d | 1) * sizeof(double);
  DMO_CUDA(cudaFuncSetAttribute(feas_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
  DMO_CUDA(cudaFuncSetAttribute(feas_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)score_smem));
  for (int j0 = 0; j0 < J; j0 += jb) {
    const int nj = std::min(jb, J - j0), s0 = j0 * FEAS_SETS, Sb = nj * FEAS_SETS;
    const int64_t p0 = (int64_t)s0 * per_set;
    {
      ProfileScope ps(ctx, "feas_scores_kernel");
      DMO_LAUNCH(feas_scores_kernel, dim3((unsigned)ceil_div(N, ROW_TILE), (unsigned)Sb), ROW_TILE, score_smem, ix.d, N, d,
                 imean.d + (int64_t)s0 * d, icomps.d + (int64_t)s0 * km * d, Z.p);
    }
    DMO_LAUNCH(feas_scaler_kernel, dim3((unsigned)km, (unsigned)Sb), FS_THREADS, 0, Z.p, N, d, ifold.d + (int64_t)j0 * N,
               osm.d + (int64_t)s0 * km, oss.d + (int64_t)s0 * km);
    DMO_LAUNCH(feas_standardise_kernel, (unsigned)std::min<int64_t>(ceil_div((int64_t)Sb * N * km, 256), ctx->sm_count * 16), 256, 0,
               Z.p, N, d, Sb, osm.d + (int64_t)s0 * km, oss.d + (int64_t)s0 * km);
    {
      ProfileScope ps(ctx, "feas_solve_kernel");
      DMO_LAUNCH(feas_solve_kernel, (unsigned)(Sb * per_set), FS_THREADS, solve_smem, Z.p, N, d, ilab.d + (int64_t)j0 * N,
                 ifold.d + (int64_t)j0 * N, iC.d, nC, max_iter, tol, ocoef.d + p0 * d, oit.d + p0, oobj.d + p0, okkt.d + p0,
                 oconv.d + p0, ocor.d + p0);
    }
    DMO_CHECK_LAUNCH();
  }
  DMO_TRY(osm.finish(ctx));
  DMO_TRY(oss.finish(ctx));
  DMO_TRY(ocoef.finish(ctx));
  DMO_TRY(oit.finish(ctx));
  DMO_TRY(oobj.finish(ctx));
  DMO_TRY(okkt.finish(ctx));
  DMO_TRY(oconv.finish(ctx));
  DMO_TRY(ocor.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_feas_create(dmo_ctx* ctx, int d, int J, const int32_t* k, const double* mean, const double* comps, const double* smean,
                    const double* sscale, const double* coef, const double* intercept, dmo_feas** out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out && k && mean && comps && smean && sscale && coef && intercept, "feas_create: null argument");
  DMO_REQUIRE(d >= 2 && d <= FEAS_MAX_D, "feas_create: d=%d outside [2, %d]", d, FEAS_MAX_D);
  DMO_REQUIRE(J >= 1 && J <= FEAS_MAX_J, "feas_create: J=%d outside [1, %d]", J, FEAS_MAX_J);
  DMO_REQUIRE(!dmo_is_device_ptr(k) && !dmo_is_device_ptr(mean) && !dmo_is_device_ptr(comps) && !dmo_is_device_ptr(smean) &&
                  !dmo_is_device_ptr(sscale) && !dmo_is_device_ptr(coef) && !dmo_is_device_ptr(intercept),
              "feas_create: the parameters are host arrays");
  const int km = d - 1;
  const int64_t st = feas_stride(d);
  std::vector<double> h((size_t)J * st, 0.0);
  for (int j = 0; j < J; ++j) {
    DMO_REQUIRE(k[j] >= 0 && k[j] <= km, "feas_create: k[%d]=%d outside [0, %d]", j, k[j], km);
    double* q = h.data() + (size_t)j * st;
    std::copy(mean + (size_t)j * d, mean + (size_t)(j + 1) * d, q);
    std::copy(comps + (size_t)j * km * d, comps + (size_t)(j + 1) * km * d, q + d);
    std::copy(smean + (size_t)j * km, smean + (size_t)(j + 1) * km, q + d + km * d);
    std::copy(sscale + (size_t)j * km, sscale + (size_t)(j + 1) * km, q + d + km * d + km);
    std::copy(coef + (size_t)j * km, coef + (size_t)(j + 1) * km, q + d + km * d + 2 * km);
    q[st - 1] = intercept[j];
  }
  dmo_feas* m = new dmo_feas;
  m->d = d;
  m->J = J;
  m->stride = st;
  int rc = m->k.alloc(ctx, J);
  if (rc == DMO_OK) rc = m->par.alloc(ctx, h.size());
  if (rc != DMO_OK) {
    delete m;
    return rc;
  }
  cudaError_t e = cudaMemcpyAsync(m->k.p, k, J * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(m->par.p, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = dmo_wait(ctx);
  if (e != cudaSuccess) {
    delete m;
    return dmo_fail(ctx, DMO_ERR_CUDA, "feas_create: upload failed: %s", cudaGetErrorString(e));
  }
  *out = m;
  return DMO_OK;
}

int dmo_feas_destroy(dmo_ctx* ctx, dmo_feas* m) {
  if (!ctx) return DMO_ERR_ARG;
  if (!m) return DMO_OK;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_CUDA(dmo_wait(ctx));
  delete m;
  return DMO_OK;
}

int dmo_feas_eval(dmo_ctx* ctx, const dmo_feas* m, const double* X, int64_t n, int d, double* rank, double* proba,
                  double* decision) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(m && (X || n == 0) && n >= 0, "feas_eval: bad arguments");
  DMO_REQUIRE(d == m->d, "feas_eval: X has %d columns, the model %d", d, m->d);
  if (n == 0) return DMO_OK;
  In<double> ix;
  Out<double> orank, opr, odec;
  DMO_TRY(ix.init(ctx, X, (size_t)n * d));
  DMO_TRY(orank.init(ctx, rank, (size_t)n));
  DMO_TRY(opr.init(ctx, proba, (size_t)n * m->J));
  DMO_TRY(odec.init(ctx, decision, (size_t)n * m->J));
  DMO_TRY(eval_launch(ctx, m, ix.d, n, orank.d, opr.d, odec.d));
  DMO_TRY(orank.finish(ctx));
  DMO_TRY(opr.finish(ctx));
  DMO_TRY(odec.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
