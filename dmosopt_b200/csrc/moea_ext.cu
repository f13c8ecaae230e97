// Optimizer-specific kernels beyond the shared sort / variation path
// (SURVEY.md section 8a rows A11 AGE-MOEA, A12 SMPSO, A13/A15 MO-CMA-ES).
//   AGE-MOEA survival_score greedy selection   dmosopt/AGEMOEA.py:377-430
//   SMPSO velocity_vector / update_position    dmosopt/SMPSO.py:311-348
//   SMPSO per-swarm polynomial mutation        dmosopt/SMPSO.py:163-182
//   CMAES sampling x = x_p + sigma_p A_p z     dmosopt/CMAES.py:263-267
//   CMAES updateCholesky (batched)             dmosopt/CMAES.py:489-537
#include <algorithm>

#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------- AGE-MOEA
// Greedy survival score of one front.  yn: (m, M) normalised objectives; nn[i] = ||yn_i||_p.
// dist(s, r) = ||yn_s - yn_r||_p / nn[s]   (the reference divides row s of the distance matrix by nn[s], :402-404)
// Repeatedly: the remaining point with the largest sum of its two smallest distances to the selected set is selected
// and receives that sum as its crowding value (:410-428).  One CTA; every thread owns a strided slice of the points and
// keeps their two smallest distances in shared memory; per step one block-wide arg-max and one distance update.
constexpr int AGE_T = 1024;
constexpr int AGE_MAXM = 16;

__device__ __forceinline__ double minkowski(const double* a, const double* b, int M, double p) {
  double s = 0.0;
  for (int j = 0; j < M; ++j) s += pow(fabs(a[j] - b[j]), p);
  return pow(s, 1.0 / p);
}

__global__ void __launch_bounds__(AGE_T) age_survival_kernel(const double* __restrict__ yn, const double* __restrict__ nn,
                                                             int m, int M, double p, const int* __restrict__ extreme,
                                                             int n_ext, double* __restrict__ d1g, double* __restrict__ d2g,
                                                             uint8_t* __restrict__ selg, double* __restrict__ crowd) {
  __shared__ double s_val[AGE_T / 32];
  __shared__ int s_idx[AGE_T / 32];
  __shared__ double s_best[AGE_MAXM + 1];
  __shared__ int s_bi;
  const int tid = threadIdx.x;
  // initialise: two smallest distances to the extreme (pre-selected) points
  for (int r = tid; r < m; r += AGE_T) {
    double a = INFINITY, b = INFINITY;
    bool sel = false;
    for (int e = 0; e < n_ext; ++e) {
      const int s = extreme[e];
      if (s == r) sel = true;
      const double dd = minkowski(yn + (int64_t)s * M, yn + (int64_t)r * M, M, p) / nn[s];
      if (dd < a) {
        b = a;
        a = dd;
      } else if (dd < b) {
        b = dd;
      }
    }
    d1g[r] = a;
    d2g[r] = b;
    selg[r] = sel ? 1 : 0;
    crowd[r] = sel ? INFINITY : 0.0;
  }
  __syncthreads();
  int n_sel = n_ext;
  const int steps = m - n_ext;
  for (int it = 0; it < steps; ++it) {
    // arg-max of (d1 + d2) [or d1 while a single point is selected], first index on ties
    double bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int r = tid; r < m; r += AGE_T) {
      if (selg[r]) continue;
      const double sc = (n_sel > 1) ? (d1g[r] + d2g[r]) : d1g[r];
      if (sc > bv || (sc == bv && r < bi)) {
        bv = sc;
        bi = r;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    if ((tid & 31) == 0) {
      s_val[tid >> 5] = bv;
      s_idx[tid >> 5] = bi;
    }
    __syncthreads();
    if (tid < 32) {
      bv = tid < AGE_T / 32 ? s_val[tid] : -INFINITY;
      bi = tid < AGE_T / 32 ? s_idx[tid] : 0x7fffffff;
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) {
          bv = ov;
          bi = oi;
        }
      }
      if (tid == 0) {
        s_bi = bi;
        selg[bi] = 1;
        crowd[bi] = bv;
        for (int j = 0; j < M; ++j) s_best[j] = yn[(int64_t)bi * M + j];
        s_best[AGE_MAXM] = nn[bi];
      }
    }
    __syncthreads();
    const int best = s_bi;
    const double nb = s_best[AGE_MAXM];
    for (int r = tid; r < m; r += AGE_T) {
      if (selg[r]) continue;
      const double dd = minkowski(s_best, yn + (int64_t)r * M, M, p) / nb;
      double a = d1g[r], b = d2g[r];
      if (dd < a) {
        b = a;
        a = dd;
      } else if (dd < b) {
        b = dd;
      }
      d1g[r] = a;
      d2g[r] = b;
    }
    (void)best;
    n_sel += 1;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------- SMPSO
// out = clip((w v + c1 r1 (l1 - x) + c2 r2 (l2 - x)) chi, -delta, +delta).  NumPy forms the differences in the common
// dtype of archive and position (SMPSO.py:338-345): float32 when both are float32 state arrays, float64 when the
// archive is the float64 x_gen that MOASMO hands to update(); diff_f32 selects which.
__global__ void smpso_velocity_kernel(const float* __restrict__ pos, const double* __restrict__ vel,
                                      const double* __restrict__ lead1, const double* __restrict__ lead2, int diff_f32,
                                      int64_t n, int d, double w, double c1r1, double c2r2, double chi,
                                      const double* __restrict__ xlb, const double* __restrict__ xub,
                                      double* __restrict__ out) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int j = (int)(t % d);
  double d1, d2;
  if (diff_f32) {
    d1 = (double)((float)lead1[j] - pos[t]);
    d2 = (double)((float)lead2[j] - pos[t]);
  } else {
    d1 = lead1[j] - (double)pos[t];
    d2 = lead2[j] - (double)pos[t];
  }
  const double delta = (xub[j] - xlb[j]) / 2;
  double v = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(w, vel[t]), __dmul_rn(c1r1, d1)), __dmul_rn(c2r2, d2)), chi);
  out[t] = np_clip(v, -delta, delta);
}

// ---------------------------------------------------------------------------------------------- batched mutation
enum : uint64_t { P_MUT_PARENT = 11, P_MUT_GENES = 12 };

__device__ __forceinline__ double mutate_gene2(double parent, double u, double di, double lb, double ub, double rate) {
  double e = __ddiv_rn(1.0, __dadd_rn(di, 1.0));
  double delta;
  if (u < rate)
    delta = __dsub_rn(pow(__dmul_rn(2.0, u), e), 1.0);
  else
    delta = __dsub_rn(1.0, pow(__dmul_rn(2.0, __dsub_rn(1.0, u)), e));
  return np_clip(__dadd_rn(parent, __dmul_rn(__dsub_rn(ub, lb), delta)), lb, ub);
}

// child c of group g mutates parent (g * group_size + randint(group_size)) of pop_x: SMPSO's per-swarm mutants
// (SMPSO.py:167-182, Generator.integers(0, popsize) per swarm and child)
__global__ void mutate_groups_kernel(const double* __restrict__ pop_x, int64_t group_size, int64_t n_groups,
                                     int64_t per_group, int d, const double* __restrict__ di,
                                     const double* __restrict__ xlb, const double* __restrict__ xub, double rate,
                                     uint64_t seed, uint64_t stream_id, double* __restrict__ out,
                                     int64_t* __restrict__ parent_out) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = n_groups * per_group;
  if (t >= total * d) return;
  const int64_t c = t / d;  // child index: g * per_group + k
  const int j = (int)(t - c * d);
  const int64_t g = c / per_group;
  Philox ph(seed);
  uint4 a = ph((uint64_t)c, (stream_id << 8) | P_MUT_PARENT);
  int64_t pi = (int64_t)(u01_53(a.x, a.y) * (double)group_size);
  if (pi >= group_size) pi = group_size - 1;
  const int64_t prow = g * group_size + pi;
  uint4 b = ph((uint64_t)t, (stream_id << 8) | P_MUT_GENES);
  const double u = u01_53(b.x, b.y);
  out[t] = mutate_gene2(pop_x[prow * d + j], u, di[j], xlb[j], xub[j], rate);
  if (j == 0 && parent_out) parent_out[c] = prow;
}

// ---------------------------------------------------------------------------------------------- MO-CMA-ES
// individuals[i] = x_p + sigma_p * (A_p @ z_i),  p = p_idx[i]          (CMAES.py:263-267)
__global__ void cmaes_sample_kernel(const double* __restrict__ parents_x, const double* __restrict__ sigmas, int sig_ld,
                                    const double* __restrict__ A, const int64_t* __restrict__ p_idx,
                                    const double* __restrict__ z, int64_t n, int d, double* __restrict__ out) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int64_t i = t / d;
  const int r = (int)(t - i * d);
  const int64_t p = p_idx[i];
  const double* Ar = A + (p * d + r) * d;
  const double* zi = z + i * d;
  double s = 0.0;
  for (int k = 0; k < d; ++k) s += Ar[k] * zi[k];
  const double sg = sig_ld == 1 ? sigmas[p] : sigmas[p * sig_ld + r];
  out[t] = parents_x[p * d + r] + sg * s;
}

// rank-one update of one individual's Cholesky factor and its inverse (CMAES.py:489-537); one block per individual
__global__ void cmaes_cholesky_kernel(double* __restrict__ A, double* __restrict__ Ainv, double* __restrict__ pc,
                                      const double* __restrict__ z, const double* __restrict__ psucc, int64_t n, int d,
                                      double cc, double ccov, double pthresh) {
  extern __shared__ double sh[];  // pc[d], w[d], wA[d]
  double* spc = sh;
  double* sw = sh + d;
  double* swA = sh + 2 * d;
  __shared__ double s_wmax, s_n2;
  const int64_t i = blockIdx.x;
  if (i >= n) return;
  double* Ai = A + i * d * d;
  double* Bi = Ainv + i * d * d;
  const double ps = psucc[i];
  double alpha;
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    double v;
    if (ps < pthresh)
      v = (1.0 - cc) * pc[i * d + k] + sqrt(cc * (2.0 - cc)) * z[i * d + k];
    else
      v = (1.0 - cc) * pc[i * d + k];
    spc[k] = v;
    pc[i * d + k] = v;
  }
  alpha = (ps < pthresh) ? (1.0 - ccov) : ((1.0 - ccov) + ccov * cc * (2.0 - cc));
  __syncthreads();
  for (int r = threadIdx.x; r < d; r += blockDim.x) {  // w = Ainv @ pc
    double s = 0.0;
    for (int k = 0; k < d; ++k) s += Bi[r * d + k] * spc[k];
    sw[r] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double mx = -INFINITY, n2 = 0.0;
    for (int k = 0; k < d; ++k) {
      mx = fmax(mx, sw[k]);
      n2 += sw[k] * sw[k];
    }
    s_wmax = mx;
    s_n2 = n2;
  }
  for (int c = threadIdx.x; c < d; c += blockDim.x) {  // wA = w @ Ainv
    double s = 0.0;
    for (int k = 0; k < d; ++k) s += sw[k] * Bi[k * d + c];
    swA[c] = s;
  }
  __syncthreads();
  if (!(s_wmax > 1e-20)) return;  // "under this threshold, the update is mostly noise"
  const double a = sqrt(alpha), n2 = s_n2;
  const double root = sqrt(1.0 + ccov / alpha * n2);
  const double b = a / n2 * (root - 1.0);
  const double c = 1.0 / (a * n2) * (1.0 - 1.0 / root);
  for (int t = threadIdx.x; t < d * d; t += blockDim.x) {
    const int r = t / d, q = t - r * d;
    Ai[t] = a * Ai[t] + b * spc[r] * sw[q];
    Bi[t] = (1.0 / a) * Bi[t] - c * sw[r] * swA[q];
  }
}

// dst[i, :] = (sel && sel[i] ? alt : src)[idx[i], :]: row gather between device-resident per-individual state arrays
// (MO-CMA-ES Cholesky factors: CMAES.py:385-411 re-assembles the parent set from old parents and updated offspring)
__global__ void gather_rows_kernel(const double* __restrict__ src, const double* __restrict__ alt, const uint8_t* __restrict__ sel,
                                   const int64_t* __restrict__ idx, int64_t n, int64_t row, double* __restrict__ dst) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * row) return;
  const int64_t i = t / row, c = t - i * row;
  const double* s = (sel && sel[i]) ? alt : src;
  dst[t] = s[idx[i] * row + c];
}

// max |x| over a device array as the bit pattern of a non-negative double (which orders like the value); exact, the
// maximum does not depend on the order of the reduction
__global__ void absmax_kernel(const double* __restrict__ x, int64_t n, unsigned long long* __restrict__ out_bits) {
  unsigned long long m = 0ull;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(fabs(x[t]));
    m = b > m ? b : m;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long v = __shfl_xor_sync(0xFFFFFFFFu, m, o);
    m = v > m ? v : m;
  }
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_bits, m);
}

// x = clip((individual / max|individuals|) * (xub - xlb) + xlb, xlb, xub): the reference's global rescale (CMAES.py:269-270)
// followed by MOEA.generate's clip (MOEA.py:155); every operation rounded separately, as NumPy evaluates it
__global__ void cmaes_rescale_kernel(double* __restrict__ x, int64_t n, int d, const unsigned long long* __restrict__ mx_bits,
                                     const double* __restrict__ xlb, const double* __restrict__ xub) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int j = (int)(t % d);
  const double mx = __longlong_as_double((long long)*mx_bits);
  const double lb = xlb[j], ub = xub[j];
  const double v = __dadd_rn(__dmul_rn(__ddiv_rn(x[t], mx), __dsub_rn(ub, lb)), lb);
  x[t] = np_clip(v, lb, ub);
}

// z[i] = ((x_gen[ci[i]] - parents_x[pi[i]]) / (xub - xlb)) / step[i]: the offspring's move in its parent's coordinates
// (CMAES.py:316-318), operations rounded one by one
__global__ void cmaes_z_kernel(const double* __restrict__ xg, const int64_t* __restrict__ ci, const double* __restrict__ px,
                               const int64_t* __restrict__ pi, const double* __restrict__ xlb, const double* __restrict__ xub,
                               const double* __restrict__ steps, int64_t n, int d, double* __restrict__ z) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int64_t i = t / d;
  const int j = (int)(t - i * d);
  const double diff = __dsub_rn(xg[ci[i] * d + j], px[pi[i] * d + j]);
  z[t] = __ddiv_rn(__ddiv_rn(diff, __dsub_rn(xub[j], xlb[j])), steps[t]);
}

// rows[seg_row[s], :] *= factors[e] for e = seg_start[s] .. seg_start[s + 1] - 1, one multiplication after the other (the
// step-size recurrences of one parent are sequential, CMAES.py:330-383); seg_row == nullptr: row s, seg_start == nullptr:
// one factor per row
__global__ void scale_rows_kernel(double* __restrict__ rows, int64_t row, int64_t n_seg, const int64_t* __restrict__ seg_row,
                                  const int64_t* __restrict__ seg_start, const double* __restrict__ factors) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_seg * row) return;
  const int64_t s = t / row, c = t - s * row;
  const int64_t r = seg_row ? seg_row[s] : s;
  const int64_t e0 = seg_start ? seg_start[s] : s, e1 = seg_start ? seg_start[s + 1] : s + 1;
  double v = rows[r * row + c];
  for (int64_t e = e0; e < e1; ++e) v = __dmul_rn(v, factors[e]);
  rows[r * row + c] = v;
}

}  // namespace

// The bodies of the CMA-ES entry points and of dmo_gather_rows / dmo_scale_rows on device arrays, without their trailing
// waits; the resident CMA-ES step (cmaes_step.cu) composes them.
int gather_rows_device(dmo_ctx* ctx, const double* src, const double* alt, const uint8_t* sel, const int64_t* idx, int64_t n,
                       int64_t row_elems, double* dst) {
  if (n == 0) return DMO_OK;
  DMO_LAUNCH(gather_rows_kernel, (unsigned)ceil_div(n * row_elems, 256), 256, 0, src, alt, sel, idx, n, row_elems, dst);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int cmaes_generate_device(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols, const double* A,
                          const int64_t* p_idx, const double* z, int64_t n, int d, const double* xlb, const double* xub, double* x_out) {
  DevBuf<unsigned long long> mx;
  DMO_TRY(mx.alloc(ctx, 1));
  DMO_CUDA(cudaMemsetAsync(mx.p, 0, sizeof(unsigned long long), ctx->stream));
  DMO_LAUNCH(cmaes_sample_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, parents_x, sigmas, sigma_cols, A, p_idx, z, n, d, x_out);
  DMO_LAUNCH(absmax_kernel, (unsigned)std::min<int64_t>(ceil_div(n * d, 256), 4 * (int64_t)ctx->sm_count), 256, 0, x_out, n * d, mx.p);
  DMO_LAUNCH(cmaes_rescale_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, x_out, n, d, mx.p, xlb, xub);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int cmaes_step_z_device(dmo_ctx* ctx, const double* x_gen, const int64_t* cand_idx, const double* parents_x, const int64_t* par_idx,
                        const double* xlb, const double* xub, const double* steps, int64_t n, int d, double* z_out) {
  if (n == 0) return DMO_OK;
  DMO_LAUNCH(cmaes_z_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, x_gen, cand_idx, parents_x, par_idx, xlb, xub, steps, n, d, z_out);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int scale_rows_device(dmo_ctx* ctx, double* rows, int64_t row_elems, int64_t n_seg, const int64_t* seg_row, const int64_t* seg_start,
                      const double* factors) {
  if (n_seg == 0) return DMO_OK;
  DMO_LAUNCH(scale_rows_kernel, (unsigned)ceil_div(n_seg * row_elems, 256), 256, 0, rows, row_elems, n_seg, seg_row, seg_start, factors);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

int cmaes_update_cholesky_device(dmo_ctx* ctx, double* A, double* Ainv, double* pc, const double* z, const double* psucc, int64_t n, int d,
                                 double cc, double ccov, double pthresh) {
  if (n == 0) return DMO_OK;
  DMO_LAUNCH(cmaes_cholesky_kernel, (unsigned)n, 64, 3 * d * sizeof(double), A, Ainv, pc, z, psucc, n, d, cc, ccov, pthresh);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

extern "C" {

int dmo_gather_rows(dmo_ctx* ctx, const double* src, const double* alt, const uint8_t* sel, const int64_t* idx, int64_t n,
                    int64_t row_elems, double* dst) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && row_elems >= 1 && src && idx && dst && (sel == nullptr || alt != nullptr), "gather_rows: bad arguments");
  DMO_REQUIRE(dmo_is_device_ptr(src) && dmo_is_device_ptr(dst) && (!alt || dmo_is_device_ptr(alt)),
              "gather_rows: src / alt / dst are device-resident arrays");
  In<int64_t> ii;
  In<uint8_t> is;
  DMO_TRY(ii.init(ctx, idx, (size_t)n));
  DMO_TRY(is.init(ctx, sel, (size_t)n));
  DMO_TRY(gather_rows_device(ctx, src, alt, is.d, ii.d, n, row_elems, dst));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_age_survival(dmo_ctx* ctx, const double* yn, const double* nn, int64_t m, int M, double p, const int32_t* extreme,
                     int n_ext, double* crowd) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(yn && nn && extreme && crowd && m > 0 && M >= 1 && M <= AGE_MAXM && n_ext >= 1 && n_ext <= m,
              "age_survival: bad arguments");
  In<double> iy, inn;
  In<int32_t> iex;
  Out<double> oc;
  DMO_TRY(iy.init(ctx, yn, (size_t)m * M));
  DMO_TRY(inn.init(ctx, nn, (size_t)m));
  DMO_TRY(iex.init(ctx, extreme, (size_t)n_ext));
  DMO_TRY(oc.init(ctx, crowd, (size_t)m));
  DevBuf<double> d1, d2;
  DevBuf<uint8_t> sel;
  DMO_TRY(d1.alloc(ctx, m));
  DMO_TRY(d2.alloc(ctx, m));
  DMO_TRY(sel.alloc(ctx, m));
  {
    ProfileScope ps(ctx, "age_survival");
    DMO_LAUNCH(age_survival_kernel, 1, AGE_T, 0, iy.d, inn.d, (int)m, M, p, (const int*)iex.d, n_ext, d1.p, d2.p, sel.p,
               oc.d);
  }
  DMO_CHECK_LAUNCH();
  DMO_TRY(oc.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_smpso_velocity(dmo_ctx* ctx, const float* position, const double* velocity, const double* leader1,
                       const double* leader2, int f32_difference, int64_t n, int d, double w, double c1, double r1,
                       double c2, double r2, double chi, const double* xlb, const double* xub, double* out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(position && velocity && leader1 && leader2 && xlb && xub && out && n > 0 && d >= 1,
              "smpso_velocity: bad arguments");
  In<float> ip;
  In<double> iv, ilb, iub, l1, l2;
  Out<double> oo;
  DMO_TRY(ip.init(ctx, position, (size_t)n * d));
  DMO_TRY(iv.init(ctx, velocity, (size_t)n * d));
  DMO_TRY(l1.init(ctx, leader1, d));
  DMO_TRY(l2.init(ctx, leader2, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(oo.init(ctx, out, (size_t)n * d));
  DMO_LAUNCH(smpso_velocity_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, ip.d, iv.d, l1.d, l2.d, f32_difference, n, d, w,
             c1 * r1, c2 * r2, chi, ilb.d, iub.d, oo.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(oo.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_mutate_groups(dmo_ctx* ctx, const double* pop_x, int64_t group_size, int64_t n_groups, int64_t per_group, int d,
                      const double* di_mutation, const double* xlb, const double* xub, double mutation_rate,
                      uint64_t seed, uint64_t stream_id, double* children, int64_t* parent_rows) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(pop_x && di_mutation && xlb && xub && children && group_size > 0 && n_groups > 0 && per_group > 0 && d >= 1,
              "mutate_groups: bad arguments");
  const int64_t total = n_groups * per_group;
  In<double> ipx, idi, ilb, iub;
  Out<double> oc;
  Out<int64_t> opar;
  DMO_TRY(ipx.init(ctx, pop_x, (size_t)(group_size * n_groups) * d));
  DMO_TRY(idi.init(ctx, di_mutation, d));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  DMO_TRY(oc.init(ctx, children, (size_t)total * d));
  DMO_TRY(opar.init(ctx, parent_rows, (size_t)total));
  DMO_LAUNCH(mutate_groups_kernel, (unsigned)ceil_div(total * d, 256), 256, 0, ipx.d, group_size, n_groups, per_group, d,
             idi.d, ilb.d, iub.d, mutation_rate, seed, stream_id, oc.d, opar.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(oc.finish(ctx));
  DMO_TRY(opar.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_cmaes_sample(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols, const double* A,
                     int64_t n_parents, const int64_t* p_idx, const double* z, int64_t n, int d, double* individuals) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(parents_x && sigmas && A && p_idx && z && individuals && n > 0 && n_parents > 0 && d >= 1 &&
                  (sigma_cols == 1 || sigma_cols == d),
              "cmaes_sample: bad arguments");
  In<double> ipx, isg, iA, iz;
  In<int64_t> ipi;
  Out<double> oo;
  DMO_TRY(ipx.init(ctx, parents_x, (size_t)n_parents * d));
  DMO_TRY(isg.init(ctx, sigmas, (size_t)n_parents * sigma_cols));
  DMO_TRY(iA.init(ctx, A, (size_t)n_parents * d * d));
  DMO_TRY(ipi.init(ctx, p_idx, (size_t)n));
  DMO_TRY(iz.init(ctx, z, (size_t)n * d));
  DMO_TRY(oo.init(ctx, individuals, (size_t)n * d));
  DMO_LAUNCH(cmaes_sample_kernel, (unsigned)ceil_div(n * d, 256), 256, 0, ipx.d, isg.d, sigma_cols, iA.d, ipi.d, iz.d, n, d,
             oo.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(oo.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_cmaes_generate(dmo_ctx* ctx, const double* parents_x, const double* sigmas, int sigma_cols, const double* A,
                       int64_t n_parents, const int64_t* p_idx, const double* z, int64_t n, int d, const double* xlb,
                       const double* xub, double* x_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(parents_x && sigmas && A && p_idx && z && xlb && xub && x_out && n > 0 && n_parents > 0 && d >= 1 &&
                  (sigma_cols == 1 || sigma_cols == d),
              "cmaes_generate: bad arguments");
  In<double> ipx, isg, iA, iz, ilb, iub;
  In<int64_t> ipi;
  Out<double> oo;
  DMO_TRY(ipx.init(ctx, parents_x, (size_t)n_parents * d));
  DMO_TRY(isg.init(ctx, sigmas, (size_t)n_parents * sigma_cols));
  DMO_TRY(iA.init(ctx, A, (size_t)n_parents * d * d));
  DMO_TRY(ipi.init(ctx, p_idx, (size_t)n));
  DMO_TRY(iz.init(ctx, z, (size_t)n * d));
  DMO_TRY(ilb.init(ctx, xlb, (size_t)d));
  DMO_TRY(iub.init(ctx, xub, (size_t)d));
  DMO_TRY(oo.init(ctx, x_out, (size_t)n * d));
  DMO_TRY(cmaes_generate_device(ctx, ipx.d, isg.d, sigma_cols, iA.d, ipi.d, iz.d, n, d, ilb.d, iub.d, oo.d));
  DMO_TRY(oo.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_cmaes_step_z(dmo_ctx* ctx, const double* x_gen, const int64_t* cand_idx, const double* parents_x,
                     const int64_t* par_idx, const double* xlb, const double* xub, const double* steps, int64_t n, int d,
                     double* z_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(x_gen && cand_idx && parents_x && par_idx && xlb && xub && steps && z_out && n > 0 && d >= 1, "cmaes_step_z: bad arguments");
  DMO_REQUIRE(dmo_is_device_ptr(x_gen) && dmo_is_device_ptr(parents_x) && dmo_is_device_ptr(steps) && dmo_is_device_ptr(z_out),
              "cmaes_step_z: x_gen / parents_x / steps / z_out are device-resident arrays");
  In<int64_t> ici, ipi;
  In<double> ilb, iub;
  DMO_TRY(ici.init(ctx, cand_idx, (size_t)n));
  DMO_TRY(ipi.init(ctx, par_idx, (size_t)n));
  DMO_TRY(ilb.init(ctx, xlb, (size_t)d));
  DMO_TRY(iub.init(ctx, xub, (size_t)d));
  DMO_TRY(cmaes_step_z_device(ctx, x_gen, ici.d, parents_x, ipi.d, ilb.d, iub.d, steps, n, d, z_out));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_scale_rows(dmo_ctx* ctx, double* rows, int64_t row_elems, int64_t n_seg, const int64_t* seg_row,
                   const int64_t* seg_start, const double* factors, int64_t n_factors) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n_seg == 0) return DMO_OK;
  DMO_REQUIRE(rows && factors && n_seg > 0 && row_elems >= 1 && n_factors >= (seg_start ? 0 : n_seg), "scale_rows: bad arguments");
  DMO_REQUIRE(dmo_is_device_ptr(rows), "scale_rows: rows is a device-resident array");
  In<int64_t> isr, iss;
  In<double> ifa;
  DMO_TRY(isr.init(ctx, seg_row, (size_t)n_seg));
  DMO_TRY(iss.init(ctx, seg_start, (size_t)n_seg + 1));
  DMO_TRY(ifa.init(ctx, factors, (size_t)n_factors));
  DMO_TRY(scale_rows_device(ctx, rows, row_elems, n_seg, isr.d, iss.d, ifa.d));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

int dmo_cmaes_update_cholesky(dmo_ctx* ctx, double* A, double* Ainv, double* pc, const double* z, const double* psucc,
                              int64_t n, int d, double cc, double ccov, double pthresh) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(A && Ainv && pc && z && psucc && n > 0 && d >= 1 && d <= 512, "cmaes_update_cholesky: bad arguments");
  // in/out arrays: stage host buffers explicitly
  const bool hostA = !dmo_is_device_ptr(A);
  DevBuf<double> dA, dB, dpc;
  double *pA = A, *pB = Ainv, *ppc = pc;
  if (hostA) {
    DMO_TRY(dA.alloc(ctx, (size_t)n * d * d));
    DMO_TRY(dB.alloc(ctx, (size_t)n * d * d));
    DMO_TRY(dpc.alloc(ctx, (size_t)n * d));
    DMO_CUDA(cudaMemcpyAsync(dA.p, A, (size_t)n * d * d * 8, cudaMemcpyHostToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(dB.p, Ainv, (size_t)n * d * d * 8, cudaMemcpyHostToDevice, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(dpc.p, pc, (size_t)n * d * 8, cudaMemcpyHostToDevice, ctx->stream));
    ctx->h2d_bytes += (uint64_t)n * d * (2 * d + 1) * 8;
    pA = dA.p;
    pB = dB.p;
    ppc = dpc.p;
  }
  In<double> iz, ips;
  DMO_TRY(iz.init(ctx, z, (size_t)n * d));
  DMO_TRY(ips.init(ctx, psucc, (size_t)n));
  DMO_TRY(cmaes_update_cholesky_device(ctx, pA, pB, ppc, iz.d, ips.d, n, d, cc, ccov, pthresh));
  if (hostA) {
    DMO_CUDA(cudaMemcpyAsync(A, pA, (size_t)n * d * d * 8, cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(Ainv, pB, (size_t)n * d * d * 8, cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(cudaMemcpyAsync(pc, ppc, (size_t)n * d * 8, cudaMemcpyDeviceToHost, ctx->stream));
    ctx->d2h_bytes += (uint64_t)n * d * (2 * d + 1) * 8;
  }
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
