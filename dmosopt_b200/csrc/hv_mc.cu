// Monte-Carlo hypervolume estimators for 2 .. 16 objectives (SURVEY.md section 8a row A16, the non-'box' branches).
//   monte_carlo  hv.AdaptiveHyperVolume._compute_standard_mc        dmosopt/hv.py:191-241
//   fpras        compute_hypervolume_fpras / _run_fpras_round        dmosopt/hv_adaptive.py:188-348
//   mcm2rv       compute_hypervolume_mcm2rv                          dmosopt/hv_adaptive.py:356-460
//   hybrid       compute_hypervolume_hybrid (+ estimate_overlap,     dmosopt/hv_adaptive.py:468-855
//                estimate_theta_bounds)
// The same random variables and stopping rules as the reference; only the random stream differs.  Every draw is Philox
// keyed by `seed`, counter = (sample index, draw index << 32 | stream_id << 8 | purpose), so a sample's whole history is a
// pure function of (seed, stream_id, purpose, sample index).  Samples are evaluated in waves; a stopping rule is applied
// in sample-index order to integer sums (exact in any order), and the work past the stopping index is discarded, so the
// result does not depend on the wave or grid sizes and is bit-identical across runs.
//
// The front the estimators see: the rows strictly inside ref, then their non-dominated subset, in row order.  Neither
// changes the volume.  The reference hands its Monte-Carlo routes the unfiltered front (hv.py:181): a row outside ref
// then has a non-positive box volume, and np.random.choice receives invalid probabilities (DESIGN.md section 4.3).
#include <math.h>
#include <stdlib.h>

#include <vector>

#include "common.cuh"

int hv_inside_nondominated(dmo_ctx* ctx, const double* dF, int64_t n, int M, const double* dref, DevBuf<double>& out,
                           int64_t* count);

namespace {

constexpr int MC_MAXM = 16;
constexpr int MC_T = 256;       // threads per block of the sampling kernels
constexpr int SCAN_T = 128;     // samples per block of the tiled dominance scan
constexpr int N_PROBES = 50;    // estimate_overlap's n_probes
constexpr int64_t WAVE_MAX = (int64_t)1 << 22;

enum : uint64_t {
  P_FPRAS_SAMPLE = 1,  // box index and the point in the box
  P_FPRAS_TRIAL = 2,   // the uniform row of trial t (four trials per Philox call)
  P_PROBE_SAMPLE = 3,  // the hybrid's level-2 probes
  P_PROBE_TRIAL = 4,
  P_MCM_SAMPLE = 5,    // MCM2RV: the point in [ideal, ref]
  P_MCM_ETA = 6,       // MCM2RV: the row of eta
  P_MC_SAMPLE = 7,     // monte_carlo: the point in [min(F), ref]
};

__device__ __forceinline__ uint64_t ctr_hi(uint64_t stream_id, uint64_t purpose, uint64_t draw) {
  return (draw << 32) | ((stream_id & 0xFFFFFFull) << 8) | purpose;
}

// uniforms u[0 .. M] of one sample: two per Philox call, u[0] first
__device__ __forceinline__ void sample_uniforms(const Philox& ph, uint64_t s, uint64_t stream_id, uint64_t purpose, int M,
                                                double* u) {
#pragma unroll
  for (int c = 0; c < (MC_MAXM + 2) / 2; ++c) {
    if (2 * c <= M) {
      const uint4 r = ph(s, ctr_hi(stream_id, purpose, (uint64_t)c));
      u[2 * c] = u01_53(r.x, r.y);
      if (2 * c + 1 <= M) u[2 * c + 1] = u01_53(r.z, r.w);
    }
  }
}

// np.random.choice(n, p=v / W): first i with cdf[i] > u (numpy: searchsorted(cdf, u, side='right'))
__device__ __forceinline__ int64_t choose_box(const double* __restrict__ cdf, int64_t n, double u) {
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// np.random.uniform(low, high): low + (high - low) * u
__device__ __forceinline__ double uniform_in(double lo, double hi, double u) { return __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), u)); }

// FPRAS point: box i with probability v_i / W, then x uniform in [f_i, ref]
__device__ __forceinline__ void fpras_point(const double* __restrict__ F, const double* __restrict__ ref, const double* __restrict__ cdf,
                                            int64_t n, int M, const Philox& ph, uint64_t s, uint64_t stream_id, uint64_t purpose,
                                            double* x) {
  double u[MC_MAXM + 1];
  sample_uniforms(ph, s, stream_id, purpose, M, u);
  const int64_t i = choose_box(cdf, n, u[0]);
#pragma unroll
  for (int j = 0; j < MC_MAXM; ++j)
    if (j < M) x[j] = uniform_in(F[i * M + j], ref[j], u[1 + j]);
}

__device__ __forceinline__ uint32_t word_of(const uint4& r, int c) { return c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w; }

// One FPRAS wave: xi of samples s0 .. s0 + S - 1 (0 = not found within `cap` trials, the rest of the budget).  Every loop
// iteration is one dominance test per lane; a lane that finishes a sample moves on to its next sample index, so the lanes
// of a warp stay converged however the geometric trial counts spread.  sums[0] += sum of xi, sums[1] += unfinished samples.
__global__ void __launch_bounds__(MC_T) fpras_wave_kernel(const double* __restrict__ F, int64_t n, int M, const double* __restrict__ ref,
                                                          const double* __restrict__ cdf, uint64_t seed, uint64_t stream_id,
                                                          uint64_t s0, int64_t S, int64_t cap, int64_t* __restrict__ xi_out,
                                                          unsigned long long* __restrict__ sums) {
  const Philox ph(seed);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double x[MC_MAXM];
  if (s < S) fpras_point(F, ref, cdf, n, M, ph, s0 + s, stream_id, P_FPRAS_SAMPLE, x);
  unsigned long long acc = 0ull, unfinished = 0ull;
  int64_t t = 0;
  uint4 rw = make_uint4(0u, 0u, 0u, 0u);
  while (s < S) {
    if ((t & 3) == 0) rw = ph(s0 + s, ctr_hi(stream_id, P_FPRAS_TRIAL, (uint64_t)(t >> 2)));
    const int64_t k = (int64_t)__umulhi(word_of(rw, (int)(t & 3)), (uint32_t)n);  // np.random.randint(0, n)
    const double* fk = F + k * M;
    bool dom = true;
#pragma unroll
    for (int j = 0; j < MC_MAXM; ++j)
      if (j < M) dom = dom && (x[j] > fk[j]);  // np.all(sample > pareto_front[k])
    ++t;
    if (dom || t >= cap) {
      xi_out[s] = dom ? t : 0;
      acc += dom ? (unsigned long long)t : 0ull;
      unfinished += dom ? 0ull : 1ull;
      s += stride;
      t = 0;
      if (s < S) fpras_point(F, ref, cdf, n, M, ph, s0 + s, stream_id, P_FPRAS_SAMPLE, x);
    }
  }
  if (acc) atomicAdd(&sums[0], acc);
  if (unfinished) atomicAdd(&sums[1], unfinished);
}

// Tiled dominance scan, one sample per thread, with a block-wide early exit: x uniform in [lo, hi]; dominated iff some row
// has f_k <= x in every coordinate (the reference's `<` or np.isclose, and hv.py:228's `>=`, both as exact <=).
// code[s] = tests | (dominated ? (eta ? 2 : 1) : 0) << 30, tests = rows scanned up to the first dominator (+1 for eta).
// sums[0] += dominated samples, sums[1] += eta, sums[2] += tests.
__global__ void __launch_bounds__(SCAN_T) dominated_wave_kernel(const double* __restrict__ F, int64_t n, int M,
                                                                const double* __restrict__ lo, const double* __restrict__ hi,
                                                                uint64_t seed, uint64_t stream_id, uint64_t purpose, int want_eta,
                                                                uint64_t s0, int64_t S, uint32_t* __restrict__ code,
                                                                unsigned long long* __restrict__ sums) {
  extern __shared__ double tile_f[];  // [SCAN_T][M]
  const Philox ph(seed);
  const int64_t s = (int64_t)blockIdx.x * SCAN_T + threadIdx.x;
  const bool live = s < S;
  double x[MC_MAXM];
  {
    double u[MC_MAXM + 1];
    sample_uniforms(ph, s0 + s, stream_id, purpose, M, u);
#pragma unroll
    for (int j = 0; j < MC_MAXM; ++j)
      if (j < M) x[j] = uniform_in(lo[j], hi[j], u[1 + j]);
  }
  bool done = !live, dominated = false;
  int64_t tests = 0;
  for (int64_t t0 = 0; t0 < n; t0 += SCAN_T) {
    if (__syncthreads_and(done ? 1 : 0)) break;
    const int cnt = (int)((n - t0) < SCAN_T ? (n - t0) : SCAN_T);
    for (int e = threadIdx.x; e < cnt * M; e += SCAN_T) tile_f[e] = F[t0 * M + e];
    __syncthreads();
    if (!done) {
      for (int r = 0; r < cnt; ++r) {
        const double* fr = tile_f + r * M;
        bool le = true;
#pragma unroll
        for (int j = 0; j < MC_MAXM; ++j)
          if (j < M) le = le && (fr[j] <= x[j]);
        ++tests;
        if (le) {
          dominated = true;
          break;
        }
      }
      done = dominated || t0 + cnt >= n;
    }
  }
  bool eta = false;
  if (live && dominated && want_eta) {  // eta: one test against a uniform random row
    const uint4 r = ph(s0 + s, ctr_hi(stream_id, P_MCM_ETA, 0));
    const int64_t k = (int64_t)__umulhi(r.x, (uint32_t)n);
    eta = true;
#pragma unroll
    for (int j = 0; j < MC_MAXM; ++j)
      if (j < M) eta = eta && (F[k * M + j] <= x[j]);
    ++tests;
  }
  if (live) {
    if (code) code[s] = (uint32_t)tests | ((uint32_t)(dominated ? (eta ? 2 : 1) : 0) << 30);
    unsigned long long a = dominated ? 1ull : 0ull, b = eta ? 1ull : 0ull;
    if (a) atomicAdd(&sums[0], a);
    if (b) atomicAdd(&sums[1], b);
    atomicAdd(&sums[2], (unsigned long long)tests);
  }
}

// estimate_overlap (hv_adaptive.py:468-522): one block per probe.  xi is the position of the first dominator in a random
// permutation of the rows; with c dominators among n rows it is drawn exactly by sequential sampling without replacement
// (the next row is a dominator with probability c / (n - t)), after the block has counted c.
__global__ void __launch_bounds__(MC_T) probe_kernel(const double* __restrict__ F, int64_t n, int M, const double* __restrict__ ref,
                                                     const double* __restrict__ cdf, uint64_t seed, uint64_t stream_id,
                                                     int64_t* __restrict__ xi_out) {
  __shared__ unsigned long long s_cnt;
  const Philox ph(seed);
  const int64_t p = blockIdx.x;
  double x[MC_MAXM];
  fpras_point(F, ref, cdf, n, M, ph, (uint64_t)p, stream_id, P_PROBE_SAMPLE, x);
  if (threadIdx.x == 0) s_cnt = 0ull;
  __syncthreads();
  unsigned long long c = 0ull;
  for (int64_t k = threadIdx.x; k < n; k += MC_T) {
    bool dom = true;
#pragma unroll
    for (int j = 0; j < MC_MAXM; ++j)
      if (j < M) dom = dom && (x[j] > F[k * M + j]);
    c += dom ? 1ull : 0ull;
  }
  if (c) atomicAdd(&s_cnt, c);
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int64_t cnt = (int64_t)s_cnt;
  int64_t xi = n;  // no dominator: the whole permutation is tested
  if (cnt > 0) {
    for (int64_t t = 0; t < n; ++t) {
      const uint4 r = ph((uint64_t)p, ctr_hi(stream_id, P_PROBE_TRIAL, (uint64_t)t));
      if (u01_53(r.x, r.y) * (double)(n - t) < (double)cnt) {
        xi = t + 1;
        break;
      }
    }
  }
  xi_out[p] = xi;
}

struct McFront {
  const double* F = nullptr;  // (n, M) device, filtered
  const double* ref = nullptr;
  const double* cdf = nullptr;
  const double* ideal = nullptr;
  int64_t n = 0;
  int M = 0;
  double W = 0.0, U = 0.0;
  uint64_t seed = 0, stream_id = 0;
};

struct FprasState {
  int64_t tests = 0, N = 0, sum_xi = 0;
  uint64_t next = 0;  // next sample index
};

int lanes(dmo_ctx* ctx) { return ctx->sm_count * 2048; }

// _run_fpras_round: continue the FPRAS sample sequence until `target` tests are spent.  The sample that straddles the
// target is discarded (its tests count), as in the reference; the next round starts at the sample after it.
int run_fpras(dmo_ctx* ctx, const McFront& f, int64_t target, FprasState& st) {
  DevBuf<int64_t> xi;
  DevBuf<unsigned long long> sums;
  DMO_TRY(sums.alloc(ctx, 2));
  std::vector<int64_t> hxi;
  while (st.tests < target) {
    const int64_t R = target - st.tests;
    int64_t S = 4096;
    if (st.N > 0) {
      const double mean = (double)st.sum_xi / (double)st.N;
      const double want = 1.05 * (double)R / mean + 64.0;
      S = want > (double)WAVE_MAX ? WAVE_MAX : (int64_t)want;
    }
    if ((size_t)S > xi.n) DMO_TRY(xi.alloc(ctx, (size_t)S));
    DMO_CUDA(cudaMemsetAsync(sums.p, 0, 2 * sizeof(unsigned long long), ctx->stream));
    const int64_t grid = ceil_div(S < lanes(ctx) ? S : lanes(ctx), MC_T);
    {
      ProfileScope ps(ctx, "hv_mc_fpras");
      DMO_LAUNCH(fpras_wave_kernel, (unsigned)grid, MC_T, 0, f.F, f.n, f.M, f.ref, f.cdf, f.seed, f.stream_id, st.next, S, R, xi.p, sums.p);
    }
    DMO_CHECK_LAUNCH();
    unsigned long long h[2];
    DMO_CUDA(cudaMemcpyAsync(h, sums.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    if (h[1] == 0 && (int64_t)h[0] <= R) {  // the whole wave fits the budget
      st.N += S;
      st.sum_xi += (int64_t)h[0];
      st.tests += (int64_t)h[0];
      st.next += (uint64_t)S;
      continue;
    }
    // the budget runs out inside this wave (a wave that fits whole took the branch above): find the stopping index in
    // sample order.  Either sample s - 1 meets the target exactly, and the next round starts at sample s, or sample s
    // straddles the target: it is discarded, its tests are spent, and the next round starts at the sample after it.
    hxi.resize((size_t)S);
    DMO_CUDA(cudaMemcpyAsync(hxi.data(), xi.p, (size_t)S * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    int64_t used = 0, s = 0;
    for (; s < S && used < R; ++s) {
      if (hxi[s] == 0 || used + hxi[s] > R) break;
      used += hxi[s];
      ++st.N;
    }
    st.sum_xi += used;
    st.tests = target;
    st.next += (uint64_t)(used < R ? s + 1 : s);
  }
  return DMO_OK;
}

// MCM2RV (hv_adaptive.py:356-460): stop when the sum of eta over the dominated samples, in sample order, reaches R
int run_mcm2rv(dmo_ctx* ctx, const McFront& f, double eps, double delta, int64_t* N_out, int64_t* S_out, int64_t* tests_out) {
  const int64_t R = (int64_t)floor((4.0 * (1.0 + eps * (1.0 - eps)) * log(2.0 / delta)) / (eps * eps * (1.0 - eps) * (1.0 - eps)));
  DevBuf<uint32_t> code;
  DevBuf<unsigned long long> sums;
  DMO_TRY(sums.alloc(ctx, 3));
  std::vector<uint32_t> hc;
  int64_t N = 0, Ssum = 0, tests = 0, attempts = 0;
  uint64_t next = 0;
  const size_t smem = (size_t)SCAN_T * f.M * sizeof(double);
  while (Ssum < R) {
    int64_t S = 65536;
    if (attempts > 0 && Ssum > 0) {
      const double want = 1.05 * (double)(R - Ssum) * (double)attempts / (double)Ssum + 64.0;
      S = want > (double)WAVE_MAX ? WAVE_MAX : (int64_t)want;
    } else if (attempts > 0) {
      S = WAVE_MAX;
    }
    if ((size_t)S > code.n) DMO_TRY(code.alloc(ctx, (size_t)S));
    DMO_CUDA(cudaMemsetAsync(sums.p, 0, 3 * sizeof(unsigned long long), ctx->stream));
    {
      ProfileScope ps(ctx, "hv_mc_mcm2rv");
      DMO_LAUNCH(dominated_wave_kernel, (unsigned)ceil_div(S, SCAN_T), SCAN_T, smem, f.F, f.n, f.M, f.ideal, f.ref, f.seed, f.stream_id,
                 (uint64_t)P_MCM_SAMPLE, 1, next, S, code.p, sums.p);
    }
    DMO_CHECK_LAUNCH();
    unsigned long long h[3];
    DMO_CUDA(cudaMemcpyAsync(h, sums.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    if (Ssum + (int64_t)h[1] < R) {
      N += (int64_t)h[0];
      Ssum += (int64_t)h[1];
      tests += (int64_t)h[2];
      attempts += S;
      next += (uint64_t)S;
      continue;
    }
    hc.resize((size_t)S);
    DMO_CUDA(cudaMemcpyAsync(hc.data(), code.p, (size_t)S * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    for (int64_t s = 0; s < S && Ssum < R; ++s) {
      const uint32_t kind = hc[s] >> 30;
      tests += (int64_t)(hc[s] & 0x3FFFFFFFu);
      ++attempts;
      if (kind == 0) continue;
      ++N;
      Ssum += kind == 2 ? 1 : 0;
    }
  }
  *N_out = N;
  *S_out = Ssum;
  *tests_out = tests;
  return DMO_OK;
}

}  // namespace

extern "C" int dmo_hypervolume_mc(dmo_ctx* ctx, const double* F, int64_t n, int M, const double* ref, int algorithm, double epsilon,
                                  double delta, int64_t n_samples, uint64_t seed, uint64_t stream_id, double* out,
                                  int64_t* samples_out, int64_t* tests_out, int* algorithm_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(out && ref && n >= 0 && M >= 2 && M <= MC_MAXM, "hypervolume_mc: bad arguments (2 <= M <= %d, got M=%d)", MC_MAXM, M);
  DMO_REQUIRE(algorithm >= DMO_HVMC_HYBRID && algorithm <= DMO_HVMC_MONTE_CARLO, "hypervolume_mc: unknown algorithm %d", algorithm);
  DMO_REQUIRE(algorithm == DMO_HVMC_MONTE_CARLO ? n_samples >= 1 : (epsilon > 0.0 && epsilon < 1.0 && delta > 0.0 && delta < 1.0),
              "hypervolume_mc: need 0 < epsilon, delta < 1 (got %g, %g) or n_samples >= 1 (got %lld)", epsilon, delta,
              (long long)n_samples);
  DMO_REQUIRE(stream_id < ((uint64_t)1 << 24), "hypervolume_mc: stream_id must be below 2^24");
  *out = 0.0;
  if (samples_out) *samples_out = 0;
  if (tests_out) *tests_out = 0;
  if (algorithm_out) *algorithm_out = 0;
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(F, "hypervolume_mc: null points");
  double h_ref[MC_MAXM];
  DMO_CUDA(cudaMemcpy(h_ref, ref, M * sizeof(double), cudaMemcpyDefault));
  In<double> f;
  DMO_TRY(f.init(ctx, F, (size_t)n * M));
  DevBuf<double> dref, front;
  DMO_TRY(dref.alloc(ctx, M));
  DMO_CUDA(cudaMemcpyAsync(dref.p, h_ref, M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  int64_t nf = 0;
  DMO_TRY(hv_inside_nondominated(ctx, f.d, n, M, dref.p, front, &nf));
  if (nf == 0) {
    DMO_CUDA(dmo_wait(ctx));
    return DMO_OK;
  }
  DMO_REQUIRE(nf < ((int64_t)1 << 32), "hypervolume_mc: front too large (%lld rows)", (long long)nf);
  // dominated_wave_kernel's per-sample record holds up to nf + 1 tests in 30 bits
  DMO_REQUIRE(algorithm == DMO_HVMC_FPRAS || algorithm == DMO_HVMC_MONTE_CARLO || nf < ((int64_t)1 << 30) - 1,
              "hypervolume_mc: front too large for mcm2rv and hybrid (%lld rows, below 2^30 - 1 needed)", (long long)nf);
  // box volumes, W, the sampling CDF, the ideal point and U: O(n M) once, in row order on the host
  std::vector<double> hF((size_t)nf * M), cdf((size_t)nf), ideal(M);
  DMO_CUDA(cudaMemcpyAsync(hF.data(), front.p, hF.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  double W = 0.0;
  for (int j = 0; j < M; ++j) ideal[j] = hF[j];
  for (int64_t i = 0; i < nf; ++i) {
    double v = 1.0;
    for (int j = 0; j < M; ++j) {
      v *= h_ref[j] - hF[i * M + j];
      ideal[j] = fmin(ideal[j], hF[i * M + j]);
    }
    W += v;
    cdf[i] = W;
  }
  for (int64_t i = 0; i < nf; ++i) cdf[i] /= W;
  double U = 1.0;
  for (int j = 0; j < M; ++j) U *= h_ref[j] - ideal[j];
  DevBuf<double> dcdf, dideal;
  DMO_TRY(dcdf.alloc(ctx, nf));
  DMO_TRY(dideal.alloc(ctx, M));
  DMO_CUDA(cudaMemcpyAsync(dcdf.p, cdf.data(), nf * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaMemcpyAsync(dideal.p, ideal.data(), M * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  McFront mf;
  mf.F = front.p;
  mf.ref = dref.p;
  mf.cdf = dcdf.p;
  mf.ideal = dideal.p;
  mf.n = nf;
  mf.M = M;
  mf.W = W;
  mf.U = U;
  mf.seed = seed;
  mf.stream_id = stream_id;

  double est = 0.0;
  int64_t samples = 0, tests = 0;
  int ran = algorithm;
  const double M1 = 8.0 * (1.0 + epsilon) * (double)nf * log(2.0 / delta) / (epsilon * epsilon);
  // a trial's Philox draw index (t / 4) has 32 bits of the counter: FPRAS budgets up to 2^34 tests
  DMO_REQUIRE(algorithm == DMO_HVMC_MONTE_CARLO || algorithm == DMO_HVMC_MCM2RV || M1 < 17179869184.0,
              "hypervolume_mc: FPRAS budget M1 = %.3g tests exceeds 2^34 (n=%lld, epsilon=%g, delta=%g); use mcm2rv or a larger epsilon",
              M1, (long long)nf, epsilon, delta);
  auto fpras_result = [&](const FprasState& st) {
    const int64_t N = st.N > 0 ? st.N : 1;
    est = (W / (double)nf) * ((double)st.sum_xi / (double)N);
    samples = N;
    tests = st.tests;
  };
  auto mcm2rv = [&](int64_t extra_tests) -> int {
    int64_t N = 0, S = 0, t = 0;
    DMO_TRY(run_mcm2rv(ctx, mf, epsilon, delta, &N, &S, &t));
    est = (W / (double)nf) * ((double)N / (double)S);
    samples = N;
    tests = t + extra_tests;
    return DMO_OK;
  };

  if (algorithm == DMO_HVMC_MONTE_CARLO) {
    // hv.py:191-241: n_samples uniform points in [min(F), ref]; redrawn while none is dominated
    DevBuf<unsigned long long> sums;
    DMO_TRY(sums.alloc(ctx, 3));
    const size_t smem = (size_t)SCAN_T * M * sizeof(double);
    unsigned long long dom = 0;
    uint64_t next = 0;
    for (int round = 0; round < 1000 && dom == 0; ++round) {
      DMO_CUDA(cudaMemsetAsync(sums.p, 0, 3 * sizeof(unsigned long long), ctx->stream));
      for (int64_t s0 = 0; s0 < n_samples; s0 += WAVE_MAX) {
        const int64_t S = n_samples - s0 < WAVE_MAX ? n_samples - s0 : WAVE_MAX;
        ProfileScope ps(ctx, "hv_mc_monte_carlo");
        DMO_LAUNCH(dominated_wave_kernel, (unsigned)ceil_div(S, SCAN_T), SCAN_T, smem, mf.F, nf, M, mf.ideal, mf.ref, seed, stream_id,
                   (uint64_t)P_MC_SAMPLE, 0, next + (uint64_t)s0, S, (uint32_t*)nullptr, sums.p);
      }
      DMO_CHECK_LAUNCH();
      unsigned long long h[3];
      DMO_CUDA(cudaMemcpyAsync(h, sums.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
      DMO_CUDA(dmo_wait(ctx));
      dom = h[0];
      tests += (int64_t)h[2];
      samples += n_samples;
      next += (uint64_t)n_samples;
    }
    est = U * ((double)dom / (double)n_samples);
  } else if (algorithm == DMO_HVMC_FPRAS) {
    FprasState st;
    DMO_TRY(run_fpras(ctx, mf, (int64_t)M1, st));
    fpras_result(st);
  } else if (algorithm == DMO_HVMC_MCM2RV) {
    DMO_TRY(mcm2rv(0));
  } else {  // hybrid (hv_adaptive.py:575-855)
    const double ratio = W / U;  // level 1: geometric pre-screening (overlap_ratio_threshold 5.0)
    if (ratio > 5.0) {
      ran = DMO_HVMC_MCM2RV;
      DMO_TRY(mcm2rv(0));
    } else if (ratio < 1.2) {
      ran = DMO_HVMC_FPRAS;
      FprasState st;
      DMO_TRY(run_fpras(ctx, mf, (int64_t)M1, st));
      fpras_result(st);
    } else {
      // level 2: E[xi] over 50 probes
      DevBuf<int64_t> pxi;
      DMO_TRY(pxi.alloc(ctx, N_PROBES));
      DMO_LAUNCH(probe_kernel, N_PROBES, MC_T, 0, mf.F, nf, M, mf.ref, mf.cdf, seed, stream_id, pxi.p);
      DMO_CHECK_LAUNCH();
      int64_t hp[N_PROBES];
      DMO_CUDA(cudaMemcpyAsync(hp, pxi.p, sizeof(hp), cudaMemcpyDeviceToHost, ctx->stream));
      DMO_CUDA(dmo_wait(ctx));
      double mean_xi = 0.0;
      for (int p = 0; p < N_PROBES; ++p) mean_xi += (double)hp[p];
      mean_xi /= N_PROBES;
      if (mean_xi > 20.0) {
        ran = DMO_HVMC_MCM2RV;
        DMO_TRY(mcm2rv(0));
      } else if (mean_xi < 5.0) {
        ran = DMO_HVMC_FPRAS;
        FprasState st;
        DMO_TRY(run_fpras(ctx, mf, (int64_t)M1, st));
        fpras_result(st);
      } else {
        // level 3: FPRAS rounds of 1, 2, 4 and 8 % of M1, then the theta bounds of estimate_theta_bounds
        const double Rv = (4.0 * (1.0 + epsilon * (1.0 - epsilon)) * log(2.0 / delta)) / (epsilon * epsilon * (1.0 - epsilon) * (1.0 - epsilon));
        auto theta = [&](double V) { return ((double)nf * (double)nf * (V * V + (U - V) * W) / (W * W)) * (Rv / M1); };
        const double fractions[4] = {0.01, 0.02, 0.04, 0.08};
        double cum = 0.0;
        FprasState st;
        bool decided = false;
        for (int r = 0; r < 4 && !decided; ++r) {
          cum += fractions[r];
          DMO_TRY(run_fpras(ctx, mf, (int64_t)(cum * M1), st));
          const int64_t N = st.N > 0 ? st.N : 1;
          const double V = (W / (double)nf) * ((double)st.sum_xi / (double)N);
          const double e1 = epsilon / sqrt(cum);
          const double th_upper = theta(V / (1.0 - e1)), th_lower = theta(V / (1.0 + e1));
          const double threshold = 1.0 - cum;
          if (th_upper < threshold * 0.85) {
            ran = DMO_HVMC_HYBRID_MCM2RV;
            DMO_TRY(mcm2rv(st.tests));
            decided = true;
          } else if (th_lower > threshold * 1.15) {
            decided = true;
          }
        }
        if (ran != DMO_HVMC_HYBRID_MCM2RV) {  // complete FPRAS to M1
          ran = DMO_HVMC_HYBRID_FPRAS;
          DMO_TRY(run_fpras(ctx, mf, (int64_t)M1, st));
          fpras_result(st);
        }
      }
    }
  }
  *out = est;
  if (samples_out) *samples_out = samples;
  if (tests_out) *tests_out = tests;
  if (algorithm_out) *algorithm_out = ran;
  return DMO_OK;
}
