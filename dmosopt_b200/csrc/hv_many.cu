// Exact hypervolume for 6 .. 8 objectives (SURVEY.md section 8a row A16; the reference routes every M < 10 to its exact box
// decomposition, dmosopt/hv.py:160-170, dmosopt/hv_box_decomposition.py:86-129).
//
// The slicing identity of hv.cu, applied recursively with limit sets (the WFG scheme):
//     HV_d(S) = sum_k (r_d - z_k) * [ vol_{d-1}(p_k) - HV_{d-1}( nds( { max(q, p_k) : q before k along axis d } ) ) ]
// (points in ascending order of their last coordinate; max = component-wise over the first d - 1 coordinates; nds = the
// non-dominated subset, which is what keeps the recursion small).  The chain sums of hv.cu (M = 4, 5) enumerate
// O(n^(M-2)) chains whatever the data; here every level filters its limit set, so fronts of a few hundred points in 6 - 8
// dimensions stay tractable.  Parallelism: the first two levels are unrolled into independent (k, j) tasks -- kernel A
// builds the limit set L_k of every point (one thread per k), kernel B gives every (k, j) pair one thread that runs the
// remaining recursion sequentially in its own arena; the terms are summed in a fixed order (deterministic).
//
// Work is exponential in the worst case (as for every exact algorithm); the front size is limited to HVM_MAX_FRONT.
#include "common.cuh"

namespace {

constexpr int HVM_MAX_FRONT = 2048;

// append q (D coordinates) to the non-dominated set L (lc points, stride D) unless a member is <= q everywhere;
// members that q dominates (q <= member everywhere) are removed
template <int D>
__device__ __forceinline__ void nds_insert(double* __restrict__ L, int& lc, const double* __restrict__ q) {
  int w = 0;
  for (int i = 0; i < lc; ++i) {
    const double* e = L + (size_t)i * D;
    bool e_le = true, q_le = true;
#pragma unroll
    for (int a = 0; a < D; ++a) {
      e_le = e_le && (e[a] <= q[a]);
      q_le = q_le && (q[a] <= e[a]);
    }
    if (e_le) {  // q adds nothing; nothing was removed before this point (a removed member would be dominated by e too)
      return;
    }
    if (!q_le) {  // keep e
      if (w != i) {
#pragma unroll
        for (int a = 0; a < D; ++a) L[(size_t)w * D + a] = e[a];
      }
      ++w;
    }
  }
#pragma unroll
  for (int a = 0; a < D; ++a) L[(size_t)w * D + a] = q[a];
  lc = w + 1;
}

template <int D>
__device__ __forceinline__ void sort_by_last(double* __restrict__ S, int cnt) {
  for (int i = 1; i < cnt; ++i) {
    double t[D];
#pragma unroll
    for (int a = 0; a < D; ++a) t[a] = S[(size_t)i * D + a];
    int j = i - 1;
    while (j >= 0 && S[(size_t)j * D + (D - 1)] > t[D - 1]) {
#pragma unroll
      for (int a = 0; a < D; ++a) S[(size_t)(j + 1) * D + a] = S[(size_t)j * D + a];
      --j;
    }
#pragma unroll
    for (int a = 0; a < D; ++a) S[(size_t)(j + 1) * D + a] = t[a];
  }
}

// HV_D of the cnt points at S (stride D, reordered in place); the levels below live behind S at n_max points per level
template <int D>
struct SetHv {
  static __device__ double run(double* __restrict__ S, int cnt, const double* __restrict__ ref, int n_max) {
    if (cnt == 0) return 0.0;
    if (cnt == 1) {
      double v = 1.0;
#pragma unroll
      for (int a = 0; a < D; ++a) v *= ref[a] - S[a];
      return v;
    }
    sort_by_last<D>(S, cnt);
    double* L = S + (size_t)n_max * D;
    double total = 0.0;
    for (int j = 0; j < cnt; ++j) {
      const double* p = S + (size_t)j * D;
      double vol = 1.0;
#pragma unroll
      for (int a = 0; a < D - 1; ++a) vol *= ref[a] - p[a];
      int lc = 0;
      for (int i = 0; i < j; ++i) {
        double q[D - 1];
#pragma unroll
        for (int a = 0; a < D - 1; ++a) q[a] = fmax(S[(size_t)i * D + a], p[a]);
        nds_insert<D - 1>(L, lc, q);
      }
      total += (ref[D - 1] - p[D - 1]) * (vol - SetHv<D - 1>::run(L, lc, ref, n_max));
    }
    return total;
  }
};

template <>
struct SetHv<2> {
  static __device__ double run(double* __restrict__ S, int cnt, const double* __restrict__ ref, int) {
    if (cnt == 0) return 0.0;
    // ascending x (insertion sort on the first coordinate), then the staircase sweep
    for (int i = 1; i < cnt; ++i) {
      const double tx = S[2 * i], ty = S[2 * i + 1];
      int j = i - 1;
      while (j >= 0 && S[2 * j] > tx) {
        S[2 * j + 2] = S[2 * j];
        S[2 * j + 3] = S[2 * j + 1];
        --j;
      }
      S[2 * j + 2] = tx;
      S[2 * j + 3] = ty;
    }
    double best = ref[1], area = 0.0;
    for (int i = 0; i < cnt; ++i)
      if (S[2 * i + 1] < best) {
        area += (ref[0] - S[2 * i]) * (best - S[2 * i + 1]);
        best = S[2 * i + 1];
      }
    return area;
  }
};

// doubles of arena one (k, j) task needs below its first limit set: levels D2, D2 - 1, .., 2
__host__ __device__ inline size_t arena_doubles(int D2, int n_max) { return (size_t)n_max * (size_t)(D2 * (D2 + 1) / 2 - 1); }

// P: the front in ascending order of its last coordinate, (n, M) row-major.  One thread per k: L_k = nds of the limit set of
// p_k against p_0 .. p_{k-1} in D1 = M - 1 dimensions, sorted by its last coordinate; cnt[k]; head[k] = (r - z_k), vol[k].
template <int D1>
__global__ void hvm_limit_kernel(const double* __restrict__ P, int n, const double* __restrict__ ref, double* __restrict__ Lbuf,
                                 int* __restrict__ cnt, double* __restrict__ head, double* __restrict__ vol) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  constexpr int M = D1 + 1;
  const double* p = P + (size_t)k * M;
  double* L = Lbuf + (size_t)k * n * D1;
  int lc = 0;
  for (int i = 0; i < k; ++i) {
    double q[D1];
#pragma unroll
    for (int a = 0; a < D1; ++a) q[a] = fmax(P[(size_t)i * M + a], p[a]);
    nds_insert<D1>(L, lc, q);
  }
  sort_by_last<D1>(L, lc);
  cnt[k] = lc;
  double v = 1.0;
#pragma unroll
  for (int a = 0; a < D1; ++a) v *= ref[a] - p[a];
  vol[k] = v;
  head[k] = ref[D1] - p[D1];
}

// one thread per (k, j): term[k][j] = (r - l_j[D1-1]) * [ vol_{D2}(l_j) - HV_{D2}( nds limit set of l_j against L_k[0 .. j-1] ) ]
template <int D2>
__global__ void hvm_pair_kernel(const double* __restrict__ Lbuf, const int* __restrict__ cnt, int n, int k0, int n_max,
                                const double* __restrict__ ref, double* __restrict__ arena, double* __restrict__ term) {
  constexpr int D1 = D2 + 1;
  const int k = k0 + blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n || j >= cnt[k]) return;
  const double* Lk = Lbuf + (size_t)k * n * D1;
  const double* l = Lk + (size_t)j * D1;
  double* A = arena + ((size_t)blockIdx.y * n_max + j) * arena_doubles(D2, n_max);
  int lc = 0;
  for (int i = 0; i < j; ++i) {
    double q[D2];
#pragma unroll
    for (int a = 0; a < D2; ++a) q[a] = fmax(Lk[(size_t)i * D1 + a], l[a]);
    nds_insert<D2>(A, lc, q);
  }
  double v = 1.0;
#pragma unroll
  for (int a = 0; a < D2; ++a) v *= ref[a] - l[a];
  term[(size_t)k * n + j] = (ref[D2] - l[D2]) * (v - SetHv<D2>::run(A, lc, ref, n_max));
}

// HV = sum_k head_k * (vol_k - sum_j term[k][j]), terms added in index order
__global__ void hvm_combine_kernel(const double* __restrict__ term, const int* __restrict__ cnt, const double* __restrict__ head,
                                   const double* __restrict__ vol, int n, double* __restrict__ out) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < cnt[k]; ++j) s += term[(size_t)k * n + j];
    acc += head[k] * (vol[k] - s);
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)blockDim.x; ++i) t += sh[i];
    *out = t;
  }
}

__global__ void hvm_gather_kernel(const double* __restrict__ F, const uint32_t* __restrict__ sidx, int n, int M, double* __restrict__ P) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n * M) return;
  const int64_t k = t / M;
  P[t] = F[(int64_t)sidx[k] * M + (t - k * M)];
}

template <int M>
int run_many(dmo_ctx* ctx, const double* dP, int n, const double* dref, double* h_out) {
  constexpr int D1 = M - 1, D2 = M - 2;
  DevBuf<double> Lbuf, head, vol, term, arena, res;
  DevBuf<int> cnt;
  DMO_TRY(Lbuf.alloc(ctx, (size_t)n * n * D1));
  DMO_TRY(head.alloc(ctx, n));
  DMO_TRY(vol.alloc(ctx, n));
  DMO_TRY(cnt.alloc(ctx, n));
  DMO_TRY(term.alloc(ctx, (size_t)n * n));
  DMO_TRY(res.alloc(ctx, 1));
  {
    ProfileScope ps(ctx, "hv_many");
    DMO_LAUNCH(hvm_limit_kernel<D1>, (unsigned)ceil_div(n, 64), 64, 0, dP, n, dref, Lbuf.p, cnt.p, head.p, vol.p);
    // largest limit set decides the arena of a task; the k range is processed in chunks that keep the arena under ~4 GiB
    std::vector<int> hc(n);
    DMO_CUDA(cudaMemcpyAsync(hc.data(), cnt.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    int n_max = 1;
    for (int k = 0; k < n; ++k) n_max = hc[k] > n_max ? hc[k] : n_max;
    const size_t per_k = (size_t)n_max * arena_doubles(D2, n_max) * sizeof(double);
    int kc = (int)(((size_t)4 << 30) / (per_k ? per_k : 1));
    if (kc < 1) kc = 1;
    if (kc > n) kc = n;
    if (kc > 65535) kc = 65535;
    DMO_TRY(arena.alloc(ctx, (size_t)kc * n_max * arena_doubles(D2, n_max)));
    for (int k0 = 0; k0 < n; k0 += kc) {
      const int kn = (n - k0) < kc ? (n - k0) : kc;
      dim3 grid((unsigned)ceil_div(n_max, 64), (unsigned)kn);
      DMO_LAUNCH(hvm_pair_kernel<D2>, grid, 64, 0, Lbuf.p, cnt.p, n, k0, n_max, dref, arena.p, term.p);
    }
    DMO_LAUNCH(hvm_combine_kernel, 1, 256, 0, term.p, cnt.p, head.p, vol.p, n, res.p);
  }
  DMO_CHECK_LAUNCH();
  DMO_CUDA(cudaMemcpyAsync(h_out, res.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // namespace

// Fnd: the non-dominated points strictly inside the reference box (device, (n, M)); sidx: their order along the last
// objective (ascending, ties by index).  M = 4 .. 8 (4 and 5 serve as a cross-check of the chain-sum kernels of hv.cu).
int hv_many_device(dmo_ctx* ctx, const double* Fnd, const uint32_t* sidx, int64_t n, int M, const double* dref, double* h_out) {
  *h_out = 0.0;
  if (n <= 0) return DMO_OK;
  DMO_REQUIRE(M >= 4 && M <= 8, "hypervolume: M=%d not supported by the limit-set recursion (4..8)", M);
  DMO_REQUIRE(n <= HVM_MAX_FRONT, "hypervolume: exact M=%d hypervolume is limited to fronts of %d points (got %lld)", M, HVM_MAX_FRONT,
              (long long)n);
  DevBuf<double> P;
  DMO_TRY(P.alloc(ctx, (size_t)n * M));
  DMO_LAUNCH(hvm_gather_kernel, (unsigned)ceil_div(n * M, 256), 256, 0, Fnd, sidx, (int)n, M, P.p);
  switch (M) {
    case 4: return run_many<4>(ctx, P.p, (int)n, dref, h_out);
    case 5: return run_many<5>(ctx, P.p, (int)n, dref, h_out);
    case 6: return run_many<6>(ctx, P.p, (int)n, dref, h_out);
    case 7: return run_many<7>(ctx, P.p, (int)n, dref, h_out);
    default: return run_many<8>(ctx, P.p, (int)n, dref, h_out);
  }
}
