// Non-dominated rank (SURVEY.md section 8a rows A1/A2; replaces dmosopt/dda.py:97-152 dda_ens).
//
// rank_i = front index = length of the longest domination chain ending at i
//        = 0 if nothing dominates i, else 1 + max{rank_j : j dominates i}.
//
// Pipeline (all on the context's stream):
//   1. per objective: radix-sort the column, give every distinct value a dense integer id
//      (order- and equality-preserving, so float64 inputs are ranked exactly with 32-bit compares);
//   2. lexicographic order of the integer vectors (LSD radix passes); in that order a point can only
//      be dominated by points before it, and identical vectors are adjacent (one "group id" each);
//      (two and three objectives, up to 1024 blocks: the segmented order of `RankSeg` below -- another linear extension
//      of the dominance order -- which lets whole tiles be skipped or answered from a per-tile staircase);
//   3. one persistent kernel evaluates the chain recurrence block by block in that order: a block of T = 128 targets
//      streams the earlier blocks through shared memory (coalesced 16-byte records, broadcast reads, one dominance
//      predicate per pair); the rank word of a record (rank + 1, 0 = not final) is its own ready flag, so a consumer
//      polls only when it catches up with the wavefront.  In-block chains and the chains entering from the predecessor
//      block are precomputed as longest-path tables (int8, breadth-first walks over 128-bit successor masks) before
//      any rank is needed, so that the serial part of a block is two packed max-plus products and one store.
//      Blocks are handed out by an atomic ticket, so a block only ever waits for blocks whose CTAs are already running
//      (no co-residency assumption, no deadlock); every wait is bounded by a watchdog that raises an error flag.
//
// Rank-0-only queries (the hypervolume's filter) take a plain block scan of the lexicographic records or, for two and three
// objectives, one test on the cell grid `grid_*`, which needs the dense ids alone.  Truncations (remove_worst: only the
// ranks of the kept rows matter) of three-objective sets peel the fronts they need off the same grid instead of running
// the chain, when those fronts are few (`rank_by_peeling`, below).
//
// Algorithmic bytes: 8 n M read + 4 n written; pair tests <= n^2 / 2 (compare / latency bound, see DESIGN.md section 4.2).
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

namespace {

constexpr int RANK_T = 128;  // targets per block == sources per shared-memory tile

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void flag_new_u64_kernel(const uint64_t* __restrict__ skeys, int64_t n, uint32_t* __restrict__ flag) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) flag[p] = (p > 0 && skeys[p] != skeys[p - 1]) ? 1u : 0u;
}

__global__ void scatter_dense_kernel(const uint32_t* __restrict__ dense, const uint32_t* __restrict__ sidx, int64_t n,
                                     uint32_t* __restrict__ R) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) R[sidx[p]] = dense[p];
}

// flag[p] = 1 iff the vector at sorted position p differs from the one at p-1
__global__ void flag_new_vec_kernel(const uint32_t* __restrict__ R, const uint32_t* __restrict__ perm, int64_t n, int M,
                                    uint32_t* __restrict__ flag) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  uint32_t f = 0;
  if (p > 0) {
    uint32_t a = perm[p], b = perm[p - 1];
    for (int j = 0; j < M; ++j) f |= (R[(int64_t)j * n + a] != R[(int64_t)j * n + b]) ? 1u : 0u;
  }
  flag[p] = f;
}

// record words: [o_1 .. o_{M-1}, gid, rank+1, pad...]; padded to W = 4*ceil((M+1)/4) words
__global__ void build_records_kernel(const uint32_t* __restrict__ R, const uint32_t* __restrict__ perm,
                                     const uint32_t* __restrict__ gid, int64_t n, int64_t npad, int M, int W,
                                     uint32_t* __restrict__ rec) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npad) return;
  uint32_t* r = rec + p * W;
  if (p < n) {
    uint32_t i = perm[p];
    for (int j = 1; j < M; ++j) r[j - 1] = R[(int64_t)j * n + i];
    r[M - 1] = gid[p];
    for (int w = M; w < W; ++w) r[w] = 0u;
  } else {
    // sentinel: larger than every real id in every objective, its own group; never dominates a real point
    for (int j = 1; j < M; ++j) r[j - 1] = 0xFFFFFFFFu;
    r[M - 1] = 0xFFFFFFFFu - (uint32_t)(p - n);
    for (int w = M; w < W; ++w) r[w] = 0u;
  }
}

__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t word_of(const uint4& a, int c) { return c == 0 ? a.x : c == 1 ? a.y : c == 2 ? a.z : a.w; }

// The rank word of a record (rank + 1, 0 = not yet final) is its own ready flag: a 4-byte store is atomic and carries
// no other data, so publication needs neither fences nor a separate flag, and consumers simply poll the word.
// ------------------------------------------------------------------------------------------------ segmented order (M <= 3)
// Any linear extension of the dominance order works for the chain recurrence.  Instead of the plain lexicographic
// order the points are ordered by (segment of objective 1, objective 2, ..., objective M, objective 1), a segment
// being a run of 1024 dense ids of objective 1 (at most 128 segments).  Sources in an earlier segment have a smaller objective-1 id than
// every target, and inside a segment the tiles are sorted by the first compare word, so for a target block with the
// band [blo, bhi] of that word a whole earlier tile is
//   * skipped        if its smallest word is > bhi (nothing in it can dominate anything in the block),
//   * "fast"         if its largest word is < blo (the first compare is known to pass and is dropped),
//   * tested in full otherwise (about one tile per segment) and, with the extra objective-1 compare, for the tiles that
//     may share a segment with the block.
// For three objectives a "fast" tile leaves a single condition, word_1(source) <= word_1(target); every block therefore
// also publishes its records as a staircase -- sorted by that word, with the running maximum of rank + 1 -- and a target
// resolves a fast tile with one 7-step binary search instead of 128 pair tests (two objectives: the tile maximum).
// Bands are compared on 8-bit floor-quantised words (conservative in both directions) held in shared memory.
struct RankSeg {
  const uint32_t* c1rec = nullptr;      // [npad] objective-1 id per position (0xFFFFFFFF for the padding)
  const uint32_t* seg_start = nullptr;  // [nseg + 1] first position whose segment is >= s
  const uint16_t* tile_q = nullptr;     // [nblocks] low byte = min, high byte = max of the quantised first compare word
  unsigned long long* stair = nullptr;  // [npad] per tile: entry t = (t-th smallest last compare word of the tile, low 32
                                        // bits; max (rank + 1) over the t+1 records with the smallest words, high 32 bits)
  int sshift = 0;                       // id1 >> sshift = segment
  int qshift = 0;                       // word >> qshift = 8-bit band coordinate (clamped to 255)
};
constexpr int RANK_SEG_MAXT = 1024;  // tiles whose bands fit the shared-memory cache (n <= 131072)

__global__ void seg_key_kernel(const uint32_t* __restrict__ R0, const uint32_t* __restrict__ perm, int64_t n, int sshift,
                               uint32_t* __restrict__ key) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) key[p] = R0[perm[p]] >> sshift;
}

__global__ void seg_c1_kernel(const uint32_t* __restrict__ R0, const uint32_t* __restrict__ perm, int64_t n, int64_t npad,
                              uint32_t* __restrict__ c1rec) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < npad) c1rec[p] = p < n ? R0[perm[p]] : 0xFFFFFFFFu;
}

__global__ void seg_start_kernel(const uint32_t* __restrict__ c1rec, int64_t n, int sshift, int nseg,
                                 uint32_t* __restrict__ seg_start) {
  int sgi = blockIdx.x * blockDim.x + threadIdx.x;
  if (sgi > nseg) return;
  int64_t lo = 0, hi = n;  // positions are sorted by segment
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((c1rec[mid] >> sshift) < (uint32_t)sgi) lo = mid + 1; else hi = mid;
  }
  seg_start[sgi] = (uint32_t)lo;
}

// one warp per tile: quantised min / max of the first compare word.  A tile whose first compare word is not ascending
// (it spans a segment boundary, or holds padding) is given the full band [0, 255]: it is then never skipped, never
// "fast", and the pair tests take the generic loop instead of the sorted-prefix loop.
__global__ void seg_tile_band_kernel(const uint32_t* __restrict__ rec, int nblocks, int T, int qshift,
                                     uint16_t* __restrict__ tile_q) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= nblocks) return;
  uint32_t lo = 255u, hi = 0u;
  bool sorted = true;
  for (int t = lane; t < T; t += 32) {
    const uint32_t w = rec[((int64_t)k * T + t) * 4];
    const uint32_t q = min(w >> qshift, 255u);
    lo = min(lo, q);
    hi = max(hi, q);
    if (t > 0) sorted = sorted && (rec[((int64_t)k * T + t - 1) * 4] <= w);
  }
  lo = __reduce_min_sync(0xFFFFFFFFu, lo);
  hi = __reduce_max_sync(0xFFFFFFFFu, hi);
  sorted = __all_sync(0xFFFFFFFFu, sorted);
  if (!sorted) {
    lo = 0u;
    hi = 255u;
  }
  if (lane == 0) tile_q[k] = (uint16_t)(lo | (hi << 8));
}

// Pair tests against a tile whose first compare word is ascending: only the prefix with word_0 <= v[0] can dominate, so
// one binary search replaces that compare and the loop stops at the longest prefix of the warp (the 32 targets of a warp
// are neighbours in the same order, their prefixes are close).
template <int M, int W, int NV, int T, bool GID>
__device__ __forceinline__ int rank_pair_tests_sorted(const uint4* tb, const uint32_t* v, uint32_t gidv, int best) {
  int p = 0;  // number of records with word_0 <= v[0]
#pragma unroll
  for (int step = T / 2; step >= 1; step >>= 1)
    if (reinterpret_cast<const uint32_t*>(&tb[(p + step - 1) * NV])[0] <= v[0]) p += step;
  if (p < T && reinterpret_cast<const uint32_t*>(&tb[p * NV])[0] <= v[0]) ++p;
  const int pmax = __reduce_max_sync(0xFFFFFFFFu, p);
  int acc[4] = {best, 0, 0, 0};
#pragma unroll 8
  for (int s = 0; s < pmax; ++s) {
    uint32_t sw[W];
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      const uint4 a4 = tb[s * NV + q];
      sw[4 * q + 0] = a4.x;
      sw[4 * q + 1] = a4.y;
      sw[4 * q + 2] = a4.z;
      sw[4 * q + 3] = a4.w;
    }
    bool dom = (s < p) && (GID ? (sw[M - 1] != gidv) : true);
#pragma unroll
    for (int j = 1; j < M - 1; ++j) dom = dom && (sw[j] <= v[j]);
    acc[s & 3] = dom ? max(acc[s & 3], (int)sw[M]) : acc[s & 3];
  }
  return max(max(acc[0], acc[1]), max(acc[2], acc[3]));
}

// 128 pair tests of one streamed tile against this thread's record.  SKIP0: the first compare word is known to pass;
// GID: the "not identical" test is needed; C1: objective 1 must be compared too (source may share the target's segment)
template <int M, int W, int NV, int T, bool SKIP0, bool GID, bool C1>
__device__ __forceinline__ int rank_pair_tests(const uint4* tb, const uint32_t* c1tb, const uint32_t* v, uint32_t gidv,
                                               uint32_t c1v, int best) {
  int acc[4] = {best, 0, 0, 0};  // four independent max chains (the predicated max is the only loop-carried dependency)
#pragma unroll 16
  for (int s = 0; s < T; ++s) {
    uint32_t sw[W];
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      const uint4 a4 = tb[s * NV + q];
      sw[4 * q + 0] = a4.x;
      sw[4 * q + 1] = a4.y;
      sw[4 * q + 2] = a4.z;
      sw[4 * q + 3] = a4.w;
    }
    bool dom = GID ? (sw[M - 1] != gidv) : true;
#pragma unroll
    for (int j = SKIP0 ? 1 : 0; j < M - 1; ++j) dom = dom && (sw[j] <= v[j]);
    if (C1) dom = dom && (c1tb[s] <= c1v);
    const int r1 = (int)sw[M];
    acc[s & 3] = dom ? max(acc[s & 3], r1) : acc[s & 3];
  }
  return max(max(acc[0], acc[1]), max(acc[2], acc[3]));
}

// Breadth-first walk by path length from the node set `f` (level `level`): table[i * DLD + col] = last level at which
// i is reached = longest path.  Each thread walks its own source; the frontier is a 128-bit set in registers.
template <int T, int DLD>
__device__ __forceinline__ void frontier_fill(int8_t* table, const uint4* succ, uint4 f, int col, int level) {
  static_assert(T == 128, "frontier sets are 128 bits wide");
  while ((f.x | f.y | f.z | f.w) != 0u) {
    uint4 nx = make_uint4(0u, 0u, 0u, 0u);
#define DMO_WALK(word, base)                           \
  for (uint32_t mm = (word); mm != 0u; mm &= mm - 1u) { \
    const int i = (base) + __ffs(mm) - 1;               \
    table[i * DLD + col] = (int8_t)level;               \
    const uint4 sc = succ[i];                           \
    nx.x |= sc.x;                                       \
    nx.y |= sc.y;                                       \
    nx.z |= sc.z;                                       \
    nx.w |= sc.w;                                       \
  }
    DMO_WALK(f.x, 0)
    DMO_WALK(f.y, 32)
    DMO_WALK(f.z, 64)
    DMO_WALK(f.w, 96)
#undef DMO_WALK
    f = nx;
    ++level;
  }
}

// max(init, max_a (vals16[a] + row[a])) over one table row of T int8 path lengths (SENT = -128 = "no path"), two
// 16-bit lanes per instruction: PRMT + AND expand a byte pair to int16 (SENT becomes -32768, so SENT + value < 0 never
// wins against init >= 0), VIADDMNMX.S16x2 does the add and the max.  Requires 0 <= vals16, init <= 32127.
template <int T>
__device__ __forceinline__ int maxplus_packed(const int8_t* row, const int16_t* vals16, int init) {
  const uint4* dr = reinterpret_cast<const uint4*>(row);
  const uint4* vr = reinterpret_cast<const uint4*>(vals16);
  unsigned acc0 = ((unsigned)init & 0xFFFFu) * 0x00010001u, acc1 = acc0;
#define DMO_EXP_LO(w) (__byte_perm((w), 0u, 0x1100) & 0x807F807Fu)
#define DMO_EXP_HI(w) (__byte_perm((w), 0u, 0x3322) & 0x807F807Fu)
#pragma unroll
  for (int c = 0; c < T / 16; ++c) {
    const uint4 dv = dr[c];
    const uint4 v0 = vr[2 * c], v1 = vr[2 * c + 1];
    acc0 = __viaddmax_s16x2(DMO_EXP_LO(dv.x), v0.x, acc0);
    acc1 = __viaddmax_s16x2(DMO_EXP_HI(dv.x), v0.y, acc1);
    acc0 = __viaddmax_s16x2(DMO_EXP_LO(dv.y), v0.z, acc0);
    acc1 = __viaddmax_s16x2(DMO_EXP_HI(dv.y), v0.w, acc1);
    acc0 = __viaddmax_s16x2(DMO_EXP_LO(dv.z), v1.x, acc0);
    acc1 = __viaddmax_s16x2(DMO_EXP_HI(dv.z), v1.y, acc1);
    acc0 = __viaddmax_s16x2(DMO_EXP_LO(dv.w), v1.z, acc0);
    acc1 = __viaddmax_s16x2(DMO_EXP_HI(dv.w), v1.w, acc1);
  }
#undef DMO_EXP_LO
#undef DMO_EXP_HI
  const unsigned m = __vmaxs2(acc0, acc1);
  return max((int)(int16_t)(m & 0xFFFFu), (int)(int16_t)(m >> 16));
}

// Above eight objectives the shared memory alone limits a CTA to four per SM, so the register cap follows that.
template <int M, int T, bool SEG>
__global__ void __launch_bounds__(T, (SEG || M > 8) ? 4 : 5) rank_chain_kernel(uint32_t* rec, int nblocks, int* __restrict__ rankS, int* ticket,
                                                                 int* errflag, RankSeg sg) {
  constexpr int W = 4 * ((M + 1 + 3) / 4);
  constexpr int NV = W / 4;
  constexpr int NW = T / 32;
  constexpr int RQ = M / 4, RC = M % 4;  // uint4 / component holding the rank word
  // Path-length tables are stored TRANSPOSED, [destination i][source], row stride T + 16 bytes: the thread that owns
  // destination i reads its whole row with 16-byte loads (stride 36 words -> the 8 threads of a quarter warp hit 8
  // distinct 4-word groups, conflict free), while the threads that fill the tables walk columns (consecutive bytes).
  constexpr int DLD = T + 16;
  constexpr int SENT = -128;  // "no in-block path"; real path lengths are 0 .. T-1 <= 127
  constexpr int PACK_LIMIT = 32000;  // ranks up to here take the packed 16-bit max-plus path
  // own block's records during table construction, then stream buffer 0.  With five uint4 per record (M == 16) it
  // would take the static shared memory past 48 KB, so there it is the kernel's dynamic shared memory instead.
  constexpr bool DYN_TILE = NV > 4;
  __shared__ uint4 tile_s[DYN_TILE ? 1 : T * NV];
  extern __shared__ uint4 tile_dyn[];
  uint4* const tile = DYN_TILE ? tile_dyn : tile_s;
  constexpr bool DBUF = NV <= 2;  // M == 8 (three uint4 per record) would exceed 48 KB of static shared memory
  __shared__ uint4 tile2[DBUF ? T * NV : 1];  // stream buffer 1
  __shared__ __align__(16) int sh_r1[T];
  __shared__ __align__(16) int16_t sh_h16[T];
  __shared__ uint4 sh_succ[T];
  __shared__ __align__(16) int8_t sD[T * DLD];
  __shared__ __align__(16) int8_t sE[T * DLD];
  __shared__ int sh_blk;
  // segmented order only: objective-1 ids of the own block and of the streamed tiles, cached tile bands
  __shared__ uint32_t c1own[SEG ? T : 1];
  __shared__ uint32_t c1t[SEG ? 2 * T : 1];
  __shared__ uint16_t sq16[SEG ? RANK_SEG_MAXT : 1];
  __shared__ uint32_t sh_band[SEG ? 2 * NW : 1];
  __shared__ uint32_t skey[SEG ? T : 1];  // the block's last compare words in ascending order (staircase keys)

  const int tid = threadIdx.x;

  for (;;) {
    if (tid == 0) sh_blk = atomicAdd(ticket, 1);
    __syncthreads();
    const int b = sh_blk;
    __syncthreads();
    if (b >= nblocks) return;
    const int64_t i = (int64_t)b * T + tid;

    // ---- own record -> registers and shared tile
    uint32_t v[W];
    {
      const uint4* src = reinterpret_cast<const uint4*>(rec + i * W);
#pragma unroll
      for (int q = 0; q < NV; ++q) {
        uint4 a = src[q];
        tile[tid * NV + q] = a;
        v[4 * q + 0] = a.x;
        v[4 * q + 1] = a.y;
        v[4 * q + 2] = a.z;
        v[4 * q + 3] = a.w;
      }
    }
    const uint32_t gidv = v[M - 1];
    uint32_t c1v = 0u;
    uint32_t wq_lo = 0u, wq_hi = 255u;  // band of this warp's 32 records (a quarter of the block's band)
    if (SEG) {
      c1v = sg.c1rec[i];
      c1own[tid] = c1v;
      const uint32_t q = min(v[0] >> sg.qshift, 255u);
      const uint32_t qlo = __reduce_min_sync(0xFFFFFFFFu, q), qhi = __reduce_max_sync(0xFFFFFFFFu, q);
      wq_lo = qlo;
      wq_hi = qhi;
      if ((tid & 31) == 0) {
        sh_band[tid >> 5] = qlo;
        sh_band[NW + (tid >> 5)] = qhi;
      }
      for (int t = tid; t < b - 1; t += T) sq16[t] = sg.tile_q[t];  // bands of every tile this block may stream
    }
    __syncthreads();
    const uint32_t first_gid = reinterpret_cast<const uint32_t*>(&tile[0])[M - 1];  // group of the block's first record
    uint32_t bq_lo = 0u, bq_hi = 255u;
    int kc = 0;  // tiles >= kc may hold sources of the block's own segment(s): full test incl. objective 1, never skipped
    int kg = 0;  // tiles >= kg may hold a copy of one of the block's vectors ("not identical" test needed)
    int spos = tid;  // position of this record in the block's staircase order
    if (SEG) {
      bq_lo = min(min(sh_band[0], sh_band[1]), min(sh_band[2], sh_band[3]));
      bq_hi = max(max(sh_band[NW], sh_band[NW + 1]), max(sh_band[NW + 2], sh_band[NW + 3]));
      kc = (int)(sg.seg_start[c1own[0] >> sg.sshift] / (uint32_t)T);
      {  // first position whose group id is >= the block's first group id (group ids grow along the order)
        int64_t lo = 0, hi = (int64_t)b * T;
        while (lo < hi) {
          const int64_t mid = (lo + hi) >> 1;
          if (rec[mid * W + (M - 1)] < first_gid) lo = mid + 1; else hi = mid;
        }
        kg = (int)(lo / T);
      }
      if (M == 3) {  // rank of the own last compare word inside the block (ties by position): 128 compares per thread
        const uint32_t key = v[1];
        int cnt = 0;
#pragma unroll 8
        for (int s = 0; s < T; ++s) {
          const uint32_t ks = reinterpret_cast<const uint32_t*>(&tile[s * NV])[1];
          cnt += (ks < key || (ks == key && s < tid)) ? 1 : 0;
        }
        spos = cnt;
        skey[spos] = key;
      } else {
        skey[tid] = 0u;
      }
    }

    // ---- in-block successor bitmasks: succ[j] = { i > j in this block : j dominates i }; independent of any rank
    {
      uint32_t sm[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        uint32_t m = 0u;
#pragma unroll 8
        for (int s = 0; s < 32; ++s) {
          const uint32_t* sp = reinterpret_cast<const uint32_t*>(&tile[(w * 32 + s) * NV]);
          bool dom = (w * 32 + s > tid) && (sp[M - 1] != gidv);
#pragma unroll
          for (int j = 0; j < M - 1; ++j) dom = dom && (v[j] <= sp[j]);
          if (SEG) dom = dom && (c1v <= c1own[w * 32 + s]);  // objective 1 is not implied by the order inside a segment
          m |= (dom ? 1u : 0u) << s;
        }
        sm[w] = m;
      }
      static_assert(NW == 4, "successor masks are stored as one uint4 per node");
      sh_succ[tid] = make_uint4(sm[0], sm[1], sm[2], sm[3]);
      // the path-length table starts as "no path"
      const uint4 fill = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
      for (int t = tid; t < T * DLD / 16; t += T) reinterpret_cast<uint4*>(sD)[t] = fill;
    }
    __syncthreads();

    // ---- in-block longest-path table, computed BEFORE any rank is needed (off the critical path):
    // D[a][i] = number of edges of the longest in-block domination chain a -> ... -> i (SENT if none, 0 for i == a).
    // Thread a walks the DAG breadth first by path length: F_l = nodes reached from a by a path of exactly l edges,
    // F_{l+1} = union of succ[i] over i in F_l; the last level that contains i is the longest path (later writes win).
    // With it the in-block resolution is one max-plus product  rank_i = max_a (best_a + D[a][i]).
    frontier_fill<T, DLD>(sD, sh_succ, sh_succ[tid], tid, 1);
    sD[tid * DLD + tid] = 0;

    // ---- predecessor table: E[s][i] = longest in-block continuation of a chain that enters this block from point s of
    // block b-1 (0 if s dominates i directly).  Same walk, seeded with the block nodes s dominates, level 0.
    {
      const uint4 fill = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
      for (int t = tid; t < T * DLD / 16; t += T) reinterpret_cast<uint4*>(sE)[t] = fill;
    }
    __syncthreads();
    if (b > 0) {
      const int64_t ps = (int64_t)(b - 1) * T + tid;
      uint32_t pv[W];
      {
        const uint4* src = reinterpret_cast<const uint4*>(rec + ps * W);
#pragma unroll
        for (int q = 0; q < NV; ++q) {
          uint4 a4 = src[q];  // static words only (ids, group); the rank word is read later with ld.relaxed
          pv[4 * q + 0] = a4.x;
          pv[4 * q + 1] = a4.y;
          pv[4 * q + 2] = a4.z;
          pv[4 * q + 3] = a4.w;
        }
      }
      const uint32_t pc1 = SEG ? sg.c1rec[ps] : 0u;
      uint32_t pm[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        uint32_t m = 0u;
#pragma unroll 8
        for (int s2 = 0; s2 < 32; ++s2) {
          const uint32_t* sp = reinterpret_cast<const uint32_t*>(&tile[(w * 32 + s2) * NV]);
          bool dom = (sp[M - 1] != pv[M - 1]);
#pragma unroll
          for (int j = 0; j < M - 1; ++j) dom = dom && (pv[j] <= sp[j]);
          if (SEG) dom = dom && (pc1 <= c1own[w * 32 + s2]);
          m |= (dom ? 1u : 0u) << s2;
        }
        pm[w] = m;
      }
      frontier_fill<T, DLD>(sE, sh_succ, make_uint4(pm[0], pm[1], pm[2], pm[3]), tid, 0);
    }
    __syncthreads();

    int best = 0;
    // ---- the last streamed tile (block b-2) is the second serial dependency: its ranks arrive one link before this
    // block's turn.  Its dominance pattern does not depend on ranks, so it is evaluated now into a 128-bit mask per
    // thread (kept in the successor-mask storage, which the table walks no longer need); when the ranks arrive only a
    // maximum over the set bits remains.
    bool sparse_b2 = false;
    if (SEG && b >= 2) {
      const int64_t p2 = (int64_t)(b - 2) * T + tid;
      tile2[tid] = *reinterpret_cast<const uint4*>(rec + p2 * W);  // static words; NV == 1 in the segmented kernels
      c1t[T + tid] = sg.c1rec[p2];
      __syncthreads();
      uint32_t mk[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        uint32_t m = 0u;
#pragma unroll 8
        for (int s2 = 0; s2 < 32; ++s2) {
          const uint32_t* sp = reinterpret_cast<const uint32_t*>(&tile2[w * 32 + s2]);
          bool dom = (sp[M - 1] != gidv) && (c1t[T + w * 32 + s2] <= c1v);
#pragma unroll
          for (int j = 0; j < M - 1; ++j) dom = dom && (sp[j] <= v[j]);
          m |= (dom ? 1u : 0u) << s2;
        }
        mk[w] = m;
      }
      sh_succ[tid] = make_uint4(mk[0], mk[1], mk[2], mk[3]);  // own slot only; all table walks finished at the barrier above
      // the set-bit walk only pays when the masks are sparse (a converged population: few dominators per point);
      // dense masks (random data) keep the pair tests, whose 128 steps pipeline better than a long dependent walk
      sparse_b2 = __syncthreads_or((__popc(mk[0]) + __popc(mk[1]) + __popc(mk[2]) + __popc(mk[3])) > 8 ? 1 : 0) == 0;
    }

    // ---- stream every earlier block except the predecessor: best = max over dominators of (rank + 1)
    // Software pipelined: the data of the next tile (static words and, speculatively, its rank word -- or its staircase
    // entry) is requested before the current tile is evaluated, and the shared tile is double buffered, so a block that is
    // behind the wavefront pays one barrier and the evaluation per tile, not an L2 round trip on top; a block at the
    // wavefront only waits for the rank word.  In the segmented order whole tiles are skipped (see RankSeg).
    {
      auto next_tile = [&](int k) {
        if (SEG) {
          const int lim = min(kc, b - 1);
          while (k < lim && (uint32_t)(sq16[k] & 0xFFu) > bq_hi) ++k;  // every source word above the block's band
        }
        return k;
      };
      // tile kinds: 2 = staircase (earlier segment, every first word below the band, no copy of a block vector),
      //             1 = pair tests incl. objective 1 (may share a segment), 0 = pair tests,
      //             3 = the last tile: maximum over the precomputed dominance mask
      auto kind_of = [&](int k) {
        if (!SEG) return 0;
        if (k == b - 2 && sparse_b2) return 3;  // sparse dominance mask precomputed above
        if (k >= kc) return 1;
        return ((uint32_t)(sq16[k] >> 8) < bq_lo && k < kg) ? 2 : 0;
      };
      uint4 cur[NV];
      uint32_t cur_c1 = 0u;
      unsigned long long cur_st = 0ull;
      auto request = [&](int k, int kind) {
        if (SEG && kind == 2) {
          cur_st = ld_relaxed_u64(sg.stair + (int64_t)k * T + tid);
        } else {
          const uint4* src = reinterpret_cast<const uint4*>(rec + ((int64_t)k * T + tid) * W);
#pragma unroll
          for (int q = 0; q < NV; ++q) cur[q] = ld_relaxed_v4(src + q);
          if (SEG && kind == 1) cur_c1 = sg.c1rec[(int64_t)k * T + tid];
        }
      };
      int k = next_tile(0);
      int kind = k < b - 1 ? kind_of(k) : 0;
      if (k < b - 1) request(k, kind);
      int pb = 0;  // stream buffer parity
      while (k < b - 1) {
        {
          unsigned spins = 0;
          if (SEG && kind == 2) {
            const unsigned long long* src = sg.stair + (int64_t)k * T + tid;
            while ((cur_st >> 32) == 0ull) {  // the owner has not published its staircase yet
              __nanosleep(spins < 8 ? 100 : 400);
              cur_st = ld_relaxed_u64(src);
              if ((++spins & 0xFFu) == 0u && (spins > (1u << 21) || ld_relaxed_u32((const uint32_t*)errflag) != 0u)) {
                atomicExch(errflag, 1);
                break;
              }
            }
          } else {
            const uint4* src = reinterpret_cast<const uint4*>(rec + ((int64_t)k * T + tid) * W);
            while (word_of(cur[RQ], RC) == 0u) {  // not final yet: this block has caught up with the wavefront
              __nanosleep(spins < 8 ? 100 : 400);
              cur[RQ] = ld_relaxed_v4(src + RQ);
              if ((++spins & 0xFFu) == 0u && (spins > (1u << 21) || ld_relaxed_u32((const uint32_t*)errflag) != 0u)) {
                atomicExch(errflag, 1);
                break;
              }
            }
          }
        }
        uint4* tb = (DBUF && pb) ? tile2 : tile;
        if (!DBUF) __syncthreads();  // single buffer: everyone must be done with the previous tile
        if (SEG && kind == 2) {
          reinterpret_cast<unsigned long long*>(tb)[tid] = cur_st;
        } else {
#pragma unroll
          for (int q = 0; q < NV; ++q) tb[tid * NV + q] = cur[q];
          if (SEG && kind == 1) c1t[pb * T + tid] = cur_c1;
        }
        // Group ids grow along the order, so a tile whose last record is in an earlier group than this block's first
        // record holds no copy of any of this block's vectors: the "not identical" test can be dropped (one compare
        // per pair less).  The owner of the tile's last record votes through the tile barrier.
        const bool last_shares = !(SEG && kind == 2) && (tid == T - 1) && (word_of(cur[(M - 1) / 4], (M - 1) % 4) >= first_gid);
        const int kn = next_tile(k + 1);
        const int kind_n = kn < b - 1 ? kind_of(kn) : 0;
        if (kn < b - 1) request(kn, kind_n);  // consumed after this tile's evaluation
        // one barrier per tile: a stream buffer is rewritten two tiles later, after the next tile's barrier
        const bool may_share_group = __syncthreads_or(last_shares ? 1 : 0) != 0;
        const uint32_t* c1tb = c1t + (SEG ? pb * T : 0);
        if (SEG && kind == 2) {
          const uint2* st = reinterpret_cast<const uint2*>(tb);  // .x = key (ascending), .y = running max of rank + 1
          if (M == 3) {
            int idx = 0;  // number of keys <= v[1]
#pragma unroll
            for (int step = T / 2; step >= 1; step >>= 1)
              if (st[idx + step - 1].x <= v[1]) idx += step;
            if (idx < T && st[idx].x <= v[1]) ++idx;  // T is a power of two: the steps cover T - 1 positions
            if (idx > 0) best = max(best, (int)st[idx - 1].y);
          } else {
            best = max(best, (int)st[T - 1].y);  // two objectives: every record of the tile dominates the block
          }
        } else if (SEG && kind == 3) {
          const uint4 mk4 = sh_succ[tid];
          const uint32_t mk[4] = {mk4.x, mk4.y, mk4.z, mk4.w};
#pragma unroll
          for (int w = 0; w < 4; ++w)
            for (uint32_t mm = mk[w]; mm != 0u; mm &= mm - 1u) {
              const int s2 = w * 32 + __ffs(mm) - 1;
              best = max(best, (int)reinterpret_cast<const uint32_t*>(&tb[s2 * NV])[M]);
            }
        } else if (kind == 1) {
          best = rank_pair_tests<M, W, NV, T, false, true, true>(tb, c1tb, v, gidv, c1v, best);
        } else if (SEG && (uint32_t)(sq16[k] & 0xFFu) > wq_hi) {
          // straddles the block's band but lies entirely above this warp's: nothing in it dominates these 32 records
        } else if (SEG && (uint32_t)(sq16[k] >> 8) < wq_lo) {  // every source word below this warp's band
          best = may_share_group ? rank_pair_tests<M, W, NV, T, true, true, false>(tb, c1tb, v, gidv, c1v, best)
                                 : rank_pair_tests<M, W, NV, T, true, false, false>(tb, c1tb, v, gidv, c1v, best);
        } else if (SEG && sq16[k] != 0xFF00u) {  // ascending first word (the full band marks the tiles that are not)
          best = may_share_group ? rank_pair_tests_sorted<M, W, NV, T, true>(tb, v, gidv, best)
                                 : rank_pair_tests_sorted<M, W, NV, T, false>(tb, v, gidv, best);
        } else {
          best = may_share_group ? rank_pair_tests<M, W, NV, T, false, true, false>(tb, c1tb, v, gidv, c1v, best)
                                 : rank_pair_tests<M, W, NV, T, false, false, false>(tb, c1tb, v, gidv, c1v, best);
        }
        // Second barrier of the tile.  The double buffering alone orders the accesses (a buffer is rewritten two tiles
        // later, after the next tile's barrier, which every reader of this tile has to reach first), but compute-sanitizer's
        // racecheck reports the read above against the next write of the same buffer as a potential WAR hazard; with this
        // barrier the tool is clean (profiles/r2_sanitizer.txt) at no measurable cost (the chain is latency bound).
        __syncthreads();
        k = kn;
        kind = kind_n;
        pb ^= 1;
      }
    }
    // ---- in-block resolution, part 1 (before the predecessor's ranks are needed):
    //   Rb_i = max_a (bulk_a + D[a][i]) folds the contributions of all blocks < b-1 through the in-block paths.
    int r = best;
    if (!__syncthreads_or(best > PACK_LIMIT)) {
      sh_h16[tid] = (int16_t)best;
      __syncthreads();
      r = maxplus_packed<T>(sD + tid * DLD, sh_h16, best);
    } else {  // more than 32000 fronts: plain 32-bit max-plus over the same table
      sh_r1[tid] = best;
      __syncthreads();
      for (int a2 = 0; a2 < T; ++a2) {
        const int dl = (int)sD[tid * DLD + a2];
        r = (dl >= 0) ? max(r, sh_r1[a2] + dl) : r;
      }
    }
    __syncthreads();

    // ---- the predecessor block is the critical dependency.  Everything that does not depend on its ranks is done
    // first: its dominance pattern (pmask) and, from it, the table  E[s][i] = longest in-block continuation of a chain that
    // enters this block from predecessor point s and ends at i  (E = max_{a : s dominates a} D[a][i], SENT if none).
    // Once the ranks r1_s = rank_s + 1 arrive the resolution is a single max-plus product
    //     rank_i = max(Rb_i, max_s (r1_s + E[s][i])),
    // i.e. the critical path per block is: poll -> one barrier -> 128 independent loads / adds / maxes -> publish.
    if (b > 0) {
      const int k = b - 1;
      // ---- critical section starts here
      bool big;
      {
        const uint32_t* rw = rec + ((int64_t)k * T + tid) * W + M;
        uint32_t r1 = ld_relaxed_u32(rw);
        unsigned spins = 0;
        while (r1 == 0u) {
          r1 = ld_relaxed_u32(rw);
          if ((++spins & 0xFFFFu) == 0u && (spins > (1u << 24) || ld_relaxed_u32((const uint32_t*)errflag) != 0u)) {
            atomicExch(errflag, 1);
            break;
          }
        }
        sh_r1[tid] = (int)r1;
        sh_h16[tid] = (int16_t)r1;
        big = (int)r1 > PACK_LIMIT || r > PACK_LIMIT;
      }
      const int any_big = __syncthreads_or(big ? 1 : 0);
      if (!any_big) {
        r = maxplus_packed<T>(sE + tid * DLD, sh_h16, r);
      } else {
        for (int s2 = 0; s2 < T; ++s2) {
          const int e = (int)sE[tid * DLD + s2];
          r = (e >= 0) ? max(r, sh_r1[s2] + e) : r;
        }
      }
    }
    st_relaxed_u32(rec + i * W + M, (uint32_t)(r + 1));  // publish: the rank word doubles as the ready flag
    rankS[i] = r;
    if (SEG) {
      // staircase of this tile for the blocks of later segments (off the critical path: they are at least a segment
      // away): running maximum of rank + 1 in ascending order of the last compare word; key and value travel in one
      // 64-bit store, a non-zero value marks the entry as published
      __syncthreads();
      sh_r1[spos] = r + 1;
      __syncthreads();
      int val = sh_r1[tid];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xFFFFFFFFu, val, off);
        if ((tid & 31) >= off) val = max(val, o);
      }
      if ((tid & 31) == 31) sh_band[tid >> 5] = (uint32_t)val;
      __syncthreads();
      for (int w = 0; w < (tid >> 5); ++w) val = max(val, (int)sh_band[w]);
      st_relaxed_u64(sg.stair + i, ((unsigned long long)(uint32_t)val << 32) | (unsigned long long)skey[tid]);
    }
    __syncthreads();
  }
}

// Rank-0 test only (filter for the hypervolume / EHVI routines): "is some point dominating me" has no dependency chain,
// so it is the bulk scan alone, with a block-wide early exit once every target of the block has found a dominator.
template <int M, int T>
__global__ void __launch_bounds__(T) nd_flag_kernel(const uint32_t* __restrict__ rec, int nblocks, int* __restrict__ flagS) {
  constexpr int W = 4 * ((M + 1 + 3) / 4);
  constexpr int NV = W / 4;
  __shared__ uint4 tile[T * NV];
  const int tid = threadIdx.x;
  const int b = blockIdx.x;
  const int64_t i = (int64_t)b * T + tid;
  uint32_t v[W];
  {
    const uint4* src = reinterpret_cast<const uint4*>(rec + i * W);
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      uint4 a = src[q];
      v[4 * q + 0] = a.x;
      v[4 * q + 1] = a.y;
      v[4 * q + 2] = a.z;
      v[4 * q + 3] = a.w;
    }
  }
  const uint32_t gidv = v[M - 1];
  bool dominated = false;
  for (int k = 0; k <= b; ++k) {
    if (__syncthreads_and(dominated ? 1 : 0)) break;
    {
      const uint4* src = reinterpret_cast<const uint4*>(rec + (int64_t)k * T * W);
#pragma unroll
      for (int q = 0; q < NV; ++q) tile[tid * NV + q] = src[tid * NV + q];
    }
    __syncthreads();
    const int lim = (k == b) ? tid : T;  // inside the own block only earlier positions can dominate
#pragma unroll 8
    for (int s = 0; s < T; ++s) {
      uint32_t sw[W];
#pragma unroll
      for (int q = 0; q < NV; ++q) {
        uint4 a = tile[s * NV + q];
        sw[4 * q + 0] = a.x;
        sw[4 * q + 1] = a.y;
        sw[4 * q + 2] = a.z;
        sw[4 * q + 3] = a.w;
      }
      bool dom = (s < lim) && (sw[M - 1] != gidv);
#pragma unroll
      for (int j = 0; j < M - 1; ++j) dom = dom && (sw[j] <= v[j]);
      dominated = dominated || dom;
    }
  }
  flagS[i] = dominated ? 1 : 0;
}

template <int M>
int launch_nd_flags(dmo_ctx* ctx, const uint32_t* rec, int nblocks, int* flagS) {
  ProfileScope ps(ctx, "nd_flags");
  DMO_LAUNCH((nd_flag_kernel<M, RANK_T>), nblocks, RANK_T, 0, rec, nblocks, flagS);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

__global__ void scatter_rank_kernel(const int* __restrict__ rankS, const uint32_t* __restrict__ perm, int64_t n,
                                    int32_t* __restrict__ rank) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) rank[perm[p]] = rankS[p];
}

__global__ void copy_u32_to_i32_kernel(const uint32_t* __restrict__ a, int64_t n, int32_t* __restrict__ out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = (int32_t)a[p];
}

template <int M, bool SEG>
int launch_chain(dmo_ctx* ctx, uint32_t* rec, int nblocks, int* rankS, int* ticket, int* errflag, const RankSeg& sg) {
  constexpr int NV = (M + 1 + 3) / 4;
  const size_t dyn = NV > 4 ? (size_t)RANK_T * NV * sizeof(uint4) : 0;  // the kernel's DYN_TILE
  if (dyn > 0)
    DMO_CUDA(cudaFuncSetAttribute(rank_chain_kernel<M, RANK_T, SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  int occ = 0;
  DMO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rank_chain_kernel<M, RANK_T, SEG>, RANK_T, dyn));
  if (occ < 1) occ = 1;
  // fewer co-resident CTAs per SM shorten the serial chain (the block on the critical path shares its SM's issue
  // slots with the others); DMO_RANK_OCC overrides for tuning
  int cap = 6;
  if (const char* e = getenv("DMO_RANK_OCC")) cap = atoi(e);
  if (cap >= 1 && occ > cap) occ = cap;
  int nctas = nblocks < occ * ctx->sm_count ? nblocks : occ * ctx->sm_count;
  {
    ProfileScope ps(ctx, "rank_chain");
    DMO_LAUNCH((rank_chain_kernel<M, RANK_T, SEG>), nctas, RANK_T, dyn, rec, nblocks, rankS, ticket, errflag, sg);
    DMO_CHECK_LAUNCH();
  }
  return DMO_OK;
}

// f(std::integral_constant<int, M>()) for a runtime objective count M in 2 .. 16: one instantiation per count
template <int MC = 2, class F>
int dispatch_m(int M, F&& f) {
  if constexpr (MC < 16) {
    if (M != MC) return dispatch_m<MC + 1>(M, f);
  }
  return f(std::integral_constant<int, MC>());
}

int bits_for(int64_t n) {
  int b = 1;
  while (((int64_t)1 << b) < n) ++b;
  return b;
}

// ------------------------------------------------------------------------------------------------ cell grid (M <= 3)
// A G x G grid over the dense ids of objectives 2 and 3 answers most "does a living point dominate me" queries with one
// table lookup.  Inside a cell the records are ordered by their objective-1 id, so the first living record of a cell
// carries its smallest living id.  A point in a cell strictly below the target's cell in both objectives dominates it iff
// its objective-1 id is <= the target's, so those cells hold a dominator iff the exclusive 2-D prefix minimum of the
// per-cell minima is <= the target's id.  Only the points in the target's own cell row and cell column need the exact
// test; two cell-ordered copies of the records (row-major and column-major) make both of them contiguous streams.
// Two objectives lay the grid over objective 2 twice: only the diagonal cells fill.
// The rank-0 filter runs one such test with every point alive; front peeling (below) runs one per front.
constexpr uint32_t PEEL_DEAD = 0xFFFFFFFFu;  // objective-1 id of a dead record, minimum of an empty cell

// cell of a dense id: the ids of an objective run from 0 to maxid (its number of distinct values - 1), which can be far below
// n (quantised or heavily tied objectives); the shift follows maxid, so the grid stays populated evenly either way
__device__ __forceinline__ int cell_shift(uint32_t maxid, int gbits) {
  const int b = 32 - __clz(maxid | 1u);
  return b > gbits ? b - gbits : 0;
}

// the three id columns a grid compares, and the largest ids of the two it is laid over (device pointers)
struct GridIds {
  const uint32_t *c0, *c1, *c2;
  const uint32_t *max1, *max2;
};

GridIds grid_ids(const uint32_t* R, const uint32_t* maxid, int64_t n, int M) {
  const int j2 = M == 3 ? 2 : 1;
  return GridIds{R, R + n, R + (size_t)j2 * n, maxid + 1, maxid + j2};
}

struct CellGrid {
  int gbits = 0;
  DevBuf<uint32_t> cstartA, cstartB;     // [G*G + 1] first slot of every cell in the row-major / column-major copy
  DevBuf<uint4> crecA, crecB;            // [n] (objective-1, -2, -3 id, row) in cell order
  DevBuf<uint32_t> pm;                   // [G*G] per-cell minimum of the living objective-1 ids, then its prefix minimum
  DevBuf<uint32_t> first, slotA, slotB;  // peeling only: first living slot of every cell, slot of every row per copy
};

__global__ void grid_key_kernel(GridIds ids, int64_t n, int gbits, uint32_t* __restrict__ key0, uint32_t* __restrict__ keyA,
                                uint32_t* __restrict__ keyB) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t G1 = (1u << gbits) - 1u;
  const uint32_t a = min(ids.c1[i] >> cell_shift(*ids.max1, gbits), G1), b = min(ids.c2[i] >> cell_shift(*ids.max2, gbits), G1);
  key0[i] = ids.c0[i];
  keyA[i] = (a << gbits) | b;
  keyB[i] = (b << gbits) | a;
}

// cell-ordered copy (ids of the three objectives, row) and, when peeling, the slot of every row in it
__global__ void grid_gather_kernel(GridIds ids, const uint32_t* __restrict__ order, int64_t n, uint4* __restrict__ crec,
                                   uint32_t* __restrict__ slot) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t i = order[t];
  crec[t] = make_uint4(ids.c0[i], ids.c1[i], ids.c2[i], i);
  if (slot != nullptr) slot[i] = (uint32_t)t;
}

// cstart[c] = first slot whose key is >= c, c = 0 .. ncell (lower bounds over the sorted keys)
__global__ void grid_start_kernel(const uint32_t* __restrict__ skey, int64_t n, int ncell, uint32_t* __restrict__ cstart) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > ncell) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (skey[mid] < (uint32_t)c) lo = mid + 1; else hi = mid;
  }
  cstart[c] = (uint32_t)lo;
}

// smallest living objective-1 id of every cell.  Peeling keeps a pointer to each cell's first living record, which only
// ever moves forward; without one (first == nullptr: every record lives) a cell's first record is its smallest.
__global__ void grid_cellmin_kernel(const uint32_t* __restrict__ cstart, const uint4* __restrict__ crec, int ncell,
                                    uint32_t* __restrict__ first, uint32_t* __restrict__ pm) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncell) return;
  uint32_t f = first != nullptr ? first[c] : cstart[c];
  const uint32_t e = cstart[c + 1];
  while (f < e && crec[f].x == PEEL_DEAD) ++f;
  if (first != nullptr) first[c] = f;
  pm[c] = f < e ? crec[f].x : PEEL_DEAD;
}

// in-place inclusive prefix minimum: pass 0 along each row of the G x G table, pass 1 along each column
__global__ void grid_prefix_min_kernel(uint32_t* __restrict__ pm, int gbits, int pass) {
  extern __shared__ uint32_t sh_scan[];
  const int G = 1 << gbits;
  const int line = blockIdx.x, t = threadIdx.x;
  const int cell = pass == 0 ? line * G + t : t * G + line;
  uint32_t v = pm[cell];
  sh_scan[t] = v;
  __syncthreads();
  for (int off = 1; off < G; off <<= 1) {
    const uint32_t o = t >= off ? sh_scan[t - off] : PEEL_DEAD;
    __syncthreads();
    v = min(v, o);
    sh_scan[t] = v;
    __syncthreads();
  }
  pm[cell] = v;
}

// dom[i] = 1 iff a living point dominates the living point i (alive == nullptr: every point lives)
template <typename OutT>
__global__ void grid_flag_kernel(GridIds ids, int64_t n, int gbits, const uint32_t* __restrict__ pm,
                                 const uint32_t* __restrict__ cstartA, const uint32_t* __restrict__ cstartB,
                                 const uint4* __restrict__ crecA, const uint4* __restrict__ crecB,
                                 const uint8_t* __restrict__ alive, OutT* __restrict__ dom_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (alive != nullptr && !alive[i])) return;
  const int G = 1 << gbits;
  const uint32_t c0 = ids.c0[i], c1 = ids.c1[i], c2 = ids.c2[i];
  const int a = (int)min(c1 >> cell_shift(*ids.max1, gbits), (uint32_t)(G - 1));
  const int b = (int)min(c2 >> cell_shift(*ids.max2, gbits), (uint32_t)(G - 1));
  // cells strictly below in both words hold different vectors: "<=" on the first objective is enough there
  bool dom = a > 0 && b > 0 && __ldg(pm + (a - 1) * G + (b - 1)) <= c0;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    if (dom) break;
    const uint4* cr = pass == 0 ? crecA : crecB;
    uint32_t t = pass == 0 ? __ldg(cstartA + a * G) : __ldg(cstartB + b * G);
    const uint32_t t1 = pass == 0 ? __ldg(cstartA + a * G + b + 1) : __ldg(cstartB + b * G + a);
    // a dead record carries PEEL_DEAD as its first id and fails the first compare
#define DMO_PEEL_TEST(q) ((q).x <= c0 && (q).y <= c1 && (q).z <= c2 && !((q).x == c0 && (q).y == c1 && (q).z == c2))
    // the few threads that get here walk hundreds of records: sixteen loads in flight per step (ncu: 9 % of the issue slots
    // busy with four, the kernel's time is the dependent-load latency of its longest walks)
    for (; t + 16 <= t1 && !dom; t += 16) {
      uint4 q[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) q[u] = __ldg(cr + t + u);
#pragma unroll
      for (int u = 0; u < 16; ++u) dom = dom || DMO_PEEL_TEST(q[u]);
    }
    for (; t + 4 <= t1 && !dom; t += 4) {
      const uint4 q0 = __ldg(cr + t), q1 = __ldg(cr + t + 1), q2 = __ldg(cr + t + 2), q3 = __ldg(cr + t + 3);
      dom = DMO_PEEL_TEST(q0) || DMO_PEEL_TEST(q1) || DMO_PEEL_TEST(q2) || DMO_PEEL_TEST(q3);
    }
    for (; t < t1 && !dom; ++t) {
      const uint4 q0 = __ldg(cr + t);
      dom = DMO_PEEL_TEST(q0);
    }
#undef DMO_PEEL_TEST
  }
  dom_out[i] = (OutT)(dom ? 1 : 0);
}

// Sorted by objective-1 id, then stably by cell for each copy, so that inside a cell the records ascend in that id.
int build_cell_grid(dmo_ctx* ctx, const GridIds& ids, int64_t n, int gbits, bool peel, CellGrid& cg) {
  cg.gbits = gbits;
  const int GG = 1 << (2 * gbits);
  const unsigned g = (unsigned)ceil_div(n, 256);
  DevBuf<uint32_t> key0, keyA, keyB, keyS[2], keyT[2], ord0, ordS[2], iota;
  DMO_TRY(key0.alloc(ctx, n));
  DMO_TRY(keyA.alloc(ctx, n));
  DMO_TRY(keyB.alloc(ctx, n));
  for (int pass = 0; pass < 2; ++pass) {
    DMO_TRY(keyS[pass].alloc(ctx, n));
    DMO_TRY(keyT[pass].alloc(ctx, n));
    DMO_TRY(ordS[pass].alloc(ctx, n));
  }
  DMO_TRY(ord0.alloc(ctx, n));
  DMO_TRY(iota.alloc(ctx, n));
  DMO_TRY(cg.cstartA.alloc(ctx, GG + 1));
  DMO_TRY(cg.cstartB.alloc(ctx, GG + 1));
  DMO_TRY(cg.crecA.alloc(ctx, n));
  DMO_TRY(cg.crecB.alloc(ctx, n));
  DMO_TRY(cg.pm.alloc(ctx, GG));
  if (peel) {
    DMO_TRY(cg.first.alloc(ctx, GG));
    DMO_TRY(cg.slotA.alloc(ctx, n));
    DMO_TRY(cg.slotB.alloc(ctx, n));
  }
  DMO_LAUNCH(grid_key_kernel, g, 256, 0, ids, n, gbits, key0.p, keyA.p, keyB.p);
  DMO_TRY(prim_iota_u32(ctx, iota.p, n));
  DMO_TRY(prim_sort_pairs_u32(ctx, key0.p, keyS[0].p, iota.p, ord0.p, n, 0, bits_for(n)));  // by objective-1 id ...
  {  // ... then stably by cell, the two copies side by side
    SideStreams side(ctx, 2);
    DMO_TRY(side.rc);
    for (int pass = 0; pass < 2; ++pass) {
      side.on(pass);
      DMO_TRY(prim_gather_u32(ctx, pass == 0 ? keyA.p : keyB.p, ord0.p, n, keyT[pass].p));
      DMO_TRY(prim_sort_pairs_u32(ctx, keyT[pass].p, keyS[pass].p, ord0.p, ordS[pass].p, n, 0, 2 * gbits));
      DMO_LAUNCH(grid_gather_kernel, g, 256, 0, ids, ordS[pass].p, n, pass == 0 ? cg.crecA.p : cg.crecB.p,
                 pass == 0 ? cg.slotA.p : cg.slotB.p);
      DMO_LAUNCH(grid_start_kernel, (unsigned)ceil_div(GG + 1, 256), 256, 0, keyS[pass].p, n, GG,
                 pass == 0 ? cg.cstartA.p : cg.cstartB.p);
    }
    side.back();
  }
  if (peel) DMO_CUDA(cudaMemcpyAsync(cg.first.p, cg.cstartA.p, (size_t)GG * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// dom[i] = 1 iff a living point dominates the living point i: per-cell minima, their 2-D prefix minimum, one flag pass
template <typename OutT>
int grid_dominated(dmo_ctx* ctx, CellGrid& cg, const GridIds& ids, int64_t n, const uint8_t* alive, OutT* dom) {
  const int G = 1 << cg.gbits, GG = G * G;
  DMO_LAUNCH(grid_cellmin_kernel, (unsigned)ceil_div(GG, 256), 256, 0, cg.cstartA.p, cg.crecA.p, GG, cg.first.p, cg.pm.p);
  DMO_LAUNCH(grid_prefix_min_kernel, G, G, G * sizeof(uint32_t), cg.pm.p, cg.gbits, 0);
  DMO_LAUNCH(grid_prefix_min_kernel, G, G, G * sizeof(uint32_t), cg.pm.p, cg.gbits, 1);
  DMO_LAUNCH((grid_flag_kernel<OutT>), (unsigned)ceil_div(n, 128), 128, 0, ids, n, cg.gbits, cg.pm.p, cg.cstartA.p, cg.cstartB.p,
             cg.crecA.p, cg.crecB.p, alive, dom);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// flag[i] = 1 iff some row dominates row i (M <= 3), written in row order
int nd_flags_cell_grid(dmo_ctx* ctx, const uint32_t* R, const uint32_t* maxid, int64_t n, int M, int32_t* d_flag01) {
  int gbits = bits_for(n) / 2;
  if (gbits < 4) gbits = 4;
  if (gbits > 9) gbits = 9;
  const GridIds ids = grid_ids(R, maxid, n, M);
  CellGrid cg;
  ProfileScope ps(ctx, "nd_flags");
  DMO_TRY(build_cell_grid(ctx, ids, n, gbits, false, cg));
  return grid_dominated(ctx, cg, ids, n, nullptr, d_flag01);
}

// ------------------------------------------------------------------------------------------------ front peeling (M == 3)
// A truncation (remove_worst: keep the best `keep` of n rows) needs the ranks of the kept rows only.  When those rows span
// few fronts -- a converging population: the bench's merged sets put the best 65 536 of 131 072 points into 7 fronts, a
// sphere-shaped set into 2 -- peeling them one by one is cheaper than the chain, whose 1024 links are serial whatever the
// data looks like.  Front k = the points of the remaining set that no remaining point dominates, found on the cell grid
// above, built once:
//   * per peel: the grid's test over the living points, then the new front is marked: rank written, its records in both
//     cell-ordered copies overwritten with an id that dominates nothing;
//   * the loop stops once `keep` rows are ranked (the others get the next rank: they are truncated away), or gives up
//     when the fronts turn out to be small (many peels ahead): the chain then runs as if nothing had happened.

// the living points nobody dominates form front k: rank, death, count
__global__ void peel_mark_kernel(int64_t n, uint8_t* __restrict__ alive, const uint8_t* __restrict__ dom, int k,
                                 int32_t* __restrict__ rank, const uint32_t* __restrict__ slotA, const uint32_t* __restrict__ slotB,
                                 uint4* __restrict__ crecA, uint4* __restrict__ crecB, unsigned long long* __restrict__ count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool mine = false;
  if (i < n && alive[i] && !dom[i]) {
    mine = true;
    rank[i] = k;
    alive[i] = 0;
    crecA[slotA[i]].x = PEEL_DEAD;
    crecB[slotB[i]].x = PEEL_DEAD;
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, mine);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (unsigned long long)__popc(m));
}

__global__ void peel_rest_kernel(int64_t n, const uint8_t* __restrict__ alive, int k, int32_t* __restrict__ rank) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && alive[i]) rank[i] = k;
}

// Is the first front worth peeling?  PEEL_PROBE evenly spaced points are tested against the whole set (every thread brings
// one point and runs it past the probes in shared memory); a probe that nobody dominates stands for n / PEEL_PROBE points of
// front 0.  A uniform cloud (front 0 = 0.05 % of the set) almost never passes, a converging population always does.
constexpr int PEEL_PROBE = 256;
__global__ void peel_probe_kernel(const uint32_t* __restrict__ R, int64_t n, unsigned* __restrict__ dominated) {
  __shared__ uint32_t sp[PEEL_PROBE][3];
  __shared__ unsigned sdom[PEEL_PROBE / 32];
  const int64_t stride = n / PEEL_PROBE;
  for (int t = threadIdx.x; t < PEEL_PROBE; t += blockDim.x) {
    const int64_t i = (int64_t)t * stride + (stride >> 1);
    sp[t][0] = R[i];
    sp[t][1] = R[n + i];
    sp[t][2] = R[2 * n + i];
  }
  if (threadIdx.x < PEEL_PROBE / 32) sdom[threadIdx.x] = 0u;
  __syncthreads();
  unsigned mine[PEEL_PROBE / 32];
#pragma unroll
  for (int w = 0; w < PEEL_PROBE / 32; ++w) mine[w] = 0u;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t a = R[j], b = R[n + j], c = R[2 * n + j];
#pragma unroll
    for (int w = 0; w < PEEL_PROBE / 32; ++w) {
      unsigned m = 0u;
#pragma unroll 8
      for (int t = 0; t < 32; ++t) {
        const uint32_t pa = sp[w * 32 + t][0], pb = sp[w * 32 + t][1], pc = sp[w * 32 + t][2];
        const bool d = a <= pa && b <= pb && c <= pc && !(a == pa && b == pb && c == pc);
        m |= d ? (1u << t) : 0u;
      }
      mine[w] |= m;
    }
  }
#pragma unroll
  for (int w = 0; w < PEEL_PROBE / 32; ++w) {
    const unsigned m = __reduce_or_sync(0xFFFFFFFFu, mine[w]);
    if ((threadIdx.x & 31) == 0 && m) atomicOr(&sdom[w], m);
  }
  __syncthreads();
  if (threadIdx.x < PEEL_PROBE / 32 && sdom[threadIdx.x]) atomicOr(&dominated[threadIdx.x], sdom[threadIdx.x]);
}

__global__ void fill_u8_kernel(uint8_t* __restrict__ a, int64_t n, uint8_t v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// *done = true: d_rank holds exact ranks for (at least) the best `keep` rows, a common larger rank for the rest
int rank_by_peeling(dmo_ctx* ctx, const uint32_t* R, const uint32_t* maxid, int64_t n, int64_t keep, int32_t* d_rank, bool* done) {
  *done = false;
  int max_peels = 14;  // the chain costs about as much as 20 peels plus the grid
  if (const char* e = getenv("DMO_RANK_PEEL")) max_peels = atoi(e);
  if (max_peels <= 0) return DMO_OK;
  ProfileScope ps(ctx, "rank_peel");
  double front_guess;  // the expected size of the front the host reads next: from the probe for front 0
  {  // probe before building anything: fewer than two undominated probes = a first front below ~1 % of the set
    DevBuf<unsigned> pd;
    DMO_TRY(pd.alloc(ctx, PEEL_PROBE / 32));
    DMO_CUDA(cudaMemsetAsync(pd.p, 0, (PEEL_PROBE / 32) * sizeof(unsigned), ctx->stream));
    const int gridp = (int)(ceil_div(n, 256) < 2 * (int64_t)ctx->sm_count ? ceil_div(n, 256) : 2 * (int64_t)ctx->sm_count);
    DMO_LAUNCH(peel_probe_kernel, gridp, 256, 0, R, n, pd.p);
    DMO_CHECK_LAUNCH();
    unsigned h[PEEL_PROBE / 32];
    DMO_CUDA(cudaMemcpyAsync(h, pd.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(dmo_wait(ctx));
    int free_probes = PEEL_PROBE;
    for (int w = 0; w < PEEL_PROBE / 32; ++w) free_probes -= __builtin_popcount(h[w]);
    if (free_probes < 2 && !(getenv("DMO_RANK_PEEL_NOPROBE") && atoi(getenv("DMO_RANK_PEEL_NOPROBE")))) return DMO_OK;
    front_guess = (double)free_probes * (double)n / PEEL_PROBE;
  }
  const int bits = bits_for(n);
  int gbits = (bits + 1) / 2;  // two cells per point at n = 131 072: measured 0.80 ms per bench step against 0.96 ms with 2^8 cells per axis
  if (gbits < 4) gbits = 4;
  if (const char* e = getenv("DMO_PEEL_GBITS")) gbits = atoi(e);
  if (gbits > 9) gbits = 9;
  const unsigned g = (unsigned)ceil_div(n, 256);
  const GridIds ids = grid_ids(R, maxid, n, 3);
  CellGrid cg;
  DMO_TRY(build_cell_grid(ctx, ids, n, gbits, true, cg));
  DevBuf<uint8_t> alive, dom;
  DevBuf<unsigned long long> count;
  DMO_TRY(alive.alloc(ctx, n));
  DMO_TRY(dom.alloc(ctx, n));
  DMO_TRY(count.alloc(ctx, 1));
  DMO_LAUNCH(fill_u8_kernel, g, 256, 0, alive.p, n, (uint8_t)1);
  DMO_CUDA(cudaMemsetAsync(count.p, 0, sizeof(unsigned long long), ctx->stream));
  DMO_TRY(dmo_lag_slots(ctx));
  // peel front j; the running count of ranked rows lands in lag_host[j & 1], lag_ev[j & 1] marks it
  auto peel = [&](int j) -> int {
    DMO_TRY(grid_dominated(ctx, cg, ids, n, alive.p, dom.p));
    DMO_LAUNCH(peel_mark_kernel, g, 256, 0, n, alive.p, dom.p, j, d_rank, cg.slotA.p, cg.slotB.p, cg.crecA.p, cg.crecB.p, count.p);
    DMO_CHECK_LAUNCH();
    DMO_CUDA(cudaMemcpyAsync(ctx->lag_host + (j & 1), count.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    DMO_CUDA(cudaEventRecord(ctx->lag_ev[j & 1], ctx->stream));
    return DMO_OK;
  };
  // When front k is not expected to complete the `keep` rows (nor, for the first front, to be small enough to give up on),
  // front k + 1 is enqueued before the host reads front k's count, so the GPU peels while the host waits and decides.  A guess that turns out
  // wrong changes no kept rank: if front k completes the `keep` rows, peel k + 1 ranks k + 1 rows peel_rest_kernel would
  // rank k + 1 anyway; if the forecast gives up, the chain overwrites every rank.  It costs one peel, which is why the
  // last front is not guessed past.
  unsigned long long ranked = 0, before = 0;
  double prev_front = 0.0;
  int k = 0, queued = 1;
  DMO_TRY(peel(0));
  for (;; ++k) {
    if (queued == k + 1 && (double)ranked + front_guess < (double)keep && (k > 0 || front_guess * 64.0 >= (double)keep)) {
      DMO_TRY(peel(k + 1));
      ++queued;
    }
    before = ranked;
    ctx->waits++;
    DMO_CUDA(cudaEventSynchronize(ctx->lag_ev[k & 1]));
    ranked = ctx->lag_host[k & 1];
    if ((int64_t)ranked >= keep || (int64_t)ranked >= n) break;
    // Give up when many peels are still ahead.  Fronts usually grow over the first few peels (the bench's sets: 2.4 k,
    // then 5 - 12 k points per front), so the forecast extrapolates the last two front sizes linearly, and the first
    // front only decides when it is tiny (a uniform cloud: 72 of 131 072 points).
    const double last = (double)(ranked - before);
    const double grow = last > prev_front ? last - prev_front : 0.0;
    bool give_up;
    if (k == 0) {
      give_up = last * 64.0 < (double)keep;
    } else {
      const double rem = (double)(keep - (int64_t)ranked);
      const double b = last + 0.5 * grow;
      const double ahead = grow > 0.0 ? (-b + sqrt(b * b + 2.0 * grow * rem)) / grow : rem / (last > 0.0 ? last : 1.0);
      give_up = (double)(k + 1) + ahead > (double)max_peels;
    }
    if (give_up) return DMO_OK;  // *done stays false: the chain takes over
    prev_front = last;
    front_guess = last + grow;
    if (queued == k + 1) {
      DMO_TRY(peel(k + 1));
      ++queued;
    }
  }
  DMO_LAUNCH(peel_rest_kernel, g, 256, 0, n, alive.p, k + 1, d_rank);
  DMO_CHECK_LAUNCH();
  *done = true;
  return DMO_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ stages of the rank
// 1. R[j * n + i] = dense id of Y[i, j] (order- and equality-preserving), maxid[j] = largest id of objective j
int dense_ids(dmo_ctx* ctx, const double* dY, int64_t n, int M, DevBuf<uint32_t>& R, DevBuf<uint32_t>& maxid) {
  DMO_REQUIRE(M >= 1 && M <= 16, "rank_nd: M=%d out of range [1,16]", M);
  DMO_REQUIRE(n < ((int64_t)1 << 31) - 4096, "rank_nd: n too large");
  const unsigned g = (unsigned)ceil_div(n, 256);
  DMO_TRY(R.alloc(ctx, (size_t)M * n));
  DMO_TRY(maxid.alloc(ctx, M));
  // the objectives are independent: each sorts on a side stream of its own (up to four at a time), so the latency-bound
  // radix passes of the columns overlap instead of queueing one column behind the other
  const int ns = M < dmo_ctx::kSide ? M : dmo_ctx::kSide;
  DevBuf<uint64_t> k0[dmo_ctx::kSide], k1[dmo_ctx::kSide];
  DevBuf<uint32_t> i0[dmo_ctx::kSide], i1[dmo_ctx::kSide], flag[dmo_ctx::kSide], dense[dmo_ctx::kSide];
  for (int s = 0; s < ns; ++s) {
    DMO_TRY(k0[s].alloc(ctx, n));
    DMO_TRY(k1[s].alloc(ctx, n));
    DMO_TRY(i0[s].alloc(ctx, n));
    DMO_TRY(i1[s].alloc(ctx, n));
    DMO_TRY(flag[s].alloc(ctx, n));
    DMO_TRY(dense[s].alloc(ctx, n));
  }
  SideStreams side(ctx, ns);
  DMO_TRY(side.rc);
  for (int j = 0; j < M; ++j) {
    const int s = j % ns;
    side.on(s);
    DMO_TRY(prim_col_keys(ctx, dY, n, M, j, k0[s].p, i0[s].p));
    DMO_TRY(prim_sort_pairs_u64(ctx, k0[s].p, k1[s].p, i0[s].p, i1[s].p, n, 0, 64));
    DMO_LAUNCH(flag_new_u64_kernel, g, 256, 0, k1[s].p, n, flag[s].p);
    DMO_TRY(prim_inclusive_sum_u32(ctx, flag[s].p, dense[s].p, n));
    DMO_LAUNCH(scatter_dense_kernel, g, 256, 0, dense[s].p, i1[s].p, n, R.p + (size_t)j * n);
    DMO_CUDA(cudaMemcpyAsync(maxid.p + j, dense[s].p + (n - 1), sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  }
  side.back();
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// 2. An order of the points in which a point can only be dominated by points before it.  sshift == 0: lexicographic
//    order (LSD passes, least significant objective first); sshift > 0: the segmented order of RankSeg, key =
//    (objective-1 id >> sshift, objective 2, ..., objective M, objective 1).  The passes are stable and start from row
//    order, so identical vectors stay in ascending row order.  *perm (position -> row) points into permA or permB.
int lex_order(dmo_ctx* ctx, const uint32_t* R, int64_t n, int M, int sshift, DevBuf<uint32_t>& permA, DevBuf<uint32_t>& permB,
              const uint32_t** perm) {
  const int bits = bits_for(n);
  const unsigned g = (unsigned)ceil_div(n, 256);
  DevBuf<uint32_t> keyA, keyB;
  DMO_TRY(permA.alloc(ctx, n));
  DMO_TRY(permB.alloc(ctx, n));
  DMO_TRY(keyA.alloc(ctx, n));
  DMO_TRY(keyB.alloc(ctx, n));
  DMO_TRY(prim_iota_u32(ctx, permA.p, n));
  uint32_t* pin = permA.p;
  uint32_t* pout = permB.p;
  auto sort_pass = [&](const uint32_t* col, int shift, int nbits) -> int {
    if (shift == 0) {
      DMO_TRY(prim_gather_u32(ctx, col, pin, n, keyA.p));
    } else {
      DMO_LAUNCH(seg_key_kernel, g, 256, 0, col, pin, n, shift, keyA.p);
    }
    DMO_TRY(prim_sort_pairs_u32(ctx, keyA.p, keyB.p, pin, pout, n, 0, nbits));
    uint32_t* t = pin;
    pin = pout;
    pout = t;
    return DMO_OK;
  };
  if (sshift > 0) {
    DMO_TRY(sort_pass(R, 0, bits));  // least significant: objective 1 itself
    for (int j = M - 1; j >= 1; --j) DMO_TRY(sort_pass(R + (size_t)j * n, 0, bits));
    DMO_TRY(sort_pass(R, sshift, bits - sshift));  // most significant: the segment
  } else {
    for (int j = M - 1; j >= 0; --j) DMO_TRY(sort_pass(R + (size_t)j * n, 0, bits));
  }
  *perm = pin;
  return DMO_OK;
}

namespace {

// The order of lex_order, the group ids of identical vectors, and the chain's padded records in that order.
struct RankOrder {
  DevBuf<uint32_t> permA, permB, rec;
  const uint32_t* perm = nullptr;  // position -> row
  int64_t nblocks = 0, npad = 0;
};

int rank_order(dmo_ctx* ctx, const uint32_t* R, int64_t n, int M, int sshift, RankOrder& o) {
  const unsigned g = (unsigned)ceil_div(n, 256);
  DMO_TRY(lex_order(ctx, R, n, M, sshift, o.permA, o.permB, &o.perm));

  // group ids (identical vectors share one)
  DevBuf<uint32_t> flag, gid;
  DMO_TRY(flag.alloc(ctx, n));
  DMO_TRY(gid.alloc(ctx, n));
  DMO_LAUNCH(flag_new_vec_kernel, g, 256, 0, R, o.perm, n, M, flag.p);
  DMO_TRY(prim_inclusive_sum_u32(ctx, flag.p, gid.p, n));

  const int W = 4 * ((M + 1 + 3) / 4);
  o.nblocks = ceil_div(n, RANK_T);
  o.npad = o.nblocks * RANK_T;
  DMO_TRY(o.rec.alloc(ctx, (size_t)o.npad * W));
  DMO_LAUNCH(build_records_kernel, (unsigned)ceil_div(o.npad, 256), 256, 0, R, o.perm, gid.p, n, o.npad, M, W, o.rec.p);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// segment shift of the chain's order: two and three objectives take the segmented order (RankSeg) from 16 to
// RANK_SEG_MAXT blocks, everything else the plain lexicographic order (0)
int seg_shift(int64_t n, int M) {
  const int bits = bits_for(n);
  int segbits = bits - 10;  // segments of 1024 dense ids of objective 1 (8 blocks), at most 128 segments
  if (segbits > 7) segbits = 7;
  if (const char* e = getenv("DMO_RANK_SEGBITS")) segbits = atoi(e);
  if (segbits < 1) segbits = 1;
  const int64_t nblocks = ceil_div(n, RANK_T);
  const bool seg = M <= 3 && nblocks >= 16 && nblocks <= RANK_SEG_MAXT && bits > segbits + 7 && getenv("DMO_RANK_NOSEG") == nullptr;
  return seg ? bits - segbits : 0;
}

// 3. the chain kernel over the records of `o`, ranks scattered back to row order
int rank_chain(dmo_ctx* ctx, const uint32_t* R, int64_t n, int M, int sshift, RankOrder& o, int32_t* d_rank) {
  const int nblocks = (int)o.nblocks;
  DevBuf<int> rankS, sync;
  DMO_TRY(rankS.alloc(ctx, o.npad));
  DMO_TRY(sync.alloc(ctx, nblocks + 2));
  DMO_CUDA(cudaMemsetAsync(sync.p, 0, (nblocks + 2) * sizeof(int), ctx->stream));
  int* ticket = sync.p + nblocks;
  int* errflag = sync.p + nblocks + 1;
  RankSeg sg;
  DevBuf<uint32_t> c1rec, seg_start;
  DevBuf<uint16_t> tile_q;
  DevBuf<unsigned long long> stair;
  if (sshift > 0) {
    const int bits = bits_for(n);
    DMO_TRY(stair.alloc(ctx, o.npad));
    DMO_CUDA(cudaMemsetAsync(stair.p, 0, (size_t)o.npad * sizeof(unsigned long long), ctx->stream));
    const int nseg = (int)(((uint32_t)(n - 1)) >> sshift) + 1;
    int qshift = bits - 8;
    if (qshift < 0) qshift = 0;
    DMO_TRY(c1rec.alloc(ctx, o.npad));
    DMO_TRY(seg_start.alloc(ctx, nseg + 1));
    DMO_TRY(tile_q.alloc(ctx, nblocks));
    DMO_LAUNCH(seg_c1_kernel, (unsigned)ceil_div(o.npad, 256), 256, 0, R, o.perm, n, o.npad, c1rec.p);
    DMO_LAUNCH(seg_start_kernel, (unsigned)ceil_div(nseg + 1, 128), 128, 0, c1rec.p, n, sshift, nseg, seg_start.p);
    DMO_LAUNCH(seg_tile_band_kernel, (unsigned)ceil_div(o.nblocks * 32, 256), 256, 0, o.rec.p, nblocks, RANK_T, qshift, tile_q.p);
    DMO_CHECK_LAUNCH();
    sg.c1rec = c1rec.p;
    sg.seg_start = seg_start.p;
    sg.tile_q = tile_q.p;
    sg.stair = stair.p;
    sg.sshift = sshift;
    sg.qshift = qshift;
    if (M == 2) {
      DMO_TRY((launch_chain<2, true>(ctx, o.rec.p, nblocks, rankS.p, ticket, errflag, sg)));
    } else {
      DMO_TRY((launch_chain<3, true>(ctx, o.rec.p, nblocks, rankS.p, ticket, errflag, sg)));
    }
  } else {
    DMO_TRY(dispatch_m(M, [&](auto m) {
      return launch_chain<decltype(m)::value, false>(ctx, o.rec.p, nblocks, rankS.p, ticket, errflag, sg);
    }));
  }
  DMO_LAUNCH(scatter_rank_kernel, (unsigned)ceil_div(n, 256), 256, 0, rankS.p, o.perm, n, d_rank);
  DMO_CHECK_LAUNCH();
  int herr = 0;
  DMO_CUDA(cudaMemcpyAsync(&herr, errflag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  if (herr) return dmo_fail(ctx, DMO_ERR_INTERNAL, "rank_nd: chain kernel watchdog tripped");
  return DMO_OK;
}

}  // namespace

// ranks that are exact for (at least) the `keep` best rows; the other rows share one larger value (see rank_by_peeling)
int rank_nd_device_keep(dmo_ctx* ctx, const double* dY, int64_t n, int M, int64_t keep, int32_t* d_rank) {
  if (n <= 0) return DMO_OK;
  DevBuf<uint32_t> R, maxid;
  DMO_TRY(dense_ids(ctx, dY, n, M, R, maxid));
  if (M == 1) {  // the dense id is the rank
    DMO_LAUNCH(copy_u32_to_i32_kernel, (unsigned)ceil_div(n, 256), 256, 0, R.p, n, d_rank);
    DMO_CHECK_LAUNCH();
    return DMO_OK;
  }
  if (M == 3 && keep > 0 && n >= 8192 && 4 * keep <= 3 * n) {  // truncation: the best `keep` rows are enough
    bool done = false;
    DMO_TRY(rank_by_peeling(ctx, R.p, maxid.p, n, keep, d_rank, &done));
    if (done) return DMO_OK;
  }
  const int sshift = seg_shift(n, M);
  RankOrder o;
  DMO_TRY(rank_order(ctx, R.p, n, M, sshift, o));
  return rank_chain(ctx, R.p, n, M, sshift, o, d_rank);
}

int rank_nd_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, int32_t* d_rank) {
  return rank_nd_device_keep(ctx, dY, n, M, 0, d_rank);
}

int nondominated_flags_device(dmo_ctx* ctx, const double* dY, int64_t n, int M, int32_t* d_flag01) {
  if (n <= 0) return DMO_OK;
  if (M == 1) return rank_nd_device(ctx, dY, n, M, d_flag01);  // the rank itself: 0 exactly for the rank-0 rows
  DevBuf<uint32_t> R, maxid;
  DMO_TRY(dense_ids(ctx, dY, n, M, R, maxid));
  if (M <= 3 && n >= 8192 && getenv("DMO_ND_BRUTE") == nullptr) return nd_flags_cell_grid(ctx, R.p, maxid.p, n, M, d_flag01);
  RankOrder o;  // the block scan over the lexicographic records
  DMO_TRY(rank_order(ctx, R.p, n, M, 0, o));
  DevBuf<int> flagS;
  DMO_TRY(flagS.alloc(ctx, o.npad));
  DMO_TRY(dispatch_m(M, [&](auto m) { return launch_nd_flags<decltype(m)::value>(ctx, o.rec.p, (int)o.nblocks, flagS.p); }));
  DMO_LAUNCH(scatter_rank_kernel, (unsigned)ceil_div(n, 256), 256, 0, flagS.p, o.perm, n, d_flag01);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

extern "C" int dmo_rank_nd(dmo_ctx* ctx, const double* Y, int64_t n, int M, int32_t* rank) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  DMO_REQUIRE(n >= 0 && M >= 1, "rank_nd: bad shape n=%lld M=%d", (long long)n, M);
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(Y && rank, "rank_nd: null pointer");
  In<double> y;
  Out<int32_t> r;
  DMO_TRY(y.init(ctx, Y, (size_t)n * M));
  DMO_TRY(r.init(ctx, rank, (size_t)n));
  DMO_TRY(rank_nd_device(ctx, y.d, n, M, r.d));
  DMO_TRY(r.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}
