// GP posterior variance on the Hopper tensor cores (DMO_GP_TENSOR, and the fast leg of DMO_GP_AUTO).
//
//   ||L^-1 K_*^T||^2 per candidate  ==  row sums of  D^2,   D[p][i] = sum_k K_*[p][k] * Linv[i][k]
//
// D is a dense (candidates x N_train) x N_train contraction, both operands k-contiguous ("TN").  It runs as warpgroup
// MMAs (wgmma.mma_async m64n256k16, fp16 inputs, fp32 accumulators in registers):
//   * split precision: every float operand x is carried as two fp16 numbers hi + lo (22 significand bits) after an
//     exact power-of-two scaling (per Linv row, per objective for K_*) that keeps both halves in fp16's normal range;
//     D accumulates hi*hi + hi*lo + lo*hi in fp32 (three MMAs per product, the lo*lo term is below fp32 resolution);
//   * a work item is 128 candidates (two consumer warpgroups x 64 rows) against 256-row blocks of Linv; each thread's
//     accumulators hold two candidate rows, so the epilogue's sum of squares is per thread plus a reduction over the
//     four lanes that share a row;
//   * Linv is lower triangular: the row block [256 j, 256 j + 256) only needs k < 256 (j + 1) -- half the MMAs skipped;
//   * operand tiles arrive by TMA (cp.async.bulk.tensor, SWIZZLE_64B) into a 4-stage shared-memory ring, completion on
//     mbarriers; one producer warp issues the loads, each consumer warp releases a slot once its MMAs have read it;
//   * persistent CTAs (one per SM) walk a list of equal-cost work items in an L2-friendly order (see below).
//
// K_* itself is produced in fp32 (relative error ~1e-6 on K_*) by kstar_mean_kernel, which accumulates the mean from the same
// kernel values (fp32 over 16 training points, then float64, slices added in a fixed order: deterministic);
// kstar_tensor_kernel + mean_split_kernel are the fallback for shapes that kernel does not take.  Predicts without
// variance never write K_*: gp_mean_direct_kernel.
//
// Accuracy contract of this path: |var - var_ref| <= 1e-5 * prior variance and |mean - mean_ref| <= 1e-5 on
// well-conditioned posteriors (tests/test_gpu_parity.py); DMO_GP_AUTO (gp.cu) measures both against the float64 path
// on probe candidates per model and recomputes in float64 what this path cannot hold to 1e-5 relative.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cudaTypedefs.h>
#include <stdlib.h>

#include "gp.cuh"

namespace {

constexpr int TN = 256;       // Linv rows per tile (wgmma N); Npad is a multiple of it
constexpr int TMV = 128;      // candidates per work item: two consumer warpgroups x wgmma M = 64
constexpr int TK = 32;        // k per pipeline stage: 64-byte rows, SWIZZLE_64B
constexpr int UK = 16;        // wgmma K for 16-bit inputs
constexpr int STAGES = 4;
constexpr int A_BYTES = TMV * TK * 2;                          // 8 KiB: K_* hi or lo
constexpr int B_BYTES = TN * TK * 2;                           // 16 KiB: Linv hi or lo
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;         // 48 KiB
constexpr size_t GEMM_SMEM = (size_t)STAGES * STAGE_BYTES + 1024 + 256;
constexpr int NTHREADS = 384;  // warpgroups 0, 1: consumers; warpgroup 2: TMA producer (one thread issues the loads)

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a protocol bug must not hang the GPU -- after ~2^22 polls the kernel flags an error and every later
// wait falls through immediately (results are then discarded by the host)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, volatile int* abort_flag) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0u) {
      if (*abort_flag) return;
      if (spins > (1u << 22)) {
        *abort_flag = 1;
        return;
      }
    }
  }
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// K-major SWIZZLE_64B shared-memory matrix descriptor (wgmma): [0,14) start address >> 4 | [16,30) leading byte
// offset >> 4 (unused for swizzled K-major: 1) | [32,46) stride byte offset >> 4 (8 rows x 64 B = 512 B between 8-row
// groups) | [62,64) layout type = 2 (SWIZZLE_64B)
__device__ __forceinline__ uint64_t make_sdesc64(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// d (+)= A[smem desc] (64 x 16) * B[smem desc]^T (256 x 16), fp16 inputs, fp32 accumulators; accumulate = 0 overwrites d.
// Thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 i + 2 (t % 4) (+ 1):
// d[4 i] = (row, col), d[4 i + 1] = (row, col + 1), d[4 i + 2] = (row + 8, col), d[4 i + 3] = (row + 8, col + 1).
__device__ __forceinline__ void wgmma_f16_m64n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// ------------------------------------------------------------------------------------------------ the contraction
// Work items and their order.  An item is (objective, 128 candidates, item q of the candidate block); the q of a
// candidate block are adjacent in the list, so the CTAs that share a K_* tile start together at k = 0 and walk k at the
// same (MMA-bound) rate: one of them pulls the tile from DRAM and the others hit it in L2.
//   * paired (default): item q owns the Linv row blocks {q, n_jt - 1 - q}, so every item costs the same n_jt + 1
//     k-blocks and a static round-robin over the persistent CTAs has a tail of at most one item;
//   * halves (DMO_GP_TC=2, the previous schedule): item 0 owns row blocks [0, j_split), item 1 [j_split, n_jt).
// Each item writes its partial sums to its own plane q of vnorm (and mnorm); var_finish_tc_kernel adds the planes in
// a fixed order.
struct GemmParams {
  int M, n_pb, n_jt, n_q;  // n_q items per candidate block
  int paired, j_split;
  int64_t k_rows, l_rows;
  const float* inv_scale;
  double* vnorm;  // [n_q][M][vn_ld]
  int64_t vn_ld;
  int* abort_flag;
  const float* zf;        // [M][l_rows] whitened targets (nullptr: the mean is not taken from this contraction)
  double* mnorm;          // [n_q][M][vn_ld] partial sums of D z
  const unsigned* ready;  // [n_pb / 2] completion counters of the K_* producer (nullptr: K_* is complete at launch)
  unsigned ready_target;
  int dbg;  // DMO_GP_DBG bits (diagnostics): 1 = no proxy fence, 2 = no nanosleep in the wait loop
};

__device__ __forceinline__ int item_blocks(const GemmParams& p, int q) {
  if (p.paired) return q == p.n_jt - 1 - q ? 1 : 2;
  return q ? p.n_jt - p.j_split : p.j_split;
}
// s-th row block of item q; in the paired schedule the short one comes first: its K_* tiles are read again right away
// by the long one
__device__ __forceinline__ int item_row_block(const GemmParams& p, int q, int s) {
  if (p.paired) return s ? p.n_jt - 1 - q : q;
  return (q ? p.j_split : 0) + s;
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(NTHREADS, 1)
    gp_var_wgmma_kernel(const __grid_constant__ CUtensorMap map_kh, const __grid_constant__ CUtensorMap map_kl,
                        const __grid_constant__ CUtensorMap map_lh, const __grid_constant__ CUtensorMap map_ll,
                        const GemmParams prm) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = (uint64_t*)(tiles + (size_t)STAGES * STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  volatile int* abort_flag = prm.abort_flag;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int per_m = prm.n_pb * prm.n_q;
  const int n_work = prm.M * per_m;

  // registers move from the producer warpgroup to the consumers (128 accumulators each): 40 + 2 x 232 per sub-partition
  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
        const int m = w / per_m, r = w - m * per_m;
        const int pb = r / prm.n_q, q = r - pb * prm.n_q;
        if (prm.ready) {  // the K_* rows of this candidate block must have been written (by another kernel, generic proxy)
          uint32_t spins = 0;
          while (ld_acquire_u32(prm.ready + (pb >> 1)) < prm.ready_target) {
            if (!(prm.dbg & 2)) __nanosleep(256);
            if ((++spins & 0xFFu) == 0u) {
              if (*abort_flag) break;
              if (spins > (1u << 23)) {  // ~2 s: the producer is not running
                *abort_flag = 2;
                break;
              }
            }
          }
          if (!(prm.dbg & 1)) asm volatile("fence.proxy.async;" ::: "memory");  // order the TMA (async proxy) reads after the acquire
        }
        const int a_row = (int)(m * prm.k_rows + (int64_t)pb * TMV);
        const int nb = item_blocks(prm, q);
        for (int s = 0; s < nb; ++s) {
          const int jt = item_row_block(prm, q, s);
          const int b_row = (int)(m * prm.l_rows + (int64_t)jt * TN);
          const int nkc = (jt + 1) * (TN / TK);
          for (int kc = 0; kc < nkc; ++kc) {
            mbar_wait(&empty[stage], phase ^ 1u, abort_flag);
            uint8_t* st = tiles + (size_t)stage * STAGE_BYTES;
            mbar_expect_tx(&full[stage], STAGE_BYTES);
            tma_load_2d(&map_kh, &full[stage], st, kc * TK, a_row);
            tma_load_2d(&map_kl, &full[stage], st + A_BYTES, kc * TK, a_row);
            tma_load_2d(&map_lh, &full[stage], st + 2 * A_BYTES, kc * TK, b_row);
            tma_load_2d(&map_ll, &full[stage], st + 2 * A_BYTES + B_BYTES, kc * TK, b_row);
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  // consumers: warpgroup wg owns candidate rows [64 wg, 64 wg + 64) of the item
  const int wg = warp >> 2;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // and row0 + 8
  const int col0 = 2 * (lane & 3);
  float acc[128];
  uint32_t stage = 0, phase = 0;
  for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
    const int m = w / per_m, r = w - m * per_m;
    const int pb = r / prm.n_q, q = r - pb * prm.n_q;
    const float* isc = prm.inv_scale + (int64_t)m * prm.l_rows;
    const float* zf = prm.zf ? prm.zf + (int64_t)m * prm.l_rows : nullptr;
    double total0 = 0.0, total1 = 0.0, mtot0 = 0.0, mtot1 = 0.0;
    const int nb = item_blocks(prm, q);
    for (int s = 0; s < nb; ++s) {
      const int jt = item_row_block(prm, q, s);
      const int nkc = (jt + 1) * (TN / TK);
      uint32_t prev = 0;
      for (int kc = 0; kc < nkc; ++kc) {
        mbar_wait(&full[stage], phase, abort_flag);
        const uint32_t sa = smem_u32(tiles + (size_t)stage * STAGE_BYTES);
        const uint32_t a_off = wg * (64 * TK * 2);
        const uint64_t a_hi = make_sdesc64(sa + a_off), a_lo = make_sdesc64(sa + A_BYTES + a_off);
        const uint64_t b_hi = make_sdesc64(sa + 2 * A_BYTES), b_lo = make_sdesc64(sa + 2 * A_BYTES + B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TK / UK; ++ks) {
          const uint64_t adv = (uint64_t)((ks * UK * 2) >> 4);
          wgmma_f16_m64n256(acc, a_hi + adv, b_hi + adv, (kc | ks) ? 1u : 0u);
          wgmma_f16_m64n256(acc, a_hi + adv, b_lo + adv, 1u);
          wgmma_f16_m64n256(acc, a_lo + adv, b_hi + adv, 1u);
        }
        wgmma_commit();
        if (kc > 0) {  // the previous k-block's MMAs are done with their slot: hand it back to the producer
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev]);
      // per 32 columns a thread holds 8 squares of each of its rows, in four fp32 partial sums folded into float64: the
      // rounding of the sum of squares stays at the 2^-24 level instead of growing with N
      const float* sc = isc + jt * TN + col0;
      const float* zc = zf ? zf + jt * TN + col0 : nullptr;
#pragma unroll
      for (int g = 0; g < TN / 32; ++g) {
        float p0[4] = {0.f, 0.f, 0.f, 0.f}, p1[4] = {0.f, 0.f, 0.f, 0.f};
        float q0[4] = {0.f, 0.f, 0.f, 0.f}, q1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = 4 * g + u;
          const float2 sv = __ldg(reinterpret_cast<const float2*>(sc + 8 * i));
          const float t00 = acc[4 * i] * sv.x, t01 = acc[4 * i + 1] * sv.y;
          const float t10 = acc[4 * i + 2] * sv.x, t11 = acc[4 * i + 3] * sv.y;
          p0[u] = fmaf(t01, t01, t00 * t00);
          p1[u] = fmaf(t11, t11, t10 * t10);
          if (zc) {  // posterior mean = D z out of the same accumulator (z = L^-1 y_n)
            const float2 zv = __ldg(reinterpret_cast<const float2*>(zc + 8 * i));
            q0[u] = fmaf(t01, zv.y, t00 * zv.x);
            q1[u] = fmaf(t11, zv.y, t10 * zv.x);
          }
        }
        total0 += ((double)p0[0] + (double)p0[1]) + ((double)p0[2] + (double)p0[3]);
        total1 += ((double)p1[0] + (double)p1[1]) + ((double)p1[2] + (double)p1[3]);
        if (zc) {
          mtot0 += ((double)q0[0] + (double)q0[1]) + ((double)q0[2] + (double)q0[3]);
          mtot1 += ((double)q1[0] + (double)q1[1]) + ((double)q1[2] + (double)q1[3]);
        }
      }
    }
    // the four lanes of a quad hold disjoint columns of the same two rows
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      total0 += __shfl_xor_sync(0xffffffffu, total0, o);
      total1 += __shfl_xor_sync(0xffffffffu, total1, o);
      mtot0 += __shfl_xor_sync(0xffffffffu, mtot0, o);
      mtot1 += __shfl_xor_sync(0xffffffffu, mtot1, o);
    }
    if ((lane & 3) == 0) {
      const int64_t o = ((int64_t)q * prm.M + m) * prm.vn_ld + (int64_t)pb * TMV + row0;
      prm.vnorm[o] = total0;
      prm.vnorm[o + 8] = total1;
      if (zf) {
        prm.mnorm[o] = mtot0;
        prm.mnorm[o + 8] = mtot1;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ operand preparation
// Linv row -> scaled fp16 hi / lo.  One block per (objective, row).
__global__ void split_linv_kernel(const double* __restrict__ Linv, int64_t Npad, int M, const int* __restrict__ k_exp,
                                  uint16_t* __restrict__ Lh, uint16_t* __restrict__ Ll, float* __restrict__ inv_scale) {
  const int64_t row = blockIdx.x;  // m * Npad + i
  const int m = (int)(row / Npad);
  const double* src = Linv + row * Npad;
  __shared__ double red[256];
  double mx = 0.0;
  for (int64_t k = threadIdx.x; k < Npad; k += blockDim.x) mx = fmax(mx, fabs(src[k]));
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  mx = red[0];
  int e = 0;
  if (mx > 0.0) e = 13 - ilogb(mx);  // scaled row maximum lands in [2^13, 2^14): far from fp16 overflow (65504)
  const double s = scalbn(1.0, e);
  for (int64_t k = threadIdx.x; k < Npad; k += blockDim.x) {
    const float x = (float)(src[k] * s);  // power-of-two scaling is exact; float keeps 24 bits
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    Lh[row * Npad + k] = __half_as_ushort(h);
    Ll[row * Npad + k] = __half_as_ushort(l);
  }
  if (threadIdx.x == 0) inv_scale[row] = (mx > 0.0) ? (float)scalbn(1.0, -e - k_exp[m]) : 0.f;
}

constexpr int KT_TN = 128, KT_TP = 32;

// c * k(r): hardware approximations (sqrt.approx / ex2.approx, relative error ~2^-22 each) are inside the 2^-22 budget
// the hi + lo fp16 split of K_* has anyway
__device__ __forceinline__ float stationary_f(float s2, int kind) {
  if (kind == DMO_KERNEL_MATERN52) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s2));
    const float K = r * 2.2360679774997896f;
    return fmaf(K, fmaf(K, 1.0f / 3.0f, 1.0f), 1.0f) * __expf(-K);
  }
  return __expf(-0.5f * s2);
}

// fp32 pairs: one correctly rounded operation per component (no FMA contraction), so a pair gives exactly what two
// scalar operations give
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// the same for a pair of squared distances
__device__ __forceinline__ float2 stationary2_f(float2 s2, int kind) {
  float2 e;
  if (kind == DMO_KERNEL_MATERN52) {
    float2 r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r.x) : "f"(s2.x));
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r.y) : "f"(s2.y));
    const float2 K = fmul2(r, make_float2(2.2360679774997896f, 2.2360679774997896f));
    const float2 one = make_float2(1.0f, 1.0f);
    const float2 p = ffma2(K, ffma2(K, make_float2(1.0f / 3.0f, 1.0f / 3.0f), one), one);
    const float2 t = fmul2(K, make_float2(-1.4426950408889634f, -1.4426950408889634f));  // exp(-K) = 2^(-K log2 e)
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(t.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(t.y));
    return fmul2(p, e);
  }
  const float2 t = fmul2(s2, make_float2(-0.5f * 1.4426950408889634f, -0.5f * 1.4426950408889634f));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(t.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(t.y));
  return e;
}

// K_* in fp32 -> scaled fp16 hi / lo.  Each thread owns two adjacent training points (their coordinates live in
// registers, results leave as packed half2), a block covers 256 training points x KT_TP candidates; the candidate
// tile is read from shared memory as 16-byte broadcasts (rows padded with zeros to DMAX coordinates, so the
// distance loops need no bounds tests and the LSU pipe carries a quarter of the instructions of scalar loads).
template <bool ISO, int DMAX>
__global__ void __launch_bounds__(KT_TN)
    kstar_tensor_kernel(const double* __restrict__ Xn, int64_t P, int64_t p_base, int64_t Pcpad,
                        const double* __restrict__ Xt, int64_t N, int d, int M, int kind,
                        const double* __restrict__ inv_ls, const double* __restrict__ constant,
                        const int* __restrict__ k_exp, int64_t ldk, int64_t plane, uint16_t* __restrict__ Kh,
                        uint16_t* __restrict__ Kl, unsigned* __restrict__ ready) {
  extern __shared__ __align__(16) float sxf[];  // [KT_TP][DMAX] candidate tile, then [M][DMAX] 1/l, [M] c * 2^kexp
  float* s_il = sxf + KT_TP * DMAX;
  float* s_c = s_il + M * DMAX;
  const int64_t n0 = ((int64_t)blockIdx.x * KT_TN + threadIdx.x) * 2;
  const int64_t pt0 = (int64_t)blockIdx.y * KT_TP;
  for (int t = threadIdx.x; t < KT_TP * DMAX; t += KT_TN) {
    const int64_t p = p_base + pt0 + t / DMAX;
    const int j = t % DMAX;
    sxf[t] = (p < P && j < d) ? (float)Xn[p * d + j] : 0.f;
  }
  for (int t = threadIdx.x; t < M * DMAX; t += KT_TN) {
    const int m = t / DMAX, j = t % DMAX;
    s_il[t] = j < d ? (float)inv_ls[m * d + j] : 0.f;
  }
  if (threadIdx.x < M) s_c[threadIdx.x] = scalbnf((float)constant[threadIdx.x], k_exp[threadIdx.x]);
  // training coordinates as pairs (two coordinates per 64-bit register pair)
  float2 xa[DMAX / 2], xb[DMAX / 2];
#pragma unroll
  for (int j = 0; j < DMAX / 2; ++j) {
    const int j0 = 2 * j, j1 = 2 * j + 1;
    xa[j] = make_float2((j0 < d && n0 < N) ? (float)Xt[n0 * d + j0] : 0.f, (j1 < d && n0 < N) ? (float)Xt[n0 * d + j1] : 0.f);
    xb[j] = make_float2((j0 < d && n0 + 1 < N) ? (float)Xt[(n0 + 1) * d + j0] : 0.f,
                        (j1 < d && n0 + 1 < N) ? (float)Xt[(n0 + 1) * d + j1] : 0.f);
  }
  __syncthreads();
  const bool live_a = n0 < N, live_b = n0 + 1 < N;
  uint32_t* Kh32 = reinterpret_cast<uint32_t*>(Kh);
  uint32_t* Kl32 = reinterpret_cast<uint32_t*>(Kl);
  for (int q = 0; q < KT_TP; ++q) {
    const int64_t pl = pt0 + q;
    if (pl >= Pcpad || n0 >= ldk) break;
    const float4* xc = reinterpret_cast<const float4*>(sxf + q * DMAX);
    float sa = 0.f, sb = 0.f;
    if (ISO) {
      float2 acc_a0 = make_float2(0.f, 0.f), acc_a1 = acc_a0, acc_b0 = acc_a0, acc_b1 = acc_a0;  // independent chains
#pragma unroll
      for (int j = 0; j < DMAX / 4; ++j) {
        const float4 c = xc[j];
        const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
        const float2 da0 = fadd2(c01, make_float2(-xa[2 * j].x, -xa[2 * j].y));
        const float2 db0 = fadd2(c01, make_float2(-xb[2 * j].x, -xb[2 * j].y));
        const float2 da1 = fadd2(c23, make_float2(-xa[2 * j + 1].x, -xa[2 * j + 1].y));
        const float2 db1 = fadd2(c23, make_float2(-xb[2 * j + 1].x, -xb[2 * j + 1].y));
        acc_a0 = ffma2(da0, da0, acc_a0);
        acc_b0 = ffma2(db0, db0, acc_b0);
        acc_a1 = ffma2(da1, da1, acc_a1);
        acc_b1 = ffma2(db1, db1, acc_b1);
      }
      sa = (acc_a0.x + acc_a0.y) + (acc_a1.x + acc_a1.y);
      sb = (acc_b0.x + acc_b0.y) + (acc_b1.x + acc_b1.y);
    }
    for (int m = 0; m < M; ++m) {
      float2 rr;
      if (ISO) {
        const float il = s_il[m * DMAX];
        const float il2 = il * il;
        rr = fmul2(make_float2(sa, sb), make_float2(il2, il2));
      } else {
        const float4* il4 = reinterpret_cast<const float4*>(s_il + m * DMAX);
        float2 acc_a = make_float2(0.f, 0.f), acc_b = acc_a;
#pragma unroll
        for (int j = 0; j < DMAX / 4; ++j) {
          const float4 c = xc[j], il = il4[j];
          const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
          const float2 i01 = make_float2(il.x, il.y), i23 = make_float2(il.z, il.w);
          const float2 da0 = fmul2(fadd2(c01, make_float2(-xa[2 * j].x, -xa[2 * j].y)), i01);
          const float2 db0 = fmul2(fadd2(c01, make_float2(-xb[2 * j].x, -xb[2 * j].y)), i01);
          const float2 da1 = fmul2(fadd2(c23, make_float2(-xa[2 * j + 1].x, -xa[2 * j + 1].y)), i23);
          const float2 db1 = fmul2(fadd2(c23, make_float2(-xb[2 * j + 1].x, -xb[2 * j + 1].y)), i23);
          acc_a = ffma2(da0, da0, acc_a);
          acc_b = ffma2(db0, db0, acc_b);
          acc_a = ffma2(da1, da1, acc_a);
          acc_b = ffma2(db1, db1, acc_b);
        }
        rr = make_float2(acc_a.x + acc_a.y, acc_b.x + acc_b.y);
      }
      const float sc = s_c[m];
      const float2 kk = fmul2(stationary2_f(rr, kind), make_float2(sc, sc));  // c * k(r), scaled by 2^kexp (exact)
      const float ka = live_a ? kk.x : 0.f;
      const float kb = live_b ? kk.y : 0.f;
      const __half2 h = __floats2half2_rn(ka, kb);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(ka - hf.x, kb - hf.y);
      const int64_t o = (m * plane + pl * ldk + n0) >> 1;
      Kh32[o] = *reinterpret_cast<const uint32_t*>(&h);
      Kl32[o] = *reinterpret_cast<const uint32_t*>(&l);
    }
  }
  if (ready) {
    // publish this block's rows to the variance kernel that is already running (v3::gp_var_tc3_kernel): every thread's
    // stores happen-before the barrier, the fence makes them visible at GPU scope before the counter moves
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      atomicAdd(ready + pt0 / 256, 1u);
    }
  }
}

// Mean-only posterior (what MOASMO.optimize asks for every generation: model.evaluate -> mean, MOASMO.py:107-108): K_* is
// never written.  A thread owns two candidates (coordinates in registers), the block walks its share of the training
// points through a shared-memory tile (16-byte broadcast reads, paired fp32 distance loops as in kstar_tensor_kernel),
// k(x, x_n) * (c alpha_n) is accumulated in fp32 over 32 training points and then folded into float64; the
// partial sums of the blockIdx.x slices are added in a fixed order by mean_finish_tc_kernel (deterministic).
constexpr int KM_T = 128, KM_Q = 256, KM_NS = 32, KM_D = 32;

__global__ void pad_xt_f32_kernel(const double* __restrict__ Xt, int64_t N, int d, int64_t Npad, float* __restrict__ Xtf) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Npad * KM_D) return;
  const int64_t n = t / KM_D;
  const int j = (int)(t % KM_D);
  Xtf[t] = (n < N && j < d) ? (float)Xt[n * d + j] : 0.f;
}

__global__ void pad_calpha_f32_kernel(const double* __restrict__ alpha, const double* __restrict__ constant, int64_t N, int M,
                                      int64_t Npad, float* __restrict__ CAf) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)M * Npad) return;
  const int m = (int)(t / Npad);
  const int64_t n = t - (int64_t)m * Npad;
  CAf[t] = n < N ? (float)(constant[m] * alpha[(int64_t)m * N + n]) : 0.f;
}

// NJ: groups of four input dimensions that are evaluated (the tile always carries KM_D = 32 zero-padded coordinates)
template <bool ISO, int MT, int NJ>
__global__ void __launch_bounds__(KM_T, 4)
    gp_mean_direct_kernel(const double* __restrict__ Xn, int64_t P, int64_t p_base, const float* __restrict__ Xtf, int64_t N,
                          int64_t Npad, int64_t n_per_block, int d, int kind, const double* __restrict__ inv_ls,
                          const double* __restrict__ constant, const double* __restrict__ alpha,
                          double* __restrict__ mpart, int64_t mp_ld) {
  __shared__ __align__(16) float s_x[KM_NS * KM_D];
  __shared__ float s_al[MT * KM_NS];  // c_m * alpha_m[n] of the tile (zero beyond N)
  __shared__ __align__(16) float s_il[MT * KM_D];
  const int t = threadIdx.x;
  const int64_t qa = (int64_t)blockIdx.y * KM_Q + t, qb = qa + KM_T;  // candidate rows inside this chunk
  float2 ca[2 * NJ], cb[2 * NJ];
  {
    const int64_t pa = p_base + qa, pb = p_base + qb;
#pragma unroll
    for (int j = 0; j < 2 * NJ; ++j) {
      const int j0 = 2 * j, j1 = 2 * j + 1;
      ca[j] = make_float2((pa < P && j0 < d) ? (float)Xn[pa * d + j0] : 0.f, (pa < P && j1 < d) ? (float)Xn[pa * d + j1] : 0.f);
      cb[j] = make_float2((pb < P && j0 < d) ? (float)Xn[pb * d + j0] : 0.f, (pb < P && j1 < d) ? (float)Xn[pb * d + j1] : 0.f);
    }
  }
  for (int i = t; i < MT * KM_D; i += KM_T) {
    const int m = i / KM_D, j = i % KM_D;
    s_il[i] = j < d ? (float)inv_ls[m * d + j] : 0.f;
  }
  double sum_a[MT], sum_b[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) sum_a[m] = sum_b[m] = 0.0;
  const int64_t n_begin = (int64_t)blockIdx.x * n_per_block;
  const int64_t n_end = n_begin + n_per_block < Npad ? n_begin + n_per_block : Npad;
  for (int64_t n0 = n_begin; n0 < n_end; n0 += KM_NS) {
    __syncthreads();  // the previous tile has been consumed
    {
      const float4* src = reinterpret_cast<const float4*>(Xtf + n0 * KM_D);
      float4* dst = reinterpret_cast<float4*>(s_x);
      dst[t] = src[t];
      dst[t + KM_T] = src[t + KM_T];
    }
    for (int i = t; i < MT * KM_NS; i += KM_T) {
      const int m = i / KM_NS;
      const int64_t n = n0 + i % KM_NS;
      s_al[i] = n < N ? (float)(constant[m] * alpha[(int64_t)m * N + n]) : 0.f;
    }
    __syncthreads();
    if (ISO) {  // one squared distance per (candidate, training point), scaled per objective
      float2 acc[MT];
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[m] = make_float2(0.f, 0.f);
#pragma unroll 2
      for (int i = 0; i < KM_NS; ++i) {
        const float4* xr = reinterpret_cast<const float4*>(s_x + i * KM_D);
        float2 a0 = make_float2(0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;  // independent chains
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const float4 c = xr[j];
          const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
          const float2 da0 = fadd2(c01, make_float2(-ca[2 * j].x, -ca[2 * j].y));
          const float2 db0 = fadd2(c01, make_float2(-cb[2 * j].x, -cb[2 * j].y));
          const float2 da1 = fadd2(c23, make_float2(-ca[2 * j + 1].x, -ca[2 * j + 1].y));
          const float2 db1 = fadd2(c23, make_float2(-cb[2 * j + 1].x, -cb[2 * j + 1].y));
          a0 = ffma2(da0, da0, a0);
          b0 = ffma2(db0, db0, b0);
          a1 = ffma2(da1, da1, a1);
          b1 = ffma2(db1, db1, b1);
        }
        const float2 r2 = make_float2((a0.x + a0.y) + (a1.x + a1.y), (b0.x + b0.y) + (b1.x + b1.y));
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const float il = s_il[m * KM_D];
          const float il2 = il * il;
          const float al = s_al[m * KM_NS + i];
          acc[m] = ffma2(stationary2_f(fmul2(r2, make_float2(il2, il2)), kind), make_float2(al, al), acc[m]);
        }
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        sum_a[m] += (double)acc[m].x;
        sum_b[m] += (double)acc[m].y;
      }
    } else {  // one length scale per dimension and objective: a pass over the tile per objective
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const float4* il4 = reinterpret_cast<const float4*>(s_il + m * KM_D);
        float2 acc = make_float2(0.f, 0.f);
#pragma unroll 2
        for (int i = 0; i < KM_NS; ++i) {
          const float4* xr = reinterpret_cast<const float4*>(s_x + i * KM_D);
          float2 aa = make_float2(0.f, 0.f), bb = aa;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const float4 c = xr[j], il = il4[j];
            const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
            const float2 i01 = make_float2(il.x, il.y), i23 = make_float2(il.z, il.w);
            const float2 da0 = fmul2(fadd2(c01, make_float2(-ca[2 * j].x, -ca[2 * j].y)), i01);
            const float2 db0 = fmul2(fadd2(c01, make_float2(-cb[2 * j].x, -cb[2 * j].y)), i01);
            const float2 da1 = fmul2(fadd2(c23, make_float2(-ca[2 * j + 1].x, -ca[2 * j + 1].y)), i23);
            const float2 db1 = fmul2(fadd2(c23, make_float2(-cb[2 * j + 1].x, -cb[2 * j + 1].y)), i23);
            aa = ffma2(da0, da0, aa);
            bb = ffma2(db0, db0, bb);
            aa = ffma2(da1, da1, aa);
            bb = ffma2(db1, db1, bb);
          }
          const float al = s_al[m * KM_NS + i];
          acc = ffma2(stationary2_f(make_float2(aa.x + aa.y, bb.x + bb.y), kind), make_float2(al, al), acc);
        }
        sum_a[m] += (double)acc.x;
        sum_b[m] += (double)acc.y;
      }
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    mpart[((int64_t)blockIdx.x * MT + m) * mp_ld + qa] = sum_a[m];
    mpart[((int64_t)blockIdx.x * MT + m) * mp_ld + qb] = sum_b[m];
  }
}

// K_* producer fused with the mean (predicts with variance): the layout of gp_mean_direct_kernel (a thread owns two
// candidates) with 16-point tiles; besides accumulating k * (c alpha) the block stages the scaled hi / lo fp16 split of
// its 256 x 16 tile per objective in shared memory (rows of 10 words: 8-byte stores of four consecutive training points
// are conflict free) and writes it out as full 32-byte sectors.  Replaces kstar_tensor_kernel + mean_split_kernel
// (1.46 + 0.72 ms at the BASELINE shape): K_* is written once and not read back for the mean.
constexpr int KF_NS = 16, KF_LD = 10;

template <bool ISO, int MT>
__global__ void __launch_bounds__(KM_T, 3)
    kstar_mean_kernel(const double* __restrict__ Xn, int64_t P, int64_t p_base, const float* __restrict__ Xtf, int64_t N,
                      int64_t Npad, int64_t n_per_block, int d, int kind, const double* __restrict__ inv_ls,
                      const double* __restrict__ constant, const int* __restrict__ k_exp, const float* __restrict__ CAf,
                      int64_t plane, uint16_t* __restrict__ Kh, uint16_t* __restrict__ Kl, double* __restrict__ mpart,
                      int64_t mp_ld) {
  extern __shared__ __align__(16) uint32_t kf_stage[];  // [MT][2][KM_Q][KF_LD] words: (objective, hi / lo, candidate row)
  __shared__ __align__(16) float s_x[KF_NS * KM_D];
  __shared__ float s_al[MT * KF_NS];  // c_m * alpha_m[n] of the tile (zero beyond N)
  __shared__ float s_live[KF_NS];     // 1 for a training point, 0 for the padding columns (written as zeros)
  __shared__ __align__(16) float s_il[MT * KM_D];
  __shared__ float s_c[MT];           // c_m * 2^kexp_m: scale of the stored K_*
  const int t = threadIdx.x;
  const int64_t q_base = (int64_t)blockIdx.y * KM_Q;
  const int64_t qa = q_base + t, qb = qa + KM_T;
  float2 ca[KM_D / 2], cb[KM_D / 2];
  {
    const int64_t pa = p_base + qa, pb = p_base + qb;
#pragma unroll
    for (int j = 0; j < KM_D / 2; ++j) {
      const int j0 = 2 * j, j1 = 2 * j + 1;
      ca[j] = make_float2((pa < P && j0 < d) ? (float)Xn[pa * d + j0] : 0.f, (pa < P && j1 < d) ? (float)Xn[pa * d + j1] : 0.f);
      cb[j] = make_float2((pb < P && j0 < d) ? (float)Xn[pb * d + j0] : 0.f, (pb < P && j1 < d) ? (float)Xn[pb * d + j1] : 0.f);
    }
  }
  for (int i = t; i < MT * KM_D; i += KM_T) {
    const int m = i / KM_D, j = i % KM_D;
    s_il[i] = j < d ? (float)inv_ls[m * d + j] : 0.f;
  }
  if (t < MT) s_c[t] = scalbnf((float)constant[t], k_exp[t]);
  double sum_a[MT], sum_b[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) sum_a[m] = sum_b[m] = 0.0;
  const int64_t n_begin = (int64_t)blockIdx.x * n_per_block;
  const int64_t n_end = n_begin + n_per_block < Npad ? n_begin + n_per_block : Npad;
  uint32_t* row_a = kf_stage + (size_t)t * KF_LD;             // + (m * 2 + arr) * KM_Q * KF_LD
  uint32_t* row_b = kf_stage + (size_t)(t + KM_T) * KF_LD;
  // the next tile's training coordinates (one float4 per thread: KF_NS * KM_D / 4 == KM_T) and c * alpha values travel
  // through registers while the current tile is being worked on: no global-load latency between two barriers
  static_assert(KF_NS * KM_D / 4 == KM_T && 6 * KF_NS <= KM_T, "tile prefetch mapping");
  float4 px = reinterpret_cast<const float4*>(Xtf + n_begin * KM_D)[t];
  float pal = t < MT * KF_NS ? CAf[(int64_t)(t / KF_NS) * Npad + n_begin + t % KF_NS] : 0.f;
  __syncthreads();  // s_il, s_c
  reinterpret_cast<float4*>(s_x)[t] = px;
  if (t < MT * KF_NS) s_al[t] = pal;
  if (t < KF_NS) s_live[t] = (n_begin + t < N) ? 1.f : 0.f;
  __syncthreads();
  for (int64_t n0 = n_begin; n0 < n_end; n0 += KF_NS) {
    const bool more = n0 + KF_NS < n_end;
    if (more) {  // in flight during the tile's arithmetic
      px = reinterpret_cast<const float4*>(Xtf + (n0 + KF_NS) * KM_D)[t];
      if (t < MT * KF_NS) pal = CAf[(int64_t)(t / KF_NS) * Npad + n0 + KF_NS + t % KF_NS];
    }
    float2 acc[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] = make_float2(0.f, 0.f);
#pragma unroll 1
    for (int i4 = 0; i4 < KF_NS; i4 += 4) {
      uint32_t wh_a[MT][2], wl_a[MT][2], wh_b[MT][2], wl_b[MT][2];  // four training points -> two half2 words each
#pragma unroll
      for (int u2 = 0; u2 < 2; ++u2) {
        float2 kv[2][MT];  // scaled kernel values of the pair of points (candidates a, b)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int i = i4 + 2 * u2 + u;
          const float4* xr = reinterpret_cast<const float4*>(s_x + i * KM_D);
          float2 r2 = make_float2(0.f, 0.f);
          if (ISO) {
            float2 a0 = make_float2(0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
#pragma unroll
            for (int j = 0; j < KM_D / 4; ++j) {
              const float4 c = xr[j];
              const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
              const float2 da0 = fadd2(c01, make_float2(-ca[2 * j].x, -ca[2 * j].y));
              const float2 db0 = fadd2(c01, make_float2(-cb[2 * j].x, -cb[2 * j].y));
              const float2 da1 = fadd2(c23, make_float2(-ca[2 * j + 1].x, -ca[2 * j + 1].y));
              const float2 db1 = fadd2(c23, make_float2(-cb[2 * j + 1].x, -cb[2 * j + 1].y));
              a0 = ffma2(da0, da0, a0);
              b0 = ffma2(db0, db0, b0);
              a1 = ffma2(da1, da1, a1);
              b1 = ffma2(db1, db1, b1);
            }
            r2 = make_float2((a0.x + a0.y) + (a1.x + a1.y), (b0.x + b0.y) + (b1.x + b1.y));
          }
          const float live = s_live[i];
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            float2 rr;
            if (ISO) {
              const float il = s_il[m * KM_D];
              const float il2 = il * il;
              rr = fmul2(r2, make_float2(il2, il2));
            } else {
              const float4* il4 = reinterpret_cast<const float4*>(s_il + m * KM_D);
              float2 aa = make_float2(0.f, 0.f), bb = aa;
#pragma unroll
              for (int j = 0; j < KM_D / 4; ++j) {
                const float4 c = xr[j], il = il4[j];
                const float2 c01 = make_float2(c.x, c.y), c23 = make_float2(c.z, c.w);
                const float2 i01 = make_float2(il.x, il.y), i23 = make_float2(il.z, il.w);
                const float2 da0 = fmul2(fadd2(c01, make_float2(-ca[2 * j].x, -ca[2 * j].y)), i01);
                const float2 db0 = fmul2(fadd2(c01, make_float2(-cb[2 * j].x, -cb[2 * j].y)), i01);
                const float2 da1 = fmul2(fadd2(c23, make_float2(-ca[2 * j + 1].x, -ca[2 * j + 1].y)), i23);
                const float2 db1 = fmul2(fadd2(c23, make_float2(-cb[2 * j + 1].x, -cb[2 * j + 1].y)), i23);
                aa = ffma2(da0, da0, aa);
                bb = ffma2(db0, db0, bb);
                aa = ffma2(da1, da1, aa);
                bb = ffma2(db1, db1, bb);
              }
              rr = make_float2(aa.x + aa.y, bb.x + bb.y);
            }
            const float2 k0 = stationary2_f(rr, kind);
            const float al = s_al[m * KF_NS + i];
            acc[m] = ffma2(k0, make_float2(al, al), acc[m]);
            const float sc = s_c[m] * live;
            kv[u][m] = fmul2(k0, make_float2(sc, sc));  // c * k(r), scaled by 2^kexp (exact); padding columns: 0
          }
        }
#pragma unroll
        for (int m = 0; m < MT; ++m) {  // pack (n, n + 1) of one candidate into half2: hi, then lo = value - hi
          const __half2 ha = __floats2half2_rn(kv[0][m].x, kv[1][m].x), hb = __floats2half2_rn(kv[0][m].y, kv[1][m].y);
          const float2 fa = __half22float2(ha), fb = __half22float2(hb);
          const __half2 la = __floats2half2_rn(kv[0][m].x - fa.x, kv[1][m].x - fa.y);
          const __half2 lb = __floats2half2_rn(kv[0][m].y - fb.x, kv[1][m].y - fb.y);
          wh_a[m][u2] = *reinterpret_cast<const uint32_t*>(&ha);
          wl_a[m][u2] = *reinterpret_cast<const uint32_t*>(&la);
          wh_b[m][u2] = *reinterpret_cast<const uint32_t*>(&hb);
          wl_b[m][u2] = *reinterpret_cast<const uint32_t*>(&lb);
        }
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const size_t oh = (size_t)(m * 2) * KM_Q * KF_LD + (i4 >> 1), ol = oh + (size_t)KM_Q * KF_LD;
        *reinterpret_cast<uint2*>(row_a + oh) = make_uint2(wh_a[m][0], wh_a[m][1]);
        *reinterpret_cast<uint2*>(row_a + ol) = make_uint2(wl_a[m][0], wl_a[m][1]);
        *reinterpret_cast<uint2*>(row_b + oh) = make_uint2(wh_b[m][0], wh_b[m][1]);
        *reinterpret_cast<uint2*>(row_b + ol) = make_uint2(wl_b[m][0], wl_b[m][1]);
      }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      sum_a[m] += (double)acc[m].x;
      sum_b[m] += (double)acc[m].y;
    }
    __syncthreads();  // the tile is staged, its inputs have been consumed
    // flush: 8-byte units, four per 32-byte row segment (a warp writes eight full sectors per instruction); thread t
    // always moves unit t & 3 of rows (t >> 2) + 32 k, so every offset below is a compile-time constant or one add
    {
      const uint32_t* src = kf_stage + (size_t)(t >> 2) * KF_LD + 2 * (t & 3);
      const int64_t row0 = (q_base + (t >> 2)) * Npad + n0 + 4 * (t & 3);
      const int64_t kstep = (int64_t)32 * Npad;
#pragma unroll
      for (int ma = 0; ma < 2 * MT; ++ma) {
        uint16_t* dst = ((ma & 1) ? Kl : Kh) + (int64_t)(ma >> 1) * plane + row0;
#pragma unroll
        for (int k = 0; k < KM_Q / 32; ++k) {
          const uint2 v = *reinterpret_cast<const uint2*>(src + (size_t)(ma * KM_Q + k * 32) * KF_LD);
          *reinterpret_cast<uint2*>(dst) = v;
          dst += kstep;
        }
      }
    }
    if (more) {  // the next tile's inputs, from the registers filled above
      reinterpret_cast<float4*>(s_x)[t] = px;
      if (t < MT * KF_NS) s_al[t] = pal;
      if (t < KF_NS) s_live[t] = (n0 + KF_NS + t < N) ? 1.f : 0.f;
    }
    __syncthreads();  // stage drained, next inputs in place
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    mpart[((int64_t)blockIdx.x * MT + m) * mp_ld + qa] = sum_a[m];
    mpart[((int64_t)blockIdx.x * MT + m) * mp_ld + qb] = sum_b[m];
  }
}

// mean[p][m] = y_std * sum_n K_*[p][n] alpha[n] + y_mean from the split K_* (hi + lo = 22 bits): HBM-bound pass,
// one warp per (objective, candidate) row, float64 accumulation in a fixed order
__global__ void mean_split_kernel(const uint16_t* __restrict__ Kh, const uint16_t* __restrict__ Kl, int64_t Pc, int64_t N,
                                  int64_t ldk, int64_t plane, int M, const int* __restrict__ k_exp,
                                  const double* __restrict__ alpha, const double* __restrict__ ymean,
                                  const double* __restrict__ ystd, int64_t p_base, double* __restrict__ mean) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= Pc * M) return;
  const int m = (int)(w / Pc);
  const int64_t pl = w - (int64_t)m * Pc;
  const uint32_t* rh = reinterpret_cast<const uint32_t*>(Kh + m * plane + pl * ldk);
  const uint32_t* rl = reinterpret_cast<const uint32_t*>(Kl + m * plane + pl * ldk);
  const double* a = alpha + (int64_t)m * N;
  double s = 0.0;
#pragma unroll 8
  for (int64_t n2 = lane; 2 * n2 < N; n2 += 32) {  // two fp16 values per 32-bit load
    const uint32_t h = rh[n2], l = rl[n2];
    const float k0 = __half2float(__ushort_as_half((uint16_t)(h & 0xFFFFu))) + __half2float(__ushort_as_half((uint16_t)(l & 0xFFFFu)));
    const float k1 = __half2float(__ushort_as_half((uint16_t)(h >> 16))) + __half2float(__ushort_as_half((uint16_t)(l >> 16)));
    const int64_t n = 2 * n2;
    s += (double)k0 * a[n];
    if (n + 1 < N) s += (double)k1 * a[n + 1];
  }
  s = warp_sum(s);
  if (lane == 0) mean[(p_base + pl) * M + m] = ystd[m] * scalbn(s, -k_exp[m]) + ymean[m];
}

// mean[p][m] = y_std * sum over the work items' partial sums of D z + y_mean (fixed order)
__global__ void mean_finish_tc_kernel(const double* __restrict__ mnorm, int nplanes, int64_t Pc, int64_t ld, int M,
                                      const double* __restrict__ ymean, const double* __restrict__ ystd, int64_t p_base,
                                      double* __restrict__ mean) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Pc * M) return;
  int64_t pl = t / M;
  int m = (int)(t - pl * M);
  double s = 0.0;
  for (int q = 0; q < nplanes; ++q) s += mnorm[((int64_t)q * M + m) * ld + pl];
  mean[(p_base + pl) * M + m] = ystd[m] * s + ymean[m];
}

__global__ void var_finish_tc_kernel(const double* __restrict__ vnorm, int nplanes, int64_t Pc, int64_t ld, int M,
                                     const double* __restrict__ constant, const double* __restrict__ noise,
                                     const double* __restrict__ ystd, int64_t p_base, double* __restrict__ var) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Pc * M) return;
  int64_t pl = t / M;
  int m = (int)(t - pl * M);
  double vn = 0.0;
  for (int q = 0; q < nplanes; ++q) vn += vnorm[((int64_t)q * M + m) * ld + pl];  // partial sums of the work items, fixed order
  double v = (constant[m] + noise[m]) - vn;
  if (v < 0.0) v = 0.0;
  double sd = sqrt(v * (ystd[m] * ystd[m]));
  var[(p_base + pl) * M + m] = sd * sd;
}

// ------------------------------------------------------------------------------------------------ host side
PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

// 2-D fp16 tensor [rows][cols] (cols contiguous), box = box_rows x box_cols
int make_map(dmo_ctx* ctx, CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
             uint32_t box_cols, CUtensorMapSwizzle swz) {
  auto fn = get_encode_fn();
  if (!fn) return dmo_fail(ctx, DMO_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return dmo_fail(ctx, DMO_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
  return DMO_OK;
}

int prepare_tensor_state(dmo_ctx* ctx, dmo_gp* gp) {
  if (gp->tensor_ready) return DMO_OK;
  const int M = gp->M;
  const int64_t Npad = gp->Npad;
  std::vector<int> kexp(M);
  for (int m = 0; m < M; ++m) {
    double c = gp->h_constant[m];
    kexp[m] = (c > 0.0) ? 13 - ilogb(c) : 13;  // scaled K_* <= 2^14
  }
  DMO_TRY(gp->Kexp.alloc(ctx, M));
  DMO_CUDA(cudaMemcpyAsync(gp->Kexp.p, kexp.data(), M * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  DMO_CUDA(cudaStreamSynchronize(ctx->stream));  // kexp is a stack vector
  DMO_TRY(gp->Lhi.alloc(ctx, (size_t)M * Npad * Npad));
  DMO_TRY(gp->Llo.alloc(ctx, (size_t)M * Npad * Npad));
  DMO_TRY(gp->Lscale.alloc(ctx, (size_t)M * Npad));
  DMO_LAUNCH(split_linv_kernel, (unsigned)(M * Npad), 256, 0, gp->Linv.p, Npad, M, gp->Kexp.p, gp->Lhi.p, gp->Llo.p,
             gp->Lscale.p);
  DMO_CHECK_LAUNCH();
  gp->tensor_ready = true;
  return DMO_OK;
}

// float copies of the training inputs and of c * alpha, zero padded to Npad (once per model)
int prepare_direct_state(dmo_ctx* ctx, dmo_gp* gp) {
  if (gp->Xtf.p && gp->CAf.p) return DMO_OK;
  const int64_t N = gp->N, Npad = gp->Npad;
  DMO_TRY(gp->Xtf.alloc(ctx, (size_t)Npad * KM_D));
  DMO_TRY(gp->CAf.alloc(ctx, (size_t)gp->M * Npad));
  DMO_LAUNCH(pad_xt_f32_kernel, (unsigned)ceil_div(Npad * KM_D, 256), 256, 0, gp->Xt.p, N, gp->d, Npad, gp->Xtf.p);
  DMO_LAUNCH(pad_calpha_f32_kernel, (unsigned)ceil_div((int64_t)gp->M * Npad, 256), 256, 0, gp->alpha.p, gp->constant.p, N, gp->M, Npad,
             gp->CAf.p);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

// Slices of the training set per candidate block for the two kernels above: the grid (slices x candidate blocks) should
// fill whole waves of `slots` resident CTAs; a slice is a multiple of `tile` points and at least 256 of them.
int64_t pick_slices(int64_t n_qb, int64_t Npad, int tile, int64_t slots, int64_t* n_per_block) {
  int64_t best = 1;
  double best_eff = -1.0;
  *n_per_block = Npad;
  const int64_t smax = Npad / 256 > 1 ? Npad / 256 : 1;
  for (int64_t sp = 1; sp <= smax; ++sp) {
    const int64_t npb = ceil_div(ceil_div(Npad, sp), (int64_t)tile) * tile;
    const int64_t ns = ceil_div(Npad, npb);
    const int64_t blocks = ns * n_qb;
    const double eff = (double)blocks / (double)(ceil_div(blocks, slots) * slots);
    if (eff > best_eff + 0.02) {  // fewer slices (fewer partial sums) unless more of them fill the waves visibly better
      best_eff = eff;
      best = ns;
      *n_per_block = npb;
    }
  }
  return best;
}

// mean-only predict without K_* in memory (d <= 32, M <= 6): see gp_mean_direct_kernel
int gp_mean_direct(dmo_ctx* ctx, dmo_gp* gp, const double* dXn, int64_t P, double* d_mean) {
  const int64_t N = gp->N, Npad = gp->Npad;
  const int M = gp->M, d = gp->d;
  DMO_TRY(prepare_direct_state(ctx, gp));
  const int64_t n_qb = ceil_div(P, KM_Q);
  int64_t n_per_block = Npad;
  const int64_t nsplit = pick_slices(n_qb, Npad, KM_NS, (int64_t)4 * ctx->sm_count, &n_per_block);
  const int64_t ld = n_qb * KM_Q;
  DevBuf<double> mpart;
  DMO_TRY(mpart.alloc(ctx, (size_t)nsplit * M * ld));
  dim3 grid((unsigned)nsplit, (unsigned)n_qb);
  {
    ProfileScope ps_(ctx, "gp_mean_direct");
#define KM_LAUNCH(ISO_, MT_)                                                                                                  \
  do {                                                                                                                      \
    if (d <= 16)                                                                                                            \
      DMO_LAUNCH((gp_mean_direct_kernel<ISO_, MT_, 4>), grid, KM_T, 0, dXn, P, (int64_t)0, gp->Xtf.p, N, Npad, n_per_block, \
                 d, gp->kernel, gp->inv_ls.p, gp->constant.p, gp->alpha.p, mpart.p, ld);                                    \
    else                                                                                                                    \
      DMO_LAUNCH((gp_mean_direct_kernel<ISO_, MT_, 8>), grid, KM_T, 0, dXn, P, (int64_t)0, gp->Xtf.p, N, Npad, n_per_block, \
                 d, gp->kernel, gp->inv_ls.p, gp->constant.p, gp->alpha.p, mpart.p, ld);                                    \
  } while (0)
#define KM_SWITCH(ISO_)        \
  switch (M) {                 \
    case 1: KM_LAUNCH(ISO_, 1); break; \
    case 2: KM_LAUNCH(ISO_, 2); break; \
    case 3: KM_LAUNCH(ISO_, 3); break; \
    case 4: KM_LAUNCH(ISO_, 4); break; \
    case 5: KM_LAUNCH(ISO_, 5); break; \
    default: KM_LAUNCH(ISO_, 6); break; \
  }
    if (gp->isotropic) {
      KM_SWITCH(true)
    } else {
      KM_SWITCH(false)
    }
#undef KM_SWITCH
#undef KM_LAUNCH
  }
  DMO_LAUNCH(mean_finish_tc_kernel, (unsigned)ceil_div(P * M, 256), 256, 0, mpart.p, (int)nsplit, P, ld, M, gp->ymean.p,
             gp->ystd.p, (int64_t)0, d_mean);
  DMO_CHECK_LAUNCH();
  return DMO_OK;  // mpart is released in stream order
}

}  // namespace

int gp_predict_tensor(dmo_ctx* ctx, dmo_gp* gp, const double* dXn, int64_t P, double* d_mean, double* d_var, bool mean_from_d) {
  const int64_t N = gp->N, Npad = gp->Npad;
  const int M = gp->M, d = gp->d;
  DMO_REQUIRE(M <= 16, "gp_predict(tensor): at most 16 objectives per model (got %d)", M);
  DMO_REQUIRE(d <= 64, "gp_predict(tensor): at most 64 input dimensions (got %d); use DMO_GP_FP64", d);
  DMO_REQUIRE(Npad % TN == 0, "gp_predict(tensor): internal padding error");
  if (!d_var && d <= KM_D && M <= 6 && !(getenv("DMO_GP_MEAN_DIRECT") && atoi(getenv("DMO_GP_MEAN_DIRECT")) == 0))
    return gp_mean_direct(ctx, gp, dXn, P, d_mean);  // nothing but the mean is wanted: K_* stays in registers
  DMO_TRY(prepare_tensor_state(ctx, gp));
  // work schedule of the contraction: 3 (default) = equal-cost paired row blocks, optionally overlapped with the K_*
  // producer; 2 = the previous schedule, two halves of the row blocks per candidate block (DMO_GP_TC=2, kept for comparison)
  int version = 3;
  if (const char* e = getenv("DMO_GP_TC")) version = atoi(e) == 2 ? 2 : 3;
  // DMO_GP_OVERLAP=1 (experimental, off by default): launch the contraction while the K_* producer is still running on
  // the context's second stream and let its TMA thread wait on per-candidate-block completion counters.  The
  // co-residency of the two kernels is not guaranteed by the hardware scheduler, so the in-line order is the product path.
  const bool overlap = version == 3 && getenv("DMO_GP_OVERLAP") && atoi(getenv("DMO_GP_OVERLAP"));
  const int dbg = getenv("DMO_GP_DBG") ? atoi(getenv("DMO_GP_DBG")) : 0;  // 4: event instead of flags, 8: mean after var
  const bool use_flags = overlap && !(dbg & 4);
  // mean from the contraction (D z) instead of the K_* alpha pass: only with the variance, version 3 and a model created from L
  mean_from_d = mean_from_d && d_var != nullptr && version == 3 && gp->z_ready;
  constexpr int64_t TMv = KM_Q;  // candidate padding: the K_* producers write 256-candidate blocks
  // candidate chunk: K_* hi/lo (2 x M x Pc x Npad fp16) within ~6 GiB
  int64_t Pc_max = ((int64_t)6 << 30) / ((int64_t)M * Npad * 4);
  Pc_max = (Pc_max / TMv) * TMv;
  if (Pc_max < TMv) Pc_max = TMv;
  const int64_t Pc_alloc = P < Pc_max ? ceil_div(P, TMv) * TMv : Pc_max;
  const int n_jt = (int)(Npad / TN);
  const int n_q = version == 3 ? (n_jt + 1) / 2 : 2;
  const int64_t n_chunks = ceil_div(P, Pc_alloc);
  const int n_pb_alloc = (int)(Pc_alloc / TMv);
  DevBuf<uint16_t> Kh, Kl;
  DevBuf<double> vnorm;
  DevBuf<int> abort_flag;
  DevBuf<unsigned> ready;
  DMO_TRY(Kh.alloc(ctx, (size_t)M * Pc_alloc * Npad));
  DMO_TRY(Kl.alloc(ctx, (size_t)M * Pc_alloc * Npad));
  DMO_TRY(vnorm.alloc(ctx, (size_t)n_q * M * Pc_alloc));
  DevBuf<double> mnorm;
  if (mean_from_d) DMO_TRY(mnorm.alloc(ctx, (size_t)n_q * M * Pc_alloc));
  DMO_TRY(abort_flag.alloc(ctx, 1));
  DMO_TRY(ready.alloc(ctx, (size_t)n_chunks * n_pb_alloc));
  DMO_CUDA(cudaMemsetAsync(abort_flag.p, 0, sizeof(int), ctx->stream));
  DMO_CUDA(cudaMemsetAsync(ready.p, 0, (size_t)n_chunks * n_pb_alloc * sizeof(unsigned), ctx->stream));
  CUtensorMap map_kh, map_kl, map_lh, map_ll;
  DMO_TRY(make_map(ctx, &map_kh, Kh.p, (uint64_t)M * Pc_alloc, (uint64_t)Npad, TMV, TK, CU_TENSOR_MAP_SWIZZLE_64B));
  DMO_TRY(make_map(ctx, &map_kl, Kl.p, (uint64_t)M * Pc_alloc, (uint64_t)Npad, TMV, TK, CU_TENSOR_MAP_SWIZZLE_64B));
  DMO_TRY(make_map(ctx, &map_lh, gp->Lhi.p, (uint64_t)M * Npad, (uint64_t)Npad, TN, TK, CU_TENSOR_MAP_SWIZZLE_64B));
  DMO_TRY(make_map(ctx, &map_ll, gp->Llo.p, (uint64_t)M * Npad, (uint64_t)Npad, TN, TK, CU_TENSOR_MAP_SWIZZLE_64B));
  DMO_CUDA(cudaFuncSetAttribute(gp_var_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM));
  const int64_t kplane = Pc_alloc * Npad;
  // K_* producer fused with the mean (d <= 32, M <= 6; DMO_GP_FUSED=0 keeps kstar_tensor_kernel + mean_split_kernel)
  // (per-dimension length scales with more than two objectives spill in the fused kernel: they keep the two-kernel route)
  const bool fused = !overlap && !mean_from_d && !(dbg & 8) && d <= KM_D && M <= 6 && (gp->isotropic || M <= 2) &&
                     !(getenv("DMO_GP_FUSED") && atoi(getenv("DMO_GP_FUSED")) == 0);
  DevBuf<double> mpart;
  if (fused) DMO_TRY(prepare_direct_state(ctx, gp));
  // producer side (K_* and the mean) on the second stream when overlapping, else in line
  cudaStream_t ps = overlap ? ctx->aux : ctx->stream;
  if (overlap) {
    DMO_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));  // allocations, memsets and Xn are ready
    DMO_CUDA(cudaStreamWaitEvent(ctx->aux, ctx->ev_fork, 0));
  }
  int64_t chunk = 0;
  for (int64_t p_base = 0; p_base < P; p_base += Pc_alloc, ++chunk) {
    const int64_t Pc = (P - p_base) < Pc_alloc ? (P - p_base) : Pc_alloc;
    const int64_t Pcpad = ceil_div(Pc, TMv) * TMv;
    unsigned* rdy = ready.p + chunk * n_pb_alloc;
    dim3 gk((unsigned)(Npad / (2 * KT_TN)), (unsigned)ceil_div(Pcpad, KT_TP));
    if (overlap && chunk > 0) {  // the K_* buffers are reused: the previous chunk's contraction must have drained them
      DMO_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
      DMO_CUDA(cudaStreamWaitEvent(ctx->aux, ctx->ev_fork, 0));
    }
    if (fused) {
      // K_* and the mean from one kernel (kstar_mean_kernel): K_* is written once and never read back for the mean
      int64_t n_per_block = Npad;
      const int64_t n_qb = Pcpad / KM_Q;
      const int64_t nsplit = pick_slices(n_qb, Npad, KF_NS, (int64_t)3 * ctx->sm_count, &n_per_block);
      DMO_TRY(mpart.alloc(ctx, (size_t)nsplit * M * Pcpad));
      dim3 gf((unsigned)nsplit, (unsigned)n_qb);
      const size_t smem = (size_t)M * 2 * KM_Q * KF_LD * sizeof(uint32_t);
      {
        ProfileScope ps_(ctx, "gp_kstar");
#define KF_LAUNCH(ISO_, MT_)                                                                                               \
  do {                                                                                                                     \
    DMO_CUDA(cudaFuncSetAttribute(kstar_mean_kernel<ISO_, MT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));  \
    DMO_LAUNCH((kstar_mean_kernel<ISO_, MT_>), gf, KM_T, smem, dXn, P, p_base, gp->Xtf.p, N, Npad, n_per_block, d,          \
               gp->kernel, gp->inv_ls.p, gp->constant.p, gp->Kexp.p, gp->CAf.p, kplane, Kh.p, Kl.p, mpart.p, Pcpad);         \
  } while (0)
#define KF_SWITCH(ISO_)                  \
  switch (M) {                           \
    case 1: KF_LAUNCH(ISO_, 1); break;   \
    case 2: KF_LAUNCH(ISO_, 2); break;   \
    case 3: KF_LAUNCH(ISO_, 3); break;   \
    case 4: KF_LAUNCH(ISO_, 4); break;   \
    case 5: KF_LAUNCH(ISO_, 5); break;   \
    default: KF_LAUNCH(ISO_, 6); break;  \
  }
        if (gp->isotropic) {
          KF_SWITCH(true)
        } else {
          KF_SWITCH(false)
        }
#undef KF_SWITCH
#undef KF_LAUNCH
      }
      DMO_LAUNCH(mean_finish_tc_kernel, (unsigned)ceil_div(Pc * M, 256), 256, 0, mpart.p, (int)nsplit, Pc, Pcpad, M, gp->ymean.p,
                 gp->ystd.p, p_base, d_mean);
    } else {
    {
        ProfileScope ps_(ctx, "gp_kstar", ps);
        const int dmax = d <= 32 ? 32 : 64;
        size_t smem = (size_t)(KT_TP * dmax + M * dmax + M) * sizeof(float);
  #define KSTAR_LAUNCH(ISO_, DM_)                                                                                   \
    DMO_LAUNCH_ON(ps, (kstar_tensor_kernel<ISO_, DM_>), gk, KT_TN, smem, dXn, P, p_base, Pcpad, gp->Xt.p, N, d, M,    \
                  gp->kernel, gp->inv_ls.p, gp->constant.p, gp->Kexp.p, Npad, kplane, Kh.p, Kl.p,                    \
                  (use_flags && d_var) ? rdy : nullptr)
        if (gp->isotropic) {
          if (d <= 32)
            KSTAR_LAUNCH(true, 32);
          else
            KSTAR_LAUNCH(true, 64);
        } else {
          if (d <= 32)
            KSTAR_LAUNCH(false, 32);
          else
            KSTAR_LAUNCH(false, 64);
        }
  #undef KSTAR_LAUNCH
      }
      if (overlap && (dbg & 4)) {  // diagnostics: the contraction waits for the whole K_* kernel by event, the mean still overlaps
        DMO_CUDA(cudaEventRecord(ctx->ev_fork, ctx->aux));
        DMO_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_fork, 0));
      }
      if (!(dbg & 8) && !mean_from_d) {
        ProfileScope ps_(ctx, "gp_mean", ps);
        DMO_LAUNCH_ON(ps, mean_split_kernel, (unsigned)ceil_div(Pc * M * 32, 256), 256, 0, Kh.p, Kl.p, Pc, N, Npad, kplane,
                      M, gp->Kexp.p, gp->alpha.p, gp->ymean.p, gp->ystd.p, p_base, d_mean);
      }
}
    if (overlap) DMO_CUDA(cudaEventRecord(ctx->ev_join, ctx->aux));
    if (d_var) {
      GemmParams prm;
      prm.M = M;
      prm.n_pb = (int)(Pcpad / TMV);
      prm.n_jt = n_jt;
      prm.n_q = n_q;
      prm.paired = version == 3;
      // halves: split the row blocks where the cumulative MMA count sum_{j < J} (j + 1) is closest to half of the total
      prm.j_split = n_jt;
      if (!prm.paired) {
        const int64_t tot = (int64_t)n_jt * (n_jt + 1) / 2;
        int64_t best_d = tot;
        for (int J = 0; J <= n_jt; ++J) {
          const int64_t dlt = llabs(2 * ((int64_t)J * (J + 1) / 2) - tot);
          if (dlt < best_d) {
            best_d = dlt;
            prm.j_split = J;
          }
        }
      }
      prm.k_rows = Pc_alloc;
      prm.l_rows = Npad;
      prm.inv_scale = gp->Lscale.p;
      prm.vnorm = vnorm.p;
      prm.vn_ld = Pc_alloc;
      prm.abort_flag = abort_flag.p;
      prm.zf = mean_from_d ? gp->Zf.p : nullptr;
      prm.mnorm = mean_from_d ? mnorm.p : nullptr;
      prm.ready = use_flags ? rdy : nullptr;
      prm.dbg = dbg;
      prm.ready_target = 8u * gk.x;  // KT_TP = 32 candidates per producer block: 8 tile rows x gk.x column blocks per 256
      const int n_work = prm.M * prm.n_pb * prm.n_q;
      const int grid = n_work < ctx->sm_count ? n_work : ctx->sm_count;
      {
        ProfileScope ps_(ctx, "gp_var");
        DMO_LAUNCH(gp_var_wgmma_kernel, grid, NTHREADS, GEMM_SMEM, map_kh, map_kl, map_lh, map_ll, prm);
      }
      DMO_LAUNCH(var_finish_tc_kernel, (unsigned)ceil_div(Pc * M, 256), 256, 0, vnorm.p, n_q, Pc, Pc_alloc, M,
                 gp->constant.p, gp->noise.p, gp->ystd.p, p_base, d_var);
      if (mean_from_d)
        DMO_LAUNCH(mean_finish_tc_kernel, (unsigned)ceil_div(Pc * M, 256), 256, 0, mnorm.p, n_q, Pc, Pc_alloc, M, gp->ymean.p,
                   gp->ystd.p, p_base, d_mean);
    }
    if (overlap) DMO_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));  // mean (and K_*) of this chunk done
    if ((dbg & 8) && !mean_from_d) {
      ProfileScope ps_(ctx, "gp_mean");
      DMO_LAUNCH(mean_split_kernel, (unsigned)ceil_div(Pc * M * 32, 256), 256, 0, Kh.p, Kl.p, Pc, N, Npad, kplane, M,
                 gp->Kexp.p, gp->alpha.p, gp->ymean.p, gp->ystd.p, p_base, d_mean);
    }
  }
  DMO_CHECK_LAUNCH();
  int h_abort = 0;
  DMO_CUDA(cudaMemcpyAsync(&h_abort, abort_flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(cudaStreamSynchronize(ctx->stream));
  if (h_abort)
    return dmo_fail(ctx, DMO_ERR_INTERNAL, "gp_predict(tensor): pipeline watchdog tripped (%s)",
                    h_abort == 2 ? "K_* producer did not deliver" : "mbarrier wait timed out");
  return DMO_OK;
}
