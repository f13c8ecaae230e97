// Device-wide sort / scan primitives (CUB, header-only, compiled into this library).
// CUB is included only in this translation unit to keep build times down.
#include <cub/cub.cuh>

#include "common.cuh"

int prim_sort_pairs_u64(dmo_ctx* ctx, const uint64_t* kin, uint64_t* kout, const uint32_t* vin,
                        uint32_t* vout, int64_t n, int begin_bit, int end_bit) {
  if (n <= 0) return DMO_OK;
  size_t tmp = 0;
  DMO_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, kin, kout, vin, vout, (int)n, begin_bit, end_bit,
                                           ctx->stream));
  DevBuf<uint8_t> t;
  DMO_TRY(t.alloc(ctx, tmp));
  DMO_CUDA(cub::DeviceRadixSort::SortPairs(t.p, tmp, kin, kout, vin, vout, (int)n, begin_bit, end_bit,
                                           ctx->stream));
  ctx->launches += 1 + (end_bit - begin_bit + 7) / 8;  // histogram + one onesweep pass per digit
  return DMO_OK;
}

int prim_sort_pairs_u32(dmo_ctx* ctx, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                        uint32_t* vout, int64_t n, int begin_bit, int end_bit) {
  if (n <= 0) return DMO_OK;
  size_t tmp = 0;
  DMO_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, kin, kout, vin, vout, (int)n, begin_bit, end_bit,
                                           ctx->stream));
  DevBuf<uint8_t> t;
  DMO_TRY(t.alloc(ctx, tmp));
  DMO_CUDA(cub::DeviceRadixSort::SortPairs(t.p, tmp, kin, kout, vin, vout, (int)n, begin_bit, end_bit,
                                           ctx->stream));
  ctx->launches += 1 + (end_bit - begin_bit + 7) / 8;
  return DMO_OK;
}

int prim_inclusive_sum_u32(dmo_ctx* ctx, const uint32_t* in, uint32_t* out, int64_t n) {
  if (n <= 0) return DMO_OK;
  size_t tmp = 0;
  DMO_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp, in, out, (int)n, ctx->stream));
  DevBuf<uint8_t> t;
  DMO_TRY(t.alloc(ctx, tmp));
  DMO_CUDA(cub::DeviceScan::InclusiveSum(t.p, tmp, in, out, (int)n, ctx->stream));
  ctx->launches += 2;
  return DMO_OK;
}

int prim_exclusive_sum_i32(dmo_ctx* ctx, const int32_t* in, int32_t* out, int64_t n) {
  if (n <= 0) return DMO_OK;
  size_t tmp = 0;
  DMO_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, in, out, (int)n, ctx->stream));
  DevBuf<uint8_t> t;
  DMO_TRY(t.alloc(ctx, tmp));
  DMO_CUDA(cub::DeviceScan::ExclusiveSum(t.p, tmp, in, out, (int)n, ctx->stream));
  ctx->launches += 2;
  return DMO_OK;
}

struct MinF64 {
  __device__ __forceinline__ double operator()(double a, double b) const { return b < a ? b : a; }
};

int prim_inclusive_min_f64(dmo_ctx* ctx, const double* in, double* out, int64_t n) {
  if (n <= 0) return DMO_OK;
  size_t tmp = 0;
  DMO_CUDA(cub::DeviceScan::InclusiveScan(nullptr, tmp, in, out, MinF64{}, (int)n, ctx->stream));
  DevBuf<uint8_t> t;
  DMO_TRY(t.alloc(ctx, tmp));
  DMO_CUDA(cub::DeviceScan::InclusiveScan(t.p, tmp, in, out, MinF64{}, (int)n, ctx->stream));
  ctx->launches += 2;
  return DMO_OK;
}

__global__ void iota_kernel(uint32_t* out, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint32_t)i;
}

int prim_iota_u32(dmo_ctx* ctx, uint32_t* out, int64_t n) {
  if (n <= 0) return DMO_OK;
  DMO_LAUNCH(iota_kernel, (unsigned)ceil_div(n, 256), 256, 0, out, n);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

__global__ void gather_u32_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, int64_t n,
                                  uint32_t* __restrict__ out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = src[idx[p]];
}

int prim_gather_u32(dmo_ctx* ctx, const uint32_t* src, const uint32_t* idx, int64_t n, uint32_t* out) {
  if (n <= 0) return DMO_OK;
  DMO_LAUNCH(gather_u32_kernel, (unsigned)ceil_div(n, 256), 256, 0, src, idx, n, out);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

__global__ void round_f32_kernel(double* a, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (double)(float)a[i];
}

int prim_round_f32(dmo_ctx* ctx, double* a, int64_t n) {
  if (n <= 0) return DMO_OK;
  DMO_LAUNCH(round_f32_kernel, (unsigned)ceil_div(n, 256), 256, 0, a, n);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

__global__ void col_key_kernel(const double* __restrict__ F, int64_t n, int M, int j, uint64_t* __restrict__ keys,
                               uint32_t* __restrict__ idx) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    keys[i] = f64_to_ordered(F[i * M + j]);
    idx[i] = (uint32_t)i;
  }
}

int prim_col_keys(dmo_ctx* ctx, const double* dF, int64_t n, int M, int j, uint64_t* keys, uint32_t* idx) {
  DMO_LAUNCH(col_key_kernel, (unsigned)ceil_div(n, 256), 256, 0, dF, n, M, j, keys, idx);
  return DMO_OK;
}

int prim_sort_by_column(dmo_ctx* ctx, const double* dF, int64_t n, int M, int j, DevBuf<uint32_t>& sidx) {
  DevBuf<uint64_t> k0, k1;
  DevBuf<uint32_t> i0;
  DMO_TRY(k0.alloc(ctx, n));
  DMO_TRY(k1.alloc(ctx, n));
  DMO_TRY(i0.alloc(ctx, n));
  DMO_TRY(sidx.alloc(ctx, n));
  DMO_TRY(prim_col_keys(ctx, dF, n, M, j, k0.p, i0.p));
  return prim_sort_pairs_u64(ctx, k0.p, k1.p, i0.p, sidx.p, n, 0, 64);
}
