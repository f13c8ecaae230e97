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
