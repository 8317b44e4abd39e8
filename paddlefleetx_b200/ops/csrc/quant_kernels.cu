// Dynamic quantisation kernels feeding the 8-bit wgmma GEMMs: per-row (per-token) abs-max scaling to int8 or fp8
// e4m3 in one pass (row kept in registers), optional SmoothQuant per-channel divisor folded in.
#include <cuda_fp8.h>

#include "pfx_common.cuh"
#include "pfx_kernels.h"

namespace pfx {

// q[r, :] = round(x[r, :] / smooth[:] / scale[r]),  scale[r] = absmax(x[r, :] / smooth) / QMAX
template <typename T, bool kFp8>
__global__ void quantize_rows_kernel(const T* __restrict__ x, const float* __restrict__ smooth, uint8_t* __restrict__ q, float* __restrict__ scale,
                                     int cols) {
  __shared__ float scratch[33];
  const int row = blockIdx.x;
  const int nvec = cols >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * cols);
  constexpr int kV = 4;
  float v[kV][8];
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < kV; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      unpack8<T>(ld_stream(xr + vi), v[i]);
      if (smooth) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] /= smooth[vi * 8 + j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[i][j]));
    }
  }
  amax = block_max(amax, scratch);
  const float qmax = kFp8 ? 448.f : 127.f;
  const float s = amax > 0.f ? amax / qmax : 1.f;
  const float inv = 1.f / s;
  if (threadIdx.x == 0) scale[row] = s;
  uint2* qr = reinterpret_cast<uint2*>(q + (size_t)row * cols);
#pragma unroll
  for (int i = 0; i < kV; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      uint8_t o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = v[i][j] * inv;
        if (kFp8) o[j] = (uint8_t)__nv_cvt_float_to_fp8(t, __NV_SATFINITE, __NV_E4M3);
        else o[j] = (uint8_t)(int8_t)max(-127, min(127, __float2int_rn(t)));
      }
      qr[vi] = *reinterpret_cast<const uint2*>(o);
    }
  }
}

cudaError_t quantize_rows(const void* x, const float* smooth, void* q, float* scale, int rows, int cols, int dtype, bool fp8, cudaStream_t st) {
  if (cols % 8 || cols > 32768) return cudaErrorInvalidValue;
  if (!rows) return cudaSuccess;
  int threads = ((cols / 8 + 3) / 4 + 31) / 32 * 32;
  if (threads < 32) threads = 32;
#define PFX_Q(T, F) quantize_rows_kernel<T, F><<<rows, threads, 0, st>>>((const T*)x, smooth, (uint8_t*)q, scale, cols)
  if (dtype == 1) { if (fp8) PFX_Q(__nv_bfloat16, true); else PFX_Q(__nv_bfloat16, false); }
  else { if (fp8) PFX_Q(__half, true); else PFX_Q(__half, false); }
#undef PFX_Q
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------- MX fp8
// x [rows, K] (bf16 / fp16) -> q e4m3 [rows, K] + E8M0 block scales, one per 32 consecutive K-elements of a row, chosen as the
// smallest power of two that brings the block's maximum inside the e4m3 range (448).  The scale bytes are written directly in the
// order the MX GEMM reads (gemm_lowp_sm90.cu): atom (row / 128, k / 128) of 512 bytes, byte
// (row % 32) * 16 + ((row % 128) / 32) * 4 + (k / 32) % 4.  One thread per 32-element block: 64 B in, 32 B + 1 B out.
namespace {
template <typename T>
__global__ void __launch_bounds__(256) quantize_mxfp8_kernel(const T* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf, int rows, int K) {
  const int kblocks = K / 32;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * kblocks) return;
  const int kb = (int)(i % kblocks);
  const int r = (int)(i / kblocks);
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)r * K + kb * 32);
  float v[32];
#pragma unroll
  for (int j = 0; j < 4; ++j) unpack8<T>(__ldg(src + j), *reinterpret_cast<float(*)[8]>(v + 8 * j));
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) amax = fmaxf(amax, fabsf(v[j]));
  int e_unb = -127;
  if (amax > 0.f) {
    int ex;
    const float m = frexpf(amax * (1.f / 448.f), &ex);       // amax / 448 = m * 2^ex, m in [0.5, 1)
    e_unb = (m == 0.5f) ? ex - 1 : ex;                       // ceil(log2(amax / 448))
    e_unb = max(-127, min(127, e_unb));
  }
  const float inv = exp2f((float)-e_unb);
  uint32_t w[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * j] * inv, v[4 * j + 1] * inv), __NV_SATFINITE, __NV_E4M3);
    const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * j + 2] * inv, v[4 * j + 3] * inv), __NV_SATFINITE, __NV_E4M3);
    w[j] = (uint32_t)lo | ((uint32_t)hi << 16);
  }
  uint4* dst = reinterpret_cast<uint4*>(q + (size_t)r * K + kb * 32);
  dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
  dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
  const size_t atom = (size_t)(r / 128) * (K / 128) + kb / 4;
  sf[atom * 512 + (size_t)(r % 32) * 16 + ((r % 128) / 32) * 4 + (kb % 4)] = (uint8_t)(e_unb + 127);
}
}  // namespace

cudaError_t quantize_mxfp8(const void* x, void* q, void* sf, int rows, int K, int dtype, cudaStream_t st) {
  if (K % 128 || rows < 1) return cudaErrorInvalidValue;
  const int64_t n = (int64_t)rows * (K / 32);
  const unsigned grid = (unsigned)((n + 255) / 256);
  if (dtype == 1) quantize_mxfp8_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, (uint8_t*)sf, rows, K);
  else if (dtype == 0) quantize_mxfp8_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (uint8_t*)q, (uint8_t*)sf, rows, K);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace pfx
