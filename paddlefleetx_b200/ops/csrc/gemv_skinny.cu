// Skinny GEMM for token-by-token decoding: y[m, n] = sum_k x[m, k] * W[n, k] (+ bias[n]),  m <= 8.
//
// With one to eight activation rows the tensor-core GEMM is idle 94+ % of a 128-row tile and, worse, covers the
// machine with only N/256 CTAs; the op is a pure weight stream.  This kernel is built for that: every warp owns
// kCols weight rows, streams them once with 16-byte no-allocate loads (two k-steps in flight per lane), keeps the
// few activation rows L1-resident, accumulates in fp32 and finishes with a shuffle reduction.  Decode GEMMs of the
// 6.7B model (N = 4096..16384, K = 4096..16384) then run at HBM speed instead of tile-quantised tensor-core speed.
// Reference: the decode path of GPTForGeneration (hybrid_model.py:1202-1339) issues cuBLAS GEMMs for these shapes.
#include "pfx_common.cuh"
#include "pfx_kernels.h"

namespace pfx {

namespace {

// Optional fusions for the decode step (every removed launch is ~5 us of a ~100 us layer): LayerNorm of the activation rows as
// a prologue (each CTA recomputes the two row statistics from the L1/L2-resident x — K reads against N*K/CTAs weight reads),
// GELU or SwiGLU, and "+ residual" in the finish.
template <typename T>
struct GemvExtra {
  const T* ln_w = nullptr;       // LayerNorm gamma (null = no norm)
  const T* ln_b = nullptr;
  float ln_eps = 1e-5f;
  const T* residual = nullptr;   // [M, N] ([M, N / 2] under SwiGLU) added after bias / activation
  int act = 0;                   // 0 none, 1 GELU(tanh), 2 SwiGLU over pair-interleaved rows: y[r, n / 2] = silu(v[r, n]) v[r, n + 1]
};

__device__ __forceinline__ float gemv_gelu_tanh(float x) {
  return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

// block = 8 warps arranged as (8 / kSplit) column groups x kSplit K-slices; a column group owns kCols weight rows.  kSwiglu selects the
// SwiGLU finish (act 2) at compile time, so that the other instantiations keep their code and registers.
template <typename T, int kRows, int kCols, int kSplit, bool kSwiglu>
__global__ void __launch_bounds__(256) gemv_skinny_kernel(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ bias,
                                                          T* __restrict__ y, int N, int K, const GemvExtra<T> ex) {
  constexpr int kGroups = 8 / kSplit;
  __shared__ float red[8][kCols * kRows];
  __shared__ float s_stat[2][kRows];
  __shared__ float s_part[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (ex.ln_w != nullptr) {      // row mean / rstd (two passes, fp32) — uniform branch
#pragma unroll 1
    for (int r = 0; r < kRows; ++r) {
      float mean = 0.f;
#pragma unroll 1
      for (int pass = 0; pass < 2; ++pass) {
        float s = 0.f;
        for (int i = threadIdx.x; i < K; i += 256) {
          const float v = to_f32<T>(x[(size_t)r * K + i]) - mean;
          s += pass ? v * v : v;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) s_part[wid] = s;
        __syncthreads();
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += s_part[i];
        __syncthreads();
        if (pass == 0) mean = t / K;
        else if (threadIdx.x == 0) { s_stat[0][r] = mean; s_stat[1][r] = rsqrtf(t / K + ex.ln_eps); }
      }
    }
    __syncthreads();
  }
  const int group = wid / kSplit, slice = wid % kSplit;
  const int n0 = (blockIdx.x * kGroups + group) * kCols;
  float acc[kCols][kRows];
#pragma unroll
  for (int c = 0; c < kCols; ++c)
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[c][r] = 0.f;
  if (n0 < N) {
    const uint4* wp[kCols];
#pragma unroll
    for (int c = 0; c < kCols; ++c) wp[c] = reinterpret_cast<const uint4*>(w + (size_t)min(n0 + c, N - 1) * K);
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    const int kvec = K >> 3;                              // 8 elements per 16-byte vector
    const int per = ((kvec + kSplit - 1) / kSplit + 31) / 32 * 32;
    const int v_lo = slice * per, v_hi = min(kvec, v_lo + per);
    constexpr int kU = 4;                                 // k-steps in flight per lane: kU * kCols 16-byte loads
    for (int v0 = v_lo + lane; v0 < v_hi; v0 += 32 * kU) {
      uint4 wr[kU][kCols];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int v = v0 + u * 32;
#pragma unroll
        for (int c = 0; c < kCols; ++c) wr[u][c] = v < v_hi ? ld_stream(wp[c] + v) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int v = v0 + u * 32;
        if (v >= v_hi) break;
        float xf[kRows][8];
#pragma unroll
        for (int r = 0; r < kRows; ++r) unpack8<T>(__ldg(xp + (size_t)r * kvec + v), xf[r]);
        if (ex.ln_w != nullptr) {
          float gw[8], gb[8];
          unpack8<T>(__ldg(reinterpret_cast<const uint4*>(ex.ln_w) + v), gw);
          unpack8<T>(__ldg(reinterpret_cast<const uint4*>(ex.ln_b) + v), gb);
#pragma unroll
          for (int r = 0; r < kRows; ++r) {
            const float mu = s_stat[0][r], rs = s_stat[1][r];
#pragma unroll
            for (int j = 0; j < 8; ++j) xf[r][j] = (xf[r][j] - mu) * rs * gw[j] + gb[j];
          }
        }
#pragma unroll
        for (int c = 0; c < kCols; ++c) {
          float wf[8];
          unpack8<T>(wr[u][c], wf);
#pragma unroll
          for (int r = 0; r < kRows; ++r)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[c][r] = fmaf(wf[j], xf[r][j], acc[c][r]);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kCols; ++c)
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      float v = acc[c][r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[wid][c * kRows + r] = v;
    }
  __syncthreads();
  if constexpr (kSwiglu) {
    // SwiGLU: a column group starts on an even weight row, so each of its column pairs (gate, up) is finished by one thread
    const int N2 = N >> 1;
    for (int t = threadIdx.x; t < kGroups * (kCols / 2) * kRows; t += blockDim.x) {
      const int g = t / ((kCols / 2) * kRows), pr = t % ((kCols / 2) * kRows), c = 2 * (pr / kRows), r = pr % kRows;
      const int n = (blockIdx.x * kGroups + g) * kCols + c;
      if (n >= N) continue;
      float a = bias ? to_f32<T>(bias[n]) : 0.f, b = bias ? to_f32<T>(bias[n + 1]) : 0.f;
#pragma unroll
      for (int s2 = 0; s2 < kSplit; ++s2) { a += red[g * kSplit + s2][c * kRows + r]; b += red[g * kSplit + s2][(c + 1) * kRows + r]; }
      float v = a * (1.f / (1.f + __expf(-a))) * b;              // the form of bias_swiglu_kernel (norm_act.cu)
      if (ex.residual != nullptr) v += to_f32<T>(ex.residual[(size_t)r * N2 + (n >> 1)]);
      y[(size_t)r * N2 + (n >> 1)] = from_f32<T>(v);
    }
  } else {
    // one thread per (group, column, row) finishes the K-slice sum and writes the output
    for (int t = threadIdx.x; t < kGroups * kCols * kRows; t += blockDim.x) {
      const int g = t / (kCols * kRows), cr = t % (kCols * kRows), c = cr / kRows, r = cr % kRows;
      const int n = (blockIdx.x * kGroups + g) * kCols + c;
      if (n >= N) continue;
      float v = bias ? to_f32<T>(bias[n]) : 0.f;
#pragma unroll
      for (int s2 = 0; s2 < kSplit; ++s2) v += red[g * kSplit + s2][cr];
      if (ex.act == 1) v = gemv_gelu_tanh(v);
      if (ex.residual != nullptr) v += to_f32<T>(ex.residual[(size_t)r * N + n]);
      y[(size_t)r * N + n] = from_f32<T>(v);
    }
  }
}

template <typename T, int kRows, int kCols, int kSplit>
cudaError_t launch_cfg(const T* x, const T* w, const T* bias, T* y, int N, int K, const GemvExtra<T>& ex, cudaStream_t st) {
  constexpr int kGroups = 8 / kSplit;
  const int groups = (N + kCols - 1) / kCols;
  if (ex.act == 2) gemv_skinny_kernel<T, kRows, kCols, kSplit, true><<<(groups + kGroups - 1) / kGroups, 256, 0, st>>>(x, w, bias, y, N, K, ex);
  else gemv_skinny_kernel<T, kRows, kCols, kSplit, false><<<(groups + kGroups - 1) / kGroups, 256, 0, st>>>(x, w, bias, y, N, K, ex);
  return cudaGetLastError();
}

int g_gemv_cols = 0, g_gemv_split = 0;      // tuning overrides (0 = heuristic), see gemv_set_tuning

template <typename T, int kRows>
cudaError_t launch_rows(const T* x, const T* w, const T* bias, T* y, int N, int K, int num_sms, const GemvExtra<T>& ex, cudaStream_t st) {
  // aim for >= ~24 warps per SM of work; split K across the warps of a block when N alone does not provide that
  const long target = (long)num_sms * 24;
  int cols = (kRows == 1) ? ((N / 4 < target / 8) ? 2 : 4) : ((kRows <= 2 || N / 4 < target) ? 2 : 4);
  if (g_gemv_cols == 2 || g_gemv_cols == 4) cols = g_gemv_cols;
  const long groups = (N + cols - 1) / cols;
  int split = 1;
  if (kRows == 1) {
    // 4 rows per warp with the block's warps split 2-way over K; very long K (FFN2) gets 8 slices
    split = K >= 16384 ? 8 : (K >= 2048 ? 2 : 1);
  } else {
    while (split < 8 && groups * split < target && K / (split * 2) >= 1024) split *= 2;
  }
  if (g_gemv_split == 1 || g_gemv_split == 2 || g_gemv_split == 4 || g_gemv_split == 8) split = g_gemv_split;
#define PFX_GV(C, S) return launch_cfg<T, kRows, C, S>(x, w, bias, y, N, K, ex, st)
  if (cols == 2) { if (split == 1) PFX_GV(2, 1); if (split == 2) PFX_GV(2, 2); if (split == 4) PFX_GV(2, 4); PFX_GV(2, 8); }
  if (split == 1) PFX_GV(4, 1); if (split == 2) PFX_GV(4, 2); if (split == 4) PFX_GV(4, 4); PFX_GV(4, 8);
#undef PFX_GV
}

// ---------------------------------------------------------------------------------------------------------------- W8A8 variant
// int8 weights (per-output-channel scale) x int8 activations (per-row scale): half the weight bytes of the bf16 stream, dot
// products on dp4a, dequantisation + bias in the finish.  Same warp layout as above (column groups x K-slices).  T (bf16 / fp16) is the
// dtype of y and bias.
template <typename T, int kRows, int kCols, int kSplit>
__global__ void __launch_bounds__(256) gemv_w8a8_kernel(const int8_t* __restrict__ x, const int8_t* __restrict__ w, const float* __restrict__ xs,
                                                        const float* __restrict__ ws, const T* __restrict__ bias,
                                                        T* __restrict__ y, int N, int K) {
  constexpr int kGroups = 8 / kSplit;
  __shared__ int red[8][kCols * kRows];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int group = wid / kSplit, slice = wid % kSplit;
  const int n0 = (blockIdx.x * kGroups + group) * kCols;
  int acc[kCols][kRows];
#pragma unroll
  for (int c = 0; c < kCols; ++c)
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[c][r] = 0;
  if (n0 < N) {
    const int4* wp[kCols];
#pragma unroll
    for (int c = 0; c < kCols; ++c) wp[c] = reinterpret_cast<const int4*>(w + (size_t)min(n0 + c, N - 1) * K);
    const int4* xp = reinterpret_cast<const int4*>(x);
    const int kvec = K >> 4;                              // 16 int8 per 16-byte vector
    const int per = ((kvec + kSplit - 1) / kSplit + 31) / 32 * 32;
    const int v_lo = slice * per, v_hi = min(kvec, v_lo + per);
    constexpr int kU = 4;
    for (int v0 = v_lo + lane; v0 < v_hi; v0 += 32 * kU) {
      int4 wr[kU][kCols];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int v = v0 + u * 32;
#pragma unroll
        for (int c = 0; c < kCols; ++c) {
          if (v < v_hi) {
            const uint4 t = ld_stream(reinterpret_cast<const uint4*>(wp[c]) + v);
            wr[u][c] = make_int4((int)t.x, (int)t.y, (int)t.z, (int)t.w);
          } else {
            wr[u][c] = make_int4(0, 0, 0, 0);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int v = v0 + u * 32;
        if (v >= v_hi) break;
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          const int4 xv = __ldg(xp + (size_t)r * kvec + v);
#pragma unroll
          for (int c = 0; c < kCols; ++c) {
            int a = acc[c][r];
            a = __dp4a(wr[u][c].x, xv.x, a);
            a = __dp4a(wr[u][c].y, xv.y, a);
            a = __dp4a(wr[u][c].z, xv.z, a);
            a = __dp4a(wr[u][c].w, xv.w, a);
            acc[c][r] = a;
          }
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kCols; ++c)
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      int v = acc[c][r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[wid][c * kRows + r] = v;
    }
  __syncthreads();
  for (int t = threadIdx.x; t < kGroups * kCols * kRows; t += blockDim.x) {
    const int g = t / (kCols * kRows), cr = t % (kCols * kRows), c = cr / kRows, r = cr % kRows;
    const int n = (blockIdx.x * kGroups + g) * kCols + c;
    if (n >= N) continue;
    int v = 0;
#pragma unroll
    for (int s2 = 0; s2 < kSplit; ++s2) v += red[g * kSplit + s2][cr];
    const float f = (float)v * xs[r] * ws[n] + (bias ? to_f32<T>(bias[n]) : 0.f);
    y[(size_t)r * N + n] = from_f32<T>(f);
  }
}

template <typename T, int kRows>
cudaError_t launch_w8a8_rows(const int8_t* x, const int8_t* w, const float* xs, const float* ws, const T* bias, T* y, int N, int K, int num_sms,
                             cudaStream_t st) {
  const long target = (long)num_sms * 24;
  const long groups = (N + 1) / 2;
  int split = 1;
  while (split < 8 && groups * split < target && K / (split * 2) >= 2048) split *= 2;
#define PFX_GW(S)                                                                                                             \
  do {                                                                                                                        \
    constexpr int kG = 8 / S;                                                                                                 \
    gemv_w8a8_kernel<T, kRows, 2, S><<<(int)((groups + kG - 1) / kG), 256, 0, st>>>(x, w, xs, ws, bias, y, N, K);                  \
    return cudaGetLastError();                                                                                                \
  } while (0)
  if (split == 1) PFX_GW(1);
  if (split == 2) PFX_GW(2);
  if (split == 4) PFX_GW(4);
  PFX_GW(8);
#undef PFX_GW
}

template <typename T>
cudaError_t launch(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int num_sms, const void* ln_w, const void* ln_b,
                   float ln_eps, const void* residual, int act, cudaStream_t st) {
  const T *xx = (const T*)x, *ww = (const T*)w, *bb = (const T*)bias;
  T* yy = (T*)y;
  GemvExtra<T> ex;
  ex.ln_w = (const T*)ln_w; ex.ln_b = (const T*)ln_b; ex.ln_eps = ln_eps; ex.residual = (const T*)residual; ex.act = act;
  switch (M) {
    case 1: return launch_rows<T, 1>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 2: return launch_rows<T, 2>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 3: return launch_rows<T, 3>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 4: return launch_rows<T, 4>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 5: return launch_rows<T, 5>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 6: return launch_rows<T, 6>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 7: return launch_rows<T, 7>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    case 8: return launch_rows<T, 8>(xx, ww, bb, yy, N, K, num_sms, ex, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t gemv_skinny(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int dtype, int num_sms, cudaStream_t st,
                        const void* ln_w, const void* ln_b, float ln_eps, const void* residual, int act) {
  if (M < 1 || M > 8 || K % 8 || ((ln_w == nullptr) != (ln_b == nullptr)) || (act == 2 && N % 2)) return cudaErrorInvalidValue;
  if (dtype == 1) return launch<__nv_bfloat16>(x, w, bias, y, M, N, K, num_sms, ln_w, ln_b, ln_eps, residual, act, st);
  if (dtype == 0) return launch<__half>(x, w, bias, y, M, N, K, num_sms, ln_w, ln_b, ln_eps, residual, act, st);
  return cudaErrorInvalidValue;
}

void gemv_set_tuning(int cols, int split) { g_gemv_cols = cols; g_gemv_split = split; }

namespace {
template <typename T>
cudaError_t launch_w8a8(const int8_t* x, const int8_t* w, const float* xs, const float* ws, const T* bb, T* yy, int M, int N, int K, int num_sms,
                        cudaStream_t st) {
  switch (M) {
    case 1: return launch_w8a8_rows<T, 1>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 2: return launch_w8a8_rows<T, 2>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 3: return launch_w8a8_rows<T, 3>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 4: return launch_w8a8_rows<T, 4>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 5: return launch_w8a8_rows<T, 5>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 6: return launch_w8a8_rows<T, 6>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    case 7: return launch_w8a8_rows<T, 7>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
    default: return launch_w8a8_rows<T, 8>(x, w, xs, ws, bb, yy, N, K, num_sms, st);
  }
}
}  // namespace

cudaError_t gemv_w8a8(const void* x, const void* w, const float* xs, const float* ws, const void* bias, void* y, int M, int N, int K, int num_sms,
                      cudaStream_t st, int dtype) {
  if (M < 1 || M > 8 || K % 16) return cudaErrorInvalidValue;
  const int8_t *xx = (const int8_t*)x, *ww = (const int8_t*)w;
  if (dtype == 1) return launch_w8a8<__nv_bfloat16>(xx, ww, xs, ws, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, M, N, K, num_sms, st);
  if (dtype == 0) return launch_w8a8<__half>(xx, ww, xs, ws, (const __half*)bias, (__half*)y, M, N, K, num_sms, st);
  return cudaErrorInvalidValue;
}

}  // namespace pfx
