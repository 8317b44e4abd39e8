// Bandwidth-bound fused kernels: LayerNorm / RMSNorm fwd+bwd, bias+GELU fwd+bwd, bias+SwiGLU fwd+bwd,
// bias + Philox-dropout + residual fwd (mask regenerated in bwd, never stored), column sums.
// Reference call sites: L8 (LayerNorm), L10 (dropout+residual), L3 (GELU) in SURVEY §2.6 — Paddle
// runs each as a separate library kernel; here every one is a single pass over HBM with 128-bit IO.
#include "pfx_common.cuh"
#include "pfx_kernels.h"
#include "pfx_ptx.cuh"

namespace pfx {

constexpr int kVPT = 4;  // 8-element vectors per thread kept in registers

// --------------------------------------------------------------------------- LayerNorm / RMSNorm fwd
template <typename T, bool kRms>
__global__ void norm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ b, T* __restrict__ y,
                                float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int cols, float eps) {
  __shared__ float scratch[33];
  const int nvec = cols >> 3;
  const int row = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * cols);
  float v[kVPT][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kVPT; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      unpack8<T>(ld_stream(xr + vi), v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += kRms ? v[i][j] * v[i][j] : v[i][j];
    }
  }
  float mean = 0.f, rstd;
  if (kRms) {
    rstd = rsqrtf(block_sum(s, scratch) / cols + eps);
  } else {
    mean = block_sum(s, scratch) / cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kVPT; ++i) {
      const int vi = threadIdx.x + i * blockDim.x;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
      }
    }
    rstd = rsqrtf(block_sum(q, scratch) / cols + eps);
  }
  if (threadIdx.x == 0) { if (mean_out) mean_out[row] = mean; rstd_out[row] = rstd; }
  uint4* yr = reinterpret_cast<uint4*>(y + (size_t)row * cols);
#pragma unroll
  for (int i = 0; i < kVPT; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      float wv[8], bv[8], o[8];
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(w) + vi), wv);
      if (!kRms && b) unpack8<T>(__ldg(reinterpret_cast<const uint4*>(b) + vi), bv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = (v[i][j] - mean) * rstd * wv[j];
        if (!kRms && b) o[j] += bv[j];
      }
      st_stream(yr + vi, pack8<T>(o));
    }
  }
}

// --------------------------------------------------------------------------- LayerNorm / RMSNorm bwd
// Persistent CTAs grid-stride over rows.  Register budget is what makes or breaks this kernel (an earlier version was
// compiled under __launch_bounds__(1024) and spilled 128-624 B/thread): x, dy and gamma stay PACKED (4 registers per
// 8 elements) and are unpacked twice instead of keeping fp32 copies of xhat and dy*gamma, the block size is a template
// parameter so ptxas gets the real bound, the next row's x / dy are prefetched before the current row's reductions so
// the CTA always has loads in flight, and the two row sums share one barrier pair.  dgamma / dbeta partials live in
// registers and are flushed once per CTA.
__device__ __forceinline__ float2 block_sum2(float a, float b, float2* scratch) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  a = warp_sum(a); b = warp_sum(b);
  __syncthreads();
  if (lane == 0) scratch[w] = make_float2(a, b);
  __syncthreads();
  float2 t = (lane < nw) ? scratch[lane] : make_float2(0.f, 0.f);
  t.x = warp_sum(t.x); t.y = warp_sum(t.y);
  return t;
}

template <typename T, bool kRms, int kVPT, int kThreads>
__global__ void __launch_bounds__(kThreads) norm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ w,
                                const float* __restrict__ mean_in, const float* __restrict__ rstd_in, T* __restrict__ dx,
                                float* __restrict__ dw_part, float* __restrict__ db_part, int rows, int cols, const T* __restrict__ dres) {
  __shared__ float2 scratch[33];
  const int nvec = cols >> 3;
  float dwp[kVPT][8], dbp[kVPT][8];
  uint4 wraw[kVPT], xn[kVPT], gn[kVPT];
#pragma unroll
  for (int i = 0; i < kVPT; ++i) {
    const int vi = threadIdx.x + i * kThreads;
#pragma unroll
    for (int j = 0; j < 8; ++j) { dwp[i][j] = 0.f; dbp[i][j] = 0.f; }
    wraw[i] = vi < nvec ? __ldg(reinterpret_cast<const uint4*>(w) + vi) : make_uint4(0, 0, 0, 0);
    xn[i] = gn[i] = make_uint4(0, 0, 0, 0);
  }
  int row = blockIdx.x;
  if (row < rows) {
#pragma unroll
    for (int i = 0; i < kVPT; ++i) {
      const int vi = threadIdx.x + i * kThreads;
      if (vi < nvec) {
        xn[i] = ld_stream(reinterpret_cast<const uint4*>(x + (size_t)row * cols) + vi);
        gn[i] = ld_stream(reinterpret_cast<const uint4*>(dy + (size_t)row * cols) + vi);
      }
    }
  }
  for (; row < rows; row += gridDim.x) {
    uint4 xc[kVPT], gc[kVPT];
#pragma unroll
    for (int i = 0; i < kVPT; ++i) { xc[i] = xn[i]; gc[i] = gn[i]; }
    const int nrow = row + gridDim.x;
    if (nrow < rows) {                            // prefetch: in flight across this row's reductions and stores
#pragma unroll
      for (int i = 0; i < kVPT; ++i) {
        const int vi = threadIdx.x + i * kThreads;
        if (vi < nvec) {
          xn[i] = ld_stream(reinterpret_cast<const uint4*>(x + (size_t)nrow * cols) + vi);
          gn[i] = ld_stream(reinterpret_cast<const uint4*>(dy + (size_t)nrow * cols) + vi);
        }
      }
    }
    const float mean = kRms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < kVPT; ++i) {
      const int vi = threadIdx.x + i * kThreads;
      if (vi < nvec) {
        float xv[8], gv[8], wv[8];
        unpack8<T>(xc[i], xv);
        unpack8<T>(gc[i], gv);
        unpack8<T>(wraw[i], wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xv[j] - mean) * rstd;
          const float gw = gv[j] * wv[j];
          s1 += gw;
          s2 += gw * xh;
          dwp[i][j] += gv[j] * xh;
          if (!kRms) dbp[i][j] += gv[j];
        }
      }
    }
    const float2 sums = block_sum2(s1, s2, scratch);
    const float c1 = kRms ? 0.f : sums.x / cols;
    const float c2 = sums.y / cols;
    uint4* dxr = reinterpret_cast<uint4*>(dx + (size_t)row * cols);
#pragma unroll
    for (int i = 0; i < kVPT; ++i) {
      const int vi = threadIdx.x + i * kThreads;
      if (vi < nvec) {
        float xv[8], gv[8], wv[8], o[8];
        unpack8<T>(xc[i], xv);
        unpack8<T>(gc[i], gv);
        unpack8<T>(wraw[i], wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (gv[j] * wv[j] - c1 - (xv[j] - mean) * rstd * c2);
        if (dres != nullptr) {      // pre-norm block: the residual branch's gradient joins here instead of in a separate add pass
          float rv[8];
          unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(dres + (size_t)row * cols) + vi), rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rv[j];
        }
        st_stream(dxr + vi, pack8<T>(o));
      }
    }
  }
#pragma unroll
  for (int i = 0; i < kVPT; ++i) {
    const int vi = threadIdx.x + i * kThreads;
    if (vi < nvec) {
      float4* dwo = reinterpret_cast<float4*>(dw_part + (size_t)blockIdx.x * cols + vi * 8);
      dwo[0] = make_float4(dwp[i][0], dwp[i][1], dwp[i][2], dwp[i][3]);
      dwo[1] = make_float4(dwp[i][4], dwp[i][5], dwp[i][6], dwp[i][7]);
      if (!kRms) {
        float4* dbo = reinterpret_cast<float4*>(db_part + (size_t)blockIdx.x * cols + vi * 8);
        dbo[0] = make_float4(dbp[i][0], dbp[i][1], dbp[i][2], dbp[i][3]);
        dbo[1] = make_float4(dbp[i][4], dbp[i][5], dbp[i][6], dbp[i][7]);
      }
    }
  }
}

// out[c] = sum_r part[r, c]   (fp32 partials -> T or fp32); block = 32 column lanes x 8 part lanes
template <typename TOut>
__global__ void reduce_partials_kernel(const float* __restrict__ part, TOut* __restrict__ out, int nparts, int cols) {
  __shared__ float red[8][33];
  const int lc = threadIdx.x & 31, lr = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lc;
  float s = 0.f;
  if (c < cols)
    for (int r = lr; r < nparts; r += 8) s += part[(size_t)r * cols + c];
  red[lr][lc] = s;
  __syncthreads();
  if (lr == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) t += red[r][lc];
    out[c] = from_f32<TOut>(t);
  }
}

static int norm_threads_vpt(int cols, int vpt) {
  const int nvec = cols / 8;
  int t = (nvec + vpt - 1) / vpt;
  t = ((t + 31) / 32) * 32;
  return t < 32 ? 32 : t;
}

static int norm_threads(int cols) {
  const int nvec = cols / 8;
  int t = (nvec + kVPT - 1) / kVPT;
  t = ((t + 31) / 32) * 32;
  if (t < 32) t = 32;
  return t;
}

template <typename T>
static cudaError_t norm_fwd_t(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int rows, int cols,
                              float eps, bool rms, cudaStream_t st) {
  const int threads = norm_threads(cols);
  if (threads > 1024 || cols % 8) return cudaErrorInvalidValue;
  if (rms) norm_fwd_kernel<T, true><<<rows, threads, 0, st>>>((const T*)x, (const T*)w, nullptr, (T*)y, nullptr, rstd, rows, cols, eps);
  else norm_fwd_kernel<T, false><<<rows, threads, 0, st>>>((const T*)x, (const T*)w, (const T*)b, (T*)y, mean, rstd, rows, cols, eps);
  return cudaGetLastError();
}

cudaError_t norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int rows, int cols, float eps,
                     int dtype, bool rms, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  return dtype == 1 ? norm_fwd_t<__nv_bfloat16>(x, w, b, y, mean, rstd, rows, cols, eps, rms, st)
                    : norm_fwd_t<__half>(x, w, b, y, mean, rstd, rows, cols, eps, rms, st);
}

int norm_bwd_num_parts(int rows, int num_sms) { int g = num_sms * 2; return rows < g ? rows : g; }

template <typename T>
static cudaError_t norm_bwd_t(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, void* dw,
                              void* db, float* workspace, int rows, int cols, bool rms, int num_sms, cudaStream_t st, const void* dres) {
  if (cols % 8 || cols > 32768) return cudaErrorInvalidValue;
  const int nvec = cols / 8;
  const int parts = norm_bwd_num_parts(rows, num_sms);
  float* dwp = workspace;
  float* dbp = workspace + (size_t)parts * cols;
#define PFX_NB(VPT, THREADS)                                                                                                              \
  do {                                                                                                                                    \
    if (rms) norm_bwd_kernel<T, true, VPT, THREADS><<<parts, THREADS, 0, st>>>((const T*)dy, (const T*)x, (const T*)w, nullptr, rstd,      \
                                                                              (T*)dx, dwp, dbp, rows, cols, (const T*)dres);              \
    else norm_bwd_kernel<T, false, VPT, THREADS><<<parts, THREADS, 0, st>>>((const T*)dy, (const T*)x, (const T*)w, mean, rstd, (T*)dx,    \
                                                                           dwp, dbp, rows, cols, (const T*)dres);                         \
  } while (0)
  if (nvec <= 128) PFX_NB(1, 128);
  else if (nvec <= 256) PFX_NB(1, 256);
  else if (nvec <= 512) PFX_NB(2, 256);
  else if (nvec <= 1024) PFX_NB(4, 256);
  else if (nvec <= 2048) PFX_NB(4, 512);
  else PFX_NB(8, 512);
#undef PFX_NB
  const int rg = (cols + 31) / 32;
  reduce_partials_kernel<T><<<rg, 256, 0, st>>>(dwp, (T*)dw, parts, cols);
  if (!rms && db) reduce_partials_kernel<T><<<rg, 256, 0, st>>>(dbp, (T*)db, parts, cols);
  return cudaGetLastError();
}

cudaError_t norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, void* dw, void* db,
                     float* workspace, int rows, int cols, int dtype, bool rms, int num_sms, cudaStream_t st, const void* dres) {
  if (rows == 0) return cudaSuccess;
  return dtype == 1 ? norm_bwd_t<__nv_bfloat16>(dy, x, w, mean, rstd, dx, dw, db, workspace, rows, cols, rms, num_sms, st, dres)
                    : norm_bwd_t<__half>(dy, x, w, mean, rstd, dx, dw, db, workspace, rows, cols, rms, num_sms, st, dres);
}

// --------------------------------------------------------------------------- bias + GELU
// exact (erf) GELU — nn.GELU's default, used by the vision models; the language models use the tanh form
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.f + erff(x * 0.7071067811865476f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}

template <typename T, bool kBwd>
__global__ void bias_gelu_kernel(const T* __restrict__ x, const T* __restrict__ bias, const T* __restrict__ dy, T* __restrict__ out,
                                 size_t total_vec, int nvec_row, bool exact) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float xv[8], bv[8], o[8];
    unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(x) + i), xv);
    if (bias) {
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(bias) + (i % nvec_row)), bv);
#pragma unroll
      for (int j = 0; j < 8; ++j) xv[j] += bv[j];
    }
    if (kBwd) {
      float gv[8];
      unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(dy) + i), gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = gv[j] * (exact ? gelu_erf_grad(xv[j]) : gelu_tanh_grad(xv[j]));
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = exact ? gelu_erf(xv[j]) : gelu_tanh(xv[j]);
    }
    st_stream(reinterpret_cast<uint4*>(out) + i, pack8<T>(o));
  }
}

static int ew_grid(size_t total_vec, int threads, int num_sms) {
  size_t g = (total_vec + threads - 1) / threads;
  const size_t cap = (size_t)num_sms * 16;
  return (int)(g < cap ? (g ? g : 1) : cap);
}

cudaError_t bias_gelu(const void* x, const void* bias, const void* dy, void* out, size_t rows, int cols, int dtype, bool bwd, int num_sms,
                      cudaStream_t st, bool exact) {
  if (cols % 8) return cudaErrorInvalidValue;
  const size_t total = rows * (size_t)(cols / 8);
  if (!total) return cudaSuccess;
  const int threads = 256, grid = ew_grid(total, threads, num_sms);
#define PFX_LAUNCH(T)                                                                                                     \
  if (bwd) bias_gelu_kernel<T, true><<<grid, threads, 0, st>>>((const T*)x, (const T*)bias, (const T*)dy, (T*)out, total, cols / 8, exact); \
  else bias_gelu_kernel<T, false><<<grid, threads, 0, st>>>((const T*)x, (const T*)bias, nullptr, (T*)out, total, cols / 8, exact);
  if (dtype == 1) { PFX_LAUNCH(__nv_bfloat16) } else { PFX_LAUNCH(__half) }
#undef PFX_LAUNCH
  return cudaGetLastError();
}

// --------------------------------------------------------------------------- bias + SwiGLU
// z [rows, 2F] holds pair-interleaved FFN1 outputs: column 2i is gate channel i, column 2i + 1 its up channel, so one thread's 16 z
// elements (two 16-byte vectors) are the 8 pairs behind one 16-byte vector of h [rows, F].  a = g + b_g, b = u + b_u, s = sigmoid(a):
//   fwd  h  = a s b
//   bwd  dg = dh b s (1 + a (1 - s)),   du = dh a s
// A saturated gate stays finite: __expf(-a) overflows to inf for a < -88, s = 1 / inf = 0 and every product above is 0 (1 - s is formed
// directly, never as e s, which would be inf * 0).  s is swiglu_sigmoid (pfx_ptx.cuh), shared with the grouped GEMM's SwiGLU epilogues.
template <typename T, bool kBwd>
__global__ void bias_swiglu_kernel(const T* __restrict__ z, const T* __restrict__ bias, const T* __restrict__ dh, T* __restrict__ out,
                                   size_t total_vec, int nvec_row) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float zv[2][8];                              // pair j: gate zv[j / 4][2 (j % 4)], up zv[j / 4][2 (j % 4) + 1]
    const uint4* zp = reinterpret_cast<const uint4*>(z) + 2 * i;
    unpack8<T>(ld_stream(zp), zv[0]);
    unpack8<T>(ld_stream(zp + 1), zv[1]);
    if (bias) {
      float bv[2][8];
      const uint4* bp = reinterpret_cast<const uint4*>(bias) + 2 * (i % nvec_row);
      unpack8<T>(__ldg(bp), bv[0]);
      unpack8<T>(__ldg(bp + 1), bv[1]);
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) zv[k][j] += bv[k][j];
    }
    if (kBwd) {
      float gv[8], o[2][8];
      unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(dh) + i), gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = j >> 2, c = 2 * (j & 3);
        const float a = zv[k][c], b = zv[k][c + 1], s = swiglu_sigmoid(a);
        o[k][c] = gv[j] * b * s * (1.f + a * (1.f - s));
        o[k][c + 1] = gv[j] * a * s;
      }
      uint4* op = reinterpret_cast<uint4*>(out) + 2 * i;
      st_stream(op, pack8<T>(o[0]));
      st_stream(op + 1, pack8<T>(o[1]));
    } else {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = j >> 2, c = 2 * (j & 3);
        o[j] = zv[k][c] * swiglu_sigmoid(zv[k][c]) * zv[k][c + 1];
      }
      st_stream(reinterpret_cast<uint4*>(out) + i, pack8<T>(o));
    }
  }
}

cudaError_t bias_swiglu(const void* z, const void* bias, const void* dh, void* out, size_t rows, int width, int dtype, bool bwd, int num_sms,
                        cudaStream_t st) {
  if (width % 8) return cudaErrorInvalidValue;
  const size_t total = rows * (size_t)(width / 8);
  if (!total) return cudaSuccess;
  const int threads = 256, grid = ew_grid(total, threads, num_sms);
#define PFX_LAUNCH(T)                                                                                                              \
  if (bwd) bias_swiglu_kernel<T, true><<<grid, threads, 0, st>>>((const T*)z, (const T*)bias, (const T*)dh, (T*)out, total, width / 8); \
  else bias_swiglu_kernel<T, false><<<grid, threads, 0, st>>>((const T*)z, (const T*)bias, nullptr, (T*)out, total, width / 8);
  if (dtype == 1) { PFX_LAUNCH(__nv_bfloat16) } else { PFX_LAUNCH(__half) }
#undef PFX_LAUNCH
  return cudaGetLastError();
}

// --------------------------------------------------------------------------- bias + dropout + residual
// fwd: y = residual + keep * (x + bias) / (1 - p)        bwd: dx = keep * dy / (1 - p)
template <typename T, bool kBwd>
__global__ void bias_dropout_add_kernel(const T* __restrict__ x, const T* __restrict__ bias, const T* __restrict__ residual,
                                        T* __restrict__ out, size_t total_vec, int nvec_row, float scale, uint32_t thresh16,
                                        uint64_t seed, uint64_t offset) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float xv[8], o[8];
    unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(x) + i), xv);
    if (!kBwd && bias) {
      float bv[8];
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(bias) + (i % nvec_row)), bv);
#pragma unroll
      for (int j = 0; j < 8; ++j) xv[j] += bv[j];
    }
    bool keep[8];
    if (thresh16 > 0) Philox::keep8(seed, offset, i, thresh16, keep);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (thresh16 == 0 || keep[j]) ? xv[j] * scale : 0.f;
    if (!kBwd && residual) {
      float rv[8];
      unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(residual) + i), rv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += rv[j];
    }
    st_stream(reinterpret_cast<uint4*>(out) + i, pack8<T>(o));
  }
}

cudaError_t bias_dropout_add(const void* x, const void* bias, const void* residual, void* out, size_t rows, int cols, float p,
                             uint64_t seed, uint64_t offset, int dtype, bool bwd, int num_sms, cudaStream_t st) {
  if (cols % 8) return cudaErrorInvalidValue;
  const size_t total = rows * (size_t)(cols / 8);
  if (!total) return cudaSuccess;
  uint32_t thresh = (uint32_t)(p * 65536.0f + 0.5f);
  if (thresh > 65535u) thresh = 65535u;
  const float scale = thresh ? 1.0f / (1.0f - thresh / 65536.0f) : 1.0f;
  const int threads = 256, grid = ew_grid(total, threads, num_sms);
#define PFX_LAUNCH(T)                                                                                                                 \
  if (bwd) bias_dropout_add_kernel<T, true><<<grid, threads, 0, st>>>((const T*)x, nullptr, nullptr, (T*)out, total, cols / 8, scale,    \
                                                                      thresh, seed, offset);                                          \
  else bias_dropout_add_kernel<T, false><<<grid, threads, 0, st>>>((const T*)x, (const T*)bias, (const T*)residual, (T*)out, total,    \
                                                                   cols / 8, scale, thresh, seed, offset);
  if (dtype == 1) { PFX_LAUNCH(__nv_bfloat16) } else { PFX_LAUNCH(__half) }
#undef PFX_LAUNCH
  return cudaGetLastError();
}

// --------------------------------------------------------------------------- column sum (bias grad)
// block = 32 column-vector lanes x 8 row lanes; grid = (ceil(cols/256), row_chunks)
template <typename T>
__global__ void colsum_partial_kernel(const T* __restrict__ x, float* __restrict__ part, int rows, int cols) {
  __shared__ float red[8][32][9];
  const int lane_c = threadIdx.x & 31, lane_r = threadIdx.x >> 5;
  const int vec = blockIdx.x * 32 + lane_c;
  const int nvec = cols >> 3;
  const int rows_per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (vec < nvec) {
    for (int r = r0 + lane_r; r < r1; r += 8) {
      float v[8];
      unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(x + (size_t)r * cols) + vec), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[lane_r][lane_c][j] = acc[j];
  __syncthreads();
  if (lane_r == 0 && vec < nvec) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) s += red[r][lane_c][j];
      part[(size_t)blockIdx.y * cols + vec * 8 + j] = s;
    }
  }
}

int colsum_num_parts(int rows) { int p = (rows + 31) / 32; return p < 1 ? 1 : (p > 256 ? 256 : p); }
static int colsum_parts_for(int rows, int cols) {
  const int gx = (cols / 8 + 31) / 32;
  int p = (592 + gx - 1) / gx;                 // aim at >= 4 CTAs per SM
  const int cap = colsum_num_parts(rows);
  if (p > cap) p = cap;
  return p < 1 ? 1 : p;
}

cudaError_t colsum(const void* x, void* out, float* workspace, int rows, int cols, int dtype, bool out_fp32, cudaStream_t st) {
  if (cols % 8) return cudaErrorInvalidValue;
  const int parts = colsum_parts_for(rows, cols);
  dim3 grid((cols / 8 + 31) / 32, parts);
  if (dtype == 1) colsum_partial_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, workspace, rows, cols);
  else colsum_partial_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, workspace, rows, cols);
  const int rt = 256, rg = (cols + 31) / 32;
  if (out_fp32) reduce_partials_kernel<float><<<rg, rt, 0, st>>>(workspace, (float*)out, parts, cols);
  else if (dtype == 1) reduce_partials_kernel<__nv_bfloat16><<<rg, rt, 0, st>>>(workspace, (__nv_bfloat16*)out, parts, cols);
  else reduce_partials_kernel<__half><<<rg, rt, 0, st>>>(workspace, (__half*)out, parts, cols);
  return cudaGetLastError();
}

}  // namespace pfx
