// Vocab-parallel-capable softmax cross-entropy (stats + in-place backward), multi-precision flat
// AdamW with device-side unscale/clip/found-inf, squared-norm reduction, fp32 main-grad accumulate.
// Reference call sites: L9 (c_softmax_with_cross_entropy), L12-L15 in SURVEY §2.6.
#include "pfx_common.cuh"
#include "pfx_kernels.h"

namespace pfx {

// ------------------------------------------------------------------ softmax-CE statistics
// One CTA per row.  Online softmax: a single pass over the logits row produces
//   row_max = max_j x_j, row_sum = sum_j exp(x_j - row_max), tgt = x[label - vocab_start] (0 if the label
// lives on another vocab shard).  The python side all-reduces (max / rescaled sum / tgt) over the
// tensor-parallel group, exactly the three tiny exchanges of ParallelCrossEntropy.
// kVec: rows are read as 16-byte vectors, which needs cols % 8 == 0 and a 16-byte aligned base (otherwise row 1 onwards is
// misaligned); the scalar instantiation reads every element through the tail loop.
// While a thread's running max is still -inf (masked logits) there is nothing to rescale: exp(-inf - -inf) would be NaN.
template <typename T, bool kVec>
__global__ void ce_stats_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels, float* __restrict__ row_max,
                                float* __restrict__ row_sum, float* __restrict__ tgt, int cols, int64_t vocab_start) {
  __shared__ float scratch[33];
  const int row = blockIdx.x;
  const T* xr = logits + (size_t)row * cols;
  const int nvec = kVec ? cols >> 3 : 0;
  float m = -INFINITY, s = 0.f;
  for (int vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
    float v[8];
    unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(xr) + vi), v);
    float lm = v[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) lm = fmaxf(lm, v[j]);
    const float nm = fmaxf(m, lm);
    if (nm == -INFINITY) continue;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(v[j] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  for (int c = nvec * 8 + threadIdx.x; c < cols; c += blockDim.x) {  // tail (cols % 8), or the whole row when !kVec
    const float v = to_f32<T>(xr[c]);
    const float nm = fmaxf(m, v);
    if (nm == -INFINITY) continue;
    s = s * __expf(m - nm) + __expf(v - nm);
    m = nm;
  }
  const float gm = block_max(m, scratch);
  const float contrib = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
  const float gs = block_sum(contrib, scratch);
  if (threadIdx.x == 0) {
    row_max[row] = gm;
    row_sum[row] = gs;
    const int64_t l = labels[row] - vocab_start;
    tgt[row] = (l >= 0 && l < cols) ? to_f32<T>(xr[l]) : 0.f;
  }
}

// dlogits (in place) = (exp(x - lse) - onehot(label)) * gscale[row]
template <typename T, bool kVec>
__global__ void ce_bwd_kernel(T* __restrict__ logits, const int64_t* __restrict__ labels, const float* __restrict__ lse,
                              const float* __restrict__ gscale, int cols, int64_t vocab_start) {
  const int row = blockIdx.x;
  T* xr = logits + (size_t)row * cols;
  const int nvec = kVec ? cols >> 3 : 0;
  const float l = lse[row], g = gscale[row];
  const int64_t lab = labels[row] - vocab_start;
  for (int vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
    float v[8];
    unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(xr) + vi), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = __expf(v[j] - l);
      if ((int64_t)(vi * 8 + j) == lab) p -= 1.f;
      v[j] = p * g;
    }
    st_stream(reinterpret_cast<uint4*>(xr) + vi, pack8<T>(v));
  }
  for (int c = nvec * 8 + threadIdx.x; c < cols; c += blockDim.x) {
    float p = __expf(to_f32<T>(xr[c]) - l);
    if ((int64_t)c == lab) p -= 1.f;
    xr[c] = from_f32<T>(p * g);
  }
}

static bool ce_vec_ok(const void* logits, int cols) { return cols % 8 == 0 && reinterpret_cast<uintptr_t>(logits) % 16 == 0; }

template <typename T>
static void ce_stats_t(const void* logits, const int64_t* labels, float* row_max, float* row_sum, float* tgt, int rows, int cols,
                       int64_t vocab_start, cudaStream_t st) {
  if (ce_vec_ok(logits, cols)) ce_stats_kernel<T, true><<<rows, 512, 0, st>>>((const T*)logits, labels, row_max, row_sum, tgt, cols, vocab_start);
  else ce_stats_kernel<T, false><<<rows, 512, 0, st>>>((const T*)logits, labels, row_max, row_sum, tgt, cols, vocab_start);
}
template <typename T>
static void ce_bwd_t(void* logits, const int64_t* labels, const float* lse, const float* gscale, int rows, int cols, int64_t vocab_start,
                     cudaStream_t st) {
  if (ce_vec_ok(logits, cols)) ce_bwd_kernel<T, true><<<rows, 512, 0, st>>>((T*)logits, labels, lse, gscale, cols, vocab_start);
  else ce_bwd_kernel<T, false><<<rows, 512, 0, st>>>((T*)logits, labels, lse, gscale, cols, vocab_start);
}

cudaError_t ce_stats(const void* logits, const int64_t* labels, float* row_max, float* row_sum, float* tgt, int rows, int cols,
                     int64_t vocab_start, int dtype, cudaStream_t st) {
  if (!rows) return cudaSuccess;
  if (dtype == 1) ce_stats_t<__nv_bfloat16>(logits, labels, row_max, row_sum, tgt, rows, cols, vocab_start, st);
  else if (dtype == 0) ce_stats_t<__half>(logits, labels, row_max, row_sum, tgt, rows, cols, vocab_start, st);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}
cudaError_t ce_bwd(void* logits, const int64_t* labels, const float* lse, const float* gscale, int rows, int cols, int64_t vocab_start,
                   int dtype, cudaStream_t st) {
  if (!rows) return cudaSuccess;
  if (dtype == 1) ce_bwd_t<__nv_bfloat16>(logits, labels, lse, gscale, rows, cols, vocab_start, st);
  else if (dtype == 0) ce_bwd_t<__half>(logits, labels, lse, gscale, rows, cols, vocab_start, st);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

// ------------------------------------------------------------------ sum of squares (deterministic two-stage)
template <typename T>
__global__ void sumsq_partial_kernel(const T* __restrict__ x, size_t n, float* __restrict__ part) {
  __shared__ float scratch[33];
  float s = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += stride) { const float v = to_f32<T>(x[i]); s += v * v; }
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
template <typename T>
__global__ void sumsq_partial_vec_kernel(const T* __restrict__ x, size_t nvec, float* __restrict__ part) {
  __shared__ float scratch[33];
  float s = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float v[8];
    unpack8<T>(ld_stream(reinterpret_cast<const uint4*>(x) + i), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[j] * v[j];
  }
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void sumsq_final_kernel(const float* __restrict__ part, int n, float* __restrict__ out, bool accumulate) {
  __shared__ float scratch[33];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += part[i];
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) out[0] = accumulate ? out[0] + s : s;
}

cudaError_t sumsq(const void* x, size_t n, float* out, float* workspace, int dtype, bool accumulate, int num_sms, cudaStream_t st) {
  int grid = num_sms * 4;
  if (grid > 1024) grid = 1024;
  if (dtype == 3) {
    sumsq_partial_kernel<float><<<grid, 512, 0, st>>>((const float*)x, n, workspace);
  } else if ((n % 8) == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0) {
    if (dtype == 1) sumsq_partial_vec_kernel<__nv_bfloat16><<<grid, 512, 0, st>>>((const __nv_bfloat16*)x, n / 8, workspace);
    else sumsq_partial_vec_kernel<__half><<<grid, 512, 0, st>>>((const __half*)x, n / 8, workspace);
  } else {
    if (dtype == 1) sumsq_partial_kernel<__nv_bfloat16><<<grid, 512, 0, st>>>((const __nv_bfloat16*)x, n, workspace);
    else sumsq_partial_kernel<__half><<<grid, 512, 0, st>>>((const __half*)x, n, workspace);
  }
  sumsq_final_kernel<<<1, 256, 0, st>>>(workspace, grid, out, accumulate);
  return cudaGetLastError();
}

// gscale = inv_loss_scale * min(1, clip_norm / (sqrt(sumsq) * inv_loss_scale + 1e-6));  found_inf = !finite(sumsq)
__global__ void clip_coef_kernel(const float* __restrict__ sq, float inv_loss_scale, float clip_norm, float* __restrict__ gscale,
                                 float* __restrict__ found_inf, float* __restrict__ gnorm) {
  const float s = sq[0];
  const bool bad = !isfinite(s);
  const float norm = sqrtf(s) * inv_loss_scale;
  float coef = 1.f;
  if (clip_norm > 0.f && !bad) coef = fminf(1.f, clip_norm / (norm + 1e-6f));
  gscale[0] = bad ? 0.f : inv_loss_scale * coef;
  found_inf[0] = bad ? 1.f : 0.f;
  if (gnorm) gnorm[0] = norm;
}
cudaError_t clip_coef(const float* sq, float inv_loss_scale, float clip_norm, float* gscale, float* found_inf, float* gnorm, cudaStream_t st) {
  clip_coef_kernel<<<1, 1, 0, st>>>(sq, inv_loss_scale, clip_norm, gscale, found_inf, gnorm);
  return cudaGetLastError();
}

// ------------------------------------------------------------------ flat multi-precision AdamW
// One launch updates a whole flat shard: fp32 master + moments, optional low-precision mirror written in
// the same pass (this mirror is what ZeRO broadcasts / the next forward reads).
// 28-32 B of traffic per element and nothing to reuse: the kernel is a pure stream.  Every thread moves two independent
// 4-element packets per iteration (16-byte accesses on the fp32 state, 8-byte on bf16 grads / weights) so that enough
// bytes are in flight per SM to cover HBM latency; the scalar tail is handled by the last threads.
template <typename TG, typename TP>
__global__ void __launch_bounds__(256) adamw_kernel(TP* __restrict__ p_lp, float* __restrict__ master, const TG* __restrict__ grad,
                                                    float* __restrict__ m, float* __restrict__ v, size_t n, float lr, float beta1, float beta2,
                                                    float eps, float wd, float bc1, float bc2, const float* __restrict__ gscale,
                                                    const float* __restrict__ found_inf) {
  if (found_inf && found_inf[0] != 0.f) return;
  const float gs = gscale ? gscale[0] : 1.f;
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  const float decay = 1.f - lr * wd, omb1 = 1.f - beta1, omb2 = 1.f - beta2;
  constexpr int kUnroll = 2;
  const size_t nvec = n >> 2;
  const size_t tid = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t nthreads = (size_t)gridDim.x * blockDim.x;
  for (size_t i0 = tid; i0 < nvec; i0 += nthreads * kUnroll) {
    float g[kUnroll][4], w[kUnroll][4], mm[kUnroll][4], vv[kUnroll][4];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t i = i0 + u * nthreads;
      if (i < nvec) {
        load4<TG>(grad + i * 4, g[u]);
        load4<float>(master + i * 4, w[u]);
        load4<float>(m + i * 4, mm[u]);
        load4<float>(v + i * 4, vv[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t i = i0 + u * nthreads;
      if (i >= nvec) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gj = g[u][j] * gs;
        mm[u][j] = beta1 * mm[u][j] + omb1 * gj;
        vv[u][j] = beta2 * vv[u][j] + omb2 * gj * gj;
        const float denom = sqrtf(vv[u][j]) * inv_sqrt_bc2 + eps;
        w[u][j] = w[u][j] * decay - step_size * mm[u][j] / denom;
      }
      store4<float>(m + i * 4, mm[u]);
      store4<float>(v + i * 4, vv[u]);
      store4<float>(master + i * 4, w[u]);
      if (p_lp) store4<TP>(p_lp + i * 4, w[u]);
    }
  }
  // tail (n % 4 elements)
  const size_t i = (nvec << 2) + tid;
  if (i < n) {
    const float gj = to_f32<TG>(grad[i]) * gs;
    const float mi = beta1 * m[i] + omb1 * gj;
    const float vi = beta2 * v[i] + omb2 * gj * gj;
    m[i] = mi; v[i] = vi;
    const float wi = master[i] * decay - step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + eps);
    master[i] = wi;
    if (p_lp) p_lp[i] = from_f32<TP>(wi);
  }
}

cudaError_t adamw_flat(void* p_lp, float* master, const void* grad, float* m, float* v, size_t n, float lr, float beta1, float beta2,
                       float eps, float wd, float bc1, float bc2, const float* gscale, const float* found_inf, int grad_dtype,
                       int lp_dtype, int num_sms, cudaStream_t st) {
  if (!n) return cudaSuccess;
  const int threads = 256;
  size_t g = (n / 8 + threads - 1) / threads;
  const size_t cap = (size_t)num_sms * 8;
  const int grid = (int)(g < cap ? (g ? g : 1) : cap);
  // vector accesses need 16-byte aligned state and 8-byte aligned low-precision pointers (flat buffers are 256 B aligned)
  if ((reinterpret_cast<uintptr_t>(master) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) return cudaErrorMisalignedAddress;
  if ((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(p_lp)) & 7) return cudaErrorMisalignedAddress;
#define PFX_ADAM(TG, TP) adamw_kernel<TG, TP><<<grid, threads, 0, st>>>((TP*)p_lp, master, (const TG*)grad, m, v, n, lr, beta1, beta2, eps, wd, bc1, bc2, gscale, found_inf)
  // a 16-bit gradient pairs with a low-precision copy of its own dtype or an fp32 one (3, also meaning "no copy")
  if ((grad_dtype == 1 && lp_dtype == 0) || (grad_dtype == 0 && lp_dtype == 1)) return cudaErrorInvalidValue;
  if (grad_dtype == 3) { if (lp_dtype == 1) PFX_ADAM(float, __nv_bfloat16); else if (lp_dtype == 0) PFX_ADAM(float, __half); else PFX_ADAM(float, float); }
  else if (grad_dtype == 1) { if (lp_dtype == 1) PFX_ADAM(__nv_bfloat16, __nv_bfloat16); else PFX_ADAM(__nv_bfloat16, float); }
  else { if (lp_dtype == 0) PFX_ADAM(__half, __half); else PFX_ADAM(__half, float); }
#undef PFX_ADAM
  return cudaGetLastError();
}

// main_grad(fp32) += grad(low precision)   — reference amp.py:44-63 hook, one pass
template <typename T>
__global__ void accumulate_kernel(float* __restrict__ dst, const T* __restrict__ src, size_t n, float scale) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += stride) dst[i] += to_f32<T>(src[i]) * scale;
}
cudaError_t accumulate_f32(float* dst, const void* src, size_t n, float scale, int dtype, int num_sms, cudaStream_t st) {
  if (!n) return cudaSuccess;
  const int threads = 256;
  size_t g = (n + threads - 1) / threads;
  const size_t cap = (size_t)num_sms * 16;
  const int grid = (int)(g < cap ? g : cap);
  if (dtype == 1) accumulate_kernel<__nv_bfloat16><<<grid, threads, 0, st>>>(dst, (const __nv_bfloat16*)src, n, scale);
  else if (dtype == 0) accumulate_kernel<__half><<<grid, threads, 0, st>>>(dst, (const __half*)src, n, scale);
  else accumulate_kernel<float><<<grid, threads, 0, st>>>(dst, (const float*)src, n, scale);
  return cudaGetLastError();
}

}  // namespace pfx
