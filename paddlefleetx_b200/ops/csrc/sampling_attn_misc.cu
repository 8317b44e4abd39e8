// Top-p (nucleus) sampling without a sort, rotary embedding, fused causal softmax.
//
// Top-p: the reference op (ppfleetx/ops/topp_sampling.cu: 6 kernels + CUB segmented radix sort + cuRAND
// states) sorts every row of the vocabulary.  Here one CTA per row does
//   (1) block arg-max with the same top-1 early-out (draw u ~ U(0,1) * top_p; if p_max >= u emit it),
//   (2) otherwise a 4-pass radix *descent* on the float bit pattern with mass histograms: it finds the
//       probability value t at which the descending cumulative mass crosses u — i.e. the token the sorted
//       prefix-sum search would have returned — in 4 reads of an L2-resident row,
//   (3) among the tokens of exactly that value, the one the sorted search reaches first (ties in index order), with no cap on
//       the number of ties.
// RNG is a stateless Philox counter (seed, offset+row): reproducible, no state tensor, graph-capturable.
#include "pfx_common.cuh"
#include "pfx_kernels.h"

namespace pfx {

constexpr int kTopPThreads = 1024;

template <typename T>
__global__ void __launch_bounds__(kTopPThreads)
topp_sampling_kernel(const T* __restrict__ probs, const float* __restrict__ top_ps, float* __restrict__ out_prob,
                     int64_t* __restrict__ out_id, int V, uint64_t seed, uint64_t offset) {
  __shared__ float hist[32][256];
  __shared__ float hist0[256];
  __shared__ float s_val[32];
  __shared__ int s_idx[32];
  __shared__ uint32_t s_prefix;
  __shared__ float s_mass_above;
  __shared__ int s_sel, s_rank;
  const int row = blockIdx.x;
  const T* pr = probs + (size_t)row * V;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

  // ---- (1) arg-max
  float bv = -1.f; int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float p = to_f32<T>(pr[i]);
    if (p > bv) { bv = p; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { s_val[w] = bv; s_idx[w] = bi; }
  __syncthreads();
  if (w == 0) {
    bv = s_val[lane]; bi = s_idx[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_val[0] = bv; s_idx[0] = bi; }
  }
  __syncthreads();
  const float pmax = s_val[0];
  const int imax = s_idx[0];
  const float u = Philox::uniform(seed, offset + row) * top_ps[row];
  if (pmax >= u) {
    if (threadIdx.x == 0) { out_prob[row] = pmax; out_id[row] = imax; }
    return;
  }

  // ---- (2) radix descent on float bits (positive floats order like their bit patterns)
  if (threadIdx.x == 0) { s_prefix = 0u; s_mass_above = 0.f; }
  uint32_t prefix_mask = 0u;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = threadIdx.x; i < 32 * 256; i += blockDim.x) (&hist[0][0])[i] = 0.f;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    // run-length privatisation: probabilities cluster in a handful of exponent bins (all of them in ONE bin for a flat
    // distribution), so each thread keeps the current bin's partial sum in a register and touches shared memory only when
    // the bin changes — the per-element shared atomics were 32-way serialised on exactly those hot bins
    int cur_bin = -1;
    float cur_sum = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float p = to_f32<T>(pr[i]);
      const uint32_t key = __float_as_uint(p);
      if ((key & prefix_mask) == prefix && p > 0.f) {
        const int bin = (int)((key >> shift) & 0xFFu);
        if (bin == cur_bin) {
          cur_sum += p;
        } else {
          if (cur_bin >= 0) atomicAdd(&hist[w][cur_bin], cur_sum);
          cur_bin = bin;
          cur_sum = p;
        }
      }
    }
    if (cur_bin >= 0) atomicAdd(&hist[w][cur_bin], cur_sum);
    __syncthreads();
    if (threadIdx.x < 256) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) s += hist[k][threadIdx.x];
      hist0[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float cum = s_mass_above;
      int chosen = -1, lowest_nonzero = -1;
      for (int b = 255; b >= 0; --b) {
        const float h = hist0[b];
        if (h > 0.f) {
          lowest_nonzero = b;
          if (cum + h >= u) { chosen = b; break; }
          cum += h;
        }
      }
      if (chosen < 0) {  // u beyond total mass through rounding: take the smallest candidate
        chosen = lowest_nonzero < 0 ? 0 : lowest_nonzero;
        cum -= hist0[chosen];
      }
      s_mass_above = cum;
      s_prefix = prefix | ((uint32_t)chosen << shift);
    }
    prefix_mask |= (0xFFu << shift);
    __syncthreads();
  }
  const uint32_t tkey = s_prefix;
  const float t = __uint_as_float(tkey);

  // ---- (3) tie number j (in index order) among the tokens of value exactly t.  Warp w owns the contiguous span
  // [w * span, (w + 1) * span) of the row and reads it 32 consecutive tokens at a time, so its reads stay coalesced and a ballot lists the
  // ties of each step in index order.  One counting pass, an exclusive scan of the 32 warp counts, then the owning warp walks its span.
  static_assert(kTopPThreads == 32 * 32, "the tie scan below is one warp wide: one count per warp");
  const int span = ((V + 31) / 32 + 31) & ~31;
  const int lo = min(V, w * span), hi = min(V, lo + span);
  int cnt = 0;
  for (int b = lo; b < hi; b += 32) {
    const int i = b + lane;
    cnt += __popc(__ballot_sync(0xffffffffu, i < hi && __float_as_uint(to_f32<T>(pr[i])) == tkey));
  }
  if (lane == 0) s_idx[w] = cnt;
  __syncthreads();
  if (w == 0) {
    const int c = s_idx[lane];
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const int ties = __shfl_sync(0xffffffffu, incl, 31);
    // the first tie whose cumulative mass reaches u: the smallest j with above + (j + 1) t >= u, evaluated in double (a product (j + 1) t
    // of a 24-bit t is exact there) rather than by an approximate fp32 division; j is clamped to the last tie when rounding overshoots
    const double need = (double)u - (double)s_mass_above;
    int j = 0;
    if (ties > 0 && t > 0.f && need > 0.0) {
      const double q = ceil(need / (double)t) - 1.0;
      j = q < 0.0 ? 0 : (q > (double)(ties - 1) ? ties - 1 : (int)q);
      while (j > 0 && (double)j * t >= need) --j;
      while (j < ties - 1 && (double)(j + 1) * t < need) ++j;
    }
    const int excl = incl - c;
    const unsigned owner = __ballot_sync(0xffffffffu, c > 0 && j >= excl && j < incl);
    if (lane == 0) s_sel = ties > 0 ? (int)__ffs(owner) - 1 : -1;
    if (ties > 0 && lane == (int)__ffs(owner) - 1) s_rank = j - excl;
  }
  __syncthreads();
  if (s_sel < 0) {                    // no token has value t (a row without positive mass): the arg-max
    if (threadIdx.x == 0) { out_prob[row] = pmax; out_id[row] = imax; }
    return;
  }
  if (w == s_sel) {
    int r = s_rank;
    for (int b = lo; b < hi; b += 32) {
      const int i = b + lane;
      const unsigned m = __ballot_sync(0xffffffffu, i < hi && __float_as_uint(to_f32<T>(pr[i])) == tkey);
      const int n = __popc(m);
      if (r < n) {
        if (lane == 0) {
          const int id = b + (int)__fns(m, 0, r + 1);
          out_prob[row] = to_f32<T>(pr[id]);
          out_id[row] = id;
        }
        break;
      }
      r -= n;
    }
  }
}

cudaError_t topp_sampling(const void* probs, const float* top_ps, float* out_prob, int64_t* out_id, int rows, int V, uint64_t seed,
                          uint64_t offset, int dtype, cudaStream_t st) {
  if (!rows) return cudaSuccess;
  if (dtype == 1) topp_sampling_kernel<__nv_bfloat16><<<rows, kTopPThreads, 0, st>>>((const __nv_bfloat16*)probs, top_ps, out_prob, out_id, V, seed, offset);
  else if (dtype == 0) topp_sampling_kernel<__half><<<rows, kTopPThreads, 0, st>>>((const __half*)probs, top_ps, out_prob, out_id, V, seed, offset);
  else topp_sampling_kernel<float><<<rows, kTopPThreads, 0, st>>>((const float*)probs, top_ps, out_prob, out_id, V, seed, offset);
  return cudaGetLastError();
}

// ------------------------------------------------------------------ rotary position embedding (NeoX halves)
// x: [tokens, heads, d]; positions: [tokens] or null (then pos = token % seq_len).  sign = +1 fwd, -1 bwd.
template <typename T>
__global__ void rope_kernel(const T* __restrict__ x, T* __restrict__ y, const int64_t* __restrict__ positions, size_t tokens, int heads,
                            int d, int seq_len, float base, float sign) {
  const int half = d >> 1;
  const size_t total = tokens * (size_t)heads * half;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int i = idx % half;
    const size_t th = idx / half;
    const size_t tok = th / heads;
    // The angle and its sine / cosine in fp64: at positions in the tens of thousands the fast-math fp32 forms (__powf, __sincosf)
    // are off by more than a 16-bit output can hide.  Double-precision functions are not replaced by --use_fast_math.
    const double pos = positions ? (double)positions[tok] : (double)(tok % seq_len);
    double sd, cd;
    sincos(pos * pow((double)base, -2.0 * i / d), &sd, &cd);
    const float sn = (float)sd * sign, cs = (float)cd;
    const T* xp = x + th * d;
    T* yp = y + th * d;
    const float a = to_f32<T>(xp[i]), b = to_f32<T>(xp[i + half]);
    yp[i] = from_f32<T>(a * cs - b * sn);
    yp[i + half] = from_f32<T>(b * cs + a * sn);
  }
}

cudaError_t rope(const void* x, void* y, const int64_t* positions, size_t tokens, int heads, int d, int seq_len, float base, bool bwd,
                 int dtype, int num_sms, cudaStream_t st) {
  const size_t total = tokens * (size_t)heads * (d / 2);
  if (!total) return cudaSuccess;
  const int threads = 256;
  size_t g = (total + threads - 1) / threads;
  const size_t cap = (size_t)num_sms * 16;
  const int grid = (int)(g < cap ? g : cap);
  const float sign = bwd ? -1.f : 1.f;
  if (dtype == 1) rope_kernel<__nv_bfloat16><<<grid, threads, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, positions, tokens, heads, d, seq_len, base, sign);
  else if (dtype == 0) rope_kernel<__half><<<grid, threads, 0, st>>>((const __half*)x, (__half*)y, positions, tokens, heads, d, seq_len, base, sign);
  else rope_kernel<float><<<grid, threads, 0, st>>>((const float*)x, (float*)y, positions, tokens, heads, d, seq_len, base, sign);
  return cudaGetLastError();
}

// ------------------------------------------------------------------ fused causal (upper-triangular masked) softmax
// x: [batch, sq, sk] scores, one warp per row; entries with col > row + (sk - sq) are masked.
template <typename T>
__global__ void causal_softmax_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int sq, int sk, float scale, size_t rows) {
  const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int r = row % sq;
  const int valid = min(sk, r + (sk - sq) + 1);
  const T* xr = x + row * sk;
  T* yr = y + row * sk;
  float m = -INFINITY;
  for (int c = lane; c < valid; c += 32) m = fmaxf(m, to_f32<T>(xr[c]) * scale);
  m = warp_max(m);
  float s = 0.f;
  for (int c = lane; c < valid; c += 32) s += __expf(to_f32<T>(xr[c]) * scale - m);
  s = warp_sum(s);
  const float inv = 1.f / s;
  for (int c = lane; c < sk; c += 32) yr[c] = from_f32<T>(c < valid ? __expf(to_f32<T>(xr[c]) * scale - m) * inv : 0.f);
}
template <typename T>
__global__ void causal_softmax_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ y, T* __restrict__ dx, int sq, int sk, float scale,
                                          size_t rows) {
  const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int r = row % sq;
  const int valid = min(sk, r + (sk - sq) + 1);
  const T* gr = dy + row * sk;
  const T* yr = y + row * sk;
  T* dr = dx + row * sk;
  float dot = 0.f;
  for (int c = lane; c < valid; c += 32) dot += to_f32<T>(gr[c]) * to_f32<T>(yr[c]);
  dot = warp_sum(dot);
  for (int c = lane; c < sk; c += 32)
    dr[c] = from_f32<T>(c < valid ? scale * to_f32<T>(yr[c]) * (to_f32<T>(gr[c]) - dot) : 0.f);
}

cudaError_t causal_softmax(const void* a, const void* b, void* out, size_t batch, int sq, int sk, float scale, bool bwd, int dtype,
                           cudaStream_t st) {
  const size_t rows = batch * sq;
  if (!rows) return cudaSuccess;
  const int threads = 256, wpb = threads / 32;
  const int grid = (int)((rows + wpb - 1) / wpb);
#define PFX_CS(T)                                                                                                      \
  if (bwd) causal_softmax_bwd_kernel<T><<<grid, threads, 0, st>>>((const T*)a, (const T*)b, (T*)out, sq, sk, scale, rows); \
  else causal_softmax_fwd_kernel<T><<<grid, threads, 0, st>>>((const T*)a, (T*)out, sq, sk, scale, rows);
  if (dtype == 1) { PFX_CS(__nv_bfloat16) } else if (dtype == 0) { PFX_CS(__half) } else { PFX_CS(float) }
#undef PFX_CS
  return cudaGetLastError();
}

}  // namespace pfx
