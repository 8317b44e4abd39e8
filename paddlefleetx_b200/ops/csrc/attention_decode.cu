// Single-query attention over a static KV cache (the decode step of generation).
//
//   out[b, h, :] = softmax(scale * q[b, h, :] . K[b, 0:L, h, :] + mask[b, 0:L]) @ V[b, 0:L, h, :]
//
// q: [B, 1, H, D], K / V: [B, Lmax, H, D] (the framework's cache layout, read in place — no gather, no transpose), mask: additive
// [B, Lmax] (0 = attend, large negative or -inf = padded / not yet written), D in {64, 128}.  A row whose L keys are all masked with
// -inf returns 0 (the flash kernels' l = 0 convention).  One CTA per (head, batch): its warps take
// keys round-robin, every lane owns D/32 contiguous channels (one 4- or 8-byte load per key), the q.k dot product is a warp
// shuffle reduction and each warp keeps a private online-softmax state (m, l, acc); the warps' partial states are merged through
// shared memory at the end.  The op is a pure stream over the cache (2 * L * D * 2 bytes per head), so several keys are in flight
// per warp.  Replaces the library SDPA call on the decode path (reference: hybrid_model.py:303-346 core attention with cache).
//
// Grouped-query attention (kGqa, a separate instantiation): the cache holds Hkv = H / G heads and query head h reads K/V head h / G.
// The grid stays (query head, batch), so the G CTAs of a group are launch-order neighbours and their cache stream is served by L2.
#include "pfx_common.cuh"
#include "pfx_kernels.h"

namespace pfx {

namespace {

constexpr int kDecWarps = 8;

// D / 8 lanes share one key (16-byte loads of 8 channels each), so a warp works on 32 / (D / 8) keys at a time and keeps
// kU such groups in flight: 8 (D = 128) or 16 (D = 64) keys = 4-8 KB per warp outstanding.  Every lane group carries its own
// online-softmax state; all states of the CTA are merged through shared memory at the end.
template <typename T, int D, bool kGqa>
__global__ void __launch_bounds__(kDecWarps * 32) attention_decode_kernel(const T* __restrict__ q, T* __restrict__ k, T* __restrict__ v,
                                                                           const T* __restrict__ mask, T* __restrict__ out, int L, int Lmax,
                                                                           int H, float scale, const int64_t* __restrict__ write_idx, int G) {
  constexpr int kLanes = D / 8;               // lanes per key
  constexpr int kKW = 32 / kLanes;            // keys per warp step
  constexpr int kStates = kDecWarps * kKW;
  constexpr int kU = 4;
  __shared__ float s_m[kStates], s_l[kStates];
  __shared__ float s_acc[kStates][D];
  const int h = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int sub = lane / kLanes, ch = (lane % kLanes) * 8;
  const int Hkv = kGqa ? H / G : H, hk = kGqa ? h / G : h, g = h - hk * (kGqa ? G : 1);    // K/V head of this query head
  // packed mode (write_idx != null): q points at the fused QKV projection [B, 1, H, 3, D]; this CTA first appends its head's new
  // key / value at cache position *write_idx (the cache write used to be two separate index_copy launches), then attends.
  // Grouped: qkv is [B, 1, Hkv, G + 2, D] (the group's G queries, then its key and value); the first CTA of a group appends, and
  // since the CTAs of one launch are unordered, none of them reads that cache row: every one takes key *write_idx from qkv instead.
  const T* qkv_row = kGqa && write_idx ? q + ((size_t)b * Hkv + hk) * (G + 2) * D : nullptr;
  const int64_t new_pos = kGqa && write_idx ? write_idx[0] : -1;
  const int q_head_stride = write_idx ? 3 * D : D;
  if (write_idx != nullptr) {
    const int64_t pos = write_idx[0];
    if (w < 2 && pos >= 0 && pos < Lmax && g == 0) {
      const T* src = kGqa ? qkv_row + (G + w) * D : q + ((size_t)b * H + h) * 3 * D + (1 + w) * D;
      T* dst = (w == 0 ? k : v) + ((size_t)b * Lmax + pos) * Hkv * D + (size_t)hk * D;
      for (int i = lane; i < D; i += 32) dst[i] = src[i];
    }
    if (!kGqa) __syncthreads();
  }
  float qv[8];
  unpack8<T>(*reinterpret_cast<const uint4*>(kGqa && write_idx ? qkv_row + g * D + ch : q + ((size_t)b * H + h) * q_head_stride + ch), qv);
#pragma unroll
  for (int i = 0; i < 8; ++i) qv[i] *= scale;
  const size_t row_stride = (size_t)Hkv * D;
  const T* kb = k + (size_t)b * Lmax * row_stride + (size_t)hk * D + ch;
  const T* vb = v + (size_t)b * Lmax * row_stride + (size_t)hk * D + ch;
  const T* mb = mask ? mask + (size_t)b * Lmax : nullptr;
  float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int t0 = w * kU * kKW; t0 < L; t0 += kDecWarps * kU * kKW) {
    uint4 rk[kU], rv[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int t = t0 + u * kKW + sub;
      if (kGqa && t == new_pos) {
        rk[u] = *reinterpret_cast<const uint4*>(qkv_row + G * D + ch);
        rv[u] = *reinterpret_cast<const uint4*>(qkv_row + (G + 1) * D + ch);
      } else if (t < L) {
        rk[u] = ld_stream(reinterpret_cast<const uint4*>(kb + (size_t)t * row_stride));
        rv[u] = ld_stream(reinterpret_cast<const uint4*>(vb + (size_t)t * row_stride));
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int t = t0 + u * kKW + sub;
      const bool live = t < L;                      // uniform inside a lane group; shuffles below stay inside the group
      float kf[8], vf[8];
      if (live) { unpack8<T>(rk[u], kf); unpack8<T>(rv[u], vf); }
      float sc = 0.f;
      if (live) {
#pragma unroll
        for (int i = 0; i < 8; ++i) sc = fmaf(qv[i], kf[i], sc);
      }
#pragma unroll
      for (int o = kLanes / 2; o > 0; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
      if (live) {
        if (mb) sc += to_f32<T>(mb[t]);
        // a state whose keys so far are all masked with -inf has m = m_new = -inf: it must stay empty (l = 0), not turn into NaN
        const float m_new = fmaxf(m, sc);
        const float corr = (m == -INFINITY) ? 0.f : __expf(m - m_new), p = (sc == -INFINITY) ? 0.f : __expf(sc - m_new);
        l = l * corr + p;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = acc[i] * corr + p * vf[i];
        m = m_new;
      }
    }
  }
  const int state = w * kKW + sub;
  if (lane % kLanes == 0) { s_m[state] = m; s_l[state] = l; }
#pragma unroll
  for (int i = 0; i < 8; ++i) s_acc[state][ch + i] = acc[i];
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float mm = -INFINITY;
#pragma unroll
    for (int i = 0; i < kStates; ++i) mm = fmaxf(mm, s_m[i]);
    float ll = 0.f, a = 0.f;
#pragma unroll
    for (int i = 0; i < kStates; ++i) {
      const float f = (s_m[i] == -INFINITY) ? 0.f : __expf(s_m[i] - mm);
      ll += s_l[i] * f;
      a += s_acc[i][c] * f;
    }
    out[((size_t)b * H + h) * D + c] = from_f32<T>(ll > 0.f ? a / ll : 0.f);
  }
}

}  // namespace

cudaError_t attention_decode(const void* q, void* k, void* v, const void* mask, void* out, int B, int H, int D, int L, int Lmax,
                             float scale, int dtype, cudaStream_t st, const int64_t* write_idx, int Hkv) {
  if (!B || !H) return cudaSuccess;
  if (Hkv == 0) Hkv = H;
  if ((D != 64 && D != 128) || L < 1 || L > Lmax || Hkv < 1 || H % Hkv != 0) return cudaErrorInvalidValue;
  const dim3 grid(H, B), block(kDecWarps * 32);
  const int G = H / Hkv;
#define PFX_AD(T, P, GQA) attention_decode_kernel<T, P, GQA><<<grid, block, 0, st>>>((const T*)q, (T*)k, (T*)v, (const T*)mask, (T*)out, L, Lmax, H, scale, write_idx, G)
#define PFX_AD_D(T, GQA) do { if (D == 128) PFX_AD(T, 128, GQA); else PFX_AD(T, 64, GQA); } while (0)
  if (dtype == 1) { if (G > 1) PFX_AD_D(__nv_bfloat16, true); else PFX_AD_D(__nv_bfloat16, false); }
  else if (dtype == 0) { if (G > 1) PFX_AD_D(__half, true); else PFX_AD_D(__half, false); }
  else return cudaErrorInvalidValue;
#undef PFX_AD_D
#undef PFX_AD
  return cudaGetLastError();
}

}  // namespace pfx
