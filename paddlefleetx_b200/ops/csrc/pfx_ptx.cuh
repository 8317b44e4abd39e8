// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), cluster helpers; the wgmma wrappers live in
// pfx_wgmma.cuh.  Everything the kernels in this directory need and nothing else — no CUTLASS.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#include "pfx_wgmma.cuh"

#ifndef PFX_HANG_GUARD
#define PFX_HANG_GUARD 1  // trap instead of spinning forever on a lost mbarrier arrival
#endif

namespace pfx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xffffffff;\n"
      "selp.b32 %0, 1, 0, px;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Register reallocation between the warpgroups of a CTA: every thread of the warpgroup executes the same instruction; the count is a
// multiple of 8 in [24, 256].
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// ------------------------------------------------------------------ cluster
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_sync() { cluster_arrive(); cluster_wait(); }
__device__ __forceinline__ uint32_t mapa(uint32_t smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(cta_rank));
  return r;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on a barrier living in another CTA of the cluster (address from mapa)
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
#if PFX_HANG_GUARD
  // try_wait suspends the warp for a hardware time slice per attempt; the guard only counts attempts (one IADD + one compare per poll — a
  // clock read per poll showed up as ~10 % of all issued instructions in the attention kernels) and looks at the clock every 4096 polls
  uint32_t polls = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 0xFFFu) == 0u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ll) __trap();  // ~2 s at H100 clocks: a lost arrival, not a slow producer.  No printf here: a function call in
                                                   // this inlined wait makes ptxas serialise every wgmma of the calling kernel (C7510)
    }
  }
#else
  while (!mbar_try_wait(bar, parity)) {}
#endif
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load into this CTA's smem, completion on this CTA's mbarrier.
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 3-D tile load (attention: [columns, sequence, batch] views with arbitrary sequence / batch strides)
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 1-D bulk copy global -> shared (size and both addresses multiples of 16 bytes), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
// smem tile += into global memory (element-wise add performed by the TMA unit / L2, fp32 tensor map): the reduction traffic of a
// split accumulation (attention dQ) without a single per-lane atomic on the SM
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------ misc math
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {   // round to nearest; beyond 65504 the result is +-inf
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// 16-bit element type chosen at compile time: kBf16 = bf16, otherwise fp16
template <bool kBf16>
__device__ __forceinline__ uint32_t pack_16x2(float lo, float hi) {
  if constexpr (kBf16) return pack_bf16x2(lo, hi);
  else return pack_f16x2(lo, hi);
}
template <bool kBf16>
__device__ __forceinline__ float2 load_16x2(const void* p) {   // two adjacent 16-bit values (4-byte aligned) as floats
  if constexpr (kBf16) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
  else return __half22float2(*reinterpret_cast<const __half2*>(p));
}
template <bool kBf16>
__device__ __forceinline__ float2 unpack_16x2(uint32_t w) {   // the two 16-bit values of a 32-bit word (low first) as floats
  if constexpr (kBf16) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
  else return __half22float2(*reinterpret_cast<const __half2*>(&w));
}
__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * x * (1.f + k1 * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.f + t);
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float x2 = x * x;
  float u = k0 * x * (1.f + k1 * x2);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  float du = k0 * (1.f + 3.f * k1 * x2);
  return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * du;
}
// sigmoid of a SwiGLU gate: for a < -88 __expf(-a) overflows to inf and s = 0 exactly, so every SwiGLU product stays finite
__device__ __forceinline__ float swiglu_sigmoid(float a) { return 1.f / (1.f + __expf(-a)); }

}  // namespace pfx
