// ZeRO collectives written against symmetric memory (symm_vmm.cpp): NVLink-SHARP multicast addresses where the fabric
// offers them, unicast peer pointers otherwise.
//
//   * reduce-scatter   multimem.ld_reduce on the calling rank's shard: the NVSwitch reads the N copies and returns their
//                      fp32-accumulated sum, so a rank receives 1/N of the bucket over its link instead of (N-1)/N, and
//                      issues one load stream instead of N.  The kernel also emits the shard's sum of squares (global
//                      grad-norm without another pass over the gradients).
//   * AdamW+broadcast  the owner updates its fp32 master shard and stores the new bf16 weights once with multimem.st;
//                      the switch replicates the store into every rank's parameter buffer (update + all-gather, one kernel,
//                      1/N of the bucket leaves each GPU instead of (N-1)/N).
//   * all-gather       same store path for plain shards (ZeRO-3 parameter gather, tests).
//   * barrier          one multimem.red (+1 on every rank's flag word) + a local acquire spin.
//
// Every kernel is 256 threads, <= 72 registers and ZERO shared memory (static included), so that a CTA takes little of an SM.  It does
// NOT fit beside a persistent wgmma GEMM CTA: that one holds 288 threads x 168 registers (about 50 K of the SM's 64 K registers), and 256 x 72
// more do not fit.  Communication CTAs therefore get SMs when a GEMM CTA retires, not a place inside a busy SM; the overlap of these kernels
// with the GEMMs has not been run on H100.
//
// Reference call sites: sharding reduce / broadcast overlap knobs, eager_engine.py:293-307 (NCCL launches in Paddle).
#include "pfx_common.cuh"
#include "pfx_kernels.h"
#include "pfx_symm.h"

#include <cstdio>

namespace pfx {

namespace {

constexpr int kMaxWorld = 16;
struct Peers { void* p[kMaxWorld]; };

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- multimem (NVLS) accessors: 16 bytes per instruction
template <typename T> __device__ __forceinline__ uint4 mm_ld_reduce(const void* mc);
template <> __device__ __forceinline__ uint4 mm_ld_reduce<__nv_bfloat16>(const void* mc) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc) : "memory");
  return r;
}
template <> __device__ __forceinline__ uint4 mm_ld_reduce<__half>(const void* mc) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc) : "memory");
  return r;
}
template <> __device__ __forceinline__ uint4 mm_ld_reduce<float>(const void* mc) {
  float4 f;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(f.x), "=f"(f.y), "=f"(f.z), "=f"(f.w) : "l"(mc) : "memory");
  return make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
}
__device__ __forceinline__ void mm_st(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
               ::"l"(mc), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

template <typename T> struct Pack { static constexpr int kElems = 16 / sizeof(T); };

template <typename T> __device__ __forceinline__ void unpack16(const uint4& raw, float (&f)[Pack<T>::kElems]) {
  if constexpr (sizeof(T) == 4) {
    f[0] = __uint_as_float(raw.x); f[1] = __uint_as_float(raw.y); f[2] = __uint_as_float(raw.z); f[3] = __uint_as_float(raw.w);
  } else {
    unpack8<T>(raw, f);
  }
}

// Write kElems fp32 values as TOut (same element count, so the byte width differs when TIn != TOut).
template <typename TOut, int kElems>
__device__ __forceinline__ void store_elems(TOut* dst, const float (&f)[kElems], bool accumulate) {
  if constexpr (sizeof(TOut) == 4) {
#pragma unroll
    for (int j = 0; j < kElems; j += 4) {
      float4 o = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
      if (accumulate) { const float4 old = *reinterpret_cast<const float4*>(dst + j); o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w; }
      *reinterpret_cast<float4*>(dst + j) = o;
    }
  } else {
    static_assert(kElems == 8, "16-bit outputs are written 8 at a time");
    float g[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = f[j];
    if (accumulate) {
      float old[8];
      unpack8<TOut>(*reinterpret_cast<const uint4*>(dst), old);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] += old[j];
    }
    *reinterpret_cast<uint4*>(dst) = pack8<TOut>(g);
  }
}

// One atomic per warp and NO shared memory: a single byte of static shared memory would make the CTA need a second kilobyte next
// to the one the system reserves per CTA, and then it no longer fits beside a GEMM CTA (measured: serialisation instead of overlap).
__device__ __forceinline__ void warp_atomic_add(float v, float* out) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(out, v);
}

// ------------------------------------------------------------------ barriers
__global__ void nvls_barrier_kernel(uint32_t* mc_flag, uint32_t* local_flag, uint32_t target) {
  if (threadIdx.x != 0) return;
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_flag), "r"(1u) : "memory");
  const long long t0 = clock64();
  while ((int32_t)(ld_acquire_sys_u32(local_flag) - target) < 0) {
    if (clock64() - t0 > 40000000000ll) { printf("pfx: nvls barrier timeout (target %u, flag %u)\n", target, ld_acquire_sys_u32(local_flag)); __trap(); }
  }
}

__global__ void p2p_flag_barrier_kernel(Peers flags, int rank, int world, uint32_t epoch) {
  const int peer = threadIdx.x;
  if (peer >= world) return;
  __threadfence_system();
  st_release_sys_u32(reinterpret_cast<uint32_t*>(flags.p[peer]) + rank, epoch);
  const uint32_t* mine = reinterpret_cast<const uint32_t*>(flags.p[rank]) + peer;
  const long long t0 = clock64();
  while ((int32_t)(ld_acquire_sys_u32(mine) - epoch) < 0) {
    if (clock64() - t0 > 40000000000ll) { printf("pfx: p2p barrier timeout (rank %d waits for %d, epoch %u)\n", rank, peer, epoch); __trap(); }
  }
}

// ------------------------------------------------------------------ reduce-scatter
// kMc: in-switch reduction through the multicast address; otherwise a pull over the unicast peer pointers in a fixed
// rank-relative order (bitwise reproducible).
template <typename TIn, typename TOut, bool kMc>
__global__ void __launch_bounds__(256) symm_reduce_scatter_kernel(const TIn* __restrict__ mc_src, Peers peers, size_t shard_off, TOut* __restrict__ out,
                                                                  size_t n, int rank, int world, float scale, bool accumulate,
                                                                  float* __restrict__ sumsq) {
  constexpr int kE = Pack<TIn>::kElems;
  constexpr int kUnroll = kMc ? 4 : 2;
  const size_t nvec = n / kE;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float sq = 0.f;
  for (size_t i0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * kUnroll) {
    float acc[kUnroll][kE];
    if constexpr (kMc) {
      uint4 raw[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t i = i0 + u * stride;
        if (i < nvec) raw[u] = mm_ld_reduce<TIn>(mc_src + shard_off + i * kE);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) unpack16<TIn>(raw[u], acc[u]);
    } else {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
#pragma unroll
        for (int j = 0; j < kE; ++j) acc[u][j] = 0.f;
      for (int p0 = 0; p0 < world; p0 += 4) {          // four peers' loads in flight per vector, then fold
        uint4 raw[kUnroll][4];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const size_t i = i0 + u * stride;
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (i < nvec && p0 + q < world)
              raw[u][q] = ld_stream(reinterpret_cast<const uint4*>(reinterpret_cast<const TIn*>(peers.p[(rank + p0 + q) % world]) + shard_off) + i);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (p0 + q < world) {
              float v[kE];
              unpack16<TIn>(raw[u][q], v);
#pragma unroll
              for (int j = 0; j < kE; ++j) acc[u][j] += v[j];
            }
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t i = i0 + u * stride;
      if (i >= nvec) continue;
#pragma unroll
      for (int j = 0; j < kE; ++j) { acc[u][j] *= scale; sq += acc[u][j] * acc[u][j]; }
      store_elems<TOut, kE>(out + i * kE, acc[u], accumulate);
    }
  }
  if (sumsq != nullptr) warp_atomic_add(sq, sumsq);
}

// ------------------------------------------------------------------ all-gather
template <bool kMc>
__global__ void __launch_bounds__(256) symm_all_gather_kernel(uint4* __restrict__ mc_dst, Peers peers, size_t dst_vec_off, const uint4* __restrict__ src,
                                                              size_t nvec, int rank, int world) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * 4) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) if (i0 + u * stride < nvec) v[u] = ld_stream(src + i0 + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const size_t i = i0 + u * stride;
      if (i >= nvec) continue;
      if constexpr (kMc) {
        mm_st(mc_dst + dst_vec_off + i, v[u]);
      } else {
        for (int p = 0; p < world; ++p) st_stream(reinterpret_cast<uint4*>(peers.p[(rank + p) % world]) + dst_vec_off + i, v[u]);
      }
    }
  }
}

// ------------------------------------------------------------------ AdamW + parameter broadcast
template <typename TG, typename TP, bool kMc>
__global__ void __launch_bounds__(256) adamw_symm_kernel(TP* __restrict__ mc_params, Peers peers, size_t shard_off, float* __restrict__ master,
                                                         const TG* __restrict__ grad, float* __restrict__ m, float* __restrict__ v, size_t n, float lr,
                                                         float beta1, float beta2, float eps, float wd, float bc1, float bc2,
                                                         const float* __restrict__ gscale, const float* __restrict__ found_inf, int rank, int world) {
  if (found_inf && found_inf[0] != 0.f) return;      // skipped step: the low-precision weights every rank holds are still current
  const float gs = gscale ? gscale[0] : 1.f;
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  const float decay = 1.f - lr * wd, omb1 = 1.f - beta1, omb2 = 1.f - beta2;
  const size_t nvec = n >> 3;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float g[8], w8[8], mm[8], vv[8];
    load4<TG>(grad + i * 8, *reinterpret_cast<float(*)[4]>(&g[0]));
    load4<TG>(grad + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&g[4]));
    load4<float>(master + i * 8, *reinterpret_cast<float(*)[4]>(&w8[0]));
    load4<float>(master + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&w8[4]));
    load4<float>(m + i * 8, *reinterpret_cast<float(*)[4]>(&mm[0]));
    load4<float>(m + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&mm[4]));
    load4<float>(v + i * 8, *reinterpret_cast<float(*)[4]>(&vv[0]));
    load4<float>(v + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&vv[4]));
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = g[j] * gs;
      mm[j] = beta1 * mm[j] + omb1 * gj;
      vv[j] = beta2 * vv[j] + omb2 * gj * gj;
      w8[j] = w8[j] * decay - step_size * mm[j] / (sqrtf(vv[j]) * inv_sqrt_bc2 + eps);
    }
    store4<float>(m + i * 8, *reinterpret_cast<float(*)[4]>(&mm[0]));
    store4<float>(m + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&mm[4]));
    store4<float>(v + i * 8, *reinterpret_cast<float(*)[4]>(&vv[0]));
    store4<float>(v + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&vv[4]));
    store4<float>(master + i * 8, *reinterpret_cast<float(*)[4]>(&w8[0]));
    store4<float>(master + i * 8 + 4, *reinterpret_cast<float(*)[4]>(&w8[4]));
    const uint4 packed = pack8<TP>(w8);
    if constexpr (kMc) {
      mm_st(reinterpret_cast<uint4*>(mc_params + shard_off) + i, packed);       // one store, replicated by the switch
    } else {
      for (int p = 0; p < world; ++p)
        st_stream(reinterpret_cast<uint4*>(reinterpret_cast<TP*>(peers.p[(rank + p) % world]) + shard_off) + i, packed);
    }
  }
}

Peers make_peers(void* const* tab, int world) {
  Peers pp{};
  if (tab) for (int i = 0; i < world && i < kMaxWorld; ++i) pp.p[i] = tab[i];
  return pp;
}

}  // namespace

cudaError_t nvls_barrier(uint32_t* mc_flag, uint32_t* local_flag, uint32_t target, cudaStream_t st) {
  nvls_barrier_kernel<<<1, 32, 0, st>>>(mc_flag, local_flag, target);
  return cudaGetLastError();
}

cudaError_t p2p_flag_barrier(uint32_t** peer_flags, int rank, int world, uint32_t epoch, cudaStream_t st) {
  if (world > kMaxWorld) return cudaErrorInvalidValue;
  p2p_flag_barrier_kernel<<<1, 32, 0, st>>>(make_peers(reinterpret_cast<void* const*>(peer_flags), world), rank, world, epoch);
  return cudaGetLastError();
}

template <typename TIn, typename TOut>
static cudaError_t rs_dispatch(const void* mc_src, const Peers& pp, size_t off, void* out, size_t n, int rank, int world, float scale, bool acc,
                               float* sumsq, int grid, cudaStream_t st) {
  if (mc_src) symm_reduce_scatter_kernel<TIn, TOut, true><<<grid, 256, 0, st>>>((const TIn*)mc_src, pp, off, (TOut*)out, n, rank, world, scale, acc, sumsq);
  else symm_reduce_scatter_kernel<TIn, TOut, false><<<grid, 256, 0, st>>>(nullptr, pp, off, (TOut*)out, n, rank, world, scale, acc, sumsq);
  return cudaGetLastError();
}

cudaError_t symm_reduce_scatter(const void* mc_src, void* const* peer_src, size_t shard_offset_elems, void* out, size_t n, int rank, int world,
                                int in_dtype, int out_dtype, float scale, bool accumulate, float* sumsq, int num_ctas, cudaStream_t st) {
  if (world > kMaxWorld || (mc_src == nullptr && peer_src == nullptr)) return cudaErrorInvalidValue;
  const size_t per = in_dtype == 3 ? 4 : 8;
  if (n % per || shard_offset_elems % per) return cudaErrorInvalidValue;
  if (!n) return cudaSuccess;
  const Peers pp = make_peers(peer_src, world);
  if (num_ctas < 1) num_ctas = 1;
  if (in_dtype == 1 && out_dtype == 1) return rs_dispatch<__nv_bfloat16, __nv_bfloat16>(mc_src, pp, shard_offset_elems, out, n, rank, world, scale, accumulate, sumsq, num_ctas, st);
  if (in_dtype == 1 && out_dtype == 3) return rs_dispatch<__nv_bfloat16, float>(mc_src, pp, shard_offset_elems, out, n, rank, world, scale, accumulate, sumsq, num_ctas, st);
  if (in_dtype == 0 && out_dtype == 0) return rs_dispatch<__half, __half>(mc_src, pp, shard_offset_elems, out, n, rank, world, scale, accumulate, sumsq, num_ctas, st);
  if (in_dtype == 0 && out_dtype == 3) return rs_dispatch<__half, float>(mc_src, pp, shard_offset_elems, out, n, rank, world, scale, accumulate, sumsq, num_ctas, st);
  if (in_dtype == 3 && out_dtype == 3) return rs_dispatch<float, float>(mc_src, pp, shard_offset_elems, out, n, rank, world, scale, accumulate, sumsq, num_ctas, st);
  return cudaErrorInvalidValue;
}

cudaError_t symm_all_gather(void* mc_dst, void* const* peer_dst, size_t dst_offset_bytes, const void* src, size_t bytes, int rank, int world,
                            int num_ctas, cudaStream_t st) {
  if (world > kMaxWorld || bytes % 16 || dst_offset_bytes % 16 || (mc_dst == nullptr && peer_dst == nullptr)) return cudaErrorInvalidValue;
  if (!bytes) return cudaSuccess;
  const Peers pp = make_peers(peer_dst, world);
  if (num_ctas < 1) num_ctas = 1;
  if (mc_dst) symm_all_gather_kernel<true><<<num_ctas, 256, 0, st>>>((uint4*)mc_dst, pp, dst_offset_bytes / 16, (const uint4*)src, bytes / 16, rank, world);
  else symm_all_gather_kernel<false><<<num_ctas, 256, 0, st>>>(nullptr, pp, dst_offset_bytes / 16, (const uint4*)src, bytes / 16, rank, world);
  return cudaGetLastError();
}

cudaError_t adamw_symm_broadcast(void* mc_params, void* const* peer_params, size_t shard_offset_elems, float* master, const void* grad, float* m,
                                 float* v, size_t n, float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2,
                                 const float* gscale, const float* found_inf, int grad_dtype, int lp_dtype, int rank, int world, int num_ctas,
                                 cudaStream_t st) {
  if (n % 8 || shard_offset_elems % 8 || world > kMaxWorld || (mc_params == nullptr && peer_params == nullptr)) return cudaErrorInvalidValue;
  if (!n) return cudaSuccess;
  const Peers pp = make_peers(peer_params, world);
  if (num_ctas < 1) num_ctas = 1;
#define PFX_AS(TG, TP)                                                                                                                         \
  do {                                                                                                                                         \
    if (mc_params) adamw_symm_kernel<TG, TP, true><<<num_ctas, 256, 0, st>>>((TP*)mc_params, pp, shard_offset_elems, master, (const TG*)grad, m, v, n, lr, beta1, beta2, eps, wd, bc1, bc2, gscale, found_inf, rank, world); \
    else adamw_symm_kernel<TG, TP, false><<<num_ctas, 256, 0, st>>>(nullptr, pp, shard_offset_elems, master, (const TG*)grad, m, v, n, lr, beta1, beta2, eps, wd, bc1, bc2, gscale, found_inf, rank, world); \
  } while (0)
  if (grad_dtype == 3 && lp_dtype == 1) PFX_AS(float, __nv_bfloat16);
  else if (grad_dtype == 3 && lp_dtype == 0) PFX_AS(float, __half);
  else if (grad_dtype == 1 && lp_dtype == 1) PFX_AS(__nv_bfloat16, __nv_bfloat16);
  else if (grad_dtype == 0 && lp_dtype == 0) PFX_AS(__half, __half);
  else return cudaErrorInvalidValue;
#undef PFX_AS
  return cudaGetLastError();
}

}  // namespace pfx
