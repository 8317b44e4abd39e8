// Small-M ("swap-AB") wgmma GEMM with split-K across a thread-block cluster, for prefill and batched decode.
//
//   y[M, N] = x[M, K] * W[N, K]^T (+ bias[N]),   3 <= M <= 128 (M <= 2 is served by gemv_skinny.cu)
//
// With so few activation rows the op is a weight stream: the regular 128x128-tile kernel would waste most of every
// wgmma and, worse, light up only N/128 SMs.  Here the roles are swapped — the WEIGHT tile is the A operand (two
// wgmma M = 64 halves of 128 weight rows), the activations are the narrow B operand (wgmma N = M rounded up to
// 16/32/64/128) and the accumulator fragment holds y^T — and K is split across the CTAs of a cluster so that
// N/128 x kSplit CTAs pull weights through TMA concurrently.  The partial accumulators are reduced through
// distributed shared memory: every CTA scatters 128/kSplit-row slices of its fp32 partial tile into the owning
// CTA's smem (st.shared::cluster), one cluster barrier, and each owner sums its kSplit slices, adds the bias and
// writes bf16 — no global workspace, no atomics, no second kernel.
//
// warp 4: TMA producer + barrier init, warps 0-3: one consumer warpgroup (products, then the reduction epilogue).
// Reference call sites: the decode / prefill linears of GPTForGeneration (hybrid_model.py:1202-1339) run cuBLAS.
#include "pfx_ptx.cuh"
#include "pfx_gemm.h"
#include "pfx_kernels.h"
#include <cudaTypedefs.h>

namespace pfx {

namespace {

constexpr int kSmTileN = 128;   // weight rows per CTA (two wgmma M = 64 halves)
constexpr int kSmBlockK = 64;
constexpr int kSmMmaK = 16;
constexpr int kSmThreads = 160;

template <int kMPad>
struct SmallMSmem {
  static constexpr int kABytes = kSmTileN * kSmBlockK * 2;
  static constexpr int kBBytes = kMPad * kSmBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRedBytes = kSmTileN * kMPad * 4;        // [kSplit][kMPad][128 / kSplit] fp32, independent of kSplit
  static constexpr int kBarrierBytes = 256;
  static constexpr int kBudget = 200 * 1024 - kRedBytes - kBarrierBytes;
  static constexpr int kStages = (kBudget / kStageBytes) > 6 ? 6 : (kBudget / kStageBytes);
  static constexpr int kTotal = 1024 + kStages * kStageBytes + kRedBytes + kBarrierBytes;
};

__device__ __forceinline__ void st_shared_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

template <typename T, int kMPad, int kSplit>
__global__ void __launch_bounds__(kSmThreads, 1)
gemm_smallm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x, const T* __restrict__ bias,
                   T* __restrict__ y, int M, int N, int K, int ab_format) {
  using S = SmallMSmem<kMPad>;
  constexpr int kStages = S::kStages;
  constexpr int kRowsPerOwner = kSmTileN / kSplit;
  static_assert(kStages >= 2, "pipeline needs at least two stages");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_ab = smem_base;
  const uint32_t smem_red = smem_base + kStages * S::kStageBytes;
  const uint32_t smem_bar = smem_red + S::kRedBytes;
  auto full_bar = [&](int s) { return smem_bar + 8u * s; };
  auto empty_bar = [&](int s) { return smem_bar + 8u * (kStages + s); };
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  const uint32_t warp = warp_id();
  const uint32_t lane = lane_id();
  const uint32_t krank = kSplit > 1 ? cluster_ctarank() : 0u;
  const int tile = blockIdx.x / kSplit;
  const int n0 = tile * kSmTileN;

  const int total_kb = (K + kSmBlockK - 1) / kSmBlockK;
  const int per = (total_kb + kSplit - 1) / kSplit;
  const int kb_lo = min((int)krank * per, total_kb);
  const int kb_hi = min(kb_lo + per, total_kb);
  const int my_kb = kb_hi - kb_lo;

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4); }
    fence_barrier_init();
  }
  if (kSplit > 1) cluster_sync(); else __syncthreads();      // also: every CTA of the cluster is running before DSMEM is touched

  if (warp == 4) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = kb_lo; kb < kb_hi; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t sa = smem_ab + stage * S::kStageBytes;
        const uint32_t fb = full_bar(stage);
        mbar_arrive_expect_tx(fb, S::kStageBytes);
        tma_load_2d(&tmap_w, fb, sa, kb * kSmBlockK, n0);
        tma_load_2d(&tmap_x, fb, sa + S::kABytes, kb * kSmBlockK, 0);
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // ---- products: acc[hw] = weight rows [64 hw, 64 hw + 64) of the tile x activations^T
    constexpr uint64_t kDesc = wgmma_desc_hi_lo(16, 1024);      // K-major, 128-byte swizzle
    float acc[2][kMPad / 2];
#pragma unroll
    for (int i = 0; i < kMPad / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    int stage = 0; uint32_t phase = 0;
    for (int kb = 0; kb < my_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_ab + stage * S::kStageBytes;
      const uint32_t sb = sa + S::kABytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kSmBlockK / kSmMmaK; ++k) {
        const uint64_t db = wgmma_desc(sb + k * kSmMmaK * 2, kDesc);
        WgmmaSS<kMPad, true, 0, 0>::mma(acc[0], wgmma_desc(sa + k * kSmMmaK * 2, kDesc), db, 1u);      // bf16 only (checked by the host wrapper)
        WgmmaSS<kMPad, true, 0, 0>::mma(acc[1], wgmma_desc(sa + 8192 + k * kSmMmaK * 2, kDesc), db, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(stage));
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
    // ---- epilogue part 1: scatter my partial tile (row n = weight row, column m = activation row) to the row owners
#pragma unroll
    for (int hw = 0; hw < 2; ++hw) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int n_local_cta = hw * 64 + (int)(warp * 16u + (lane >> 2)) + 8 * hh;                   // 0..127 inside the tile
        const int owner = n_local_cta / kRowsPerOwner;
        const int n_in_owner = n_local_cta % kRowsPerOwner;
        const uint32_t red_remote = kSplit > 1 ? mapa(smem_red, (uint32_t)owner) : smem_red;
#pragma unroll
        for (int j = 0; j < kMPad / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = 8 * j + (int)(lane & 3u) * 2 + e;
            if (m < M) {
              const uint32_t off = (uint32_t)((((int)krank * kMPad + m) * kRowsPerOwner + n_in_owner) * 4);
              const float val = acc[hw][4 * j + 2 * hh + e];
              if (kSplit > 1) st_shared_cluster_f32(red_remote + off, val);
              else *reinterpret_cast<float*>(smem_gen + (smem_red - smem_base) + off) = val;
            }
          }
        }
      }
    }
  }

  if (kSplit > 1) cluster_sync(); else __syncthreads();

  if (warp < 4) {
    // ---- epilogue part 2: this CTA owns rows [krank * R, (krank + 1) * R) of the tile: sum the kSplit partials, bias, store
    const float* red = reinterpret_cast<const float*>(smem_gen + (smem_red - smem_base));
    const int t = (int)threadIdx.x;
    const int row0 = n0 + (int)krank * kRowsPerOwner;
    for (int idx = t; idx < M * kRowsPerOwner; idx += 128) {
      const int m = idx / kRowsPerOwner, nl = idx % kRowsPerOwner;
      const int n = row0 + nl;
      if (n >= N) continue;
      float v = bias ? __bfloat162float(bias[n]) : 0.f;
#pragma unroll
      for (int s = 0; s < kSplit; ++s) v += red[(s * kMPad + m) * kRowsPerOwner + nl];
      y[(size_t)m * N + n] = __float2bfloat16(v);
    }
  }
}

template <int kMPad, int kSplit>
cudaError_t launch_smallm(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, cudaStream_t st) {
  using S = SmallMSmem<kMPad>;
  CUtensorMap tw, tx;
  bool ok = make_tmap_2d(&tw, w, 2, 1, (uint64_t)K, (uint64_t)N, (uint64_t)K * 2, kSmBlockK, kSmTileN);
  ok &= make_tmap_2d(&tx, x, 2, 1, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kSmBlockK, kMPad);
  if (!ok) return cudaErrorInvalidValue;
  auto kern = gemm_smallm_kernel<__nv_bfloat16, kMPad, kSplit>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int tiles = (N + kSmTileN - 1) / kSmTileN;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(tiles * kSplit);
  cfg.blockDim = dim3(kSmThreads);
  cfg.dynamicSmemBytes = S::kTotal;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kSplit; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, tw, tx, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, M, N, K, 1);
}

template <int kMPad>
cudaError_t launch_split(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int split, cudaStream_t st) {
  switch (split) {
    case 1: return launch_smallm<kMPad, 1>(x, w, bias, y, M, N, K, st);
    case 2: return launch_smallm<kMPad, 2>(x, w, bias, y, M, N, K, st);
    case 4: return launch_smallm<kMPad, 4>(x, w, bias, y, M, N, K, st);
    default: return launch_smallm<kMPad, 8>(x, w, bias, y, M, N, K, st);
  }
}

}  // namespace

cudaError_t gemm_smallm(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int dtype, int split, int num_sms,
                        cudaStream_t st) {
  if (dtype != 1 || M < 1 || M > 128 || K % 8 || N % 8) return cudaErrorInvalidValue;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15) return cudaErrorMisalignedAddress;
  if (split <= 0) {        // enough CTAs to cover the machine, but keep >= 4 k-blocks per CTA
    const int tiles = (N + kSmTileN - 1) / kSmTileN;
    const int total_kb = (K + kSmBlockK - 1) / kSmBlockK;
    split = 1;
    while (split < 8 && tiles * split < num_sms && total_kb / (split * 2) >= 4) split *= 2;
  }
  if (M <= 16) return launch_split<16>(x, w, bias, y, M, N, K, split, st);
  if (M <= 32) return launch_split<32>(x, w, bias, y, M, N, K, split, st);
  if (M <= 64) return launch_split<64>(x, w, bias, y, M, N, K, split, st);
  return launch_split<128>(x, w, bias, y, M, N, K, split, st);
}

}  // namespace pfx
