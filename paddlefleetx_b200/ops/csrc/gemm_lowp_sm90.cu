// 8-bit wgmma GEMMs for sm_90a: int8 x int8 -> int32 (the W8A8 inference GEMM behind the QAT / SmoothQuant export) and
// fp8 e4m3 x e4m3 -> fp32 (the scaled TP GEMM).
//
//   D[M,N] (bf16 or fp16) = (A_q[M,K] * B_q[N,K]^T) * row_scale[M] * col_scale[N] (+ bias[N], same dtype as D)
//
// Same pipeline as gemm_sm90.cu (TMA producer warp, two consumer warpgroups with the accumulator fragment in registers, swizzled smem
// staging + TMA store, persistent grouped raster, 128 x 128 tiles) with the 8-bit specifics: 128 elements per 128-byte swizzle row
// (BLOCK_K = 128), wgmma K = 32, integer accumulators are converted with I2F in the epilogue and the per-token / per-channel
// dequantisation scales are applied there, so the int32 / fp32 product never touches HBM.  Reference: L23 in SURVEY §2.6
// (Paddle-Inference / TensorRT int8 passes — no in-tree kernel in the reference).
//
// fp8 accumulation: the tensor core does not keep a full fp32 sum across an fp8 wgmma chain.  On an H100 a 128-K chain of positive
// terms loses up to 2^-10 of their sum, and one chain over K = 16384 lost 25 % (tests/test_gpu_lowp_kernels.py).  Kind 2 therefore runs
// one chain per k-block (128 K, one stage) into a fresh partial and adds it to the fp32 accumulator in registers.
//
// kKind 3 = MX block-scaled fp8: every 32 K-elements of every row of A and B carry their own E8M0 scale (2^(e - 127)).  Hopper's tensor
// core has no block-scale mode, so each K = 32 wgmma writes a fresh partial product and the consumer threads fold it into the fp32
// accumulator with the two scales of its (row, column, K block).  The quantiser (quant_kernels.cu) writes the scale bytes as one
// 512-byte atom per (128 rows, 128 K): byte (r % 32) * 16 + (r / 32) * 4 + k32 — a stage needs one 512-byte bulk copy per operand.
#include <type_traits>

#include "pfx_ptx.cuh"
#include "pfx_gemm.h"
#include <cudaTypedefs.h>

namespace pfx {
namespace lowp {

constexpr int kBlockM = 128;
constexpr int kBlockN = 128;
constexpr int kBlockK = 128;      // 8-bit elements: 128 B = one swizzle span
constexpr int kMmaK = 32;
constexpr int kNumThreads = 288;  // warps 0-7 = two consumer warpgroups, warp 8 = TMA producer
constexpr int kGroupM = 16;
constexpr int kStoreCols = 64;

template <bool kMx = false>
struct Smem {
  static constexpr int kABytes = kBlockM * kBlockK;
  static constexpr int kBBytes = kBlockN * kBlockK;
  static constexpr int kSfBytes = 512;                      // one scale-factor atom (128 rows x 4 K-blocks of 32) per operand, MX only
  static constexpr int kStageBytes = kABytes + kBBytes + (kMx ? 1024 : 0);   // 1 KB keeps the next stage on a swizzle-atom boundary
  static constexpr int kEpiBytes = kBlockM * kStoreCols * 2;
  static constexpr int kBudget = 227 * 1024 - 1024 - 1024 - 2 * kEpiBytes;
  static constexpr int kStages = (kBudget / kStageBytes) > 6 ? 6 : (kBudget / kStageBytes);
  static constexpr int kTotal = 1024 + kStages * kStageBytes + 2 * kEpiBytes + 1024;
};

__device__ __forceinline__ void tile_of(int tile, int num_m, int num_n, int& m_blk, int& n_blk) {
  const int per_group = kGroupM * num_n;
  const int group = tile / per_group;
  const int first = group * kGroupM;
  const int gm = min(kGroupM, num_m - first);
  const int in = tile - group * per_group;
  m_blk = first + in % gm;
  n_blk = in / gm;
}

__device__ __forceinline__ float e8m0_to_float(uint32_t e) { return __uint_as_float(e == 0u ? 0x00400000u : e << 23); }

// kKind: 1 = int8 (s32 accumulate), 2 = fp8 e4m3 (f32 accumulate, promoted per k-block), 3 = MX fp8 (per-32 block scales folded in by
// the consumers).  kBf16: D and bias are bf16, otherwise fp16.
template <int kKind, bool kBf16>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_lowp_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_d, const float* __restrict__ row_scale, const float* __restrict__ col_scale,
                 const void* __restrict__ bias, int M, int N, int K, const uint8_t* __restrict__ sfa, const uint8_t* __restrict__ sfb) {
  constexpr bool kMx = kKind == 3;
  using S = Smem<kMx>;
  using Acc = std::conditional_t<kKind == 1, int32_t, float>;
  constexpr int kStages = S::kStages;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_epi = smem_base + kStages * S::kStageBytes;
  const uint32_t smem_bar = smem_epi + 2 * S::kEpiBytes;
  auto full_bar = [&](int s) { return smem_bar + 8u * s; };
  auto empty_bar = [&](int s) { return smem_bar + 8u * (kStages + s); };
  const uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  const uint32_t warp = warp_id(), lane = lane_id();
  const int num_m = (M + kBlockM - 1) / kBlockM, num_n = (N + kBlockN - 1) / kBlockN;
  const int num_tiles = num_m * num_n, num_kb = (K + kBlockK - 1) / kBlockK;
  const int num_ctas = gridDim.x, cta_id = blockIdx.x;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmap_a); tma_prefetch_desc(&tmap_b); tma_prefetch_desc(&tmap_d);
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = cta_id; tile < num_tiles; tile += num_ctas) {
        int m_blk, n_blk; tile_of(tile, num_m, num_n, m_blk, n_blk);
        const int m_idx = m_blk * kBlockM, n_idx = n_blk * kBlockN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * S::kStageBytes, sb = sa + S::kABytes, fb = full_bar(stage);
          mbar_arrive_expect_tx(fb, S::kABytes + S::kBBytes + (kMx ? 2 * S::kSfBytes : 0));
          tma_load_2d(&tmap_a, fb, sa, kb * kBlockK, m_idx); tma_load_2d(&tmap_b, fb, sb, kb * kBlockK, n_idx);
          if constexpr (kMx) {      // the stage's two scale-factor atoms
            bulk_load_1d(sb + S::kBBytes, sfa + ((size_t)m_blk * num_kb + kb) * S::kSfBytes, S::kSfBytes, fb);
            bulk_load_1d(sb + S::kBBytes + S::kSfBytes, sfb + ((size_t)n_blk * num_kb + kb) * S::kSfBytes, S::kSfBytes, fb);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    const uint32_t wg = warp >> 2;
    const uint32_t row_lo = wg * 64u + (warp & 3u) * 16u + (lane >> 2);   // this thread's rows inside the CTA tile: row_lo and row_lo + 8
    const uint32_t col_in8 = (lane & 3u) * 2u;
    const bool is_store_thread = threadIdx.x == 0;
    constexpr uint64_t kDesc = wgmma_desc_hi_lo(16, 1024);
    int stage = 0; uint32_t phase = 0, store_iter = 0;
    for (int tile = cta_id; tile < num_tiles; tile += num_ctas) {
      int m_blk, n_blk; tile_of(tile, num_m, num_n, m_blk, n_blk);
      const int row0 = m_blk * kBlockM, col_tile = n_blk * kBlockN;
      Acc acc[kBlockN / 2];
      if constexpr (kKind != 1) {
#pragma unroll
        for (int i = 0; i < kBlockN / 2; ++i) acc[i] = 0;
      }
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa = smem_base + stage * S::kStageBytes + wg * 8192u, sb = smem_base + stage * S::kStageBytes + S::kABytes;
        if constexpr (kMx) {
          const uint8_t* sf = smem_gen + stage * S::kStageBytes + S::kABytes + S::kBBytes;     // A atom, then B atom
#pragma unroll
          for (int k = 0; k < kBlockK / kMmaK; ++k) {
            float part[kBlockN / 2];
            wgmma_fence();
            Wgmma8<kBlockN, false>::mma(part, wgmma_desc(sa + k * kMmaK, kDesc), wgmma_desc(sb + k * kMmaK, kDesc), 0u);
            wgmma_commit();
            float sa_f[2];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) { const uint32_t r = row_lo + 8u * hh; sa_f[hh] = e8m0_to_float(sf[(r % 32u) * 16u + (r / 32u) * 4u + k]); }
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < kBlockN / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint32_t c = 8u * j + col_in8 + e;
                const float sb_f = e8m0_to_float(sf[S::kSfBytes + (c % 32u) * 16u + (c / 32u) * 4u + k]);
                acc[4 * j + e] += part[4 * j + e] * (sa_f[0] * sb_f);
                acc[4 * j + 2 + e] += part[4 * j + 2 + e] * (sa_f[1] * sb_f);
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(stage));
        } else if constexpr (kKind == 2) {
          float part[kBlockN / 2];
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / kMmaK; ++k)
            Wgmma8<kBlockN, false>::mma(part, wgmma_desc(sa + k * kMmaK, kDesc), wgmma_desc(sb + k * kMmaK, kDesc), k != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
#pragma unroll
          for (int i = 0; i < kBlockN / 2; ++i) acc[i] += part[i];
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(stage));
        } else {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / kMmaK; ++k)        // 32 B per K = 32 step
            Wgmma8<kBlockN, true>::mma(acc, wgmma_desc(sa + k * kMmaK, kDesc), wgmma_desc(sb + k * kMmaK, kDesc), (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          if (prev_stage >= 0) {
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(empty_bar(prev_stage));
          }
          prev_stage = stage;
        }
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      if constexpr (kKind == 1) {
        wgmma_wait<0>();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
      }
      float rs[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) { const int grow = row0 + (int)row_lo + 8 * hh; rs[hh] = (row_scale && grow < M) ? row_scale[grow] : 1.f; }
#pragma unroll
      for (int c = 0; c < kBlockN / kStoreCols; ++c) {
        const int col0 = col_tile + c * kStoreCols;
        const int cb = col0 + (int)col_in8;
        float v[32];                              // v[4 j + e]: row row_lo + 8 (e / 2), column cb + 8 j + (e % 2)
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = (kKind == 1 ? __int2float_rn((int)acc[c * 32 + i]) : (float)acc[c * 32 + i]) * rs[(i >> 1) & 1];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (cb + 8 * j < N) {
            if (col_scale) {
              const float2 cs = __ldg(reinterpret_cast<const float2*>(col_scale + cb + 8 * j));
              v[4 * j] *= cs.x; v[4 * j + 1] *= cs.y; v[4 * j + 2] *= cs.x; v[4 * j + 3] *= cs.y;
            }
            if (bias) {
              const float2 f = load_16x2<kBf16>(static_cast<const uint16_t*>(bias) + cb + 8 * j);
              v[4 * j] += f.x; v[4 * j + 1] += f.y; v[4 * j + 2] += f.x; v[4 * j + 3] += f.y;
            }
          }
        }
        const uint32_t buf = store_iter & 1u;
        if (store_iter >= 2) {
          if (is_store_thread) tma_store_wait_read<1>();
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const uint32_t r = row_lo + 8u * hh;
          const uint32_t sbase = smem_epi + buf * S::kEpiBytes + r * 128u + col_in8 * 2u;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + (((uint32_t)j ^ (r & 7u)) << 4)), "r"(pack_16x2<kBf16>(v[4 * j + 2 * hh], v[4 * j + 2 * hh + 1])) : "memory");
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (is_store_thread) {
          if (col0 < N && row0 < M) tma_store_2d(&tmap_d, smem_epi + buf * S::kEpiBytes, col0, row0);
          tma_store_commit();
        }
        ++store_iter;
      }
    }
    if (is_store_thread) tma_store_wait<0>();
  }
}

template <int kKind, bool kBf16>
static cudaError_t launch(const LowpGemmArgs& g, cudaStream_t stream) {
  using S = Smem<kKind == 3>;
  if (kKind == 3 && (g.sfa == nullptr || g.sfb == nullptr || g.K % kBlockK != 0)) return cudaErrorInvalidValue;
  CUtensorMap ta, tb, td;
  bool ok = make_tmap_2d(&ta, g.a, 1, 2, g.K, g.M, (uint64_t)g.lda, kBlockK, kBlockM);
  ok &= make_tmap_2d(&tb, g.b, 1, 2, g.K, g.N, (uint64_t)g.ldb, kBlockK, kBlockN);
  ok &= make_tmap_2d(&td, g.d, 2, kBf16 ? 1 : 0, g.N, g.M, (uint64_t)g.ldd * 2, kStoreCols, kBlockM);
  if (!ok) return cudaErrorInvalidValue;
  auto kern = gemm_lowp_kernel<kKind, kBf16>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int tiles = ((g.M + kBlockM - 1) / kBlockM) * ((g.N + kBlockN - 1) / kBlockN);
  int ctas = g.num_sms;
  if (ctas > tiles) ctas = tiles;
  if (ctas < 1) ctas = 1;
  kern<<<ctas, kNumThreads, S::kTotal, stream>>>(ta, tb, td, g.row_scale, g.col_scale, g.bias, g.M, g.N, g.K,
                                                 reinterpret_cast<const uint8_t*>(g.sfa), reinterpret_cast<const uint8_t*>(g.sfb));
  return cudaGetLastError();
}

}  // namespace lowp

cudaError_t gemm_lowp_wgmma(const LowpGemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return cudaSuccess;
  if (g.kind == 3) return g.out_fp16 ? cudaErrorInvalidValue : lowp::launch<3, true>(g, stream);
  if (g.kind == 1) return g.out_fp16 ? lowp::launch<1, false>(g, stream) : lowp::launch<1, true>(g, stream);
  if (g.kind == 2) return g.out_fp16 ? lowp::launch<2, false>(g, stream) : lowp::launch<2, true>(g, stream);
  return cudaErrorInvalidValue;
}

}  // namespace pfx
