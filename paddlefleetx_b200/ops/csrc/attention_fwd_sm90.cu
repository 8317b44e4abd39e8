// Flash-style attention forward on wgmma / TMA (sm_90a), bf16 or fp16 (a template parameter), head_dim 64 or 128, causal or full, optional dropout.
//
//   O[b, s, h, :] = softmax(scale * Q[b, s, h, :] . K[b, :, h, :]^T (+ causal mask)) (dropout) @ V[b, :, h, :]
//
// Inputs / output are [B, S, H, D] VIEWS (3-D tensor maps over {columns, S, B}): contiguous tensors, the q / k / v slices of a packed
// projection output and sequence-major storage are all read in place.
//
// One CTA owns a 64-query tile of one (batch, head) at a time (persistent over the work items, longest causal tiles first):
//   warp 4    TMA producer: the Q tile once per work item, then K / V tiles of 128 keys through a 2-stage mbarrier ring
//   warps 0-3 one consumer warpgroup: S = Q K^T (wgmma m64n128k16, both operands from shared memory) into registers; online softmax on
//             the accumulator fragment (a query row lives in the four lanes of a quad: two shuffles per row statistic), exp2 with the
//             scale folded into one FFMA, dropout (counter hash, pfx_attn.cuh); P V with P fed to wgmma straight from REGISTERS (the
//             accumulator fragment of S is the A fragment of the next product, so probabilities never touch shared memory) and V read
//             as the MN-major B operand; O accumulates in registers.
// Shared memory per CTA is 72 KB (D = 64) or 144 KB (D = 128); registers allow two CTAs per SM at D = 64 and one at D = 128 (the launcher
// asks the occupancy calculator and sizes the persistent grid to what is resident).
// Causal tiles above the diagonal are never loaded; masks are applied only on diagonal / ragged tiles.  Output O (the inputs' type) and the row-wise
// log-sum-exp (fp32, [B, H, S]) are written from registers.  Reference call site: flash_attention in hybrid_model.py:284-301
// (FlashAttention-2 library on Ampere mma.sync).
#include <climits>
#include <cstdio>

#include "pfx_ptx.cuh"
#include "pfx_gemm.h"
#include "pfx_kernels.h"
#include "pfx_attn.h"
#include "pfx_attn.cuh"
#include <cudaTypedefs.h>

namespace pfx {

namespace {

constexpr int kFaThreads = 160;       // warps 0-3 consumer warpgroup, warp 4 TMA producer
constexpr int kFaQ = 64;              // queries per tile (one wgmma M)
constexpr int kFaKv = 128;            // keys per KV tile

template <int kD>
struct FaSmem {
  static constexpr int kQBytes = kFaQ * kD * 2;
  static constexpr int kKBytes = kFaKv * kD * 2;
  static constexpr int kVBytes = kFaKv * kD * 2;
  static constexpr int kStageBytes = kKBytes + kVBytes;
  static constexpr int kStages = 2;
  static constexpr int kBarBytes = 128;
  static constexpr int kAlignSlack = 1024;
  static constexpr int kUsed = kQBytes + kStages * kStageBytes + kBarBytes;
  static constexpr int kTotal = kAlignSlack + kUsed;
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

__device__ __forceinline__ void tma3(const CUtensorMap* m, bool swapped, uint32_t bar, uint32_t dst, int col, int s, int b) {
  if (swapped) tma_load_3d(m, bar, dst, col, b, s); else tma_load_3d(m, bar, dst, col, s, b);
}

// kBf16: bf16 operands and output, otherwise fp16.  kGqa: G = H / Hkv > 1 query heads share one K/V head (a separate instantiation, so
// the multi-head kernels are compiled exactly as without it); query head h loads Q at column (h / G) * gs_q + (h % G) * hs_q and K / V
// of head h / G.  The work order keeps the heads of one batch adjacent, so the G query heads of a group stream the same K / V tiles
// at about the same time and share them through L2.
// kDoc (with kCausal, Sq == Sk): query i attends keys [doc.key_start[b, i], i] (AttnDocMask).  A 64-query tile starts at key tile
// tile_min / 128 in the producer and the consumers alike, and only tiles with key0 < tile_max (plus the diagonal / ragged ones) pay
// per-element compares.
template <int kD, bool kCausal, bool kBf16, bool kGqa, bool kDoc = false>
__global__ void __launch_bounds__(kFaThreads, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                     uint16_t* __restrict__ out, int64_t o_sb, int64_t o_ss, int64_t o_sh, float* __restrict__ lse, int B, int Sq, int Sk, int H,
                     float scale_log2, int hs_q, int hs_k, int hs_v, uint32_t swapped, uint32_t drop_thresh16, float inv_keep, uint64_t seed,
                     int G, int gs_q, AttnDocMask doc) {
  static_assert(!kDoc || kCausal, "the document mask is a causal mask with a per-row lower key bound");
  using S = FaSmem<kD>;
  constexpr int kPanels = kD / 64;                 // 64-element (128-byte) column panels of a D-wide tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_q = smem_base;
  const uint32_t smem_kv = smem_q + S::kQBytes;
  const uint32_t smem_bar = smem_kv + S::kStages * S::kStageBytes;
  const uint32_t q_full = smem_bar, q_empty = smem_bar + 8;
  auto kv_full = [&](int s) { return smem_bar + 8u * (2 + s); };
  auto kv_empty = [&](int s) { return smem_bar + 8u * (4 + s); };

  const uint32_t warp = warp_id(), lane = lane_id();
  const int n_q_tiles = (Sq + kFaQ - 1) / kFaQ;
  const int n_kv_all = (Sk + kFaKv - 1) / kFaKv;
  const int hb_count = H * B;
  const int n_items = n_q_tiles * hb_count;
  // item w -> (query tile, h, b): all (h, b) of the longest tile first, then the next shorter one, ...
  auto item_tile = [&](int w) { return n_q_tiles - 1 - w / hb_count; };
  auto tile_n_kv = [&](int q_tile) {                 // key tiles a query tile attends to
    return kCausal ? min(n_kv_all, (q_tile * kFaQ + kFaQ - 1 + (Sk - Sq)) / kFaKv + 1) : n_kv_all;
  };
  auto tile_j0 = [&](int q_tile, int b) {            // first key tile a query tile attends to
    return kDoc ? __ldg(doc.tile_min + (size_t)b * n_q_tiles + q_tile) / kFaKv : 0;
  };

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1); mbar_init(q_empty, 4);
    for (int s2 = 0; s2 < S::kStages; ++s2) { mbar_init(kv_full(s2), 1); mbar_init(kv_empty(s2), 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ==== TMA producer
    if (elect_one()) {
      uint32_t t = 0;                                   // KV tiles issued so far (all items): ring stage / phase
      int it = 0;
      for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
        const int q_tile = item_tile(w), hb = w % hb_count, h = hb % H, b = hb / H;
        const int n_kv = tile_n_kv(q_tile);
        const int q_col = kGqa ? (h / G) * gs_q + (h % G) * hs_q : h * hs_q;
        const int hk = kGqa ? h / G : h;
        mbar_wait(q_empty, ((uint32_t)it & 1u) ^ 1u);
        mbar_arrive_expect_tx(q_full, S::kQBytes);
        for (int p = 0; p < kPanels; ++p) tma3(&tmap_q, swapped & 1u, q_full, smem_q + p * (kFaQ * 128), q_col + p * 64, q_tile * kFaQ, b);
        for (int j = tile_j0(q_tile, b); j < n_kv; ++j, ++t) {
          const int stage = t & 1;
          mbar_wait(kv_empty(stage), ((t >> 1) & 1u) ^ 1u);
          const uint32_t sk = smem_kv + stage * S::kStageBytes, sv = sk + S::kKBytes;
          mbar_arrive_expect_tx(kv_full(stage), S::kStageBytes);
          const int key0 = j * kFaKv;
          for (int p = 0; p < kPanels; ++p) tma3(&tmap_k, swapped & 2u, kv_full(stage), sk + p * (kFaKv * 128), hk * hs_k + p * 64, key0, b);
          for (int kb = 0; kb < 2; ++kb)            // V as the MN-major B operand: [64 keys x 64 channels] boxes, channel chunks 8 KB apart
            for (int nc = 0; nc < kPanels; ++nc)
              tma3(&tmap_v, swapped & 4u, kv_full(stage), sv + (kb * kPanels + nc) * 8192, hk * hs_v + nc * 64, key0 + kb * 64, b);
        }
      }
    }
  } else {
    // ==== consumer warpgroup: products, softmax, epilogue
    constexpr uint64_t kDescK = wgmma_desc_hi_lo(16, 1024);        // K-major, 128-byte swizzle
    constexpr uint64_t kDescMN = wgmma_desc_hi_lo(8192, 1024);     // MN-major: 64-channel chunks 8 KB apart
    const int row_lo = (int)(warp * 16u + (lane >> 2));            // this thread's query rows inside the tile: row_lo and row_lo + 8
    const int col_in8 = (int)(lane & 3u) * 2;                      // ... and its column pair inside every 8-column group
    uint32_t t = 0;
    int it = 0;
    for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
      const int q_tile = item_tile(w), hb = w % hb_count, h = hb % H, b = hb / H;
      const int n_kv = tile_n_kv(q_tile);
      const int q0 = q_tile * kFaQ;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // per row (row_lo, row_lo + 8): running maximum (log2 units), this thread's part of the row sum
      float o[kD / 2];
#pragma unroll
      for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
      const uint32_t rng_key = attn_rng_key(seed, (uint32_t)(b * H + h));
      const uint32_t rng_pairs = ((uint32_t)Sk + 1u) >> 1;
      int doc_max = 0, doc_ks[2] = {0, 0};            // kDoc: the tile's largest key_start, and that of this thread's two rows
      if constexpr (kDoc) {
        doc_max = __ldg(doc.tile_max + (size_t)b * n_q_tiles + q_tile);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row_g = q0 + row_lo + 8 * hh;
          doc_ks[hh] = row_g < Sq ? __ldg(doc.key_start + (size_t)b * Sq + row_g) : 0;
        }
      }
      mbar_wait(q_full, (uint32_t)it & 1u);
      for (int j = tile_j0(q_tile, b); j < n_kv; ++j, ++t) {
        const int stage = t & 1;
        const uint32_t sk = smem_kv + stage * S::kStageBytes, sv = sk + S::kKBytes;
        mbar_wait(kv_full(stage), (t >> 1) & 1u);
        float s[kFaKv / 2];                        // s[4 g + e]: row row_lo + 8 (e / 2), key 8 g + col_in8 + (e % 2)
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kD / 16; ++k) {
          const uint32_t offq = (k / 4) * (kFaQ * 128) + (k % 4) * 32, offk = (k / 4) * (kFaKv * 128) + (k % 4) * 32;
          WgmmaSS<kFaKv, kBf16, 0, 0>::mma(s, wgmma_desc(smem_q + offq, kDescK), wgmma_desc(sk + offk, kDescK), k != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        const int key0 = j * kFaKv;
        const bool need_mask = (kCausal && key0 + kFaKv - 1 > q0 + (Sk - Sq)) || (key0 + kFaKv > Sk) || (kDoc && key0 < doc_max);
        if (need_mask) {
#pragma unroll
          for (int i = 0; i < kFaKv / 2; ++i) {
            const int cg = key0 + 8 * (i >> 2) + col_in8 + (i & 1);
            const int row_g = q0 + row_lo + 8 * ((i >> 1) & 1);
            if (cg >= Sk || (kCausal && cg > row_g + (Sk - Sq)) || (kDoc && cg < doc_ks[(i >> 1) & 1])) s[i] = -INFINITY;
          }
        }
        float f[2], m_use[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float mx = -INFINITY;
#pragma unroll
          for (int g = 0; g < kFaKv / 8; ++g) mx = fmaxf(mx, fmaxf(s[4 * g + 2 * hh], s[4 * g + 2 * hh + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m_run[hh], mx * scale_log2);       // log2 units from here on
          f[hh] = (m_run[hh] == -INFINITY) ? 0.f : exp2f(m_run[hh] - m_new);
          m_run[hh] = m_new;
          m_use[hh] = (m_new == -INFINITY) ? 0.f : m_new;
          l_run[hh] *= f[hh];
        }
#pragma unroll
        for (int i = 0; i < kD / 2; ++i) o[i] *= f[(i >> 1) & 1];
        uint32_t pw[kFaKv / 4];                    // the probabilities as packed 16-bit pairs, in wgmma A-fragment order
#pragma unroll
        for (int g = 0; g < kFaKv / 8; ++g) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float p0 = exp2f(fmaf(s[4 * g + 2 * hh], scale_log2, -m_use[hh]));
            float p1 = exp2f(fmaf(s[4 * g + 2 * hh + 1], scale_log2, -m_use[hh]));
            l_run[hh] += p0 + p1;
            if (drop_thresh16 != 0u) {               // the row sum keeps every probability; only the P V product sees the mask
              const uint32_t kg = (uint32_t)(key0 + 8 * g + col_in8);
              const uint32_t bits = attn_rng_pair(rng_key, (uint32_t)(q0 + row_lo + 8 * hh), kg >> 1, rng_pairs);
              if ((bits & 0xFFFFu) < drop_thresh16) p0 = 0.f;
              if ((bits >> 16) < drop_thresh16) p1 = 0.f;
            }
            pw[2 * g + hh] = pack_16x2<kBf16>(p0, p1);
          }
        }
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kFaKv / 16; ++k) {
          const uint32_t b_off = (k / 4) * (kPanels * 8192) + (k % 4) * 2048;              // V: 64-key blocks, 16 keys = 2 KB
          const uint32_t a[4] = {pw[4 * k], pw[4 * k + 1], pw[4 * k + 2], pw[4 * k + 3]};
          WgmmaRS<kD, 1, kBf16>::mma(o, a, wgmma_desc(sv + b_off, kDescMN), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(kv_empty(stage));
      }
      if (lane == 0) mbar_arrive(q_empty);          // every product that reads the Q tile has retired
      // item epilogue: normalise by the full row sum (the four lanes of a quad hold the parts of a row)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float l_all = l_run[hh];
        l_all += __shfl_xor_sync(0xffffffffu, l_all, 1);
        l_all += __shfl_xor_sync(0xffffffffu, l_all, 2);
        const int row_g = q0 + row_lo + 8 * hh;
        const float inv = l_all > 0.f ? inv_keep / l_all : 0.f;
        if (row_g < Sq) {
          uint16_t* dst = out + (size_t)b * o_sb + (size_t)row_g * o_ss + (size_t)h * o_sh + col_in8;
#pragma unroll
          for (int g = 0; g < kD / 8; ++g)
            *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack_16x2<kBf16>(o[4 * g + 2 * hh] * inv, o[4 * g + 2 * hh + 1] * inv);
          if (lse != nullptr && (lane & 3u) == 0)
            lse[((size_t)b * H + h) * Sq + row_g] = (l_all > 0.f) ? (m_run[hh] + log2f(l_all)) * 0.6931471805599453f : -INFINITY;
        }
      }
    }
  }
}

template <int kD, bool kCausal, bool kBf16, bool kGqa, bool kDoc = false>
cudaError_t launch_fa(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H, int Hkv,
                      float scale, AttnDropout drop, cudaStream_t st, AttnDocMask doc = AttnDocMask{}) {
  using S = FaSmem<kD>;
  CUtensorMap tq, tk, tv;
  bool sq = false, sk = false, sv = false;
  const int G = H / Hkv;
  // the maps' inner extent reaches the furthest column a head reads
  const uint64_t inner_q = kGqa ? (uint64_t)(Hkv - 1) * q.sg + (uint64_t)(G - 1) * q.sh + kD : (uint64_t)(H - 1) * q.sh + kD;
  auto inner = [&](const AttnView& t) { return (uint64_t)(Hkv - 1) * t.sh + kD; };
  constexpr int dt = kBf16 ? 1 : 0;
  bool ok = make_tmap_bshd(&tq, q.ptr, dt, inner_q, Sq, B, (uint64_t)q.ss * 2, (uint64_t)q.sb * 2, 64, kFaQ, &sq);
  ok &= make_tmap_bshd(&tk, k.ptr, dt, inner(k), Sk, B, (uint64_t)k.ss * 2, (uint64_t)k.sb * 2, 64, kFaKv, &sk);
  ok &= make_tmap_bshd(&tv, v.ptr, dt, inner(v), Sk, B, (uint64_t)v.ss * 2, (uint64_t)v.sb * 2, 64, 64, &sv);
  if (!ok) return cudaErrorInvalidValue;
  auto kern = attention_fwd_kernel<kD, kCausal, kBf16, kGqa, kDoc>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int ctas_per_sm = 1;      // resident CTAs per SM (registers and shared memory): the persistent grid must not exceed them
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, kFaThreads, S::kTotal) != cudaSuccess || ctas_per_sm < 1) ctas_per_sm = 1;
  const long items = (long)((Sq + kFaQ - 1) / kFaQ) * H * B;
  const int grid = (int)(items < (long)sms * ctas_per_sm ? items : (long)sms * ctas_per_sm);
  const uint32_t thresh = drop.p > 0.f ? (uint32_t)(drop.p * 65536.f + 0.5f) : 0u;
  const float inv_keep = drop.p > 0.f ? 1.f / (1.f - drop.p) : 1.f;
  const uint32_t swapped = (sq ? 1u : 0u) | (sk ? 2u : 0u) | (sv ? 4u : 0u);
  kern<<<grid, kFaThreads, S::kTotal, st>>>(tq, tk, tv, (uint16_t*)const_cast<void*>(out.ptr), out.sb, out.ss, out.sh, lse, B, Sq, Sk, H,
                                            scale * 1.4426950408889634f, (int)q.sh, (int)k.sh, (int)v.sh, swapped, thresh, inv_keep, drop.seed, G, (int)q.sg, doc);
  return cudaGetLastError();
}

template <bool kBf16, bool kGqa>
cudaError_t launch_fa_dt(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                         int Hkv, int D, float scale, bool causal, AttnDropout drop, cudaStream_t st) {
  if (D == 128) return causal ? launch_fa<128, true, kBf16, kGqa>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, scale, drop, st)
                              : launch_fa<128, false, kBf16, kGqa>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, scale, drop, st);
  return causal ? launch_fa<64, true, kBf16, kGqa>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, scale, drop, st)
                : launch_fa<64, false, kBf16, kGqa>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, scale, drop, st);
}

template <bool kBf16, bool kGqa>
cudaError_t launch_fa_doc(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int S, int H, int Hkv, int D,
                          float scale, AttnDropout drop, const AttnDocMask& doc, cudaStream_t st) {
  if (D == 128) return launch_fa<128, true, kBf16, kGqa, true>(q, k, v, out, lse, B, S, S, H, Hkv, scale, drop, st, doc);
  return launch_fa<64, true, kBf16, kGqa, true>(q, k, v, out, lse, B, S, S, H, Hkv, scale, drop, st, doc);
}

}  // namespace

cudaError_t attention_fwd_v2(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                             int Hkv, int D, float scale, bool causal, AttnDropout drop, int dtype, cudaStream_t st) {
  if ((D != 64 && D != 128) || (dtype != 0 && dtype != 1) || B < 1 || Sq < 1 || Sk < 1 || (causal && Sk < Sq)) return cudaErrorInvalidValue;
  if (H < 1 || Hkv < 1 || H % Hkv != 0 || (Hkv < H && q.sg % 8)) return cudaErrorInvalidValue;
  for (const AttnView* t : {&q, &k, &v, &out})
    if (t->ptr == nullptr || (reinterpret_cast<uintptr_t>(t->ptr) % 16) || t->sb % 8 || t->ss % 8 || t->sh % 8) return cudaErrorInvalidValue;
  if (Hkv < H)
    return dtype == 1 ? launch_fa_dt<true, true>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, D, scale, causal, drop, st)
                      : launch_fa_dt<false, true>(q, k, v, out, lse, B, Sq, Sk, H, Hkv, D, scale, causal, drop, st);
  return dtype == 1 ? launch_fa_dt<true, false>(q, k, v, out, lse, B, Sq, Sk, H, H, D, scale, causal, drop, st)
                    : launch_fa_dt<false, false>(q, k, v, out, lse, B, Sq, Sk, H, H, D, scale, causal, drop, st);
}

cudaError_t attention_fwd_doc(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int S, int H, int Hkv,
                              int D, float scale, AttnDropout drop, const AttnDocMask& doc, int dtype, cudaStream_t st) {
  if ((D != 64 && D != 128) || (dtype != 0 && dtype != 1) || B < 1 || S < 1) return cudaErrorInvalidValue;
  if (H < 1 || Hkv < 1 || H % Hkv != 0 || (Hkv < H && q.sg % 8)) return cudaErrorInvalidValue;
  if (doc.key_start == nullptr || doc.tile_min == nullptr || doc.tile_max == nullptr) return cudaErrorInvalidValue;
  for (const AttnView* t : {&q, &k, &v, &out})
    if (t->ptr == nullptr || (reinterpret_cast<uintptr_t>(t->ptr) % 16) || t->sb % 8 || t->ss % 8 || t->sh % 8) return cudaErrorInvalidValue;
  if (Hkv < H)
    return dtype == 1 ? launch_fa_doc<true, true>(q, k, v, out, lse, B, S, H, Hkv, D, scale, drop, doc, st)
                      : launch_fa_doc<false, true>(q, k, v, out, lse, B, S, H, Hkv, D, scale, drop, doc, st);
  return dtype == 1 ? launch_fa_doc<true, false>(q, k, v, out, lse, B, S, H, H, D, scale, drop, doc, st)
                    : launch_fa_doc<false, false>(q, k, v, out, lse, B, S, H, H, D, scale, drop, doc, st);
}

// ---- document-mask bounds: key_start[b, i] = clamp(i - pos[b, i], 0, i) (or clamp(src, 0, i) when src already holds key starts), and
// the minimum / maximum of key_start over every 64-query tile.  One 64-thread block per (tile, b).
__global__ void attn_doc_bounds_kernel(const int64_t* __restrict__ src, int from_positions, int S, int n_tiles, int* __restrict__ key_start,
                                       int* __restrict__ tile_min, int* __restrict__ tile_max) {
  __shared__ int red[2][2];
  const int b = blockIdx.y, i = blockIdx.x * 64 + threadIdx.x;
  int lo = INT_MAX, hi = 0;
  if (i < S) {
    const int64_t x = src[(size_t)b * S + i];
    const int64_t ks = from_positions ? (int64_t)i - x : x;
    const int v = (int)(ks < 0 ? 0 : (ks > i ? i : ks));
    key_start[(size_t)b * S + i] = v;
    lo = hi = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = lo; red[1][threadIdx.x >> 5] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    tile_min[(size_t)b * n_tiles + blockIdx.x] = min(red[0][0], red[0][1]);
    tile_max[(size_t)b * n_tiles + blockIdx.x] = max(red[1][0], red[1][1]);
  }
}

cudaError_t attention_doc_bounds(const int64_t* src, bool from_positions, int B, int S, int* key_start, int* tile_min, int* tile_max, cudaStream_t st) {
  if (src == nullptr || B < 1 || S < 1 || B > 65535) return cudaErrorInvalidValue;
  const int n_tiles = (S + 63) / 64;
  attn_doc_bounds_kernel<<<dim3(n_tiles, B), 64, 0, st>>>(src, from_positions ? 1 : 0, S, n_tiles, key_start, tile_min, tile_max);
  return cudaGetLastError();
}

cudaError_t attention_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Sq, int Sk, int H, int D, float scale,
                          bool causal, cudaStream_t st) {
  const int64_t hd = (int64_t)H * D;
  const AttnView vq{q, (int64_t)Sq * hd, hd, D}, vk{k, (int64_t)Sk * hd, hd, D}, vv{v, (int64_t)Sk * hd, hd, D}, vo{out, (int64_t)Sq * hd, hd, D};
  return attention_fwd_v2(vq, vk, vv, vo, lse, B, Sq, Sk, H, H, D, scale, causal, AttnDropout{0.f, 0}, 1, st);
}

}  // namespace pfx
