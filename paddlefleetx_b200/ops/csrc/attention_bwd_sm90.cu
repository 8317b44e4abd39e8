// Flash-attention backward on wgmma / TMA (sm_90a), bf16 or fp16 (a template parameter), head_dim 128 or 64, causal or full, optional dropout.
//
// One CTA owns a tile of 64 keys of one (batch, head) and walks the 64-query tiles that attend to it.  The score tile is computed
// TRANSPOSED (keys on the wgmma M rows, queries on the columns), so that its accumulator fragment is directly the A fragment of the
// two products that accumulate over queries — P^T and dS^T never leave registers for them:
//
//     S^T  = K_j Q_i^T                      [64 k x 64 q]     A = K_j  (K-major),   B = Q_i  (K-major)
//     dP^T = V_j dO_i^T                     [64 k x 64 q]     A = V_j  (K-major),   B = dO_i (K-major)
//     P^T  = exp2(S^T * c - lse_i)   masked, dropout applied
//     dS^T = P^T o (drop(dP^T) - delta_i) * scale
//     dV  += P_drop^T dO_i                  [64 k x D]        A = P^T  (REGISTERS), B = dO_i (MN-major)     persistent accumulator
//     dK  += dS^T Q_i                       [64 k x D]        A = dS^T (REGISTERS), B = Q_i  (MN-major)     persistent accumulator
//     dQ   = dS K_j                         [64 q x D]        A = dS^T in shared memory read MN-major, B = K_j (MN-major)
//
// The same shared-memory tiles serve as K-major and MN-major operands (a 128-byte-swizzled [rows x 64] panel is both), so Q_i,
// dO_i, K_j, V_j are loaded once by TMA straight from the framework layout ([B, S, H, D] views, packed QKV included).  dQ is accumulated
// across key tiles in an fp32 workspace: each dQ tile goes registers -> shared memory and ONE TMA reduce-add (cp.reduce.async.bulk.tensor)
// folds it into global memory; the workspace is converted to the inputs' type afterwards; lse (log2 units) and delta = rowsum(dO o O) come from a small
// preprocessing kernel.
//
// Warp roles (160 threads): warp 4 TMA producer (K/V once, then a 3-stage ring of Q_i / dO_i / lse_i / delta_i), warps 0-3 one consumer
// warpgroup that issues the five products and does the softmax-gradient math on the fragments.
// Reference call site: flash_attention in hybrid_model.py:284-301 (FlashAttention-2 library, mma.sync on Ampere).
#include <cstdio>

#include "pfx_ptx.cuh"
#include "pfx_common.cuh"
#include "pfx_gemm.h"
#include "pfx_attn.h"
#include "pfx_attn.cuh"

namespace pfx {

namespace {

constexpr int kBwThreads = 160;
constexpr int kKv = 64;             // keys per CTA
constexpr int kQt = 64;             // queries per inner iteration

template <int kHd>                  // head dim: 128 (two 64-channel panels per tile) or 64 (one)
struct BwSmem {
  static constexpr int kPanels = kHd / 64;
  static constexpr int kKBytes = kKv * kHd * 2;          // [64 x 64] panels of 8 KB
  static constexpr int kQBytes = kQt * kHd * 2;          // [64 x 64] panels of 8 KB
  static constexpr int kDsBytes = kKv * kQt * 2;         // 8 KB: one [64 x 64] panel
  static constexpr int kStatBytes = 2 * kQt * 4;         // lse2 + delta of one query tile
  static constexpr int kStages = 3;                      // Q_i / dO_i / stats ring
  static constexpr int kDqBytes = kQt * kHd * 4;         // dQ tile [64 q][kHd d] fp32, row-major (TMA reduce source)
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kOffK + kKBytes;
  static constexpr int kOffQ = kOffV + kKBytes;
  static constexpr int kOffDo = kOffQ + kStages * kQBytes;
  static constexpr int kOffDs = kOffDo + kStages * kQBytes;
  static constexpr int kOffDq = kOffDs + kDsBytes;
  static constexpr int kOffStat = kOffDq + kDqBytes;
  static constexpr int kOffBar = kOffStat + kStages * kStatBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kUsed = kOffBar + kBarBytes;
  static constexpr int kTotal = kUsed + 1024;            // alignment slack
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

struct BwOut { void* ptr; int64_t sb, ss, sh; };

struct BwParams {
  const float* lse2;       // [B*H, Sq_pad], log2 units, +inf in the padding
  const float* delta;      // [B*H, Sq_pad]
  float* dq_acc;           // [B, Sq, H, D] fp32
  BwOut dk, dv;
  int B, Sq, Sk, H, Sq_pad;
  int hs_q, hs_k, hs_v, hs_do;        // head strides (elements) of the four TMA views
  uint32_t swapped;                    // bit t: tensor map t (q, k, v, do) has {cols, B, S} coordinate order
  float scale, scale_log2;
  int causal;
  uint32_t drop_thresh16;              // 0 = no dropout
  float inv_keep;
  uint64_t seed;
  int G, gs_q;                         // grouped-query instantiation only: query heads per K/V head, q stride between groups
  AttnDocMask doc;                     // document-mask instantiation only
};

__device__ __forceinline__ void tma_tile(const CUtensorMap* m, bool swapped, uint32_t bar, uint32_t dst, int col, int s, int b) {
  if (swapped) tma_load_3d(m, bar, dst, col, b, s); else tma_load_3d(m, bar, dst, col, s, b);
}

// kBf16: bf16 operands and gradients, otherwise fp16.  kGqa: G = H / Hkv > 1 query heads share one K/V head (a separate instantiation,
// so the multi-head kernels are compiled exactly as without it).  The CTA then owns a key tile of one (batch, K/V head) and walks the
// query tiles of all G heads of the group in turn, with each head's lse / delta, dropout key, Q column and dQ column, while dK / dV
// stay in registers: they are exact sums written once, with no atomics, and deterministic.
// kDoc (causal, Sq == Sk): query i attends keys [doc.key_start[b, i], i].  A query tile whose tile_min lies past the key tile's last key
// holds no pair of it: the producer does not load it and the consumers do not wait for it (both skip by the same rule, for every head of
// a group).  The ring slots count only the tiles that run.  key_start need not be monotone: the rule uses the tile's minimum.
template <int kHd, bool kBf16, bool kGqa, bool kDoc = false>
__global__ void __launch_bounds__(kBwThreads, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                     const __grid_constant__ CUtensorMap tmap_do, const __grid_constant__ CUtensorMap tmap_dq, const __grid_constant__ BwParams prm) {
  using S = BwSmem<kHd>;
  constexpr int kPanels = S::kPanels;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t s_k = smem_base + S::kOffK, s_v = smem_base + S::kOffV, s_q = smem_base + S::kOffQ, s_do = smem_base + S::kOffDo;
  const uint32_t s_ds = smem_base + S::kOffDs, s_dq = smem_base + S::kOffDq, s_stat = smem_base + S::kOffStat;
  const uint32_t s_bar = smem_base + S::kOffBar;
  auto bar = [&](int i) { return s_bar + 8u * i; };
  const uint32_t kv_full = bar(0);
  auto q_full = [&](int s) { return bar(1 + s); };           // 3 stages
  auto q_empty = [&](int s) { return bar(4 + s); };

  const uint32_t warp = warp_id(), lane = lane_id();
  // CTA order: the key tiles of ONE (batch, head) are neighbours in launch order, so the CTAs that stream the same Q / dO tiles and reduce
  // into the same dQ rows run at the same time and meet in L2.  Within a head the tiles ascend: under a causal mask the first ones carry
  // the most work.
  const int n_kv_tiles = (prm.Sk + kKv - 1) / kKv;
  const int bh = blockIdx.x / n_kv_tiles;         // (batch, K/V head)
  const int j = blockIdx.x - bh * n_kv_tiles;
  const int Hkv = kGqa ? prm.H / prm.G : prm.H;
  const int h = bh % Hkv, b = bh / Hkv;           // h: the K/V head (= the query head without grouping)
  const int k0 = j * kKv;
  const int off = prm.Sk - prm.Sq;                // query q attends keys <= q + off
  const int n_q_tiles = (prm.Sq + kQt - 1) / kQt;
  const int i_begin = prm.causal ? max(0, k0 - off) / kQt : 0;
  const int n_head_iter = n_q_tiles - i_begin;    // >= 1 for every key tile that holds a valid key
  const int n_iter = kGqa ? n_head_iter * prm.G : n_head_iter;
  // iteration it -> (query head, first query): the query tiles of the group's first head, then the next head's, ...
  auto iter_head = [&](int it) { return kGqa ? h * prm.G + it / n_head_iter : h; };
  auto iter_q0 = [&](int it) { return (i_begin + (kGqa ? it % n_head_iter : it)) * kQt; };
  // kDoc: the tile bounds of iteration it + 1 are loaded while iteration it runs, which keeps their latency off the loop
  struct DocBounds { int lo, hi; };
  auto doc_bounds = [&](int it) -> DocBounds {
    if (!kDoc || it >= n_iter) return DocBounds{0, 0};
    const size_t o = (size_t)b * n_q_tiles + iter_q0(it) / kQt;
    return DocBounds{__ldg(prm.doc.tile_min + o), __ldg(prm.doc.tile_max + o)};
  };

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v); tma_prefetch_desc(&tmap_do); tma_prefetch_desc(&tmap_dq);
    mbar_init(kv_full, 1);
    for (int s = 0; s < S::kStages; ++s) { mbar_init(q_full(s), 1); mbar_init(q_empty(s), 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ==== TMA producer
    if (elect_one()) {
      mbar_arrive_expect_tx(kv_full, 2 * S::kKBytes);
      for (int p = 0; p < kPanels; ++p) {
        tma_tile(&tmap_k, prm.swapped & 2u, kv_full, s_k + p * 8192, h * prm.hs_k + p * 64, k0, b);
        tma_tile(&tmap_v, prm.swapped & 4u, kv_full, s_v + p * 8192, h * prm.hs_v + p * 64, k0, b);
      }
      int n_run = 0;                                  // kDoc: query tiles loaded so far (the ring slot)
      DocBounds nxt = doc_bounds(0);
      for (int it = 0; it < n_iter; ++it) {
        const int q0 = iter_q0(it);
        const DocBounds cur = nxt;
        if constexpr (kDoc) nxt = doc_bounds(it + 1);
        if (kDoc && cur.lo > k0 + kKv - 1) continue;
        const int slot = kDoc ? n_run++ : it;
        const int st = slot % S::kStages;
        const int hq = iter_head(it);
        const int q_col = kGqa ? h * prm.gs_q + (hq - h * prm.G) * prm.hs_q : h * prm.hs_q;
        mbar_wait(q_empty(st), (((uint32_t)(slot / S::kStages)) & 1u) ^ 1u);
        mbar_arrive_expect_tx(q_full(st), 2 * S::kQBytes + S::kStatBytes);
        for (int p = 0; p < kPanels; ++p) {
          tma_tile(&tmap_q, prm.swapped & 1u, q_full(st), s_q + st * S::kQBytes + p * 8192, q_col + p * 64, q0, b);
          tma_tile(&tmap_do, prm.swapped & 8u, q_full(st), s_do + st * S::kQBytes + p * 8192, hq * prm.hs_do + p * 64, q0, b);
        }
        const size_t so = (kGqa ? (size_t)b * prm.H + hq : (size_t)bh) * prm.Sq_pad + q0;
        bulk_load_1d(s_stat + st * S::kStatBytes, prm.lse2 + so, kQt * 4, q_full(st));
        bulk_load_1d(s_stat + st * S::kStatBytes + kQt * 4, prm.delta + so, kQt * 4, q_full(st));
      }
    }
  } else {
    // ==== consumer warpgroup
    constexpr uint64_t kDescK = wgmma_desc_hi_lo(16, 1024);
    constexpr uint64_t kDescMN = wgmma_desc_hi_lo(8192, 1024);        // 64-wide MN chunks 8 KB apart (all panels here are [64 x 64])
    const int k_row = (int)(warp * 16u + (lane >> 2));                // this thread's key rows inside the tile: k_row and k_row + 8
    const int col_in8 = (int)(lane & 3u) * 2;                         // ... and its query / channel pair inside every 8-column group
    const uint32_t pairs = ((uint32_t)prm.Sk + 1u) >> 1;
    uint32_t key = attn_rng_key(prm.seed, (uint32_t)(kGqa ? b * prm.H + h * prm.G : bh));
    const bool drop = prm.drop_thresh16 != 0;
    const float p_to_pdrop = prm.inv_keep / prm.scale;
    const bool leader = threadIdx.x == 0;
    float dv[kHd / 2], dk[kHd / 2];
#pragma unroll
    for (int i = 0; i < kHd / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    mbar_wait(kv_full, 0);
    int n_run = 0;
    DocBounds nxt = doc_bounds(0);
    for (int it = 0; it < n_iter; ++it) {
      const int q0 = iter_q0(it);
      const DocBounds cur = nxt;
      if constexpr (kDoc) nxt = doc_bounds(it + 1);
      if (kDoc && cur.lo > k0 + kKv - 1) continue;   // never the diagonal tile i_begin (its tile_min <= its first query = k0)
      const int slot = kDoc ? n_run++ : it;
      const int st = slot % S::kStages;
      const int hq = iter_head(it);
      if (kGqa && it != 0 && q0 == i_begin * kQt) key = attn_rng_key(prm.seed, (uint32_t)(b * prm.H + hq));   // next head of the group
      const uint32_t sq = s_q + st * S::kQBytes, sdo = s_do + st * S::kQBytes;
      mbar_wait(q_full(st), ((uint32_t)(slot / S::kStages)) & 1u);
      float s[kQt / 2], dp[kQt / 2];                                  // [4 g + e]: key k_row + 8 (e / 2), query 8 g + col_in8 + (e % 2)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kHd / 16; ++kk) {
        const uint32_t o = (kk / 4) * 8192 + (kk % 4) * 32;
        WgmmaSS<kQt, kBf16, 0, 0>::mma(s, wgmma_desc(s_k + o, kDescK), wgmma_desc(sq + o, kDescK), kk != 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < kHd / 16; ++kk) {
        const uint32_t o = (kk / 4) * 8192 + (kk % 4) * 32;
        WgmmaSS<kQt, kBf16, 0, 0>::mma(dp, wgmma_desc(s_v + o, kDescK), wgmma_desc(sdo + o, kDescK), kk != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      const float* lse_s = reinterpret_cast<const float*>(smem_gen + (s_stat - smem_base) + st * S::kStatBytes);
      const float* dl_s = lse_s + kQt;
      // masks are decided per tile (warp-uniform branches): only diagonal / ragged tiles pay per-element compares
      const bool tile_mask = (prm.causal && (k0 + kKv - 1 > q0 + off)) || (k0 + kKv > prm.Sk) ||
                             (kDoc && k0 < cur.hi);
      uint32_t pw[kQt / 4], dsw[kQt / 4];                             // P_drop^T and dS^T as packed 16-bit pairs, in wgmma A-fragment order
#pragma unroll
      for (int g = 0; g < kQt / 8; ++g) {
        const int qc = 8 * g + col_in8;
        const float2 ls = *reinterpret_cast<const float2*>(lse_s + qc), dl = *reinterpret_cast<const float2*>(dl_s + qc);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kg = k0 + k_row + 8 * hh;
          float p0 = exp2f(fmaf(s[4 * g + 2 * hh], prm.scale_log2, -ls.x)) * prm.scale;      // P * scale (the softmax scale is folded in here once)
          float p1 = exp2f(fmaf(s[4 * g + 2 * hh + 1], prm.scale_log2, -ls.y)) * prm.scale;
          if (tile_mask) {
            if (kg >= prm.Sk || (prm.causal && kg > q0 + qc + off)) p0 = 0.f;
            if (kg >= prm.Sk || (prm.causal && kg > q0 + qc + 1 + off)) p1 = 0.f;
            if constexpr (kDoc) {                  // rows past Sq have P = 0 already (lse2 = +inf)
              const int* ks = prm.doc.key_start + (size_t)b * prm.Sq;
              if (q0 + qc < prm.Sq && kg < __ldg(ks + q0 + qc)) p0 = 0.f;
              if (q0 + qc + 1 < prm.Sq && kg < __ldg(ks + q0 + qc + 1)) p1 = 0.f;
            }
          }
          float d0 = dp[4 * g + 2 * hh], d1 = dp[4 * g + 2 * hh + 1];
          float pd0 = p0 * p_to_pdrop, pd1 = p1 * p_to_pdrop;
          if (drop) {
            const bool keep0 = attn_keep(attn_rng_pair(key, (uint32_t)(q0 + qc), (uint32_t)kg >> 1, pairs), (uint32_t)kg, prm.drop_thresh16);
            const bool keep1 = attn_keep(attn_rng_pair(key, (uint32_t)(q0 + qc + 1), (uint32_t)kg >> 1, pairs), (uint32_t)kg, prm.drop_thresh16);
            d0 = keep0 ? d0 * prm.inv_keep : 0.f; d1 = keep1 ? d1 * prm.inv_keep : 0.f;
            if (!keep0) pd0 = 0.f;
            if (!keep1) pd1 = 0.f;
          }
          pw[2 * g + hh] = pack_16x2<kBf16>(pd0, pd1);
          dsw[2 * g + hh] = pack_16x2<kBf16>(p0 * (d0 - dl.x), p1 * (d1 - dl.y));                 // dS^T * scale = (P scale) o (drop(dP) - delta)
        }
      }
      // dS^T -> shared memory ([64 k x 64 q] 16-bit panel, 128-byte swizzle) for the dQ product; the previous tile's dQ product has retired
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t r = (uint32_t)(k_row + 8 * hh);
        const uint32_t dst_row = s_ds + (r / 8u) * 1024u + (r % 8u) * 128u + (uint32_t)col_in8 * 2u;
#pragma unroll
        for (int g = 0; g < kQt / 8; ++g)
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst_row + (((uint32_t)g ^ (r % 8u)) << 4)), "r"(dsw[2 * g + hh]) : "memory");
      }
      fence_proxy_async_smem();
      if (leader) tma_store_wait_read<0>();                     // the previous tile's reduce has finished reading the dQ staging buffer
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float dq[kHd / 2];                                          // [4 g + e]: query k_row + 8 (e / 2) (same lane mapping, rows are queries here), channel 8 g + col_in8 + (e % 2)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kQt / 16; ++kk) {
        const uint32_t a[4] = {pw[4 * kk], pw[4 * kk + 1], pw[4 * kk + 2], pw[4 * kk + 3]};
        WgmmaRS<kHd, 1, kBf16>::mma(dv, a, wgmma_desc(sdo + kk * 2048, kDescMN), 1u);
      }
#pragma unroll
      for (int kk = 0; kk < kQt / 16; ++kk) {
        const uint32_t a[4] = {dsw[4 * kk], dsw[4 * kk + 1], dsw[4 * kk + 2], dsw[4 * kk + 3]};
        WgmmaRS<kHd, 1, kBf16>::mma(dk, a, wgmma_desc(sq + kk * 2048, kDescMN), 1u);
      }
#pragma unroll
      for (int kk = 0; kk < kKv / 16; ++kk)
        WgmmaSS<kHd, kBf16, 1, 1>::mma(dq, wgmma_desc(s_ds + kk * 2048, kDescMN), wgmma_desc(s_k + kk * 2048, kDescMN), kk != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(q_empty(st));
      // dQ tile: registers -> staging [64 q][kHd d] fp32 -> one TMA reduce-add
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t row = s_dq + (uint32_t)(k_row + 8 * hh) * (kHd * 4u) + (uint32_t)col_in8 * 4u;
#pragma unroll
        for (int g = 0; g < kHd / 8; ++g)
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(row + g * 32u), "f"(dq[4 * g + 2 * hh]), "f"(dq[4 * g + 2 * hh + 1]) : "memory");
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (leader) {
        // rows of the 2-D [B*Sq, H*D] view; query rows past Sq of a ragged tile carry exact zeros (P = 0 there), rows past the tensor are dropped
        tma_reduce_add_2d(&tmap_dq, s_dq, hq * kHd, b * prm.Sq + q0);
        tma_store_commit();
      }
    }
    if (leader) tma_store_wait<0>();
    // ---- epilogue: dV and dK of this key tile
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int kg = k0 + k_row + 8 * hh;
      if (kg < prm.Sk) {
        uint16_t* pv = reinterpret_cast<uint16_t*>(prm.dv.ptr) + (size_t)b * prm.dv.sb + (size_t)kg * prm.dv.ss + (size_t)h * prm.dv.sh + col_in8;
        uint16_t* pk = reinterpret_cast<uint16_t*>(prm.dk.ptr) + (size_t)b * prm.dk.sb + (size_t)kg * prm.dk.ss + (size_t)h * prm.dk.sh + col_in8;
#pragma unroll
        for (int g = 0; g < kHd / 8; ++g) {
          *reinterpret_cast<uint32_t*>(pv + 8 * g) = pack_16x2<kBf16>(dv[4 * g + 2 * hh], dv[4 * g + 2 * hh + 1]);
          *reinterpret_cast<uint32_t*>(pk + 8 * g) = pack_16x2<kBf16>(dk[4 * g + 2 * hh], dk[4 * g + 2 * hh + 1]);
        }
      }
    }
  }
}

// ---- preprocessing: delta = rowsum(dO o O), lse in log2 units; both padded to a multiple of 64 queries per (b, h)
template <int kHd, bool kBf16>
__global__ void attn_bwd_prep_kernel(const uint16_t* __restrict__ o, int64_t o_sb, int64_t o_ss, int64_t o_sh, const uint16_t* __restrict__ dout,
                                     int64_t d_sb, int64_t d_ss, int64_t d_sh, const float* __restrict__ lse, float* __restrict__ lse2,
                                     float* __restrict__ delta, int B, int Sq, int H, int Sq_pad) {
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // (b, s_pad, h)
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)B * Sq_pad * H) return;
  const int h = (int)(w % H);
  const int s = (int)((w / H) % Sq_pad);
  const int b = (int)(w / ((int64_t)H * Sq_pad));
  const size_t oi = ((size_t)b * H + h) * Sq_pad + s;
  if (s >= Sq) {
    if (lane == 0) { lse2[oi] = INFINITY; delta[oi] = 0.f; }
    return;
  }
  constexpr int kPer = kHd / 32;                         // channels per lane (4 or 2)
  const uint16_t* a2 = o + b * o_sb + s * o_ss + h * o_sh + lane * kPer;
  const uint16_t* g2 = dout + b * d_sb + s * d_ss + h * d_sh + lane * kPer;
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < kPer / 2; ++i) {
    const float2 x = load_16x2<kBf16>(a2 + 2 * i), y = load_16x2<kBf16>(g2 + 2 * i);
    acc += x.x * y.x + x.y * y.y;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    delta[oi] = acc;
    lse2[oi] = lse[((size_t)b * H + h) * Sq + s] * 1.4426950408889634f;
  }
}

// ---- dq: fp32 accumulator -> 16-bit view
template <bool kBf16, bool kGqa>    // kGqa: dq is a grouped view, head h at (h / G) * sg + (h % G) * sh
__global__ void attn_bwd_dq_convert_kernel(const float* __restrict__ acc, uint16_t* __restrict__ dq, int64_t sb, int64_t ss, int64_t sh, int B, int Sq, int H, int kHd,
                                           int G, int64_t sg) {
  const int64_t n8 = (int64_t)B * Sq * H * (kHd / 8);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % (kHd / 8));
    const int64_t row = i / (kHd / 8);                 // (b, s, h)
    const int h = (int)(row % H);
    const int s = (int)((row / H) % Sq);
    const int b = (int)(row / ((int64_t)H * Sq));
    const float4 x = *reinterpret_cast<const float4*>(acc + i * 8), y = *reinterpret_cast<const float4*>(acc + i * 8 + 4);
    uint4 v;
    v.x = pack_16x2<kBf16>(x.x, x.y); v.y = pack_16x2<kBf16>(x.z, x.w); v.z = pack_16x2<kBf16>(y.x, y.y); v.w = pack_16x2<kBf16>(y.z, y.w);
    const int64_t ho = kGqa ? (h / G) * sg + (h % G) * sh : h * sh;
    *reinterpret_cast<uint4*>(dq + b * sb + s * ss + ho + c * 8) = v;
  }
}

bool view_ok(const AttnView& t) {
  return t.ptr != nullptr && (reinterpret_cast<uintptr_t>(t.ptr) % 16) == 0 && t.sb % 8 == 0 && t.ss % 8 == 0 && t.sh % 8 == 0;
}

// H: the view's heads.  G > 1: a grouped query view of H = Hkv * G heads (see AttnView)
bool make_map(CUtensorMap* m, const AttnView& t, int dtype, int B, int S, int H, int D, uint32_t box_rows, bool* swapped, int G = 1) {
  const uint64_t inner = G > 1 ? (uint64_t)(H / G - 1) * t.sg + (uint64_t)(G - 1) * t.sh + D : (uint64_t)(H - 1) * t.sh + D;
  return make_tmap_bshd(m, t.ptr, dtype, inner, (uint64_t)S, (uint64_t)B, (uint64_t)t.ss * 2, (uint64_t)t.sb * 2, 64, box_rows, swapped);
}

}  // namespace

template <int kHd, bool kBf16, bool kGqa, bool kDoc = false>
static cudaError_t attention_bwd_impl(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                                      const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                                      int Sk, int H, int Hkv, float scale, bool causal, AttnDropout drop, cudaStream_t st,
                                      const AttnDocMask& doc = AttnDocMask{}) {
  const int G = H / Hkv;
  constexpr int D = kHd;
  constexpr int dt = kBf16 ? 1 : 0;
  using S = BwSmem<kHd>;
  const int Sq_pad = (Sq + kQt - 1) / kQt * kQt;
  cudaError_t e = cudaMemsetAsync(dq_acc, 0, (size_t)B * Sq * H * kHd * sizeof(float), st);
  if (e != cudaSuccess) return e;
  {
    const int64_t warps = (int64_t)B * Sq_pad * H;
    const int wpb = 8;
    attn_bwd_prep_kernel<kHd, kBf16><<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, st>>>(
        (const uint16_t*)out.ptr, out.sb, out.ss, out.sh, (const uint16_t*)dout.ptr, dout.sb, dout.ss, dout.sh, lse, lse2, delta, B, Sq, H, Sq_pad);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  CUtensorMap tq, tk, tv, tdo, tdq;
  bool sq = false, sk = false, sv = false, sdo = false;
  bool ok = make_map(&tq, q, dt, B, Sq, H, D, kQt, &sq, G) && make_map(&tk, k, dt, B, Sk, Hkv, D, kKv, &sk) && make_map(&tv, v, dt, B, Sk, Hkv, D, kKv, &sv) &&
            make_map(&tdo, dout, dt, B, Sq, H, D, kQt, &sdo) &&
            make_tmap_2d_plain(&tdq, dq_acc, 3, (uint64_t)H * kHd, (uint64_t)B * Sq, (uint64_t)H * kHd * 4, kHd, kQt);
  if (!ok) return cudaErrorInvalidValue;
  BwParams prm{};
  prm.lse2 = lse2; prm.delta = delta; prm.dq_acc = dq_acc;
  prm.dk = BwOut{const_cast<void*>(dk.ptr), dk.sb, dk.ss, dk.sh};
  prm.dv = BwOut{const_cast<void*>(dv.ptr), dv.sb, dv.ss, dv.sh};
  prm.B = B; prm.Sq = Sq; prm.Sk = Sk; prm.H = H; prm.Sq_pad = Sq_pad;
  prm.hs_q = (int)q.sh; prm.hs_k = (int)k.sh; prm.hs_v = (int)v.sh; prm.hs_do = (int)dout.sh;
  prm.G = G; prm.gs_q = (int)q.sg;
  prm.swapped = (sq ? 1u : 0u) | (sk ? 2u : 0u) | (sv ? 4u : 0u) | (sdo ? 8u : 0u);
  prm.scale = scale; prm.scale_log2 = scale * 1.4426950408889634f;
  prm.causal = causal ? 1 : 0;
  prm.drop_thresh16 = drop.p > 0.f ? (uint32_t)(drop.p * 65536.f + 0.5f) : 0u;
  prm.inv_keep = drop.p > 0.f ? 1.f / (1.f - drop.p) : 1.f;
  prm.seed = drop.seed;
  prm.doc = doc;
  static bool attr_set = false;
  if (!attr_set) {
    if ((e = cudaFuncSetAttribute(attention_bwd_kernel<kHd, kBf16, kGqa, kDoc>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal)) != cudaSuccess) return e;
    attr_set = true;
  }
  const int n_kv = (Sk + kKv - 1) / kKv;
  attention_bwd_kernel<kHd, kBf16, kGqa, kDoc><<<(unsigned)(n_kv * B * Hkv), kBwThreads, S::kTotal, st>>>(tq, tk, tv, tdo, tdq, prm);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  attn_bwd_dq_convert_kernel<kBf16, kGqa><<<1184, 256, 0, st>>>(dq_acc, (uint16_t*)const_cast<void*>(dq.ptr), dq.sb, dq.ss, dq.sh, B, Sq, H, kHd, G, dq.sg);
  return cudaGetLastError();
}

cudaError_t attention_bwd(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                          const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                          int Sk, int H, int Hkv, int D, float scale, bool causal, AttnDropout drop, int dtype, cudaStream_t st) {
  if ((D != 64 && D != 128) || (dtype != 0 && dtype != 1) || B < 1 || Sq < 1 || Sk < 1 || (causal && Sk < Sq)) return cudaErrorInvalidValue;
  if (H < 1 || Hkv < 1 || H % Hkv != 0 || (Hkv < H && (q.sg % 8 || dq.sg % 8))) return cudaErrorInvalidValue;
  for (const AttnView* t : {&q, &k, &v, &out, &dout, &dq, &dk, &dv}) if (!view_ok(*t)) return cudaErrorInvalidValue;
#define PFX_BWD(HD, BF, GQA) attention_bwd_impl<HD, BF, GQA>(q, k, v, out, dout, lse, dq, dk, dv, dq_acc, lse2, delta, B, Sq, Sk, H, Hkv, scale, causal, drop, st)
  if (Hkv < H) {
    if (dtype == 1) return D == 128 ? PFX_BWD(128, true, true) : PFX_BWD(64, true, true);
    return D == 128 ? PFX_BWD(128, false, true) : PFX_BWD(64, false, true);
  }
  if (dtype == 1) return D == 128 ? PFX_BWD(128, true, false) : PFX_BWD(64, true, false);
  return D == 128 ? PFX_BWD(128, false, false) : PFX_BWD(64, false, false);
#undef PFX_BWD
}

cudaError_t attention_bwd_doc(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                              const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int S,
                              int H, int Hkv, int D, float scale, AttnDropout drop, const AttnDocMask& doc, int dtype, cudaStream_t st) {
  if ((D != 64 && D != 128) || (dtype != 0 && dtype != 1) || B < 1 || S < 1) return cudaErrorInvalidValue;
  if (H < 1 || Hkv < 1 || H % Hkv != 0 || (Hkv < H && (q.sg % 8 || dq.sg % 8))) return cudaErrorInvalidValue;
  if (doc.key_start == nullptr || doc.tile_min == nullptr || doc.tile_max == nullptr) return cudaErrorInvalidValue;
  for (const AttnView* t : {&q, &k, &v, &out, &dout, &dq, &dk, &dv}) if (!view_ok(*t)) return cudaErrorInvalidValue;
#define PFX_BWD(HD, BF, GQA) \
  attention_bwd_impl<HD, BF, GQA, true>(q, k, v, out, dout, lse, dq, dk, dv, dq_acc, lse2, delta, B, S, S, H, Hkv, scale, true, drop, st, doc)
  if (Hkv < H) {
    if (dtype == 1) return D == 128 ? PFX_BWD(128, true, true) : PFX_BWD(64, true, true);
    return D == 128 ? PFX_BWD(128, false, true) : PFX_BWD(64, false, true);
  }
  if (dtype == 1) return D == 128 ? PFX_BWD(128, true, false) : PFX_BWD(64, true, false);
  return D == 128 ? PFX_BWD(128, false, false) : PFX_BWD(64, false, false);
#undef PFX_BWD
}

}  // namespace pfx
