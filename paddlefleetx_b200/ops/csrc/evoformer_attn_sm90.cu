// Evoformer gated attention on wgmma / TMA (sm_90a): the attention primitive of AlphaFold2 / HelixFold
// (reference ppfleetx/models/protein_folding/attentions.py:35-180, its ``fused_gate_attention`` path :126-142).
//
//   logits[g, h, q, k] = scale * Q[g, q, h, :] . K[g, k, h, :] + mask_bias[g, k] + pair_bias[g / groups_per_pair, h, q, k]
//   O[g, q, h, :]      = softmax_k(logits) @ V[g, k, h, :]  *  sigmoid(gate[g, q, h, :])
//
// g runs over batch x {MSA sequences | residues} (thousands of independent small attentions), the head width is 32, H is 4 or 8.  The
// reference materialises the [g, h, q, k] logits in HBM three times (bias add, softmax, gating are separate ops); here they live in
// registers only.
//
// A 32-wide head is half of a 128-byte swizzle row, so one CTA owns a PAIR of heads of one 64-query tile: the Q / K / V tiles are
// loaded as [rows x 64] (both heads, one TMA box each) and each of the two consumer warpgroups takes one head: S_x = Q_x K_x^T runs over
// the two wgmma K-steps that belong to head x, and P_x V is issued at N = 64 over both heads' channels — only the 32 columns of head x
// are stored.  That wastes half of a product the tensor core is not short of and keeps every operand in the layouts the flash-attention
// kernel already runs on (K-major / MN-major, 128-byte swizzle, P from registers).
//   warp 8    TMA producer: Q tile once per work item, K / V tiles of 128 keys through a 2-stage ring
//   warps 0-7 two consumer warpgroups (head x = warpgroup): products, biases added on the accumulator fragment (mask bias: one value per
//             key, pair bias: bf16 pairs of this row), online softmax, P from registers; the epilogue multiplies by sigmoid(gate)
// Output O (bf16, [g, q, h, 32]) and the row-wise log-sum-exp ([g, h, q] fp32, for the backward).
#include <cstdio>

#include "pfx_ptx.cuh"
#include "pfx_common.cuh"
#include "pfx_gemm.h"
#include "pfx_kernels.h"
#include "pfx_attn.h"
#include <cudaTypedefs.h>

namespace pfx {

namespace {

constexpr int kEvThreads = 288;       // warps 0-7 two consumer warpgroups (one head each), warp 8 TMA producer
constexpr int kEvQ = 64;              // queries per tile
constexpr int kEvKv = 128;            // keys per KV tile
constexpr int kEvD = 64;              // two heads of 32 channels = one 128-byte row
constexpr int kEvHead = 32;

struct EvSmem {
  static constexpr int kQBytes = kEvQ * kEvD * 2;
  static constexpr int kKBytes = kEvKv * kEvD * 2;
  static constexpr int kVBytes = kEvKv * kEvD * 2;
  static constexpr int kStageBytes = kKBytes + kVBytes;
  static constexpr int kStages = 2;
  static constexpr int kBarBytes = 128;
  static constexpr int kAlignSlack = 1024;
  static constexpr int kUsed = kQBytes + kStages * kStageBytes + kBarBytes;
  static constexpr int kTotal = kAlignSlack + kUsed;
};

struct EvParams {
  __nv_bfloat16* out;          // [G, Sq, H, 32]
  float* lse;                  // [G, H, Sq] natural log, or nullptr
  const float* mask_bias;      // [G, Sk] fp32 or nullptr
  const __nv_bfloat16* pair_bias;   // [G / groups_per_pair, H, Sq, Sk] bf16 or nullptr
  const __nv_bfloat16* gate;   // [G, Sq, H, 32] pre-sigmoid logits or nullptr
  int G, Sq, Sk, H, groups_per_pair;
  float scale_log2;
};

__global__ void __launch_bounds__(kEvThreads, 1)
evoformer_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                          const __grid_constant__ EvParams prm) {
  using S = EvSmem;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_q = smem_base;
  const uint32_t smem_kv = smem_q + S::kQBytes;
  const uint32_t smem_bar = smem_kv + S::kStages * S::kStageBytes;
  const uint32_t q_full = smem_bar, q_empty = smem_bar + 8;
  auto kv_full = [&](int s) { return smem_bar + 8u * (2 + s); };
  auto kv_empty = [&](int s) { return smem_bar + 8u * (4 + s); };

  const uint32_t warp = warp_id(), lane = lane_id();
  const int Sq = prm.Sq, Sk = prm.Sk, H = prm.H;
  const int n_q_tiles = (Sq + kEvQ - 1) / kEvQ;
  const int n_kv = (Sk + kEvKv - 1) / kEvKv;
  const int n_hp = H / 2;                              // head pairs
  const int n_items = prm.G * n_hp * n_q_tiles;        // item -> (g, head pair, query tile): the tiles of one group are neighbours (K / V stay in L2)
  auto item_qt = [&](int w) { return w % n_q_tiles; };
  auto item_hp = [&](int w) { return (w / n_q_tiles) % n_hp; };
  auto item_g = [&](int w) { return w / (n_q_tiles * n_hp); };

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1); mbar_init(q_empty, 8);
    for (int s2 = 0; s2 < S::kStages; ++s2) { mbar_init(kv_full(s2), 1); mbar_init(kv_empty(s2), 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ==== TMA producer
    if (elect_one()) {
      uint32_t t = 0;
      int it = 0;
      for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
        const int g = item_g(w), col = item_hp(w) * kEvD, q0 = item_qt(w) * kEvQ;
        mbar_wait(q_empty, ((uint32_t)it & 1u) ^ 1u);
        mbar_arrive_expect_tx(q_full, S::kQBytes);
        tma_load_3d(&tmap_q, q_full, smem_q, col, q0, g);
        for (int j = 0; j < n_kv; ++j, ++t) {
          const int stage = t & 1;
          mbar_wait(kv_empty(stage), ((t >> 1) & 1u) ^ 1u);
          const uint32_t sk = smem_kv + stage * S::kStageBytes, sv = sk + S::kKBytes;
          mbar_arrive_expect_tx(kv_full(stage), S::kStageBytes);
          const int key0 = j * kEvKv;
          tma_load_3d(&tmap_k, kv_full(stage), sk, col, key0, g);
          for (int kb = 0; kb < 2; ++kb)            // V as the MN-major B operand: [64 keys x 64 channels] boxes
            tma_load_3d(&tmap_v, kv_full(stage), sv + kb * 8192, col, key0 + kb * 64, g);
        }
      }
    }
  } else {
    // ==== consumers: warpgroup x = head x of the pair
    constexpr uint64_t kDescK = wgmma_desc_hi_lo(16, 1024);        // K-major, 128-byte swizzle
    constexpr uint64_t kDescMN = wgmma_desc_hi_lo(8192, 1024);     // MN-major (a single 64-channel chunk)
    constexpr float kLog2e = 1.4426950408889634f;
    const int x = (int)(warp >> 2);
    const int row_lo = (int)((warp & 3u) * 16u + (lane >> 2));     // this thread's query rows inside the tile: row_lo and row_lo + 8
    const int col_in8 = (int)(lane & 3u) * 2;
    uint32_t t = 0;
    int it = 0;
    for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
      const int g = item_g(w), hp = item_hp(w), q0 = item_qt(w) * kEvQ;
      const int head = 2 * hp + x;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      float o[kEvD / 2];                          // both heads' channels; [32 x, 32 x + 32) are head x's
#pragma unroll
      for (int i = 0; i < kEvD / 2; ++i) o[i] = 0.f;
      const float* mb_row = prm.mask_bias ? prm.mask_bias + (size_t)g * Sk : nullptr;
      const __nv_bfloat16* pb_rows[2] = {nullptr, nullptr};
      if (prm.pair_bias) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row_c = min(q0 + row_lo + 8 * hh, Sq - 1);   // rows past Sq of a ragged tile: read a valid bias row, never stored
          pb_rows[hh] = prm.pair_bias + (((size_t)(g / prm.groups_per_pair) * H + head) * Sq + row_c) * Sk;
        }
      }
      mbar_wait(q_full, (uint32_t)it & 1u);
      for (int j = 0; j < n_kv; ++j, ++t) {
        const int stage = t & 1;
        const uint32_t sk = smem_kv + stage * S::kStageBytes, sv = sk + S::kKBytes;
        mbar_wait(kv_full(stage), (t >> 1) & 1u);
        float s[kEvKv / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {               // S_x = Q[:, 32 x : 32 x + 32] K[:, 32 x : 32 x + 32]^T: the two K-steps of head x
          const uint32_t off = (uint32_t)(2 * x + k) * 32u;
          WgmmaSS<kEvKv, true, 0, 0>::mma(s, wgmma_desc(smem_q + off, kDescK), wgmma_desc(sk + off, kDescK), k != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        const int key0 = j * kEvKv;
        const bool pair_ok = (Sk % 2) == 0;         // bf16 / fp32 pair loads need an even row length
#pragma unroll
        for (int gi = 0; gi < kEvKv / 8; ++gi) {
          const int c = key0 + 8 * gi + col_in8;
          float mb0 = 0.f, mb1 = 0.f;
          if (mb_row) {
            if (pair_ok && c + 1 < Sk) { const float2 f = __ldg(reinterpret_cast<const float2*>(mb_row + c)); mb0 = f.x; mb1 = f.y; }
            else { if (c < Sk) mb0 = __ldg(mb_row + c); if (c + 1 < Sk) mb1 = __ldg(mb_row + c + 1); }
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float b0 = mb0, b1 = mb1;
            if (prm.pair_bias) {
              if (pair_ok && c + 1 < Sk) { const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(pb_rows[hh] + c)); b0 += f.x; b1 += f.y; }
              else { if (c < Sk) b0 += __bfloat162float(pb_rows[hh][c]); if (c + 1 < Sk) b1 += __bfloat162float(pb_rows[hh][c + 1]); }
            }
            s[4 * gi + 2 * hh] = (c < Sk) ? fmaf(s[4 * gi + 2 * hh], prm.scale_log2, b0 * kLog2e) : -INFINITY;          // logits in log2 units
            s[4 * gi + 2 * hh + 1] = (c + 1 < Sk) ? fmaf(s[4 * gi + 2 * hh + 1], prm.scale_log2, b1 * kLog2e) : -INFINITY;
          }
        }
        float f[2], m_use[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float mx = -INFINITY;
#pragma unroll
          for (int gi = 0; gi < kEvKv / 8; ++gi) mx = fmaxf(mx, fmaxf(s[4 * gi + 2 * hh], s[4 * gi + 2 * hh + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m_run[hh], mx);
          f[hh] = (m_run[hh] == -INFINITY) ? 0.f : exp2f(m_run[hh] - m_new);
          m_run[hh] = m_new;
          m_use[hh] = (m_new == -INFINITY) ? 0.f : m_new;
          l_run[hh] *= f[hh];
        }
#pragma unroll
        for (int i = 0; i < kEvD / 2; ++i) o[i] *= f[(i >> 1) & 1];
        uint32_t pw[kEvKv / 4];
#pragma unroll
        for (int gi = 0; gi < kEvKv / 8; ++gi) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float p0 = exp2f(s[4 * gi + 2 * hh] - m_use[hh]), p1 = exp2f(s[4 * gi + 2 * hh + 1] - m_use[hh]);
            l_run[hh] += p0 + p1;
            pw[2 * gi + hh] = pack_bf16x2(p0, p1);
          }
        }
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kEvKv / 16; ++k) {
          const uint32_t b_off = (k / 4) * 8192 + (k % 4) * 2048;
          const uint32_t a[4] = {pw[4 * k], pw[4 * k + 1], pw[4 * k + 2], pw[4 * k + 3]};
          WgmmaRS<kEvD, 1>::mma(o, a, wgmma_desc(sv + b_off, kDescMN), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(kv_empty(stage));
      }
      if (lane == 0) mbar_arrive(q_empty);
      // item epilogue: O_x / l, gate, store head x's 32 channels
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float l_all = l_run[hh];
        l_all += __shfl_xor_sync(0xffffffffu, l_all, 1);
        l_all += __shfl_xor_sync(0xffffffffu, l_all, 2);
        const int row_g = q0 + row_lo + 8 * hh;
        const float inv = l_all > 0.f ? 1.f / l_all : 0.f;
        if (row_g < Sq) {
          const size_t base = (((size_t)g * Sq + row_g) * H + head) * kEvHead + col_in8;
#pragma unroll
          for (int jj = 0; jj < kEvHead / 8; ++jj) {
            float v0 = (x ? o[4 * (4 + jj) + 2 * hh] : o[4 * jj + 2 * hh]) * inv;            // static register indices
            float v1 = (x ? o[4 * (4 + jj) + 2 * hh + 1] : o[4 * jj + 2 * hh + 1]) * inv;
            if (prm.gate) {
              const float2 gt = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(prm.gate + base + 8 * jj));
              v0 *= 1.f / (1.f + __expf(-gt.x)); v1 *= 1.f / (1.f + __expf(-gt.y));
            }
            *reinterpret_cast<uint32_t*>(prm.out + base + 8 * jj) = pack_bf16x2(v0, v1);
          }
          if (prm.lse != nullptr && (lane & 3u) == 0)
            prm.lse[((size_t)g * H + head) * Sq + row_g] = (l_all > 0.f) ? (m_run[hh] + log2f(l_all)) * 0.6931471805599453f : -INFINITY;
        }
      }
    }
  }
}


// Backward.  Same transposed formulation as attention_bwd_sm90.cu (keys on the wgmma M rows, 64-query inner tiles, P^T and dS^T fed to
// the accumulating products from registers, dQ by TMA reduce-add), specialised for a 32-wide head: one CTA = (group, head, 64-key
// tile); the [.. x 64] TMA tiles carry the head PAIR, the two wgmma K-steps of this head select its half for S^T / dP^T, the N = 64
// products (dV, dK, dQ) compute the other head's columns as a by-product that is never read.
//   logits^T = scale K Q^T + mask_bias[k] + pair_bias[q, k]      P^T = exp2(logits^T log2e - lse2[q])
//   dV  += P^T dO'                 dO' = dOut * sigmoid(gate)   (written once by the prep kernel, with dGate and delta = rowsum(dOut o out))
//   dS^T = P^T o (dP^T - delta[q])      dP^T = V dO'^T
//   dK  += scale dS^T Q      dQ = scale dS K      dPairBias[q, k] += dS (fp32 red.add: the groups that share a pair bias collide here)
constexpr int kEbThreads = 160;       // warps 0-3 consumer warpgroup, warp 4 TMA producer
constexpr int kEbKv = 64, kEbQt = 64;

struct EbSmem {
  static constexpr int kKBytes = kEbKv * kEvD * 2;          //  8 KB: K / V tile of the head pair
  static constexpr int kQBytes = kEbQt * kEvD * 2;          //  8 KB: Q / dO' tile
  static constexpr int kDsBytes = kEbKv * kEbQt * 2;        //  8 KB
  static constexpr int kStatBytes = 2 * kEbQt * 4;
  static constexpr int kStages = 3;
  static constexpr int kDqBytes = kEbQt * kEvHead * 4;      //  8 KB: dQ tile [64 q][32 d] fp32
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kOffK + kKBytes;
  static constexpr int kOffQ = kOffV + kKBytes;
  static constexpr int kOffDo = kOffQ + kStages * kQBytes;
  static constexpr int kOffDs = kOffDo + kStages * kQBytes;
  static constexpr int kOffDq = kOffDs + kDsBytes;
  static constexpr int kOffStat = kOffDq + kDqBytes;
  static constexpr int kOffBar = kOffStat + kStages * kStatBytes;
  static constexpr int kTotal = kOffBar + 256 + 1024;
};

struct EbParams {
  const float* lse2;                 // [G*H, Sq_pad] log2 units, +inf in the padding
  const float* delta;                // [G*H, Sq_pad]
  const float* mask_bias;            // [G, Sk] or null
  const __nv_bfloat16* pair_bias;    // [G / gpp, H, Sq, Sk] or null
  float* dpair;                      // fp32 [G / gpp, H, Sq, Sk] or null
  __nv_bfloat16* dk;                 // [G, Sk, H, 32]
  __nv_bfloat16* dv;
  int G, Sq, Sk, H, Sq_pad, gpp;
  float scale, scale_log2;
};

__global__ void __launch_bounds__(kEbThreads, 1)
evoformer_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                          const __grid_constant__ CUtensorMap tmap_do, const __grid_constant__ CUtensorMap tmap_dq, const __grid_constant__ EbParams prm) {
  using S = EbSmem;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t s_k = smem_base + S::kOffK, s_v = smem_base + S::kOffV, s_q = smem_base + S::kOffQ, s_do = smem_base + S::kOffDo;
  const uint32_t s_ds = smem_base + S::kOffDs, s_dq = smem_base + S::kOffDq, s_stat = smem_base + S::kOffStat;
  const uint32_t s_bar = smem_base + S::kOffBar;
  auto bar = [&](int i) { return s_bar + 8u * i; };
  const uint32_t kv_full = bar(0);
  auto q_full = [&](int s) { return bar(1 + s); };
  auto q_empty = [&](int s) { return bar(4 + s); };

  const uint32_t warp = warp_id(), lane = lane_id();
  const int n_kv_tiles = (prm.Sk + kEbKv - 1) / kEbKv;
  const int gh = blockIdx.x / n_kv_tiles;            // (group, head): its key tiles are neighbours in launch order (shared Q / dO' in L2)
  const int j = blockIdx.x - gh * n_kv_tiles;
  const int h = gh % prm.H, g = gh / prm.H;
  const int hx = h & 1, col = (h >> 1) * kEvD;        // head inside its pair; first column of the pair
  const int k0 = j * kEbKv;
  const int n_iter = (prm.Sq + kEbQt - 1) / kEbQt;

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v); tma_prefetch_desc(&tmap_do); tma_prefetch_desc(&tmap_dq);
    mbar_init(kv_full, 1);
    for (int s2 = 0; s2 < S::kStages; ++s2) { mbar_init(q_full(s2), 1); mbar_init(q_empty(s2), 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ==== TMA producer
    if (elect_one()) {
      mbar_arrive_expect_tx(kv_full, 2 * S::kKBytes);
      tma_load_3d(&tmap_k, kv_full, s_k, col, k0, g);
      tma_load_3d(&tmap_v, kv_full, s_v, col, k0, g);
      for (int it = 0; it < n_iter; ++it) {
        const int st = it % S::kStages, q0 = it * kEbQt;
        mbar_wait(q_empty(st), (((uint32_t)(it / S::kStages)) & 1u) ^ 1u);
        mbar_arrive_expect_tx(q_full(st), 2 * S::kQBytes + S::kStatBytes);
        tma_load_3d(&tmap_q, q_full(st), s_q + st * S::kQBytes, col, q0, g);
        tma_load_3d(&tmap_do, q_full(st), s_do + st * S::kQBytes, col, q0, g);
        const size_t so = (size_t)gh * prm.Sq_pad + q0;
        bulk_load_1d(s_stat + st * S::kStatBytes, prm.lse2 + so, kEbQt * 4, q_full(st));
        bulk_load_1d(s_stat + st * S::kStatBytes + kEbQt * 4, prm.delta + so, kEbQt * 4, q_full(st));
      }
    }
  } else {
    // ==== consumer warpgroup
    constexpr float kLog2e = 1.4426950408889634f;
    constexpr uint64_t kDescK = wgmma_desc_hi_lo(16, 1024);
    constexpr uint64_t kDescMN = wgmma_desc_hi_lo(8192, 1024);
    const int k_row = (int)(warp * 16u + (lane >> 2));               // this thread's key rows inside the tile: k_row and k_row + 8
    const int col_in8 = (int)(lane & 3u) * 2;
    const size_t pair_base = ((size_t)(g / prm.gpp) * prm.H + h) * prm.Sq;     // row index base of [.., Sq, Sk]
    const bool leader = threadIdx.x == 0;
    float mb2[2];
    int kc[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      kc[hh] = min(k0 + k_row + 8 * hh, prm.Sk - 1);                 // clamped key index for bias loads
      mb2[hh] = prm.mask_bias ? __ldg(prm.mask_bias + (size_t)g * prm.Sk + kc[hh]) * kLog2e : 0.f;
    }
    float dv[kEvD / 2], dk[kEvD / 2];
#pragma unroll
    for (int i = 0; i < kEvD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    mbar_wait(kv_full, 0);
    for (int it = 0; it < n_iter; ++it) {
      const int st = it % S::kStages;
      const int q0 = it * kEbQt;
      const uint32_t sq = s_q + st * S::kQBytes, sdo = s_do + st * S::kQBytes;
      mbar_wait(q_full(st), ((uint32_t)(it / S::kStages)) & 1u);
      float s[kEbQt / 2], dp[kEbQt / 2];                             // [4 gi + e]: key k_row + 8 (e / 2), query 8 gi + col_in8 + (e % 2)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {                 // the two K-steps (32 channels) of this head inside the pair's 128-byte rows
        const uint32_t off = (uint32_t)(2 * hx + kk) * 32u;
        WgmmaSS<kEbQt, true, 0, 0>::mma(s, wgmma_desc(s_k + off, kDescK), wgmma_desc(sq + off, kDescK), kk != 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const uint32_t off = (uint32_t)(2 * hx + kk) * 32u;
        WgmmaSS<kEbQt, true, 0, 0>::mma(dp, wgmma_desc(s_v + off, kDescK), wgmma_desc(sdo + off, kDescK), kk != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      const float* lse_s = reinterpret_cast<const float*>(smem_gen + (s_stat - smem_base) + st * S::kStatBytes);
      const float* dl_s = lse_s + kEbQt;
      uint32_t pw[kEbQt / 4], dsw[kEbQt / 4];
#pragma unroll
      for (int gi = 0; gi < kEbQt / 8; ++gi) {
        const int qc = 8 * gi + col_in8;
        const float2 ls = *reinterpret_cast<const float2*>(lse_s + qc), dl = *reinterpret_cast<const float2*>(dl_s + qc);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kg = k0 + k_row + 8 * hh;
          const bool k_valid = kg < prm.Sk;
          float b0 = mb2[hh], b1 = mb2[hh];
          if (prm.pair_bias) {
            b0 = fmaf(__bfloat162float(prm.pair_bias[(pair_base + min(q0 + qc, prm.Sq - 1)) * prm.Sk + kc[hh]]), kLog2e, b0);
            b1 = fmaf(__bfloat162float(prm.pair_bias[(pair_base + min(q0 + qc + 1, prm.Sq - 1)) * prm.Sk + kc[hh]]), kLog2e, b1);
          }
          float p0 = exp2f(fmaf(s[4 * gi + 2 * hh], prm.scale_log2, b0) - ls.x);      // lse2 = +inf past Sq -> 0
          float p1 = exp2f(fmaf(s[4 * gi + 2 * hh + 1], prm.scale_log2, b1) - ls.y);
          if (!k_valid) { p0 = 0.f; p1 = 0.f; }
          pw[2 * gi + hh] = pack_bf16x2(p0, p1);
          const float ds0 = p0 * (dp[4 * gi + 2 * hh] - dl.x), ds1 = p1 * (dp[4 * gi + 2 * hh + 1] - dl.y);
          if (prm.dpair != nullptr && k_valid) {                 // dPairBias[q, k] += dS
            if (q0 + qc < prm.Sq) red_add_f32(prm.dpair + (pair_base + q0 + qc) * prm.Sk + kg, ds0);
            if (q0 + qc + 1 < prm.Sq) red_add_f32(prm.dpair + (pair_base + q0 + qc + 1) * prm.Sk + kg, ds1);
          }
          dsw[2 * gi + hh] = pack_bf16x2(ds0 * prm.scale, ds1 * prm.scale);
        }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t r = (uint32_t)(k_row + 8 * hh);
        const uint32_t dst_row = s_ds + (r / 8u) * 1024u + (r % 8u) * 128u + (uint32_t)col_in8 * 2u;
#pragma unroll
        for (int gi = 0; gi < kEbQt / 8; ++gi)
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst_row + (((uint32_t)gi ^ (r % 8u)) << 4)), "r"(dsw[2 * gi + hh]) : "memory");
      }
      fence_proxy_async_smem();
      if (leader) tma_store_wait_read<0>();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float dq[kEvD / 2];                                          // rows are queries here; both heads' channels
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kEbQt / 16; ++kk) {
        const uint32_t a[4] = {pw[4 * kk], pw[4 * kk + 1], pw[4 * kk + 2], pw[4 * kk + 3]};
        WgmmaRS<kEvD, 1>::mma(dv, a, wgmma_desc(sdo + kk * 2048, kDescMN), 1u);
      }
#pragma unroll
      for (int kk = 0; kk < kEbQt / 16; ++kk) {
        const uint32_t a[4] = {dsw[4 * kk], dsw[4 * kk + 1], dsw[4 * kk + 2], dsw[4 * kk + 3]};
        WgmmaRS<kEvD, 1>::mma(dk, a, wgmma_desc(sq + kk * 2048, kDescMN), 1u);
      }
#pragma unroll
      for (int kk = 0; kk < kEbKv / 16; ++kk)
        WgmmaSS<kEvD, true, 1, 1>::mma(dq, wgmma_desc(s_ds + kk * 2048, kDescMN), wgmma_desc(s_k + kk * 2048, kDescMN), kk != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(q_empty(st));
      // this head's 32 channels of the dQ tile: registers -> staging [64 q][32 d] fp32 -> one TMA reduce-add
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t row = s_dq + (uint32_t)(k_row + 8 * hh) * (kEvHead * 4u) + (uint32_t)col_in8 * 4u;
#pragma unroll
        for (int jj = 0; jj < kEvHead / 8; ++jj) {
          const float v0 = hx ? dq[4 * (4 + jj) + 2 * hh] : dq[4 * jj + 2 * hh], v1 = hx ? dq[4 * (4 + jj) + 2 * hh + 1] : dq[4 * jj + 2 * hh + 1];
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(row + jj * 32u), "f"(v0), "f"(v1) : "memory");
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (leader) {
        tma_reduce_add_2d(&tmap_dq, s_dq, h * kEvHead, g * prm.Sq + q0);
        tma_store_commit();
      }
    }
    if (leader) tma_store_wait<0>();
    // ---- epilogue: dV and dK rows of this key tile, this head's 32 channels
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int kg = k0 + k_row + 8 * hh;
      if (kg < prm.Sk) {
        const size_t base = (((size_t)g * prm.Sk + kg) * prm.H + h) * kEvHead + col_in8;
#pragma unroll
        for (int jj = 0; jj < kEvHead / 8; ++jj) {
          const int a0 = 4 * jj + 2 * hh, a1 = 4 * (4 + jj) + 2 * hh;                         // static register indices
          *reinterpret_cast<uint32_t*>(prm.dv + base + 8 * jj) = pack_bf16x2(hx ? dv[a1] : dv[a0], hx ? dv[a1 + 1] : dv[a0 + 1]);
          *reinterpret_cast<uint32_t*>(prm.dk + base + 8 * jj) = pack_bf16x2(hx ? dk[a1] : dk[a0], hx ? dk[a1 + 1] : dk[a0 + 1]);
        }
      }
    }
  }
}

// prep: dO' = dOut * sigmoid(gate) (bf16), dGate = dOut * out * (1 - sigmoid(gate)), delta = rowsum(dOut o out), lse -> log2 units (padded)
__global__ void evoformer_bwd_prep_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ gate,
                                          const float* __restrict__ lse, __nv_bfloat16* __restrict__ do_pre, __nv_bfloat16* __restrict__ dgate,
                                          float* __restrict__ lse2, float* __restrict__ delta, int G, int Sq, int H, int Sq_pad) {
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // (g, s_pad, h)
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)G * Sq_pad * H) return;
  const int h = (int)(w % H);
  const int s = (int)((w / H) % Sq_pad);
  const int g = (int)(w / ((int64_t)H * Sq_pad));
  const size_t oi = ((size_t)g * H + h) * Sq_pad + s;
  if (s >= Sq) {
    if (lane == 0) { lse2[oi] = INFINITY; delta[oi] = 0.f; }
    return;
  }
  const size_t e = (((size_t)g * Sq + s) * H + h) * kEvHead + lane;
  const float o = __bfloat162float(out[e]), d = __bfloat162float(dout[e]);
  float sig = 1.f;
  if (gate != nullptr) {
    sig = 1.f / (1.f + __expf(-__bfloat162float(gate[e])));
    dgate[e] = __float2bfloat16(d * o * (1.f - sig));
  }
  do_pre[e] = __float2bfloat16(d * sig);
  const float acc = warp_sum(d * o);
  if (lane == 0) {
    delta[oi] = acc;
    lse2[oi] = lse[((size_t)g * H + h) * Sq + s] * 1.4426950408889634f;
  }
}

__global__ void evoformer_f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n8) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = *reinterpret_cast<const float4*>(src + i * 8), b = *reinterpret_cast<const float4*>(src + i * 8 + 4);
    uint4 v;
    v.x = pack_bf16x2(a.x, a.y); v.y = pack_bf16x2(a.z, a.w); v.z = pack_bf16x2(b.x, b.y); v.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(dst + i * 8) = v;
  }
}

}  // namespace

// q [G, Sq, H, 32], k / v [G, Sk, H, 32], out [G, Sq, H, 32] bf16 contiguous; mask_bias [G, Sk] fp32 (or null); pair_bias [G / groups_per_pair,
// H, Sq, Sk] bf16 (or null); gate [G, Sq, H, 32] bf16 pre-sigmoid (or null); lse [G, H, Sq] fp32 (or null).  H even.
cudaError_t evoformer_attention_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const float* mask_bias, const void* pair_bias,
                                    const void* gate, int G, int Sq, int Sk, int H, int groups_per_pair, float scale, cudaStream_t st) {
  if (G < 1 || Sq < 1 || Sk < 1 || H < 2 || (H & 1) || groups_per_pair < 1 || G % groups_per_pair) return cudaErrorInvalidValue;
  for (const void* p : {q, k, v, (const void*)out})
    if (p == nullptr || (reinterpret_cast<uintptr_t>(p) % 16)) return cudaErrorInvalidValue;
  using S = EvSmem;
  const uint64_t row = (uint64_t)H * kEvHead;           // elements per (g, position)
  CUtensorMap tq, tk, tv;
  bool sw = false;
  bool ok = make_tmap_bshd(&tq, q, 1, row, Sq, G, row * 2, (uint64_t)Sq * row * 2, 64, kEvQ, &sw);
  ok &= !sw;
  ok &= make_tmap_bshd(&tk, k, 1, row, Sk, G, row * 2, (uint64_t)Sk * row * 2, 64, kEvKv, &sw);
  ok &= !sw;
  ok &= make_tmap_bshd(&tv, v, 1, row, Sk, G, row * 2, (uint64_t)Sk * row * 2, 64, 64, &sw);
  ok &= !sw;
  if (!ok) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(evoformer_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long items = (long)G * (H / 2) * ((Sq + kEvQ - 1) / kEvQ);
  int per_sm = 1;           // resident CTAs per SM (registers bound it): the persistent grid must not exceed them
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, evoformer_attn_fwd_kernel, kEvThreads, S::kTotal) != cudaSuccess || per_sm < 1) per_sm = 1;
  const int grid = (int)(items < (long)per_sm * sms ? items : (long)per_sm * sms);
  EvParams prm{};
  prm.out = (__nv_bfloat16*)out; prm.lse = lse; prm.mask_bias = mask_bias; prm.pair_bias = (const __nv_bfloat16*)pair_bias;
  prm.gate = (const __nv_bfloat16*)gate; prm.G = G; prm.Sq = Sq; prm.Sk = Sk; prm.H = H; prm.groups_per_pair = groups_per_pair;
  prm.scale_log2 = scale * 1.4426950408889634f;
  evoformer_attn_fwd_kernel<<<grid, kEvThreads, S::kTotal, st>>>(tq, tk, tv, prm);
  return cudaGetLastError();
}

// Backward.  Workspaces: do_pre bf16 like q, dq_acc fp32 [G, Sq, H, 32], lse2 / delta fp32 [G*H, round_up(Sq, 64)].  dpair (fp32, zeroed by
// the caller) accumulates the pair-bias gradient over the groups; dgate is written only when gate != null.
cudaError_t evoformer_attention_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const void* gate, const float* lse,
                                    const float* mask_bias, const void* pair_bias, void* dq, void* dk, void* dv, void* dgate, float* dpair,
                                    void* do_pre, float* dq_acc, float* lse2, float* delta, int G, int Sq, int Sk, int H, int groups_per_pair,
                                    float scale, cudaStream_t st) {
  if (G < 1 || Sq < 1 || Sk < 1 || H < 2 || (H & 1) || groups_per_pair < 1 || G % groups_per_pair) return cudaErrorInvalidValue;
  using S = EbSmem;
  const int Sq_pad = (Sq + kEbQt - 1) / kEbQt * kEbQt;
  const uint64_t row = (uint64_t)H * kEvHead;
  cudaError_t e = cudaMemsetAsync(dq_acc, 0, (size_t)G * Sq * row * sizeof(float), st);
  if (e != cudaSuccess) return e;
  {
    const int64_t warps = (int64_t)G * Sq_pad * H;
    evoformer_bwd_prep_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, (const __nv_bfloat16*)gate, lse,
                                                                           (__nv_bfloat16*)do_pre, (__nv_bfloat16*)dgate, lse2, delta, G, Sq, H, Sq_pad);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  CUtensorMap tq, tk, tv, tdo, tdq;
  bool sw = false, ok = true;
  ok &= make_tmap_bshd(&tq, q, 1, row, Sq, G, row * 2, (uint64_t)Sq * row * 2, 64, kEbQt, &sw); ok &= !sw;
  ok &= make_tmap_bshd(&tk, k, 1, row, Sk, G, row * 2, (uint64_t)Sk * row * 2, 64, kEbKv, &sw); ok &= !sw;
  ok &= make_tmap_bshd(&tv, v, 1, row, Sk, G, row * 2, (uint64_t)Sk * row * 2, 64, kEbKv, &sw); ok &= !sw;
  ok &= make_tmap_bshd(&tdo, do_pre, 1, row, Sq, G, row * 2, (uint64_t)Sq * row * 2, 64, kEbQt, &sw); ok &= !sw;
  ok &= make_tmap_2d_plain(&tdq, dq_acc, 3, row, (uint64_t)G * Sq, row * 4, kEvHead, kEbQt);
  if (!ok) return cudaErrorInvalidValue;
  EbParams prm{};
  prm.lse2 = lse2; prm.delta = delta; prm.mask_bias = mask_bias; prm.pair_bias = (const __nv_bfloat16*)pair_bias; prm.dpair = dpair;
  prm.dk = (__nv_bfloat16*)dk; prm.dv = (__nv_bfloat16*)dv;
  prm.G = G; prm.Sq = Sq; prm.Sk = Sk; prm.H = H; prm.Sq_pad = Sq_pad; prm.gpp = groups_per_pair;
  prm.scale = scale; prm.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    if ((e = cudaFuncSetAttribute(evoformer_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal)) != cudaSuccess) return e;
    attr_set = true;
  }
  const int n_kv = (Sk + kEbKv - 1) / kEbKv;
  evoformer_attn_bwd_kernel<<<(unsigned)((int64_t)n_kv * G * H), kEbThreads, S::kTotal, st>>>(tq, tk, tv, tdo, tdq, prm);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  evoformer_f32_to_bf16_kernel<<<1184, 256, 0, st>>>(dq_acc, (__nv_bfloat16*)dq, (int64_t)G * Sq * (int64_t)row / 8);
  return cudaGetLastError();
}

}  // namespace pfx
