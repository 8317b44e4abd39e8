// Flash-attention kernels (attention_fwd_sm90.cu, attention_bwd_sm90.cu): host interface and the shared dropout generator.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace pfx {

// A [B, S, H, D] 16-bit view with D contiguous; strides in elements.  Covers contiguous tensors, the q / k / v slices of a packed
// [B, S, H, 3, D] projection output and sequence-major ([S, B, ...]) storage without any copy.
//
// Grouped-query attention (Hkv K/V heads, G = H / Hkv query heads per K/V head): k / v / dk / dv have Hkv heads; q and dq are
// addressed per query head h as (h / G) * sg + (h % G) * sh, which also covers the q slice of a packed [B, S, Hkv, G + 2, D]
// projection output (no uniform head stride there).  sg is read only when G > 1; a uniform view has sg = G * sh.
struct AttnView {
  const void* ptr;
  int64_t sb, ss, sh;
  int64_t sg = 0;
};

struct AttnDropout {
  float p;            // drop probability (0 = off)
  uint64_t seed;      // counter-hash key; the element (b, h, q, k) keeps iff hash16(seed, b*H+h, q, k) >= p * 65536
};

// O = softmax(scale * Q K^T + causal) (dropout) V;  lse = row-wise log-sum-exp (natural log) [B, H, Sq] fp32.
// dtype: 1 = bf16, 0 = fp16, for every view of the call (the flash kernels are compiled for both).
// H query heads, Hkv K/V heads (H % Hkv == 0); query head h reads K/V head h / (H / Hkv).  LSE, out and the dropout key stay per query
// head, so a grouped call drops the same elements as an H-head call with K/V repeated per group.
cudaError_t attention_fwd_v2(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                             int Hkv, int D, float scale, bool causal, AttnDropout drop, int dtype, cudaStream_t st);

// Intra-document mask for packed sequences: query i of batch row b attends the keys [key_start[b, i], i] when causal (self-attention,
// Sq == Sk, 0 <= key_start[b, i] <= i), or [key_start[b, i], Sk) when not (0 <= key_start[b, i] <= Sk; Sk leaves the row empty: out = 0,
// lse = -inf).  tile_min / tile_max hold the minimum / maximum of key_start over each 64-query tile ([B, ceil(Sq / 64)]); the kernels
// skip whole key tiles from them and compare per element only on boundary tiles.
struct AttnDocMask {
  const int* key_start;     // int32 [B, Sq]
  const int* tile_min;      // int32 [B, ceil(Sq / 64)]
  const int* tile_max;
};

// Writes key_start = clamp(i - src[b, i], 0, i) when from_positions (src = position ids, which restart at 0 at each document), or
// clamp(src[b, i], 0, i) otherwise, and the per-tile bounds of AttnDocMask.  src int64 [B, S].
cudaError_t attention_doc_bounds(const int64_t* src, bool from_positions, int B, int S, int* key_start, int* tile_min, int* tile_max, cudaStream_t st);

// Ring attention's document blocks: for every source rank src of a ring of c (this rank r), the block's key_start in its own key coordinates
// and tile bounds, from this rank's zigzag-local position ids pos int64 [B, s_l] (s_l = 2h: global chunks r and 2c - 1 - r).  The blocks
// are src == r: all rows x both own chunks (causal); src < r: all rows x chunk src; src > r: rows [h, 2h) x chunks src and 2c - 1 - src.
// out holds, per src in turn, key_start [B, rows], tile_min [B, ceil(rows / 64)], tile_max [B, ceil(rows / 64)] (rows = s_l or h).
cudaError_t attention_ring_doc_bounds(const int64_t* pos, int B, int s_l, int c, int r, int* out, cudaStream_t st);

// attention_fwd_v2 under a document mask (separate kernel instantiations): causal with Sq == Sk, or non-causal with any Sq, Sk.
cudaError_t attention_fwd_doc(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                              int Hkv, int D, float scale, bool causal, AttnDropout drop, const AttnDocMask& doc, int dtype, cudaStream_t st);

// Backward.  Workspace: dq_acc fp32 [B, Sq, H, D] (zeroed by the call), lse2 / delta fp32 [B, H, round_up(Sq, 64)].
// dq / dk / dv may be strided views (e.g. slices of one packed [B, S, H, 3, D] gradient buffer).  D is 64 or 128; dtype as above.
// With Hkv < H one CTA per (batch, K/V head, key tile) walks the query tiles of every head of the group, so dk / dv are written once.
cudaError_t attention_bwd(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                          const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                          int Sk, int H, int Hkv, int D, float scale, bool causal, AttnDropout drop, int dtype, cudaStream_t st);

// attention_bwd under a document mask (causal with Sq == Sk, or non-causal): a key tile skips every query tile whose tile_min lies past its
// last key; a key tile that no query reaches writes dk = dv = 0.
cudaError_t attention_bwd_doc(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                              const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                              int Sk, int H, int Hkv, int D, float scale, bool causal, AttnDropout drop, const AttnDocMask& doc, int dtype,
                              cudaStream_t st);

// Key-padding mask for bidirectional attention: query i of batch row b attends key j iff bit j % 32 of key_bits[b, j / 32] is set (any
// pattern).  key_end[b] = 1 + the last valid key: key tiles at or past it are never loaded.  key_dense[b] = the first invalid key (Sk
// when there is none): key tiles entirely below it need no per-element compare.  A row with no valid key has every bit of [0, Sk) set
// (softmax is unchanged by one additive constant on every logit), so key_end >= 1 always.  Bits at or past Sk are 0.
struct AttnKeyPad {
  const uint32_t* key_bits;  // [B, ceil(Sk / 32)]
  const int* key_end;        // int32 [B]
  const int* key_dense;      // int32 [B]
};

// Writes AttnKeyPad from a [B, S] tensor in one launch: valid = (src != pad_id) when from_ids, else (src != 0).
// src_dtype: 0 = bool / uint8, 1 = int32, 2 = int64, 3 = float32, 4 = float16, 5 = bfloat16.
cudaError_t attention_key_pad_bounds(const void* src, int src_dtype, bool from_ids, int64_t pad_id, int B, int S, uint32_t* key_bits, int* key_end,
                                     int* key_dense, cudaStream_t st);

// attention_fwd_v2 / attention_bwd, non-causal multi-head (H == Hkv), under a key-padding mask (separate kernel instantiations).
cudaError_t attention_fwd_keypad(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                                 int D, float scale, AttnDropout drop, const AttnKeyPad& pad, int dtype, cudaStream_t st);
cudaError_t attention_bwd_keypad(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                                 const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                                 int Sk, int H, int D, float scale, AttnDropout drop, const AttnKeyPad& pad, int dtype, cudaStream_t st);

// Evoformer gated attention (head width 32, H even): softmax(scale QK^T + mask_bias[g, k] + pair_bias[g / groups_per_pair, h, q, k]) V * sigmoid(gate).
// q / out / gate [G, Sq, H, 32], k / v [G, Sk, H, 32] bf16 contiguous; mask_bias fp32 [G, Sk]; pair_bias bf16; stats fp32 [2, G, H, Sq]: the
// row maximum of the logits and log2 of the row sum relative to it (log2 units; log-sum-exp = (stats[0] + stats[1]) ln 2).
cudaError_t evoformer_attention_fwd(const void* q, const void* k, const void* v, void* out, float* stats, const float* mask_bias, const void* pair_bias,
                                    const void* gate, int G, int Sq, int Sk, int H, int groups_per_pair, float scale, cudaStream_t st);

// Backward of the above.  do_pre (bf16 like q), dq_acc (fp32 like q), m2 / delta / l2 (fp32 [G*H, round_up(Sq, 64)]) are workspaces; dpair is
// an fp32 accumulator [G / groups_per_pair, H, Sq, Sk] zeroed by the caller (null = no pair-bias gradient); dgate may be null when gate is.
cudaError_t evoformer_attention_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const void* gate, const float* stats,
                                    const float* mask_bias, const void* pair_bias, void* dq, void* dk, void* dv, void* dgate, float* dpair,
                                    void* do_pre, float* dq_acc, float* m2, float* delta, float* l2, int G, int Sq, int Sk, int H, int groups_per_pair,
                                    float scale, cudaStream_t st);

}  // namespace pfx
