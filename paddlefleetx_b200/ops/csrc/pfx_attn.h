// Flash-attention kernels (attention_fwd_sm90.cu, attention_bwd_sm90.cu): host interface and the shared dropout generator.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace pfx {

// A [B, S, H, D] bf16 view with D contiguous; strides in elements.  Covers contiguous tensors, the q / k / v slices of a packed
// [B, S, H, 3, D] projection output and sequence-major ([S, B, ...]) storage without any copy.
struct AttnView {
  const void* ptr;
  int64_t sb, ss, sh;
};

struct AttnDropout {
  float p;            // drop probability (0 = off)
  uint64_t seed;      // counter-hash key; the element (b, h, q, k) keeps iff hash16(seed, b*H+h, q, k) >= p * 65536
};

// O = softmax(scale * Q K^T + causal) (dropout) V;  lse = row-wise log-sum-exp (natural log) [B, H, Sq] fp32
cudaError_t attention_fwd_v2(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, float* lse, int B, int Sq, int Sk, int H,
                             int D, float scale, bool causal, AttnDropout drop, cudaStream_t st);

// Backward.  Workspace: dq_acc fp32 [B, Sq, H, D] (zeroed by the call), lse2 / delta fp32 [B, H, round_up(Sq, 64)].
// dq / dk / dv may be strided views (e.g. slices of one packed [B, S, H, 3, D] gradient buffer).  D must be 128.
cudaError_t attention_bwd(const AttnView& q, const AttnView& k, const AttnView& v, const AttnView& out, const AttnView& dout, const float* lse,
                          const AttnView& dq, const AttnView& dk, const AttnView& dv, float* dq_acc, float* lse2, float* delta, int B, int Sq,
                          int Sk, int H, int D, float scale, bool causal, AttnDropout drop, cudaStream_t st);

// Evoformer gated attention (head width 32, H even): softmax(scale QK^T + mask_bias[g, k] + pair_bias[g / groups_per_pair, h, q, k]) V * sigmoid(gate).
// q / out / gate [G, Sq, H, 32], k / v [G, Sk, H, 32] bf16 contiguous; mask_bias fp32 [G, Sk]; pair_bias bf16; lse fp32 [G, H, Sq].
cudaError_t evoformer_attention_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const float* mask_bias, const void* pair_bias,
                                    const void* gate, int G, int Sq, int Sk, int H, int groups_per_pair, float scale, cudaStream_t st);

// Backward of the above.  do_pre (bf16 like q), dq_acc (fp32 like q), lse2 / delta (fp32 [G*H, round_up(Sq, 64)]) are workspaces; dpair is an
// fp32 accumulator [G / groups_per_pair, H, Sq, Sk] zeroed by the caller (null = no pair-bias gradient); dgate may be null when gate is.
cudaError_t evoformer_attention_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const void* gate, const float* lse,
                                    const float* mask_bias, const void* pair_bias, void* dq, void* dk, void* dv, void* dgate, float* dpair,
                                    void* do_pre, float* dq_acc, float* lse2, float* delta, int G, int Sq, int Sk, int H, int groups_per_pair,
                                    float scale, cudaStream_t st);

}  // namespace pfx
