// C++ launch interface of the non-GEMM kernels.  dtype codes: 0 = fp16, 1 = bf16, 3 = fp32.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace pfx {

cudaError_t norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int rows, int cols, float eps,
                     int dtype, bool rms, cudaStream_t st);
int norm_bwd_num_parts(int rows, int num_sms);
cudaError_t norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, void* dw, void* db,
                     float* workspace, int rows, int cols, int dtype, bool rms, int num_sms, cudaStream_t st, const void* dres = nullptr);

cudaError_t bias_gelu(const void* x, const void* bias, const void* dy, void* out, size_t rows, int cols, int dtype, bool bwd, int num_sms,
                      cudaStream_t st, bool exact = false);
cudaError_t bias_dropout_add(const void* x, const void* bias, const void* residual, void* out, size_t rows, int cols, float p,
                             uint64_t seed, uint64_t offset, int dtype, bool bwd, int num_sms, cudaStream_t st);
int colsum_num_parts(int rows);
cudaError_t colsum(const void* x, void* out, float* workspace, int rows, int cols, int dtype, bool out_fp32, cudaStream_t st);

cudaError_t ce_stats(const void* logits, const int64_t* labels, float* row_max, float* row_sum, float* tgt, int rows, int cols,
                     int64_t vocab_start, int dtype, cudaStream_t st);
cudaError_t ce_bwd(void* logits, const int64_t* labels, const float* lse, const float* gscale, int rows, int cols, int64_t vocab_start,
                   int dtype, cudaStream_t st);

cudaError_t sumsq(const void* x, size_t n, float* out, float* workspace, int dtype, bool accumulate, int num_sms, cudaStream_t st);
cudaError_t clip_coef(const float* sq, float inv_loss_scale, float clip_norm, float* gscale, float* found_inf, float* gnorm, cudaStream_t st);
cudaError_t adamw_flat(void* p_lp, float* master, const void* grad, float* m, float* v, size_t n, float lr, float beta1, float beta2,
                       float eps, float wd, float bc1, float bc2, const float* gscale, const float* found_inf, int grad_dtype,
                       int lp_dtype, int num_sms, cudaStream_t st);
cudaError_t accumulate_f32(float* dst, const void* src, size_t n, float scale, int dtype, int num_sms, cudaStream_t st);

cudaError_t topp_sampling(const void* probs, const float* top_ps, float* out_prob, int64_t* out_id, int rows, int V, uint64_t seed,
                          uint64_t offset, int dtype, cudaStream_t st);
cudaError_t rope(const void* x, void* y, const int64_t* positions, size_t tokens, int heads, int d, int seq_len, float base, bool bwd,
                 int dtype, int num_sms, cudaStream_t st);
cudaError_t causal_softmax(const void* a, const void* b, void* out, size_t batch, int sq, int sk, float scale, bool bwd, int dtype,
                           cudaStream_t st);

// MX fp8: e4m3 values + E8M0 scale per 32 K-elements; sf = [ceil(rows / 128), K / 128, 512] bytes in the GEMM copy order (zero-initialised by the caller)
cudaError_t quantize_mxfp8(const void* x, void* q, void* sf, int rows, int K, int dtype, cudaStream_t st);
cudaError_t quantize_rows(const void* x, const float* smooth, void* q, float* scale, int rows, int cols, int dtype, bool fp8, cudaStream_t st);

// ---- peer-memory collectives (comm_p2p.cu): every pointer table lives in device memory
cudaError_t p2p_barrier(uint32_t** signal_pads, int rank, int world, uint32_t epoch_slot, cudaStream_t st);
cudaError_t p2p_reduce_scatter(void** peer_bufs, void* out, size_t shard_elems, int rank, int world, int in_dtype, int out_dtype,
                               bool accumulate, float scale, int num_sms, cudaStream_t st);
cudaError_t slot_reduce(const void* staging, void* out, const void* bias, size_t slot_elems, int world, int cols, int dtype, int num_sms,
                        cudaStream_t st);
cudaError_t p2p_all_gather(void** peer_bufs, const void* src, size_t shard_elems, int rank, int world, int dtype, int num_sms,
                           cudaStream_t st);
cudaError_t adamw_p2p_broadcast(void** peer_param_bufs, size_t shard_offset, float* master, const void* grad, float* m, float* v, size_t n,
                                float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2, const float* gscale,
                                const float* found_inf, int grad_dtype, int lp_dtype, int world, int num_sms, cudaStream_t st);

// gemv_skinny.cu — decode-time y = x W^T (+b) for <= 8 activation rows
cudaError_t gemv_skinny(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int dtype, int num_sms, cudaStream_t st,
                        const void* ln_w = nullptr, const void* ln_b = nullptr, float ln_eps = 1e-5f, const void* residual = nullptr, int act = 0);

void gemv_set_tuning(int cols, int split);
cudaError_t gemv_w8a8(const void* x, const void* w, const float* xs, const float* ws, const void* bias, void* y, int M, int N, int K, int num_sms,
                      cudaStream_t st);

// gemm_smallm_sm90.cu — swap-AB wgmma GEMM, split-K over a cluster with DSMEM reduction (1 <= M <= 128, bf16)
cudaError_t gemm_smallm(const void* x, const void* w, const void* bias, void* y, int M, int N, int K, int dtype, int split, int num_sms,
                        cudaStream_t st);

// attention_fwd_sm90.cu — flash-style attention forward (wgmma / TMA), [B,S,H,D] bf16, D in {64,128}
cudaError_t attention_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Sq, int Sk, int H, int D, float scale,
                          bool causal, cudaStream_t st);

// attention_decode.cu — single-query attention over the static KV cache
cudaError_t attention_decode(const void* q, void* k, void* v, const void* mask, void* out, int B, int H, int D, int L, int Lmax,
                             float scale, int dtype, cudaStream_t st, const int64_t* write_idx = nullptr);


// embedding.cu — fused word (+ position) look-up; deterministic sorted scatter-add gradient (workspace: next_pow2(tokens) 64-bit keys)
cudaError_t embedding_fwd(const int64_t* ids, const void* w, const int64_t* pos, const void* pw, void* out, int64_t tokens, int hidden,
                          int64_t vocab_start, int64_t rows, int dtype, cudaStream_t st);
int embedding_bwd_max_tokens();
cudaError_t embedding_bwd(const int64_t* ids, const void* dout, void* dw, unsigned long long* workspace, int64_t tokens, int hidden,
                          int64_t vocab_start, int64_t rows, int dtype, int grad_dtype, bool accumulate, cudaStream_t st);

// moe_kernels.cu — expert-parallel dispatch / combine over peer memory
cudaError_t moe_route(const int64_t* gate_idx, int num_slots, int total_experts, int* slot_rank, int* counts, cudaStream_t st);
cudaError_t moe_dispatch(const void* src, const float* scale, const int64_t* gate_idx, const int* slot_rank, const int* counts, int* slot_loc,
                         int* seg, void** peer_recv, void** peer_cnt, void** peer_flags, unsigned* block_counter, int num_slots, int src_div,
                         int H, int e_local, int world, int rank, int align, int cap_rows, uint32_t epoch, int dtype, int num_ctas,
                         cudaStream_t st);
cudaError_t moe_tile_table(const int* seg, int e_local, int align, int cap_rows, int* tile_group, int* seg2, int* sticky, cudaStream_t st);
cudaError_t grouped_colsum(const void* x, const int* seg2, int groups, int N, void* out, int dtype, cudaStream_t st);
cudaError_t moe_combine(void** peer_src, const int* slot_loc, const float* weights, void* out, void* rows, void** peer_flags, int T, int topk,
                        int H, int world, int rank, uint32_t epoch, int dtype, int num_ctas, cudaStream_t st);

}  // namespace pfx
