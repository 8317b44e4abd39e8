// Host-side C++ interface of the wgmma GEMM family (no torch headers: keeps .cu compiles fast).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace pfx {

// EPI_BIAS_GELU_DUAL: D = acc + bias (the pre-activation the backward needs) AND D2 = gelu(D), two TMA stores per tile (FFN1 forward).
// EPI_DGELU:          D = acc * gelu'(aux) with aux = the saved pre-activation [M, N] (FFN2 dgrad producing dL/d(pre-activation)).
enum Epilogue : int { EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_GELU = 2, EPI_GELU = 3, EPI_BIAS_GELU_DUAL = 4, EPI_DGELU = 5 };

// Peer-memory communication descriptor of the fused GEMM+collective modes (passed to the kernel by value).
struct GemmComm {
  void* peer_out[8];          // mode 3: per destination rank, staging base [world][rows_per_rank][ldd] (bf16)
  void* peer_gather[8];       // AG mode: per rank, gathered A buffer [world * rows_per_rank][K]
  uint32_t* peer_flags[8];    // AG mode: per rank, chunk flags [world][chunks]
  const uint32_t* my_flags;   // AG mode: this rank's flags (local)
  const void* a_local;        // AG mode: this rank's A shard [rows_per_rank][K]
  int rows_per_rank;          // rows of the M dimension owned by one rank (0 = no comm)
  int chunk_rows;             // AG mode: rows per flag
  int my_rank, world;
  int ag_world;               // > 1 enables the all-gather -> GEMM mode
  int num_comm_ctas;          // AG mode: CTAs reserved for the push role
  uint32_t epoch;             // AG mode: value that marks "chunk present" for this call
};

// Grouped (mixture-of-experts) modes: ONE launch covers every expert, and what each tile works on comes from a table in DEVICE memory that the
// dispatch kernel wrote — the host never learns the per-expert token counts.
//   mode 1  rows grouped: A / D are the expert-major token buffer [cap_rows, *] whose 128-row blocks each belong to one expert (or to none:
//           -1, tile skipped); B (and bias) are the experts' weights stacked along their outer dimension, the tile's block picks the slice.
//           Serves forward (B K-major: [G*N, K]) and dgrad (B MN-major: [G*K, N]).
//   mode 2  K grouped: D[g] = A_g^T B_g over the token rows of expert g (wgrad).  A [rows, m_per_group] and B [rows, N] are both MN-major,
//           D is the stacked weight gradient [G*m_per_group, N]; seg = (row start, padded row count) per expert.
struct GemmGroup {
  const int* tile_group = nullptr;   // mode 1: [ceil(M / 128)] expert of each 128-row block, -1 = unused
  const int* seg = nullptr;          // mode 2: [2 * groups]
  int mode = 0;
  int groups = 0;
  int b_group_stride = 0;            // mode 1: rows of stacked B per expert (N if B is K-major, K if MN-major)
  int m_per_group = 0;               // mode 2: rows of D per expert
  int row_align = 128;               // mode 1: alignment of the expert blocks (256 allows the 2-CTA tile)
};

struct GemmArgs {
  const void* a;     // K-major: [M, K] row-major (lda = row stride, elements); MN-major: [K, M]
  const void* b;     // K-major: [N, K] row-major;                              MN-major: [K, N]
  void* d;           // [M, N] row-major, ldd = row stride (elements)
  const void* bias;  // [N] bf16 or nullptr
  void* d2 = nullptr;         // EPI_BIAS_GELU_DUAL: second output [M, N] (same dtype / ldd as d)
  const void* aux = nullptr;  // EPI_DGELU: pre-activation [M, N] (same dtype as the operands), row stride ld_aux
  int ld_aux = 0;
  int M, N, K;
  int lda, ldb, ldd;
  bool a_kmajor, b_kmajor;
  int out_mode;      // 0 = same dtype as inputs (TMA store), 1 = fp32 store, 2 = fp32 accumulate, 3 = peer scatter (GEMM->RS)
  int epilogue;      // Epilogue
  int ab_format;     // 0 = fp16, 1 = bf16
  int num_sms;
  int config;        // 0 = auto
  GemmComm comm;     // zero-initialised = plain GEMM
  GemmGroup group;   // mode 0 = plain GEMM
};

cudaError_t gemm_wgmma(const GemmArgs& args, cudaStream_t stream);

// 8-bit GEMM: D(bf16)[M,N] = (A_q[M,K] * B_q[N,K]^T) * row_scale[M] * col_scale[N] (+ bias[N]); both operands K-major.
struct LowpGemmArgs {
  const void* a; const void* b; void* d;
  const float* row_scale;   // [M] or nullptr
  const float* col_scale;   // [N] or nullptr
  const void* bias;         // [N] bf16 or nullptr
  int M, N, K, lda, ldb, ldd;
  int kind;                 // 1 = int8 (kind::i8), 2 = fp8 e4m3 (kind::f8f6f4), 3 = MX block-scaled fp8 e4m3 (kind::mxf8f6f4.block_scale)
  int num_sms, config;
  const void* sfa = nullptr;   // kind 3: E8M0 scale bytes of A / B, one 512-byte atom per (128 rows, 128 K): [row_blocks, K / 128, 512]
  const void* sfb = nullptr;
};
cudaError_t gemm_lowp_wgmma(const LowpGemmArgs& args, cudaStream_t stream);

// hit / miss counters of the tensor-map descriptor cache (diagnostics)
void tmap_cache_stats(uint64_t* hits, uint64_t* misses);

bool make_tmap_2d(CUtensorMap* map, const void* ptr, int elem_bytes, int dtype_code, uint64_t inner, uint64_t outer,
                  uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer);

// 2-D row-major tensor without shared-memory swizzle (plain row-major box in smem): fp32 reduction targets.
bool make_tmap_2d_plain(CUtensorMap* map, const void* ptr, int dtype_code, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                        uint32_t box_inner, uint32_t box_outer);

// 3-D tensor map over a [B, S, H, D] activation view (D contiguous, `inner` = columns spanned by one (b, s) row): dims are
// {inner, S, B} or — when the batch stride is the smaller one (sequence-major [S, B, ...] storage) — {inner, B, S}; `*swapped`
// tells the kernel which coordinate order to pass.  Box = {box_cols, box_rows along S, 1}, 128-byte swizzle.
bool make_tmap_bshd(CUtensorMap* map, const void* ptr, int dtype_code, uint64_t inner, uint64_t S, uint64_t B, uint64_t s_stride_bytes,
                    uint64_t b_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool* swapped);

}  // namespace pfx
