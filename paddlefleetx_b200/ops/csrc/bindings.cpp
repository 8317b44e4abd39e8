// pybind11 / torch glue for the sm_90a kernel library.  All kernels run on the current CUDA stream.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <string>
#include <vector>

#include "pfx_gemm.h"
#include "pfx_kernels.h"
#include "pfx_symm.h"
#include "pfx_attn.h"

namespace {

inline int dtype_code(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kHalf: return 0;
    case at::kBFloat16: return 1;
    case at::kFloat: return 3;
    default: TORCH_CHECK(false, "pfx: unsupported dtype ", t.scalar_type());
  }
}
inline bool is_16bit(const at::Tensor& t) { return t.scalar_type() == at::kBFloat16 || t.scalar_type() == at::kHalf; }
// The bandwidth-bound kernels are compiled for bf16 and fp16 only; any other dtype would be reinterpreted as one of them.
inline void check_16bit(const at::Tensor& t, const char* op, const char* name) {
  TORCH_CHECK(is_16bit(t), op, ": ", name, " must be bf16 or fp16, got ", t.scalar_type());
}
inline void check_like(const at::Tensor& t, const at::Tensor& ref, const char* op, const char* name) {
  TORCH_CHECK(t.scalar_type() == ref.scalar_type(), op, ": ", name, " dtype ", t.scalar_type(), " differs from ", ref.scalar_type());
}
inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
inline int num_sms() {
  static int n = 0;
  if (!n) n = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  return n;
}
#define PFX_CUDA_CHECK(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    TORCH_CHECK(_e == cudaSuccess, "pfx CUDA error: ", cudaGetErrorString(_e), " at ", #expr); \
  } while (0)
#define PFX_CHECK_CUDA_CONTIG(t) TORCH_CHECK((t).is_cuda() && (t).is_contiguous(), #t " must be a contiguous CUDA tensor")

// ------------------------------------------------------------------------------- GEMM
// d[M,N] (+)= op(a) * op(b)^T.  a: [M,K] if a_kmajor else [K,M]; b: [N,K] if b_kmajor else [K,N].
at::Tensor gemm(const at::Tensor& a, const at::Tensor& b, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> out, bool a_kmajor,
                bool b_kmajor, int64_t epilogue, int64_t out_mode, int64_t config) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2, "gemm: 2-D CUDA tensors expected");
  TORCH_CHECK(a.scalar_type() == b.scalar_type() && (a.scalar_type() == at::kBFloat16 || a.scalar_type() == at::kHalf),
              "gemm: bf16/fp16 operands expected");
  TORCH_CHECK(a.stride(1) == 1 && b.stride(1) == 1, "gemm: innermost dim must be contiguous");
  const c10::cuda::CUDAGuard guard(a.device());
  const int64_t M = a_kmajor ? a.size(0) : a.size(1);
  const int64_t K = a_kmajor ? a.size(1) : a.size(0);
  const int64_t N = b_kmajor ? b.size(0) : b.size(1);
  const int64_t Kb = b_kmajor ? b.size(1) : b.size(0);
  TORCH_CHECK(K == Kb, "gemm: K mismatch ", K, " vs ", Kb);
  TORCH_CHECK(a.stride(0) % 8 == 0 && b.stride(0) % 8 == 0, "gemm: row strides must be multiples of 8 elements (16 B)");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(a.data_ptr()) % 16) == 0 && (reinterpret_cast<uintptr_t>(b.data_ptr()) % 16) == 0,
              "gemm: operands must be 16-byte aligned");
  at::Tensor d;
  if (out.has_value()) {
    d = *out;
    TORCH_CHECK(d.is_cuda() && d.dim() == 2 && d.size(0) == M && d.size(1) == N && d.stride(1) == 1, "gemm: bad out tensor");
  } else {
    TORCH_CHECK(out_mode != 2, "gemm: accumulate mode needs an out tensor");
    d = at::empty({M, N}, a.options().dtype(out_mode == 0 ? a.scalar_type() : at::kFloat));
  }
  if (out_mode == 0) {
    TORCH_CHECK(d.scalar_type() == a.scalar_type() && N % 8 == 0 && d.stride(0) % 8 == 0, "gemm: bf16 out needs N % 8 == 0");
  } else {
    TORCH_CHECK(d.scalar_type() == at::kFloat && N % 4 == 0 && d.stride(0) % 4 == 0, "gemm: fp32 out needs N % 4 == 0");
  }
  pfx::GemmArgs g{};
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr();
  g.bias = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == a.scalar_type() && bias->numel() == N && bias->is_contiguous(), "gemm: bias must be [N] of the operands' dtype (",
                a.scalar_type(), "), got ", bias->scalar_type());
    TORCH_CHECK(N % 8 == 0, "gemm: bias epilogue needs N % 8 == 0");
    g.bias = bias->data_ptr();
  } else {
    TORCH_CHECK(epilogue == pfx::EPI_NONE || epilogue == pfx::EPI_GELU, "gemm: bias epilogue without bias");
  }
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.lda = (int)a.stride(0); g.ldb = (int)b.stride(0); g.ldd = (int)d.stride(0);
  g.a_kmajor = a_kmajor; g.b_kmajor = b_kmajor;
  g.out_mode = (int)out_mode; g.epilogue = (int)epilogue;
  g.ab_format = a.scalar_type() == at::kBFloat16 ? 1 : 0;
  g.num_sms = num_sms(); g.config = (int)config;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return d;
}

// FFN1 forward in one kernel: z = x W^T + b (kept for the backward) and g = gelu(z), both written by the GEMM epilogue.
std::vector<at::Tensor> gemm_bias_gelu_dual(const at::Tensor& x, const at::Tensor& w, const at::Tensor& bias) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1), "gemm_bias_gelu_dual: x [M,K], w [N,K]");
  TORCH_CHECK(is_16bit(x) && w.scalar_type() == x.scalar_type() && bias.scalar_type() == x.scalar_type() && bias.numel() == w.size(0) &&
              bias.is_contiguous(), "gemm_bias_gelu_dual: bf16 or fp16 operands of one dtype, bias [N]");
  TORCH_CHECK(w.size(0) % 8 == 0 && x.size(1) % 8 == 0, "gemm_bias_gelu_dual: N, K multiples of 8");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor z = at::empty({x.size(0), w.size(0)}, x.options()), gl = at::empty({x.size(0), w.size(0)}, x.options());
  pfx::GemmArgs g{};
  g.a = x.data_ptr(); g.b = w.data_ptr(); g.d = z.data_ptr(); g.d2 = gl.data_ptr(); g.bias = bias.data_ptr();
  g.M = (int)x.size(0); g.N = (int)w.size(0); g.K = (int)x.size(1);
  g.lda = (int)x.stride(0); g.ldb = (int)w.stride(0); g.ldd = (int)z.stride(0);
  g.a_kmajor = true; g.b_kmajor = true; g.out_mode = 0; g.epilogue = pfx::EPI_BIAS_GELU_DUAL; g.ab_format = dtype_code(x); g.num_sms = num_sms(); g.config = 0;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return {z, gl};
}

// FFN2 dgrad with the GELU derivative applied in the epilogue: dz = (dy W) * gelu'(z);  w is [K = out_features, N = in_features].
at::Tensor gemm_dgelu(const at::Tensor& dy, const at::Tensor& w, const at::Tensor& z, int64_t config) {
  TORCH_CHECK(dy.is_cuda() && dy.dim() == 2 && w.dim() == 2 && z.dim() == 2 && dy.is_contiguous() && w.is_contiguous() && z.is_contiguous(), "gemm_dgelu: contiguous 2-D");
  TORCH_CHECK(dy.size(1) == w.size(0) && z.size(0) == dy.size(0) && z.size(1) == w.size(1), "gemm_dgelu: dy [M,K], w [K,N], z [M,N]");
  TORCH_CHECK(is_16bit(dy) && w.scalar_type() == dy.scalar_type() && z.scalar_type() == dy.scalar_type(), "gemm_dgelu: bf16 or fp16 operands of one dtype");
  TORCH_CHECK(w.size(1) % 8 == 0 && w.size(0) % 8 == 0, "gemm_dgelu: N, K multiples of 8");
  const c10::cuda::CUDAGuard guard(dy.device());
  at::Tensor dz = at::empty_like(z);
  pfx::GemmArgs g{};
  g.a = dy.data_ptr(); g.b = w.data_ptr(); g.d = dz.data_ptr(); g.aux = z.data_ptr(); g.ld_aux = (int)z.stride(0);
  g.M = (int)dy.size(0); g.N = (int)w.size(1); g.K = (int)dy.size(1);
  g.lda = (int)dy.stride(0); g.ldb = (int)w.stride(0); g.ldd = (int)dz.stride(0);
  g.a_kmajor = true; g.b_kmajor = false; g.out_mode = 0; g.epilogue = pfx::EPI_DGELU; g.ab_format = dtype_code(dy); g.num_sms = num_sms(); g.config = (int)config;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return dz;
}


// ------------------------------------------------------------------------------- fused GEMM + collectives
// GEMM -> reduce-scatter, phase 1: every tile of a*op(b)^T goes straight to the owner rank's staging slot over NVLink.
void gemm_rs_scatter(const at::Tensor& a, const at::Tensor& b, const std::vector<int64_t>& peer_staging, int64_t my_rank, int64_t rows_per_rank,
                     bool a_kmajor, bool b_kmajor, int64_t config) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm_rs: bf16 CUDA operands");
  const c10::cuda::CUDAGuard guard(a.device());
  const int64_t M = a_kmajor ? a.size(0) : a.size(1), K = a_kmajor ? a.size(1) : a.size(0), N = b_kmajor ? b.size(0) : b.size(1);
  const int world = (int)peer_staging.size();
  TORCH_CHECK(world >= 2 && world <= 8 && M == rows_per_rank * world && N % 8 == 0, "gemm_rs: bad partition");
  pfx::GemmArgs g{};
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = nullptr; g.bias = nullptr;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.lda = (int)a.stride(0); g.ldb = (int)b.stride(0); g.ldd = (int)N;
  g.a_kmajor = a_kmajor; g.b_kmajor = b_kmajor; g.out_mode = 3; g.epilogue = pfx::EPI_NONE; g.ab_format = 1;
  g.num_sms = num_sms(); g.config = (int)config;
  for (int i = 0; i < world; ++i) g.comm.peer_out[i] = reinterpret_cast<void*>((uintptr_t)peer_staging[i]);
  g.comm.rows_per_rank = (int)rows_per_rank; g.comm.my_rank = (int)my_rank; g.comm.world = world; g.comm.ag_world = 0;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
}
at::Tensor slot_reduce(const at::Tensor& staging, c10::optional<at::Tensor> bias, int64_t world) {
  PFX_CHECK_CUDA_CONTIG(staging);
  const c10::cuda::CUDAGuard guard(staging.device());
  const int64_t cols = staging.size(-1), rows = staging.numel() / cols / world;
  auto out = at::empty({rows, cols}, staging.options());
  PFX_CUDA_CHECK(pfx::slot_reduce(staging.data_ptr(), out.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr,
                                  (size_t)rows * cols, (int)world, (int)cols, dtype_code(staging), num_sms(), cur_stream()));
  return out;
}
// all-gather -> GEMM in one kernel: d[M,N] = gathered(a_local)[M,K] * b[N,K]^T (+bias).  `gathered` is this rank's symmetric
// gather buffer (peers push their shards into it), flags / peer pointers come from the symmetric allocator.
at::Tensor gemm_ag(const at::Tensor& a_local, const at::Tensor& b, const at::Tensor& gathered, const std::vector<int64_t>& peer_gather,
                   const std::vector<int64_t>& peer_flags, const at::Tensor& my_flags, c10::optional<at::Tensor> bias, int64_t my_rank,
                   int64_t chunk_rows, int64_t num_comm_ctas, int64_t epoch, bool b_kmajor, int64_t config) {
  TORCH_CHECK(a_local.is_cuda() && a_local.is_contiguous() && a_local.scalar_type() == at::kBFloat16, "gemm_ag: a_local bf16 contiguous");
  const c10::cuda::CUDAGuard guard(a_local.device());
  const int world = (int)peer_gather.size();
  const int64_t rows = a_local.size(0), K = a_local.size(1), M = rows * world, N = b_kmajor ? b.size(0) : b.size(1);
  TORCH_CHECK(gathered.size(0) == M && gathered.size(1) == K && gathered.is_contiguous(), "gemm_ag: gathered buffer shape");
  TORCH_CHECK(rows % chunk_rows == 0 && N % 8 == 0 && K % 8 == 0, "gemm_ag: bad shapes");
  auto d = at::empty({M, N}, a_local.options());
  pfx::GemmArgs g{};
  g.a = gathered.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr();
  g.bias = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.lda = (int)K; g.ldb = (int)b.stride(0); g.ldd = (int)N;
  g.a_kmajor = true; g.b_kmajor = b_kmajor; g.out_mode = 0; g.epilogue = g.bias ? pfx::EPI_BIAS : pfx::EPI_NONE; g.ab_format = 1;
  g.num_sms = num_sms(); g.config = (int)config;
  for (int i = 0; i < world; ++i) {
    g.comm.peer_gather[i] = reinterpret_cast<void*>((uintptr_t)peer_gather[i]);
    g.comm.peer_flags[i] = reinterpret_cast<uint32_t*>((uintptr_t)peer_flags[i]);
  }
  g.comm.my_flags = reinterpret_cast<const uint32_t*>(my_flags.data_ptr());
  g.comm.a_local = a_local.data_ptr();
  g.comm.rows_per_rank = (int)rows; g.comm.chunk_rows = (int)chunk_rows; g.comm.my_rank = (int)my_rank; g.comm.world = world;
  g.comm.ag_world = world; g.comm.num_comm_ctas = (int)num_comm_ctas; g.comm.epoch = (uint32_t)epoch;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return d;
}

// ------------------------------------------------------------------------------- 8-bit GEMMs
// The quantiser keeps a row in registers: cols % 8 == 0 and cols <= 32768.
std::vector<at::Tensor> quantize_rows(const at::Tensor& x, c10::optional<at::Tensor> smooth, bool fp8) {
  PFX_CHECK_CUDA_CONTIG(x);
  check_16bit(x, "quantize_rows", "x");
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t cols = x.size(-1), rows = cols ? x.numel() / cols : 0;
  TORCH_CHECK(cols % 8 == 0 && cols > 0 && cols <= 32768, "quantize_rows: x needs 8 <= cols <= 32768 with cols % 8 == 0, got ", cols);
  auto q = at::empty(x.sizes(), x.options().dtype(fp8 ? at::kFloat8_e4m3fn : at::kChar));
  auto scale = at::empty({rows}, x.options().dtype(at::kFloat));
  const float* sm = nullptr;
  at::Tensor smc;
  if (smooth.has_value() && smooth->defined()) {
    TORCH_CHECK(smooth->device() == x.device() && smooth->numel() == cols, "quantize_rows: smooth must be [", cols, "] on ", x.device(), ", got ",
                smooth->sizes(), " on ", smooth->device());
    smc = smooth->to(at::kFloat).contiguous(); sm = smc.data_ptr<float>();
  }
  PFX_CUDA_CHECK(pfx::quantize_rows(x.data_ptr(), sm, q.data_ptr(), scale.data_ptr<float>(), (int)rows, (int)cols, dtype_code(x), fp8, cur_stream()));
  return {q, scale};
}
// out_dtype: bf16 (default) or fp16; bias must have the output dtype.
at::Tensor gemm_lowp(const at::Tensor& a, const at::Tensor& b, c10::optional<at::Tensor> row_scale, c10::optional<at::Tensor> col_scale,
                     c10::optional<at::Tensor> bias, int64_t config, c10::optional<at::ScalarType> out_dtype) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous(), "gemm_lowp: contiguous 2-D CUDA operands");
  TORCH_CHECK(a.scalar_type() == b.scalar_type() && (a.scalar_type() == at::kChar || a.scalar_type() == at::kFloat8_e4m3fn), "gemm_lowp: int8 or fp8-e4m3 operands");
  const c10::cuda::CUDAGuard guard(a.device());
  const int64_t M = a.size(0), K = a.size(1), N = b.size(0);
  TORCH_CHECK(b.size(1) == K && K % 16 == 0 && N % 8 == 0, "gemm_lowp: K % 16 == 0 and N % 8 == 0 required");
  const at::ScalarType od = out_dtype.value_or(at::kBFloat16);
  TORCH_CHECK(od == at::kBFloat16 || od == at::kHalf, "gemm_lowp: out_dtype must be bf16 or fp16, got ", od);
  auto d = at::empty({M, N}, a.options().dtype(od));
  pfx::LowpGemmArgs g{};
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr(); g.out_fp16 = od == at::kHalf;
  at::Tensor rs, cs;
  if (row_scale.has_value() && row_scale->defined()) { rs = row_scale->to(at::kFloat).contiguous(); TORCH_CHECK(rs.numel() == M); g.row_scale = rs.data_ptr<float>(); }
  if (col_scale.has_value() && col_scale->defined()) { cs = col_scale->to(at::kFloat).contiguous(); TORCH_CHECK(cs.numel() == N); g.col_scale = cs.data_ptr<float>(); }
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->scalar_type() == od && bias->numel() == N, "gemm_lowp: bias must be a contiguous [",
                N, "] CUDA tensor of the output dtype ", od, ", got ", bias->scalar_type(), " ", bias->sizes());
    g.bias = bias->data_ptr();
  }
  g.M = (int)M; g.N = (int)N; g.K = (int)K; g.lda = (int)K; g.ldb = (int)K; g.ldd = (int)N;
  g.kind = a.scalar_type() == at::kChar ? 1 : 2;
  g.num_sms = num_sms(); g.config = (int)config;
  PFX_CUDA_CHECK(pfx::gemm_lowp_wgmma(g, cur_stream()));
  return d;
}

// MX block-scaled fp8: quantiser and GEMM.  quantize_mxfp8(x [R, K]) -> (q e4m3 [R, K], sf uint8 [ceil(R / 128), K / 128, 512])
std::vector<at::Tensor> quantize_mxfp8(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && x.size(1) % 128 == 0, "quantize_mxfp8: contiguous [R, K], K % 128 == 0");
  check_16bit(x, "quantize_mxfp8", "x");
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t R = x.size(0), K = x.size(1);
  at::Tensor q = at::empty({R, K}, x.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor sf = at::zeros({(R + 127) / 128, K / 128, 512}, x.options().dtype(at::kByte));
  PFX_CUDA_CHECK(pfx::quantize_mxfp8(x.data_ptr(), q.data_ptr(), sf.data_ptr(), (int)R, (int)K, dtype_code(x), cur_stream()));
  return {q, sf};
}
// d [M, N] bf16 = (A_q * 2^(sfa - 127)) (B_q * 2^(sfb - 127))^T (+ bias): each K = 32 partial product is scaled by its two block scales and
// summed in fp32 registers (Hopper's tensor core has no block-scale mode)
at::Tensor gemm_mxfp8(const at::Tensor& a, const at::Tensor& sfa, const at::Tensor& b, const at::Tensor& sfb, c10::optional<at::Tensor> bias) {
  TORCH_CHECK(a.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous() && a.scalar_type() == at::kFloat8_e4m3fn &&
              b.scalar_type() == at::kFloat8_e4m3fn, "gemm_mxfp8: contiguous e4m3 operands");
  const int64_t M = a.size(0), K = a.size(1), N = b.size(0);
  TORCH_CHECK(b.size(1) == K && K % 128 == 0 && N % 8 == 0, "gemm_mxfp8: K % 128 == 0, N % 8 == 0");
  TORCH_CHECK(sfa.scalar_type() == at::kByte && sfb.scalar_type() == at::kByte && sfa.is_contiguous() && sfb.is_contiguous() &&
              sfa.numel() == ((M + 127) / 128) * (K / 128) * 512 && sfb.numel() == ((N + 127) / 128) * (K / 128) * 512, "gemm_mxfp8: scale tensors");
  const c10::cuda::CUDAGuard guard(a.device());
  auto d = at::empty({M, N}, a.options().dtype(at::kBFloat16));
  pfx::LowpGemmArgs g{};
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr(); g.sfa = sfa.data_ptr(); g.sfb = sfb.data_ptr();
  if (bias.has_value() && bias->defined()) { TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N); g.bias = bias->data_ptr(); }
  g.M = (int)M; g.N = (int)N; g.K = (int)K; g.lda = (int)K; g.ldb = (int)K; g.ldd = (int)N;
  g.kind = 3; g.num_sms = num_sms(); g.config = 0;
  PFX_CUDA_CHECK(pfx::gemm_lowp_wgmma(g, cur_stream()));
  return d;
}

// ------------------------------------------------------------------------------- norms
std::vector<at::Tensor> norm_fwd(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> b, double eps, bool rms) {
  PFX_CHECK_CUDA_CONTIG(x); PFX_CHECK_CUDA_CONTIG(w);
  check_16bit(x, "norm_fwd", "x");
  const int64_t cols = x.size(-1), rows = x.numel() / cols;
  TORCH_CHECK(cols % 8 == 0 && cols <= 32768, "norm_fwd: the row length must be a multiple of 8 and at most 32768, got ", cols);
  check_like(w, x, "norm_fwd", "w");
  TORCH_CHECK(w.numel() == cols, "norm_fwd: w has ", w.numel(), " elements for rows of ", cols);
  if (b.has_value() && b->defined()) {
    PFX_CHECK_CUDA_CONTIG(*b);
    check_like(*b, x, "norm_fwd", "b");
    TORCH_CHECK(b->numel() == cols, "norm_fwd: b has ", b->numel(), " elements for rows of ", cols);
  }
  const c10::cuda::CUDAGuard guard(x.device());
  auto y = at::empty_like(x);
  auto fopt = x.options().dtype(at::kFloat);
  auto mean = rms ? at::empty({0}, fopt) : at::empty({rows}, fopt);
  auto rstd = at::empty({rows}, fopt);
  PFX_CUDA_CHECK(pfx::norm_fwd(x.data_ptr(), w.data_ptr(), (b.has_value() && b->defined()) ? b->data_ptr() : nullptr, y.data_ptr(),
                               rms ? nullptr : mean.data_ptr<float>(), rstd.data_ptr<float>(), (int)rows, (int)cols, (float)eps,
                               dtype_code(x), rms, cur_stream()));
  return {y, mean, rstd};
}

std::vector<at::Tensor> norm_bwd(const at::Tensor& dy, const at::Tensor& x, const at::Tensor& w, const at::Tensor& mean,
                                 const at::Tensor& rstd, bool rms, bool has_bias, c10::optional<at::Tensor> dres) {
  // dres: gradient of the residual branch that bypasses the norm (pre-norm block): dx = norm_bwd(dy) + dres in the same pass
  PFX_CHECK_CUDA_CONTIG(dy); PFX_CHECK_CUDA_CONTIG(x); PFX_CHECK_CUDA_CONTIG(w);
  check_16bit(x, "norm_bwd", "x");
  check_like(dy, x, "norm_bwd", "dy");
  check_like(w, x, "norm_bwd", "w");
  TORCH_CHECK(dy.sizes() == x.sizes(), "norm_bwd: dy shape ", dy.sizes(), " differs from x ", x.sizes());
  TORCH_CHECK(x.size(-1) % 8 == 0 && x.size(-1) <= 32768, "norm_bwd: the row length must be a multiple of 8 and at most 32768, got ",
              x.size(-1));
  TORCH_CHECK(w.numel() == x.size(-1), "norm_bwd: w has ", w.numel(), " elements for rows of ", x.size(-1));
  const bool with_res = dres.has_value() && dres->defined();
  if (with_res) TORCH_CHECK(dres->is_contiguous() && dres->sizes() == x.sizes() && dres->scalar_type() == x.scalar_type(), "norm_bwd: dres");
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t cols = x.size(-1), rows = x.numel() / cols;
  auto dx = at::empty_like(x);
  auto dw = at::empty_like(w);
  auto db = (has_bias && !rms) ? at::empty_like(w) : at::empty({0}, w.options());
  const int parts = pfx::norm_bwd_num_parts((int)rows, num_sms());
  auto ws = at::empty({2 * (int64_t)parts * cols}, x.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::norm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), rms ? nullptr : mean.data_ptr<float>(), rstd.data_ptr<float>(),
                               dx.data_ptr(), dw.data_ptr(), (has_bias && !rms) ? db.data_ptr() : nullptr, ws.data_ptr<float>(), (int)rows,
                               (int)cols, dtype_code(x), rms, num_sms(), cur_stream(), with_res ? dres->data_ptr() : nullptr));
  return {dx, dw, db};
}

// ------------------------------------------------------------------------------- activations / dropout
static void check_same_dtype(const at::Tensor& x, const c10::optional<at::Tensor>& t, const char* what) {
  if (t.has_value() && t->defined())
    TORCH_CHECK(t->scalar_type() == x.scalar_type(), what, ": operand dtype ", t->scalar_type(), " differs from activation dtype ", x.scalar_type());
}
at::Tensor bias_gelu_fwd(const at::Tensor& x, c10::optional<at::Tensor> bias, bool exact) {
  PFX_CHECK_CUDA_CONTIG(x);
  check_16bit(x, "bias_gelu", "x");
  check_same_dtype(x, bias, "bias_gelu");
  const c10::cuda::CUDAGuard guard(x.device());
  auto y = at::empty_like(x);
  const int64_t cols = x.size(-1);
  PFX_CUDA_CHECK(pfx::bias_gelu(x.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr, nullptr, y.data_ptr(),
                                x.numel() / cols, (int)cols, dtype_code(x), false, num_sms(), cur_stream(), exact));
  return y;
}
at::Tensor bias_gelu_bwd(const at::Tensor& dy, const at::Tensor& x, c10::optional<at::Tensor> bias, bool exact) {
  PFX_CHECK_CUDA_CONTIG(x); PFX_CHECK_CUDA_CONTIG(dy);
  check_16bit(x, "bias_gelu_bwd", "x");
  check_same_dtype(x, bias, "bias_gelu_bwd");
  TORCH_CHECK(dy.scalar_type() == x.scalar_type(), "bias_gelu_bwd: dy dtype");
  const c10::cuda::CUDAGuard guard(x.device());
  auto dx = at::empty_like(x);
  const int64_t cols = x.size(-1);
  PFX_CUDA_CHECK(pfx::bias_gelu(x.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr, dy.data_ptr(),
                                dx.data_ptr(), x.numel() / cols, (int)cols, dtype_code(x), true, num_sms(), cur_stream(), exact));
  return dx;
}
// SwiGLU over pair-interleaved z [.., 2F] (column 2i gate channel i, 2i + 1 its up channel) -> h [.., F]
at::Tensor bias_swiglu_fwd(const at::Tensor& z, c10::optional<at::Tensor> bias) {
  PFX_CHECK_CUDA_CONTIG(z);
  check_16bit(z, "bias_swiglu", "z");
  check_same_dtype(z, bias, "bias_swiglu");
  const int64_t cols = z.size(-1);
  TORCH_CHECK(cols % 16 == 0, "bias_swiglu: z needs 2F columns with F % 8 == 0, got ", cols);
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->is_contiguous() && bias->numel() == cols, "bias_swiglu: bias has ", bias->numel(), " elements for rows of ", cols);
  const c10::cuda::CUDAGuard guard(z.device());
  auto sizes = z.sizes().vec();
  sizes.back() = cols / 2;
  auto h = at::empty(sizes, z.options());
  PFX_CUDA_CHECK(pfx::bias_swiglu(z.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr, nullptr, h.data_ptr(),
                                  z.numel() / cols, (int)(cols / 2), dtype_code(z), false, num_sms(), cur_stream()));
  return h;
}
at::Tensor bias_swiglu_bwd(const at::Tensor& dh, const at::Tensor& z, c10::optional<at::Tensor> bias) {
  PFX_CHECK_CUDA_CONTIG(z); PFX_CHECK_CUDA_CONTIG(dh);
  check_16bit(z, "bias_swiglu_bwd", "z");
  check_same_dtype(z, bias, "bias_swiglu_bwd");
  check_like(dh, z, "bias_swiglu_bwd", "dh");
  const int64_t cols = z.size(-1);
  TORCH_CHECK(cols % 16 == 0, "bias_swiglu_bwd: z needs 2F columns with F % 8 == 0, got ", cols);
  TORCH_CHECK(dh.dim() == z.dim() && dh.size(-1) * 2 == cols && dh.numel() * 2 == z.numel(), "bias_swiglu_bwd: dh ", dh.sizes(),
              " does not match z ", z.sizes());
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->is_contiguous() && bias->numel() == cols, "bias_swiglu_bwd: bias has ", bias->numel(), " elements for rows of ", cols);
  const c10::cuda::CUDAGuard guard(z.device());
  auto dz = at::empty_like(z);
  PFX_CUDA_CHECK(pfx::bias_swiglu(z.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr, dh.data_ptr(),
                                  dz.data_ptr(), z.numel() / cols, (int)(cols / 2), dtype_code(z), true, num_sms(), cur_stream()));
  return dz;
}
at::Tensor bias_dropout_add_fwd(const at::Tensor& x, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> residual, double p,
                                int64_t seed, int64_t offset) {
  PFX_CHECK_CUDA_CONTIG(x);
  check_16bit(x, "bias_dropout_add", "x");
  check_same_dtype(x, bias, "bias_dropout_add");
  check_same_dtype(x, residual, "bias_dropout_add");
  const c10::cuda::CUDAGuard guard(x.device());
  auto y = at::empty_like(x);
  const int64_t cols = x.size(-1);
  if (residual.has_value() && residual->defined()) PFX_CHECK_CUDA_CONTIG(*residual);
  PFX_CUDA_CHECK(pfx::bias_dropout_add(x.data_ptr(), (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr,
                                       (residual.has_value() && residual->defined()) ? residual->data_ptr() : nullptr, y.data_ptr(),
                                       x.numel() / cols, (int)cols, (float)p, (uint64_t)seed, (uint64_t)offset, dtype_code(x), false,
                                       num_sms(), cur_stream()));
  return y;
}
at::Tensor dropout_bwd(const at::Tensor& dy, double p, int64_t seed, int64_t offset) {
  PFX_CHECK_CUDA_CONTIG(dy);
  check_16bit(dy, "dropout_bwd", "dy");
  const c10::cuda::CUDAGuard guard(dy.device());
  auto dx = at::empty_like(dy);
  const int64_t cols = dy.size(-1);
  PFX_CUDA_CHECK(pfx::bias_dropout_add(dy.data_ptr(), nullptr, nullptr, dx.data_ptr(), dy.numel() / cols, (int)cols, (float)p,
                                       (uint64_t)seed, (uint64_t)offset, dtype_code(dy), true, num_sms(), cur_stream()));
  return dx;
}
at::Tensor colsum(const at::Tensor& x, bool out_fp32) {
  PFX_CHECK_CUDA_CONTIG(x);
  check_16bit(x, "colsum", "x");
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t cols = x.size(-1), rows = x.numel() / cols;
  auto out = at::empty({cols}, x.options().dtype(out_fp32 ? at::kFloat : x.scalar_type()));
  auto ws = at::empty({(int64_t)pfx::colsum_num_parts((int)rows) * cols}, x.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::colsum(x.data_ptr(), out.data_ptr(), ws.data_ptr<float>(), (int)rows, (int)cols, dtype_code(x), out_fp32, cur_stream()));
  return out;
}

// ------------------------------------------------------------------------------- loss
std::vector<at::Tensor> ce_stats(const at::Tensor& logits, const at::Tensor& labels, int64_t vocab_start) {
  PFX_CHECK_CUDA_CONTIG(logits); PFX_CHECK_CUDA_CONTIG(labels);
  check_16bit(logits, "ce_stats", "logits");
  TORCH_CHECK(labels.scalar_type() == at::kLong, "labels must be int64");
  const c10::cuda::CUDAGuard guard(logits.device());
  const int64_t cols = logits.size(-1), rows = logits.numel() / cols;
  TORCH_CHECK(labels.numel() == rows, "ce_stats: ", labels.numel(), " labels for ", rows, " rows");
  auto fopt = logits.options().dtype(at::kFloat);
  auto mx = at::empty({rows}, fopt), sm = at::empty({rows}, fopt), tg = at::empty({rows}, fopt);
  PFX_CUDA_CHECK(pfx::ce_stats(logits.data_ptr(), labels.data_ptr<int64_t>(), mx.data_ptr<float>(), sm.data_ptr<float>(),
                               tg.data_ptr<float>(), (int)rows, (int)cols, vocab_start, dtype_code(logits), cur_stream()));
  return {mx, sm, tg};
}
void ce_bwd_(at::Tensor& logits, const at::Tensor& labels, const at::Tensor& lse, const at::Tensor& gscale, int64_t vocab_start) {
  PFX_CHECK_CUDA_CONTIG(logits); PFX_CHECK_CUDA_CONTIG(labels); PFX_CHECK_CUDA_CONTIG(lse); PFX_CHECK_CUDA_CONTIG(gscale);
  check_16bit(logits, "ce_bwd_", "logits");
  const c10::cuda::CUDAGuard guard(logits.device());
  const int64_t cols = logits.size(-1), rows = logits.numel() / cols;
  TORCH_CHECK(labels.scalar_type() == at::kLong && labels.numel() == rows, "ce_bwd_: labels must be int64 with one entry per row");
  TORCH_CHECK(lse.scalar_type() == at::kFloat && gscale.scalar_type() == at::kFloat && lse.numel() == rows && gscale.numel() == rows);
  PFX_CUDA_CHECK(pfx::ce_bwd(logits.data_ptr(), labels.data_ptr<int64_t>(), lse.data_ptr<float>(), gscale.data_ptr<float>(), (int)rows,
                             (int)cols, vocab_start, dtype_code(logits), cur_stream()));
}

// ------------------------------------------------------------------------------- optimizer
void sumsq_(const at::Tensor& x, at::Tensor& out, bool accumulate) {
  PFX_CHECK_CUDA_CONTIG(x);
  const c10::cuda::CUDAGuard guard(x.device());
  auto ws = at::empty({1024}, x.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::sumsq(x.data_ptr(), (size_t)x.numel(), out.data_ptr<float>(), ws.data_ptr<float>(), dtype_code(x), accumulate,
                            num_sms(), cur_stream()));
}
void clip_coef_(const at::Tensor& sq, double inv_loss_scale, double clip_norm, at::Tensor& gscale, at::Tensor& found_inf, at::Tensor& gnorm) {
  const c10::cuda::CUDAGuard guard(sq.device());
  PFX_CUDA_CHECK(pfx::clip_coef(sq.data_ptr<float>(), (float)inv_loss_scale, (float)clip_norm, gscale.data_ptr<float>(),
                                found_inf.data_ptr<float>(), gnorm.data_ptr<float>(), cur_stream()));
}
void adamw_flat_(c10::optional<at::Tensor> p_lp, at::Tensor& master, const at::Tensor& grad, at::Tensor& m, at::Tensor& v, double lr,
                 double beta1, double beta2, double eps, double wd, int64_t step, c10::optional<at::Tensor> gscale,
                 c10::optional<at::Tensor> found_inf, int64_t cta_budget) {
  // cta_budget > 0: grid size cap (the kernel is launched with cta_budget CTAs instead of 8 per SM) — used when the update runs on a side
  // stream underneath GEMMs and must not take the whole memory system
  PFX_CHECK_CUDA_CONTIG(master); PFX_CHECK_CUDA_CONTIG(grad); PFX_CHECK_CUDA_CONTIG(m); PFX_CHECK_CUDA_CONTIG(v);
  const c10::cuda::CUDAGuard guard(master.device());
  const size_t n = master.numel();
  TORCH_CHECK((size_t)grad.numel() == n && (size_t)m.numel() == n && (size_t)v.numel() == n, "adamw: size mismatch");
  const float bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  const bool has_lp = p_lp.has_value() && p_lp->defined();
  if (has_lp) {
    PFX_CHECK_CUDA_CONTIG(*p_lp);
    TORCH_CHECK((size_t)p_lp->numel() == n, "adamw: p_lp has ", p_lp->numel(), " elements, master has ", n);
    TORCH_CHECK(!is_16bit(grad) || !is_16bit(*p_lp) || p_lp->scalar_type() == grad.scalar_type(), "adamw: a ", grad.scalar_type(),
                " grad needs p_lp of the same dtype or fp32, got ", p_lp->scalar_type());
  }
  PFX_CUDA_CHECK(pfx::adamw_flat(has_lp ? p_lp->data_ptr() : nullptr, master.data_ptr<float>(), grad.data_ptr(), m.data_ptr<float>(),
                                 v.data_ptr<float>(), n, (float)lr, (float)beta1, (float)beta2, (float)eps, (float)wd, bc1, bc2,
                                 (gscale.has_value() && gscale->defined()) ? gscale->data_ptr<float>() : nullptr,
                                 (found_inf.has_value() && found_inf->defined()) ? found_inf->data_ptr<float>() : nullptr,
                                 dtype_code(grad), has_lp ? dtype_code(*p_lp) : 3, cta_budget > 0 ? (int)((cta_budget + 7) / 8) : num_sms(), cur_stream()));
}
void accumulate_f32_(at::Tensor& dst, const at::Tensor& src, double scale) {
  const c10::cuda::CUDAGuard guard(dst.device());
  TORCH_CHECK(dst.scalar_type() == at::kFloat && dst.numel() == src.numel() && dst.is_contiguous() && src.is_contiguous());
  PFX_CUDA_CHECK(pfx::accumulate_f32(dst.data_ptr<float>(), src.data_ptr(), (size_t)src.numel(), (float)scale, dtype_code(src), num_sms(),
                                     cur_stream()));
}

// ------------------------------------------------------------------------------- sampling / rope / softmax
std::vector<at::Tensor> topp_sampling(const at::Tensor& probs, const at::Tensor& top_ps, int64_t seed, int64_t offset) {
  PFX_CHECK_CUDA_CONTIG(probs);
  const c10::cuda::CUDAGuard guard(probs.device());
  const int64_t V = probs.size(-1), rows = probs.numel() / V;
  auto tp = top_ps.to(at::kFloat).contiguous();
  TORCH_CHECK(tp.numel() == rows, "top_ps must have one entry per row");
  auto out_p = at::empty({rows, 1}, probs.options().dtype(at::kFloat));
  auto out_i = at::empty({rows, 1}, probs.options().dtype(at::kLong));
  PFX_CUDA_CHECK(pfx::topp_sampling(probs.data_ptr(), tp.data_ptr<float>(), out_p.data_ptr<float>(), out_i.data_ptr<int64_t>(), (int)rows,
                                    (int)V, (uint64_t)seed, (uint64_t)offset, dtype_code(probs), cur_stream()));
  return {out_p.to(probs.scalar_type()), out_i};
}
at::Tensor rope(const at::Tensor& x, c10::optional<at::Tensor> positions, int64_t seq_len, double base, bool bwd) {
  PFX_CHECK_CUDA_CONTIG(x);
  TORCH_CHECK(x.dim() >= 3, "rope: [..., heads, d]");
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t d = x.size(-1), heads = x.size(-2), tokens = x.numel() / (d * heads);
  TORCH_CHECK(d % 2 == 0, "rope: head dim must be even, got ", d);
  auto y = at::empty_like(x);
  const int64_t* pos = nullptr;
  at::Tensor pc;
  if (positions.has_value() && positions->defined()) {
    pc = positions->to(at::kLong).contiguous();
    TORCH_CHECK(pc.numel() == tokens, "rope: ", pc.numel(), " positions for ", tokens, " tokens");
    pos = pc.data_ptr<int64_t>();
  }
  PFX_CUDA_CHECK(pfx::rope(x.data_ptr(), y.data_ptr(), pos, (size_t)tokens, (int)heads, (int)d, (int)seq_len, (float)base, bwd,
                           dtype_code(x), num_sms(), cur_stream()));
  return y;
}
at::Tensor causal_softmax_fwd(const at::Tensor& x, double scale) {
  PFX_CHECK_CUDA_CONTIG(x);
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t sk = x.size(-1), sq = x.size(-2), batch = x.numel() / (sk * sq);
  auto y = at::empty_like(x);
  PFX_CUDA_CHECK(pfx::causal_softmax(x.data_ptr(), nullptr, y.data_ptr(), (size_t)batch, (int)sq, (int)sk, (float)scale, false,
                                     dtype_code(x), cur_stream()));
  return y;
}
at::Tensor causal_softmax_bwd(const at::Tensor& dy, const at::Tensor& y, double scale) {
  PFX_CHECK_CUDA_CONTIG(dy); PFX_CHECK_CUDA_CONTIG(y);
  check_like(dy, y, "causal_softmax_bwd", "dy");
  TORCH_CHECK(dy.sizes() == y.sizes(), "causal_softmax_bwd: dy shape ", dy.sizes(), " differs from y ", y.sizes());
  const c10::cuda::CUDAGuard guard(y.device());
  const int64_t sk = y.size(-1), sq = y.size(-2), batch = y.numel() / (sk * sq);
  auto dx = at::empty_like(y);
  PFX_CUDA_CHECK(pfx::causal_softmax(dy.data_ptr(), y.data_ptr(), dx.data_ptr(), (size_t)batch, (int)sq, (int)sk, (float)scale, true,
                                     dtype_code(y), cur_stream()));
  return dx;
}

// ------------------------------------------------------------------------------- symmetric memory (CUDA IPC)
// Buffers are raw cudaMalloc allocations (the caching allocator's blocks cannot be IPC-exported piecewise).
py::tuple ipc_alloc(int64_t nbytes) {
  void* p = nullptr;
  PFX_CUDA_CHECK(cudaMalloc(&p, (size_t)nbytes));
  PFX_CUDA_CHECK(cudaMemset(p, 0, (size_t)nbytes));
  cudaIpcMemHandle_t h;
  PFX_CUDA_CHECK(cudaIpcGetMemHandle(&h, p));
  return py::make_tuple((int64_t) reinterpret_cast<uintptr_t>(p), py::bytes(reinterpret_cast<const char*>(&h), sizeof(h)));
}
int64_t ipc_open(const std::string& handle) {
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle.data(), sizeof(h));
  void* p = nullptr;
  PFX_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return (int64_t) reinterpret_cast<uintptr_t>(p);
}
void ipc_close(int64_t ptr) { cudaIpcCloseMemHandle(reinterpret_cast<void*>((uintptr_t)ptr)); }
void ipc_free(int64_t ptr) { cudaFree(reinterpret_cast<void*>((uintptr_t)ptr)); }
at::Tensor tensor_from_ptr(int64_t ptr, std::vector<int64_t> sizes, at::ScalarType dtype, int64_t device) {
  auto opts = at::TensorOptions().dtype(dtype).device(at::kCUDA, (c10::DeviceIndex)device);
  return at::from_blob(reinterpret_cast<void*>((uintptr_t)ptr), sizes, [](void*) {}, opts);
}

static std::vector<void*> to_ptrs(const std::vector<int64_t>& v) {
  std::vector<void*> out;
  for (auto x : v) out.push_back(reinterpret_cast<void*>((uintptr_t)x));
  return out;
}
void p2p_barrier(const std::vector<int64_t>& pads, int64_t rank, int64_t slot) {
  auto pp = to_ptrs(pads);
  PFX_CUDA_CHECK(pfx::p2p_barrier(reinterpret_cast<uint32_t**>(pp.data()), (int)rank, (int)pads.size(), (uint32_t)slot, cur_stream()));
}
void p2p_reduce_scatter(const std::vector<int64_t>& peer_bufs, at::Tensor& out, int64_t rank, int64_t in_dtype, bool accumulate,
                        double scale, int64_t num_ctas) {
  auto pp = to_ptrs(peer_bufs);
  PFX_CUDA_CHECK(pfx::p2p_reduce_scatter(pp.data(), out.data_ptr(), (size_t)out.numel(), (int)rank, (int)peer_bufs.size(), (int)in_dtype,
                                         dtype_code(out), accumulate, (float)scale, (int)num_ctas, cur_stream()));
}
void p2p_all_gather(const std::vector<int64_t>& peer_bufs, const at::Tensor& src, int64_t rank, int64_t num_ctas) {
  auto pp = to_ptrs(peer_bufs);
  PFX_CUDA_CHECK(pfx::p2p_all_gather(pp.data(), src.data_ptr(), (size_t)src.numel(), (int)rank, (int)peer_bufs.size(), dtype_code(src),
                                     (int)num_ctas, cur_stream()));
}
void adamw_p2p_broadcast_(const std::vector<int64_t>& peer_param_bufs, int64_t shard_offset, at::Tensor& master, const at::Tensor& grad,
                          at::Tensor& m, at::Tensor& v, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                          c10::optional<at::Tensor> gscale, c10::optional<at::Tensor> found_inf, int64_t lp_dtype, int64_t num_ctas) {
  auto pp = to_ptrs(peer_param_bufs);
  const float bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  PFX_CUDA_CHECK(pfx::adamw_p2p_broadcast(pp.data(), (size_t)shard_offset, master.data_ptr<float>(), grad.data_ptr(), m.data_ptr<float>(),
                                          v.data_ptr<float>(), (size_t)master.numel(), (float)lr, (float)beta1, (float)beta2, (float)eps,
                                          (float)wd, bc1, bc2,
                                          (gscale.has_value() && gscale->defined()) ? gscale->data_ptr<float>() : nullptr,
                                          (found_inf.has_value() && found_inf->defined()) ? found_inf->data_ptr<float>() : nullptr,
                                          dtype_code(grad), (int)lp_dtype, (int)peer_param_bufs.size(), (int)num_ctas, cur_stream()));
}

// ------------------------------------------------------------------------------- symmetric memory (cuMem VMM + multicast)
py::dict vmm_caps() {
  const pfx::vmm::Caps c = pfx::vmm::query_caps();
  py::dict d;
  d["vmm"] = c.vmm; d["fd_export"] = c.fd_export; d["multicast"] = c.multicast; d["granularity"] = (int64_t)c.granularity;
  return d;
}
int64_t vmm_mc_granularity(int64_t world, int64_t bytes, bool recommended) {
  return (int64_t)pfx::vmm::multicast_granularity((int)world, (size_t)bytes, recommended);
}
py::tuple vmm_arena_alloc(int64_t bytes) {
  int64_t ptr = 0; int fd = -1; std::string err;
  TORCH_CHECK(pfx::vmm::arena_alloc((size_t)bytes, &ptr, &fd, &err), "pfx vmm: ", err);
  return py::make_tuple(ptr, (int64_t)fd);
}
int64_t vmm_arena_import(int64_t fd, int64_t bytes) {
  int64_t ptr = 0; std::string err;
  TORCH_CHECK(pfx::vmm::arena_import((int)fd, (size_t)bytes, &ptr, &err), "pfx vmm: ", err);
  return ptr;
}
py::tuple vmm_mc_create(int64_t bytes, int64_t world) {
  int64_t id = 0; int fd = -1; std::string err;
  TORCH_CHECK(pfx::vmm::mc_create((size_t)bytes, (int)world, &id, &fd, &err), "pfx vmm: ", err);
  return py::make_tuple(id, (int64_t)fd);
}
int64_t vmm_mc_import(int64_t fd) {
  int64_t id = 0; std::string err;
  TORCH_CHECK(pfx::vmm::mc_import((int)fd, &id, &err), "pfx vmm: ", err);
  return id;
}
void vmm_mc_add_device(int64_t id) {
  std::string err;
  TORCH_CHECK(pfx::vmm::mc_add_device(id, &err), "pfx vmm: ", err);
}
int64_t vmm_mc_bind_and_map(int64_t id, int64_t arena_ptr, int64_t bytes) {
  int64_t ptr = 0; std::string err;
  TORCH_CHECK(pfx::vmm::mc_bind_and_map(id, arena_ptr, (size_t)bytes, &ptr, &err), "pfx vmm: ", err);
  return ptr;
}
void vmm_unmap(int64_t ptr) { pfx::vmm::unmap(ptr); }

static std::vector<void*> to_ptrs2(const std::vector<int64_t>& v) {
  std::vector<void*> out;
  for (auto x : v) out.push_back(reinterpret_cast<void*>((uintptr_t)x));
  return out;
}
void nvls_barrier(int64_t mc_flag, int64_t local_flag, int64_t target) {
  PFX_CUDA_CHECK(pfx::nvls_barrier(reinterpret_cast<uint32_t*>((uintptr_t)mc_flag), reinterpret_cast<uint32_t*>((uintptr_t)local_flag),
                                   (uint32_t)target, cur_stream()));
}
void p2p_flag_barrier(const std::vector<int64_t>& peer_flags, int64_t rank, int64_t epoch) {
  auto pp = to_ptrs2(peer_flags);
  PFX_CUDA_CHECK(pfx::p2p_flag_barrier(reinterpret_cast<uint32_t**>(pp.data()), (int)rank, (int)pp.size(), (uint32_t)epoch, cur_stream()));
}
// out = scale * sum over ranks of bucket[shard_offset : shard_offset + out.numel()]; mc_src = 0 selects the unicast pull
void symm_reduce_scatter(int64_t mc_src, const std::vector<int64_t>& peer_src, int64_t shard_offset, at::Tensor& out, int64_t rank, int64_t in_dtype,
                         double scale, bool accumulate, c10::optional<at::Tensor> sumsq, int64_t num_ctas) {
  auto pp = to_ptrs2(peer_src);
  float* sq = (sumsq.has_value() && sumsq->defined()) ? sumsq->data_ptr<float>() : nullptr;
  PFX_CUDA_CHECK(pfx::symm_reduce_scatter(reinterpret_cast<const void*>((uintptr_t)mc_src), pp.empty() ? nullptr : pp.data(), (size_t)shard_offset,
                                          out.data_ptr(), (size_t)out.numel(), (int)rank, (int)pp.size(), (int)in_dtype, dtype_code(out),
                                          (float)scale, accumulate, sq, (int)num_ctas, cur_stream()));
}
void symm_all_gather(int64_t mc_dst, const std::vector<int64_t>& peer_dst, int64_t dst_offset_bytes, const at::Tensor& src, int64_t rank,
                     int64_t num_ctas) {
  auto pp = to_ptrs2(peer_dst);
  PFX_CUDA_CHECK(pfx::symm_all_gather(reinterpret_cast<void*>((uintptr_t)mc_dst), pp.empty() ? nullptr : pp.data(), (size_t)dst_offset_bytes,
                                      src.data_ptr(), (size_t)src.numel() * src.element_size(), (int)rank, (int)pp.size(), (int)num_ctas, cur_stream()));
}
void adamw_symm_broadcast_(int64_t mc_params, const std::vector<int64_t>& peer_params, int64_t shard_offset, at::Tensor& master, const at::Tensor& grad,
                           at::Tensor& m, at::Tensor& v, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                           c10::optional<at::Tensor> gscale, c10::optional<at::Tensor> found_inf, int64_t lp_dtype, int64_t rank, int64_t num_ctas) {
  auto pp = to_ptrs2(peer_params);
  const float bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  PFX_CUDA_CHECK(pfx::adamw_symm_broadcast(reinterpret_cast<void*>((uintptr_t)mc_params), pp.empty() ? nullptr : pp.data(), (size_t)shard_offset,
                                           master.data_ptr<float>(), grad.data_ptr(), m.data_ptr<float>(), v.data_ptr<float>(), (size_t)master.numel(),
                                           (float)lr, (float)beta1, (float)beta2, (float)eps, (float)wd, bc1, bc2,
                                           (gscale.has_value() && gscale->defined()) ? gscale->data_ptr<float>() : nullptr,
                                           (found_inf.has_value() && found_inf->defined()) ? found_inf->data_ptr<float>() : nullptr,
                                           dtype_code(grad), (int)lp_dtype, (int)rank, (int)pp.size(), (int)num_ctas, cur_stream()));
}

at::Tensor gemv_skinny(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1), "gemv_skinny: x [M,K], w [N,K]");
  TORCH_CHECK(x.scalar_type() == w.scalar_type(), "gemv_skinny: dtype mismatch");
  at::Tensor y = at::empty({x.size(0), w.size(0)}, x.options());
  const void* b = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  PFX_CUDA_CHECK(pfx::gemv_skinny(x.data_ptr(), w.data_ptr(), b, y.data_ptr(), (int)x.size(0), (int)w.size(0), (int)x.size(1), dtype_code(x),
                                  at::cuda::getCurrentDeviceProperties()->multiProcessorCount, cur_stream()));
  return y;
}

at::Tensor gemv_fused(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> ln_w,
                      c10::optional<at::Tensor> ln_b, double ln_eps, c10::optional<at::Tensor> residual, int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1), "gemv_fused: x [M,K], w [N,K]");
  TORCH_CHECK(x.scalar_type() == w.scalar_type(), "gemv_fused: dtype mismatch");
  TORCH_CHECK(act >= 0 && act <= 2, "gemv_fused: act must be 0 (none), 1 (GELU) or 2 (SwiGLU), got ", act);
  TORCH_CHECK(act != 2 || w.size(0) % 2 == 0, "gemv_fused: SwiGLU needs an even number of weight rows (gate, up pairs), got ", w.size(0));
  at::Tensor y = at::empty({x.size(0), act == 2 ? w.size(0) / 2 : w.size(0)}, x.options());
  auto ptr = [](const c10::optional<at::Tensor>& t) -> const void* { return (t.has_value() && t->defined()) ? t->data_ptr() : nullptr; };
  if (residual.has_value() && residual->defined())
    TORCH_CHECK(residual->is_contiguous() && residual->numel() == y.numel() && residual->scalar_type() == x.scalar_type(), "gemv_fused: residual [M,N]");
  if (ln_w.has_value() && ln_w->defined())
    TORCH_CHECK(ln_w->numel() == x.size(1) && ln_b.has_value() && ln_b->numel() == x.size(1) && ln_w->scalar_type() == x.scalar_type(), "gemv_fused: ln params [K]");
  PFX_CUDA_CHECK(pfx::gemv_skinny(x.data_ptr(), w.data_ptr(), ptr(bias), y.data_ptr(), (int)x.size(0), (int)w.size(0), (int)x.size(1), dtype_code(x),
                                  at::cuda::getCurrentDeviceProperties()->multiProcessorCount, cur_stream(), ptr(ln_w), ptr(ln_b), (float)ln_eps,
                                  ptr(residual), (int)act));
  return y;
}

at::Tensor gemv_w8a8(const at::Tensor& xq, const at::Tensor& wq, const at::Tensor& xs, const at::Tensor& ws, c10::optional<at::Tensor> bias,
                     c10::optional<at::ScalarType> out_dtype) {
  TORCH_CHECK(xq.is_cuda() && xq.scalar_type() == at::kChar && wq.scalar_type() == at::kChar && xq.is_contiguous() && wq.is_contiguous() &&
              xq.dim() == 2 && wq.dim() == 2 && xq.size(1) == wq.size(1), "gemv_w8a8: int8 x [M,K], w [N,K]");
  TORCH_CHECK(wq.is_cuda() && wq.device() == xq.device(), "gemv_w8a8: wq must be on ", xq.device());
  // the kernel reads xq and wq rows with 16-byte loads
  TORCH_CHECK(reinterpret_cast<uintptr_t>(xq.data_ptr()) % 16 == 0, "gemv_w8a8: xq must be 16-byte aligned");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(wq.data_ptr()) % 16 == 0, "gemv_w8a8: wq must be 16-byte aligned");
  TORCH_CHECK(xs.is_cuda() && xs.is_contiguous() && xs.scalar_type() == at::kFloat && xs.numel() == xq.size(0), "gemv_w8a8: xs must be a contiguous [",
              xq.size(0), "] float CUDA tensor");
  TORCH_CHECK(ws.is_cuda() && ws.is_contiguous() && ws.scalar_type() == at::kFloat && ws.numel() == wq.size(0), "gemv_w8a8: ws must be a contiguous [",
              wq.size(0), "] float CUDA tensor");
  const c10::cuda::CUDAGuard guard(xq.device());
  const bool has_bias = bias.has_value() && bias->defined();
  const at::ScalarType od = out_dtype.value_or(at::kBFloat16);
  TORCH_CHECK(od == at::kBFloat16 || od == at::kHalf, "gemv_w8a8: out_dtype must be bf16 or fp16, got ", od);
  if (has_bias)
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->scalar_type() == od && bias->numel() == wq.size(0), "gemv_w8a8: bias must be a contiguous [",
                wq.size(0), "] CUDA tensor of the output dtype ", od, ", got ", bias->scalar_type(), " ", bias->sizes());
  at::Tensor y = at::empty({xq.size(0), wq.size(0)}, xq.options().dtype(od));
  const void* b = has_bias ? bias->data_ptr() : nullptr;
  PFX_CUDA_CHECK(pfx::gemv_w8a8(xq.data_ptr(), wq.data_ptr(), xs.data_ptr<float>(), ws.data_ptr<float>(), b, y.data_ptr(), (int)xq.size(0),
                                (int)wq.size(0), (int)xq.size(1), num_sms(), cur_stream(), od == at::kHalf ? 0 : 1));
  return y;
}

at::Tensor gemm_smallm(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, int64_t split) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1), "gemm_smallm: x [M,K], w [N,K]");
  TORCH_CHECK(is_16bit(x) && w.scalar_type() == x.scalar_type(), "gemm_smallm: bf16 or fp16 operands of one dtype");
  const bool has_bias = bias.has_value() && bias->defined();
  if (has_bias) TORCH_CHECK(bias->scalar_type() == x.scalar_type() && bias->is_contiguous() && bias->numel() == w.size(0), "gemm_smallm: bias [N] of the operands' dtype");
  at::Tensor y = at::empty({x.size(0), w.size(0)}, x.options());
  const void* b = has_bias ? bias->data_ptr() : nullptr;
  PFX_CUDA_CHECK(pfx::gemm_smallm(x.data_ptr(), w.data_ptr(), b, y.data_ptr(), (int)x.size(0), (int)w.size(0), (int)x.size(1), dtype_code(x), (int)split,
                                  at::cuda::getCurrentDeviceProperties()->multiProcessorCount, cur_stream()));
  return y;
}

at::Tensor attention_decode(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, c10::optional<at::Tensor> mask, int64_t L, double scale) {
  // q [B,1,H,D]; k, v [B,Lmax,Hkv,D] (contiguous cache, H % Hkv == 0); mask additive [B,Lmax] in the same dtype, or none
  PFX_CHECK_CUDA_CONTIG(q); PFX_CHECK_CUDA_CONTIG(k); PFX_CHECK_CUDA_CONTIG(v);
  TORCH_CHECK(q.dim() == 4 && q.size(1) == 1 && k.dim() == 4 && k.sizes() == v.sizes() && k.size(0) == q.size(0) &&
              k.size(3) == q.size(3) && k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(), "attention_decode: shape mismatch");
  TORCH_CHECK(k.size(2) >= 1 && q.size(2) % k.size(2) == 0, "attention_decode: q has ", q.size(2), " heads, which is not a multiple of the ",
              k.size(2), " cache heads");
  const c10::cuda::CUDAGuard guard(q.device());
  const void* mp = nullptr;
  at::Tensor mc;
  if (mask.has_value() && mask->defined()) {
    mc = mask->reshape({q.size(0), -1}).to(q.scalar_type()).contiguous();
    TORCH_CHECK(mc.size(1) == k.size(1), "attention_decode: mask must cover the whole cache");
    mp = mc.data_ptr();
  }
  auto out = at::empty_like(q);
  PFX_CUDA_CHECK(pfx::attention_decode(q.data_ptr(), k.data_ptr(), v.data_ptr(), mp, out.data_ptr(), (int)q.size(0), (int)q.size(2), (int)q.size(3),
                                       (int)L, (int)k.size(1), (float)scale, dtype_code(q), cur_stream(), nullptr, (int)k.size(2)));
  return out;
}

std::vector<at::Tensor> attention_fwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, bool causal, double scale) {
  // q [B,Sq,H,D], k/v [B,Sk,H,D], contiguous bf16 -> (out [B,Sq,H,D], lse [B,H,Sq] fp32)
  PFX_CHECK_CUDA_CONTIG(q); PFX_CHECK_CUDA_CONTIG(k); PFX_CHECK_CUDA_CONTIG(v);
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && k.sizes() == v.sizes() && q.size(0) == k.size(0) && q.size(2) == k.size(2) && q.size(3) == k.size(3),
              "attention_fwd: shape mismatch");
  TORCH_CHECK(q.scalar_type() == at::kBFloat16 && k.scalar_type() == at::kBFloat16 && v.scalar_type() == at::kBFloat16, "attention_fwd: bf16 only");
  const c10::cuda::CUDAGuard guard(q.device());
  auto out = at::empty_like(q);
  auto lse = at::empty({q.size(0), q.size(2), q.size(1)}, q.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::attention_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr<float>(), (int)q.size(0), (int)q.size(1),
                                    (int)k.size(1), (int)q.size(2), (int)q.size(3), (float)scale, causal, cur_stream()));
  return {out, lse};
}


// out[t] = w[ids[t] - vocab_start] (zero for foreign ids) (+ pos_w[pos[t]])
at::Tensor embedding_fwd(const at::Tensor& ids, const at::Tensor& w, c10::optional<at::Tensor> pos, c10::optional<at::Tensor> pos_w, int64_t vocab_start) {
  PFX_CHECK_CUDA_CONTIG(ids); PFX_CHECK_CUDA_CONTIG(w);
  TORCH_CHECK(ids.scalar_type() == at::kLong && w.dim() == 2, "embedding_fwd: int64 ids, 2-D weight");
  const bool with_pos = pos.has_value() && pos->defined();
  if (with_pos) {
    TORCH_CHECK(pos_w.has_value() && pos_w->defined() && pos->is_contiguous() && pos_w->is_contiguous() && pos->numel() == ids.numel() &&
                pos->scalar_type() == at::kLong && pos_w->scalar_type() == w.scalar_type() && pos_w->size(1) == w.size(1), "embedding_fwd: position operands");
  }
  const c10::cuda::CUDAGuard guard(w.device());
  auto sizes = ids.sizes().vec();
  sizes.push_back(w.size(1));
  auto out = at::empty(sizes, w.options());
  PFX_CUDA_CHECK(pfx::embedding_fwd(ids.data_ptr<int64_t>(), w.data_ptr(), with_pos ? pos->data_ptr<int64_t>() : nullptr, with_pos ? pos_w->data_ptr() : nullptr,
                                    out.data_ptr(), ids.numel(), (int)w.size(1), vocab_start, w.size(0), dtype_code(w), cur_stream()));
  return out;
}
int64_t embedding_bwd_max_tokens() { return pfx::embedding_bwd_max_tokens(); }
// dw[ids[t] - vocab_start] (+)= sum over equal ids of dout[t]   (rows that do not occur are left untouched)
void embedding_bwd_(const at::Tensor& ids, const at::Tensor& dout, at::Tensor& dw, int64_t vocab_start, bool accumulate) {
  PFX_CHECK_CUDA_CONTIG(ids); PFX_CHECK_CUDA_CONTIG(dout); PFX_CHECK_CUDA_CONTIG(dw);
  TORCH_CHECK(ids.scalar_type() == at::kLong && dw.dim() == 2 && dout.numel() == ids.numel() * dw.size(1), "embedding_bwd_: shape mismatch");
  const c10::cuda::CUDAGuard guard(dw.device());
  int64_t n2 = 2;
  while (n2 < ids.numel()) n2 <<= 1;
  auto ws = at::empty({n2}, ids.options());
  PFX_CUDA_CHECK(pfx::embedding_bwd(ids.data_ptr<int64_t>(), dout.data_ptr(), dw.data_ptr(), reinterpret_cast<unsigned long long*>(ws.data_ptr<int64_t>()),
                                    ids.numel(), (int)dw.size(1), vocab_start, dw.size(0), dtype_code(dout), dtype_code(dw), accumulate, cur_stream()));
}

static pfx::AttnView attn_view(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.dim() == 4 && is_16bit(t) && t.stride(3) == 1, name, ": [B,S,H,D] bf16 or fp16 CUDA view with contiguous D expected");
  TORCH_CHECK(t.stride(0) % 8 == 0 && t.stride(1) % 8 == 0 && t.stride(2) % 8 == 0 && (reinterpret_cast<uintptr_t>(t.data_ptr()) % 16) == 0,
              name, ": strides must be multiples of 8 elements and the base 16-byte aligned");
  return pfx::AttnView{t.data_ptr(), t.stride(0), t.stride(1), t.stride(2)};
}

// Query heads of q (or dq): [B,S,H,D], or [B,S,Hkv,G,D] for the query part of a packed [B,S,Hkv,G+2,D] grouped projection output.
static int64_t attn_q_heads(const at::Tensor& t) { return t.dim() == 5 ? t.size(2) * t.size(3) : t.size(2); }

// The view of q / dq when k / v have Hkv heads: a [B,S,H,D] view (group stride G * head stride) or a [B,S,Hkv,G,D] view.
static pfx::AttnView attn_qview(const at::Tensor& t, const char* name, int64_t Hkv) {
  if (t.dim() != 5) {
    pfx::AttnView v = attn_view(t, name);
    v.sg = (t.size(2) / Hkv) * t.stride(2);
    return v;
  }
  TORCH_CHECK(t.is_cuda() && is_16bit(t) && t.stride(4) == 1, name, ": [B,S,Hkv,G,D] bf16 or fp16 CUDA view with contiguous D expected");
  TORCH_CHECK(t.size(2) == Hkv, name, ": a [B,S,Hkv,G,D] view needs one group per K/V head (", t.size(2), " groups, ", Hkv, " K/V heads)");
  TORCH_CHECK(t.stride(0) % 8 == 0 && t.stride(1) % 8 == 0 && t.stride(2) % 8 == 0 && t.stride(3) % 8 == 0 &&
              (reinterpret_cast<uintptr_t>(t.data_ptr()) % 16) == 0, name, ": strides must be multiples of 8 elements and the base 16-byte aligned");
  return pfx::AttnView{t.data_ptr(), t.stride(0), t.stride(1), t.stride(3), t.stride(2)};
}

// k / v heads against the query heads of q: returns Hkv (H % Hkv == 0 is required)
static int64_t attn_kv_heads(const at::Tensor& q, const at::Tensor& k, const char* fn) {
  TORCH_CHECK(q.dim() == 4 || q.dim() == 5, fn, ": q must be [B,S,H,D] or [B,S,Hkv,G,D]");
  TORCH_CHECK(k.dim() == 4, fn, ": k must be [B,S,Hkv,D]");
  const int64_t H = attn_q_heads(q), Hkv = k.size(2);
  TORCH_CHECK(Hkv >= 1 && H % Hkv == 0, fn, ": q has ", H, " heads, which is not a multiple of the ", Hkv, " K/V heads");
  return Hkv;
}

// Flash attention forward on [B,S,H,D] bf16 or fp16 views (no copies for packed-QKV slices / sequence-major storage); optional dropout keyed by `seed`.
// Grouped-query attention: k / v may have Hkv heads with H % Hkv == 0, and q may be the [B,S,Hkv,G,D] query part of a packed projection.
std::vector<at::Tensor> attention_fwd_v2(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, bool causal, double scale, double dropout_p,
                                         int64_t seed) {
  const int64_t Hkv = attn_kv_heads(q, k, "attention_fwd_v2");
  const int64_t H = attn_q_heads(q), D = q.size(q.dim() - 1);
  TORCH_CHECK(k.sizes() == v.sizes() && q.size(0) == k.size(0) && D == k.size(3), "attention_fwd_v2: shape mismatch");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(), "attention_fwd_v2: q, k, v must have one dtype");
  const c10::cuda::CUDAGuard guard(q.device());
  auto out = at::empty({q.size(0), q.size(1), H, D}, q.options());
  auto lse = at::empty({q.size(0), H, q.size(1)}, q.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::attention_fwd_v2(attn_qview(q, "q", Hkv), attn_view(k, "k"), attn_view(v, "v"), attn_view(out, "out"), lse.data_ptr<float>(),
                                       (int)q.size(0), (int)q.size(1), (int)k.size(1), (int)H, (int)Hkv, (int)D, (float)scale, causal,
                                       pfx::AttnDropout{(float)dropout_p, (uint64_t)seed}, dtype_code(q), cur_stream()));
  return {out, lse};
}

// Flash attention backward (head_dim 64 or 128, bf16 or fp16): writes dq / dk / dv into the given (possibly strided) views.
void attention_bwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& out, const at::Tensor& dout, const at::Tensor& lse,
                   at::Tensor& dq, at::Tensor& dk, at::Tensor& dv, bool causal, double scale, double dropout_p, int64_t seed) {
  const int64_t Hkv = attn_kv_heads(q, k, "attention_bwd");
  const int64_t H = attn_q_heads(q), D = q.size(q.dim() - 1);
  TORCH_CHECK(D == 128 || D == 64, "attention_bwd: head_dim must be 64 or 128");
  TORCH_CHECK(k.sizes() == v.sizes() && q.size(0) == k.size(0) && D == k.size(3), "attention_bwd: k / v shape mismatch");
  TORCH_CHECK(k.sizes() == dk.sizes() && k.sizes() == dv.sizes(), "attention_bwd: dk / dv must have the shape of k");
  TORCH_CHECK(q.sizes() == dq.sizes(), "attention_bwd: dq must have the shape of q");
  const std::vector<int64_t> o_shape{q.size(0), q.size(1), H, D};
  TORCH_CHECK(out.sizes() == at::IntArrayRef(o_shape) && dout.sizes() == at::IntArrayRef(o_shape), "attention_bwd: out / dout must be [B,Sq,H,D]");
  TORCH_CHECK(lse.is_cuda() && lse.is_contiguous() && lse.scalar_type() == at::kFloat && lse.numel() == q.size(0) * q.size(1) * H, "attention_bwd: lse");
  for (const at::Tensor* t : std::initializer_list<const at::Tensor*>{&k, &v, &out, &dout, &dq, &dk, &dv})
    TORCH_CHECK(t->scalar_type() == q.scalar_type(), "attention_bwd: q, k, v, out, dout and the gradients must have one dtype");
  const c10::cuda::CUDAGuard guard(q.device());
  const int64_t B = q.size(0), Sq = q.size(1), Sk = k.size(1);
  const int64_t sq_pad = (Sq + 63) / 64 * 64;
  auto f32 = q.options().dtype(at::kFloat);
  auto dq_acc = at::empty({B, Sq, H, D}, f32);
  auto stats = at::empty({2, B * H * sq_pad}, f32);
  PFX_CUDA_CHECK(pfx::attention_bwd(attn_qview(q, "q", Hkv), attn_view(k, "k"), attn_view(v, "v"), attn_view(out, "out"), attn_view(dout, "dout"),
                                    lse.data_ptr<float>(), attn_qview(dq, "dq", Hkv), attn_view(dk, "dk"), attn_view(dv, "dv"), dq_acc.data_ptr<float>(),
                                    stats[0].data_ptr<float>(), stats[1].data_ptr<float>(), (int)B, (int)Sq, (int)Sk, (int)H, (int)Hkv, (int)D, (float)scale,
                                    causal, pfx::AttnDropout{(float)dropout_p, (uint64_t)seed}, dtype_code(q), cur_stream()));
}

// Document-mask bounds from int64 [B, S] position ids (from_positions: key_start = clamp(i - pos, 0, i)) or key starts (clamped into
// [0, i]): returns (key_start int32 [B, S], tile_min, tile_max int32 [B, ceil(S / 64)]), computed by one kernel.
std::vector<at::Tensor> attention_doc_bounds(const at::Tensor& src, bool from_positions) {
  TORCH_CHECK(src.is_cuda() && src.dim() == 2 && src.is_contiguous() && src.scalar_type() == at::kLong, "attention_doc_bounds: int64 [B, S] CUDA tensor");
  TORCH_CHECK(src.size(0) >= 1 && src.size(0) <= 65535 && src.size(1) >= 1, "attention_doc_bounds: 1 <= B <= 65535 and S >= 1");
  const c10::cuda::CUDAGuard guard(src.device());
  const int64_t B = src.size(0), S = src.size(1), T = (S + 63) / 64;
  auto i32 = src.options().dtype(at::kInt);
  auto ks = at::empty({B, S}, i32), tmin = at::empty({B, T}, i32), tmax = at::empty({B, T}, i32);
  PFX_CUDA_CHECK(pfx::attention_doc_bounds(src.data_ptr<int64_t>(), from_positions, (int)B, (int)S, ks.data_ptr<int>(), tmin.data_ptr<int>(),
                                           tmax.data_ptr<int>(), cur_stream()));
  return {ks, tmin, tmax};
}

static pfx::AttnDocMask attn_doc(const at::Tensor& ks, const at::Tensor& tmin, const at::Tensor& tmax, int64_t B, int64_t S, const char* fn) {
  const int64_t T = (S + 63) / 64;
  for (const at::Tensor* t : {&ks, &tmin, &tmax})
    TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == at::kInt, fn, ": document bounds must be contiguous int32 CUDA tensors");
  TORCH_CHECK(ks.numel() == B * S && tmin.numel() == B * T && tmax.numel() == B * T, fn, ": document bounds must be [B, S] and [B, ceil(S / 64)]");
  return pfx::AttnDocMask{ks.data_ptr<int>(), tmin.data_ptr<int>(), tmax.data_ptr<int>()};
}

// Causal flash attention under a document mask (self-attention, Sq == Sk): query i attends keys [key_start[b, i], i].  The bounds come
// from attention_doc_bounds.  Views as in attention_fwd_v2.
std::vector<at::Tensor> attention_fwd_doc(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& key_start,
                                          const at::Tensor& tile_min, const at::Tensor& tile_max, double scale, double dropout_p, int64_t seed) {
  const int64_t Hkv = attn_kv_heads(q, k, "attention_fwd_doc");
  const int64_t H = attn_q_heads(q), D = q.size(q.dim() - 1);
  TORCH_CHECK(k.sizes() == v.sizes() && q.size(0) == k.size(0) && q.size(1) == k.size(1) && D == k.size(3),
              "attention_fwd_doc: shape mismatch (self-attention: q and k have one sequence length)");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(), "attention_fwd_doc: q, k, v must have one dtype");
  const pfx::AttnDocMask doc = attn_doc(key_start, tile_min, tile_max, q.size(0), q.size(1), "attention_fwd_doc");
  const c10::cuda::CUDAGuard guard(q.device());
  auto out = at::empty({q.size(0), q.size(1), H, D}, q.options());
  auto lse = at::empty({q.size(0), H, q.size(1)}, q.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::attention_fwd_doc(attn_qview(q, "q", Hkv), attn_view(k, "k"), attn_view(v, "v"), attn_view(out, "out"), lse.data_ptr<float>(),
                                        (int)q.size(0), (int)q.size(1), (int)H, (int)Hkv, (int)D, (float)scale,
                                        pfx::AttnDropout{(float)dropout_p, (uint64_t)seed}, doc, dtype_code(q), cur_stream()));
  return {out, lse};
}

// Backward of attention_fwd_doc: writes dq / dk / dv into the given (possibly strided) views.
void attention_bwd_doc(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& out, const at::Tensor& dout, const at::Tensor& lse,
                       at::Tensor& dq, at::Tensor& dk, at::Tensor& dv, const at::Tensor& key_start, const at::Tensor& tile_min, const at::Tensor& tile_max,
                       double scale, double dropout_p, int64_t seed) {
  const int64_t Hkv = attn_kv_heads(q, k, "attention_bwd_doc");
  const int64_t H = attn_q_heads(q), D = q.size(q.dim() - 1);
  TORCH_CHECK(D == 128 || D == 64, "attention_bwd_doc: head_dim must be 64 or 128");
  TORCH_CHECK(k.sizes() == v.sizes() && q.size(0) == k.size(0) && q.size(1) == k.size(1) && D == k.size(3), "attention_bwd_doc: k / v shape mismatch");
  TORCH_CHECK(k.sizes() == dk.sizes() && k.sizes() == dv.sizes(), "attention_bwd_doc: dk / dv must have the shape of k");
  TORCH_CHECK(q.sizes() == dq.sizes(), "attention_bwd_doc: dq must have the shape of q");
  const std::vector<int64_t> o_shape{q.size(0), q.size(1), H, D};
  TORCH_CHECK(out.sizes() == at::IntArrayRef(o_shape) && dout.sizes() == at::IntArrayRef(o_shape), "attention_bwd_doc: out / dout must be [B,S,H,D]");
  TORCH_CHECK(lse.is_cuda() && lse.is_contiguous() && lse.scalar_type() == at::kFloat && lse.numel() == q.size(0) * q.size(1) * H, "attention_bwd_doc: lse");
  for (const at::Tensor* t : std::initializer_list<const at::Tensor*>{&k, &v, &out, &dout, &dq, &dk, &dv})
    TORCH_CHECK(t->scalar_type() == q.scalar_type(), "attention_bwd_doc: q, k, v, out, dout and the gradients must have one dtype");
  const pfx::AttnDocMask doc = attn_doc(key_start, tile_min, tile_max, q.size(0), q.size(1), "attention_bwd_doc");
  const c10::cuda::CUDAGuard guard(q.device());
  const int64_t B = q.size(0), S = q.size(1);
  const int64_t s_pad = (S + 63) / 64 * 64;
  auto f32 = q.options().dtype(at::kFloat);
  auto dq_acc = at::empty({B, S, H, D}, f32);
  auto stats = at::empty({2, B * H * s_pad}, f32);
  PFX_CUDA_CHECK(pfx::attention_bwd_doc(attn_qview(q, "q", Hkv), attn_view(k, "k"), attn_view(v, "v"), attn_view(out, "out"), attn_view(dout, "dout"),
                                        lse.data_ptr<float>(), attn_qview(dq, "dq", Hkv), attn_view(dk, "dk"), attn_view(dv, "dv"), dq_acc.data_ptr<float>(),
                                        stats[0].data_ptr<float>(), stats[1].data_ptr<float>(), (int)B, (int)S, (int)H, (int)Hkv, (int)D, (float)scale,
                                        pfx::AttnDropout{(float)dropout_p, (uint64_t)seed}, doc, dtype_code(q), cur_stream()));
}

at::Tensor attention_decode_packed(const at::Tensor& qkv, at::Tensor& k, at::Tensor& v, c10::optional<at::Tensor> mask, const at::Tensor& write_idx,
                                   double scale) {
  // qkv [B,1,Hkv,G+2,D] (fused projection output: per K/V head its G queries, key and value; G = 1 is [B,1,H,3,D]); appends this step's
  // K/V at cache position write_idx[0] and attends over the whole cache [B,Lmax,Hkv,D]
  PFX_CHECK_CUDA_CONTIG(qkv); PFX_CHECK_CUDA_CONTIG(k); PFX_CHECK_CUDA_CONTIG(v);
  TORCH_CHECK(qkv.dim() == 5 && qkv.size(1) == 1 && qkv.size(3) >= 3 && k.dim() == 4 && k.sizes() == v.sizes() && k.size(0) == qkv.size(0) &&
              k.size(2) == qkv.size(2) && k.size(3) == qkv.size(4) && k.scalar_type() == qkv.scalar_type() && v.scalar_type() == qkv.scalar_type(),
              "attention_decode_packed: shape mismatch (qkv [B,1,Hkv,G+2,D], caches [B,Lmax,Hkv,D])");
  TORCH_CHECK(write_idx.is_cuda() && write_idx.scalar_type() == at::kLong && write_idx.numel() == 1, "attention_decode_packed: write_idx");
  const c10::cuda::CUDAGuard guard(qkv.device());
  const void* mp = nullptr;
  at::Tensor mc;
  if (mask.has_value() && mask->defined()) {
    mc = mask->reshape({qkv.size(0), -1}).to(qkv.scalar_type()).contiguous();
    TORCH_CHECK(mc.size(1) == k.size(1), "attention_decode_packed: mask must cover the whole cache");
    mp = mc.data_ptr();
  }
  const int64_t Hkv = qkv.size(2), H = Hkv * (qkv.size(3) - 2);
  auto out = at::empty({qkv.size(0), 1, H, qkv.size(4)}, qkv.options());
  PFX_CUDA_CHECK(pfx::attention_decode(qkv.data_ptr(), k.data_ptr(), v.data_ptr(), mp, out.data_ptr(), (int)qkv.size(0), (int)H,
                                       (int)qkv.size(4), (int)k.size(1), (int)k.size(1), (float)scale, dtype_code(qkv), cur_stream(),
                                       write_idx.data_ptr<int64_t>(), (int)Hkv));
  return out;
}

// ---- MoE dispatch / combine over peer memory
std::vector<at::Tensor> moe_route(const at::Tensor& gate_idx, int64_t total_experts) {
  TORCH_CHECK(gate_idx.is_cuda() && gate_idx.scalar_type() == at::kLong && gate_idx.is_contiguous(), "gate_idx: contiguous int64 CUDA tensor");
  auto iopt = gate_idx.options().dtype(at::kInt);
  at::Tensor slot_rank = at::empty({gate_idx.numel()}, iopt), counts = at::empty({total_experts}, iopt);
  PFX_CUDA_CHECK(pfx::moe_route(gate_idx.data_ptr<int64_t>(), (int)gate_idx.numel(), (int)total_experts, slot_rank.data_ptr<int>(),
                                counts.data_ptr<int>(), cur_stream()));
  return {slot_rank, counts};
}
std::vector<at::Tensor> moe_dispatch(const at::Tensor& src, c10::optional<at::Tensor> scale, const at::Tensor& gate_idx,
                                     const at::Tensor& slot_rank, const at::Tensor& counts, const std::vector<int64_t>& peer_recv,
                                     const std::vector<int64_t>& peer_cnt, const std::vector<int64_t>& peer_flags, at::Tensor& block_counter,
                                     int64_t src_div, int64_t e_local, int64_t rank, int64_t align, int64_t cap_rows, int64_t epoch,
                                     int64_t num_ctas) {
  TORCH_CHECK(src.is_cuda() && src.is_contiguous() && src.dim() == 2, "src: contiguous [rows, H]");
  const int world = (int)peer_recv.size();
  auto iopt = gate_idx.options().dtype(at::kInt);
  at::Tensor slot_loc = at::empty({gate_idx.numel()}, iopt), seg = at::empty({2 * e_local + 2}, iopt);
  auto pr = to_ptrs(peer_recv), pc = to_ptrs(peer_cnt), pf = to_ptrs(peer_flags);
  const float* sc = (scale.has_value() && scale->defined()) ? scale->data_ptr<float>() : nullptr;
  PFX_CUDA_CHECK(pfx::moe_dispatch(src.data_ptr(), sc, gate_idx.data_ptr<int64_t>(), slot_rank.data_ptr<int>(), counts.data_ptr<int>(),
                                   slot_loc.data_ptr<int>(), seg.data_ptr<int>(), pr.data(), pc.data(), pf.data(),
                                   reinterpret_cast<unsigned*>(block_counter.data_ptr<int>()), (int)gate_idx.numel(), (int)src_div,
                                   (int)src.size(1), (int)e_local, world, (int)rank, (int)align, (int)cap_rows, (uint32_t)epoch,
                                   dtype_code(src), (int)num_ctas, cur_stream()));
  return {slot_loc, seg};
}
// Evoformer gated attention forward: q [G, Sq, H, 32], k / v [G, Sk, H, 32]; returns (out [G, Sq, H, 32], stats [2, G, H, Sq]: row maximum and
// log2 row sum, log2 units)
std::vector<at::Tensor> evoformer_attention_fwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, c10::optional<at::Tensor> mask_bias,
                                                c10::optional<at::Tensor> pair_bias, c10::optional<at::Tensor> gate, int64_t groups_per_pair, double scale) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 4 && k.dim() == 4 && v.dim() == 4 && q.is_contiguous() && k.is_contiguous() && v.is_contiguous(), "evoformer_attention: contiguous [G, S, H, 32]");
  TORCH_CHECK(q.scalar_type() == at::kBFloat16 && k.scalar_type() == at::kBFloat16 && v.scalar_type() == at::kBFloat16, "evoformer_attention: bf16");
  const int64_t G = q.size(0), Sq = q.size(1), H = q.size(2), Sk = k.size(1);
  TORCH_CHECK(q.size(3) == 32 && k.size(3) == 32 && v.size(3) == 32 && H % 2 == 0 && k.size(0) == G && v.size(0) == G && k.size(2) == H && v.size(2) == H && v.size(1) == Sk,
              "evoformer_attention: head width 32, even head count, matching shapes");
  const c10::cuda::CUDAGuard guard(q.device());
  const float* mb = nullptr; const void* pb = nullptr; const void* gt = nullptr;
  if (mask_bias.has_value() && mask_bias->defined()) {
    TORCH_CHECK(mask_bias->scalar_type() == at::kFloat && mask_bias->is_contiguous() && mask_bias->numel() == G * Sk, "evoformer_attention: mask_bias fp32 [G, Sk]");
    mb = mask_bias->data_ptr<float>();
  }
  if (pair_bias.has_value() && pair_bias->defined()) {
    TORCH_CHECK(pair_bias->scalar_type() == at::kBFloat16 && pair_bias->is_contiguous() && G % groups_per_pair == 0 &&
                pair_bias->numel() == (G / groups_per_pair) * H * Sq * Sk, "evoformer_attention: pair_bias bf16 [G / groups_per_pair, H, Sq, Sk]");
    pb = pair_bias->data_ptr();
  }
  if (gate.has_value() && gate->defined()) {
    TORCH_CHECK(gate->scalar_type() == at::kBFloat16 && gate->is_contiguous() && gate->numel() == q.numel(), "evoformer_attention: gate bf16 like q");
    gt = gate->data_ptr();
  }
  at::Tensor out = at::empty_like(q), stats = at::empty({2, G, H, Sq}, q.options().dtype(at::kFloat));
  PFX_CUDA_CHECK(pfx::evoformer_attention_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), stats.data_ptr<float>(), mb, pb, gt, (int)G, (int)Sq,
                                              (int)Sk, (int)H, (int)groups_per_pair, (float)scale, cur_stream()));
  return {out, stats};
}

// Evoformer gated attention backward: returns (dq, dk, dv, dgate or empty, dpair fp32 or empty)
std::vector<at::Tensor> evoformer_attention_bwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, const at::Tensor& out, const at::Tensor& dout,
                                                const at::Tensor& stats, c10::optional<at::Tensor> mask_bias, c10::optional<at::Tensor> pair_bias,
                                                c10::optional<at::Tensor> gate, int64_t groups_per_pair, double scale, bool need_dpair) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 4 && q.is_contiguous() && k.is_contiguous() && v.is_contiguous() && out.is_contiguous() && dout.is_contiguous() &&
              q.scalar_type() == at::kBFloat16 && dout.scalar_type() == at::kBFloat16 && out.sizes() == q.sizes() && dout.sizes() == q.sizes(),
              "evoformer_attention_bwd: contiguous bf16 [G, S, H, 32] operands");
  const int64_t G = q.size(0), Sq = q.size(1), H = q.size(2), Sk = k.size(1);
  TORCH_CHECK(q.size(3) == 32 && H % 2 == 0 && stats.scalar_type() == at::kFloat && stats.is_contiguous() && stats.numel() == 2 * G * H * Sq,
              "evoformer_attention_bwd: shapes (stats: the forward's [2, G, H, Sq])");
  const c10::cuda::CUDAGuard guard(q.device());
  const bool has_gate = gate.has_value() && gate->defined(), has_pb = pair_bias.has_value() && pair_bias->defined(), has_mb = mask_bias.has_value() && mask_bias->defined();
  if (has_mb) TORCH_CHECK(mask_bias->scalar_type() == at::kFloat && mask_bias->is_contiguous() && mask_bias->numel() == G * Sk, "mask_bias fp32 [G, Sk]");
  if (has_pb) TORCH_CHECK(pair_bias->scalar_type() == at::kBFloat16 && pair_bias->is_contiguous() && pair_bias->numel() == (G / groups_per_pair) * H * Sq * Sk, "pair_bias");
  if (has_gate) TORCH_CHECK(gate->scalar_type() == at::kBFloat16 && gate->is_contiguous() && gate->numel() == q.numel(), "gate");
  auto fopt = q.options().dtype(at::kFloat);
  at::Tensor dq = at::empty_like(q), dk = at::empty_like(k), dv = at::empty_like(v);
  at::Tensor dgate = has_gate ? at::empty_like(q) : at::empty({0}, q.options());
  at::Tensor dpair = (has_pb && need_dpair) ? at::zeros({G / groups_per_pair, H, Sq, Sk}, fopt) : at::empty({0}, fopt);
  at::Tensor do_pre = at::empty_like(q), dq_acc = at::empty({G, Sq, H, 32}, fopt);
  const int64_t sq_pad = (Sq + 63) / 64 * 64;
  at::Tensor m2 = at::empty({G * H, sq_pad}, fopt), delta = at::empty({G * H, sq_pad}, fopt), l2 = at::empty({G * H, sq_pad}, fopt);
  PFX_CUDA_CHECK(pfx::evoformer_attention_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), dout.data_ptr(), has_gate ? gate->data_ptr() : nullptr,
                                              stats.data_ptr<float>(), has_mb ? mask_bias->data_ptr<float>() : nullptr, has_pb ? pair_bias->data_ptr() : nullptr,
                                              dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), has_gate ? dgate.data_ptr() : nullptr,
                                              dpair.numel() ? dpair.data_ptr<float>() : nullptr, do_pre.data_ptr(), dq_acc.data_ptr<float>(),
                                              m2.data_ptr<float>(), delta.data_ptr<float>(), l2.data_ptr<float>(), (int)G, (int)Sq, (int)Sk, (int)H, (int)groups_per_pair,
                                              (float)scale, cur_stream()));
  return {dq, dk, dv, dgate, dpair};
}

// tile table + K segments of the grouped expert GEMMs, from the dispatch kernel's segment table (all on the device)
std::vector<at::Tensor> moe_tile_table(const at::Tensor& seg, int64_t e_local, int64_t align, int64_t cap_rows, at::Tensor& sticky) {
  TORCH_CHECK(seg.is_cuda() && seg.scalar_type() == at::kInt && seg.numel() == 2 * e_local + 2 && sticky.scalar_type() == at::kInt, "moe_tile_table: bad seg");
  at::Tensor tile_group = at::empty({cap_rows / 128}, seg.options()), seg2 = at::empty({2 * e_local}, seg.options());
  PFX_CUDA_CHECK(pfx::moe_tile_table(seg.data_ptr<int>(), (int)e_local, (int)align, (int)cap_rows, tile_group.data_ptr<int>(), seg2.data_ptr<int>(),
                                     sticky.data_ptr<int>(), cur_stream()));
  return {tile_group, seg2};
}

// Grouped expert GEMM, rows grouped: d[r, :] = a[r, :] . B[g(r)]^T (+ bias[g(r)]) for the expert g(r) that owns row block r / 128.
//   b: [G, N, K] (b_kmajor: forward) or [G, K, N] (dgrad).  epilogue: EPI_NONE / EPI_BIAS / EPI_BIAS_GELU_DUAL (out2) / EPI_DGELU (aux).
at::Tensor gemm_grouped(const at::Tensor& a, const at::Tensor& b, c10::optional<at::Tensor> bias, const at::Tensor& tile_group, at::Tensor& out,
                        bool b_kmajor, int64_t epilogue, c10::optional<at::Tensor> out2, c10::optional<at::Tensor> aux, int64_t row_align) {
  TORCH_CHECK(a.is_cuda() && a.dim() == 2 && b.dim() == 3 && a.is_contiguous() && b.is_contiguous() && out.is_contiguous(), "gemm_grouped: a [M,K], b [G,*,*] contiguous");
  TORCH_CHECK(is_16bit(a) && b.scalar_type() == a.scalar_type() && out.scalar_type() == a.scalar_type(), "gemm_grouped: bf16 or fp16 operands of one dtype");
  const int64_t M = a.size(0), K = a.size(1), G = b.size(0);
  const int64_t N = b_kmajor ? b.size(1) : b.size(2);
  TORCH_CHECK((b_kmajor ? b.size(2) : b.size(1)) == K, "gemm_grouped: K mismatch");
  TORCH_CHECK(M % 128 == 0 && tile_group.numel() == M / 128 && tile_group.scalar_type() == at::kInt, "gemm_grouped: tile table must cover M / 128 blocks");
  TORCH_CHECK(out.dim() == 2 && out.size(0) == M && out.size(1) == N && N % 8 == 0 && K % 64 == 0, "gemm_grouped: out [M, N], N % 8 == 0, K % 64 == 0");
  const c10::cuda::CUDAGuard guard(a.device());
  pfx::GemmArgs g{};
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = out.data_ptr();
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == a.scalar_type() && bias->numel() == G * N && bias->is_contiguous(), "gemm_grouped: bias [G, N] of the operands' dtype");
    g.bias = bias->data_ptr();
  } else {
    TORCH_CHECK(epilogue == pfx::EPI_NONE || epilogue == pfx::EPI_DGELU, "gemm_grouped: bias epilogue without bias");
  }
  if (epilogue == pfx::EPI_BIAS_GELU_DUAL) {
    TORCH_CHECK(out2.has_value() && out2->is_contiguous() && out2->sizes() == out.sizes() && out2->scalar_type() == a.scalar_type(), "gemm_grouped: out2 like out");
    g.d2 = out2->data_ptr();
  }
  if (epilogue == pfx::EPI_DGELU) {
    TORCH_CHECK(aux.has_value() && aux->is_contiguous() && aux->sizes() == out.sizes() && aux->scalar_type() == a.scalar_type(), "gemm_grouped: aux like out");
    g.aux = aux->data_ptr(); g.ld_aux = (int)N;
  }
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.lda = (int)K; g.ldb = (int)(b_kmajor ? K : N); g.ldd = (int)N;
  g.a_kmajor = true; g.b_kmajor = b_kmajor; g.out_mode = 0; g.epilogue = (int)epilogue; g.ab_format = dtype_code(a); g.num_sms = num_sms(); g.config = 0;
  g.group.mode = 1; g.group.tile_group = tile_group.data_ptr<int>(); g.group.groups = (int)G; g.group.b_group_stride = (int)(b_kmajor ? N : K);
  g.group.row_align = (int)row_align;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return out;
}

// Grouped expert wgrad: out[g] = dy[rows of g]^T . x[rows of g]   (dy [R, Mg], x [R, N], out [G, Mg, N], all bf16 or all fp16; seg2 = (start, padded count) per expert)
at::Tensor gemm_grouped_wgrad(const at::Tensor& dy, const at::Tensor& x, const at::Tensor& seg2, at::Tensor& out) {
  TORCH_CHECK(dy.is_cuda() && dy.dim() == 2 && x.dim() == 2 && out.dim() == 3 && dy.is_contiguous() && x.is_contiguous() && out.is_contiguous(), "gemm_grouped_wgrad: contiguous");
  TORCH_CHECK(is_16bit(dy) && x.scalar_type() == dy.scalar_type() && out.scalar_type() == dy.scalar_type(), "gemm_grouped_wgrad: bf16 or fp16 operands of one dtype");
  const int64_t R = dy.size(0), Mg = dy.size(1), N = x.size(1), G = out.size(0);
  TORCH_CHECK(x.size(0) == R && out.size(1) == Mg && out.size(2) == N && seg2.numel() == 2 * G && seg2.scalar_type() == at::kInt, "gemm_grouped_wgrad: shapes");
  TORCH_CHECK(Mg % 128 == 0 && N % 8 == 0, "gemm_grouped_wgrad: Mg % 128 == 0, N % 8 == 0");
  const c10::cuda::CUDAGuard guard(dy.device());
  pfx::GemmArgs g{};
  g.a = dy.data_ptr(); g.b = x.data_ptr(); g.d = out.data_ptr();
  g.M = (int)(G * Mg); g.N = (int)N; g.K = (int)R;
  g.lda = (int)Mg; g.ldb = (int)N; g.ldd = (int)N;
  g.a_kmajor = false; g.b_kmajor = false; g.out_mode = 0; g.epilogue = pfx::EPI_NONE; g.ab_format = dtype_code(dy); g.num_sms = num_sms(); g.config = 0;
  g.group.mode = 2; g.group.seg = seg2.data_ptr<int>(); g.group.groups = (int)G; g.group.m_per_group = (int)Mg;
  PFX_CUDA_CHECK(pfx::gemm_wgmma(g, cur_stream()));
  return out;
}

at::Tensor grouped_colsum(const at::Tensor& x, const at::Tensor& seg2, int64_t groups) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && seg2.numel() == 2 * groups && seg2.scalar_type() == at::kInt, "grouped_colsum: x [R, N], seg2 [2G]");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor out = at::empty({groups, x.size(1)}, x.options());
  PFX_CUDA_CHECK(pfx::grouped_colsum(x.data_ptr(), seg2.data_ptr<int>(), (int)groups, (int)x.size(1), out.data_ptr(), dtype_code(x), cur_stream()));
  return out;
}

void moe_combine(const std::vector<int64_t>& peer_src, const at::Tensor& slot_loc, c10::optional<at::Tensor> weights, at::Tensor& out,
                 c10::optional<at::Tensor> rows, const std::vector<int64_t>& peer_flags, int64_t topk, int64_t rank, int64_t epoch,
                 int64_t num_ctas) {
  auto ps = to_ptrs(peer_src), pf = to_ptrs(peer_flags);
  const float* w = (weights.has_value() && weights->defined()) ? weights->data_ptr<float>() : nullptr;
  void* r = (rows.has_value() && rows->defined()) ? rows->data_ptr() : nullptr;
  PFX_CUDA_CHECK(pfx::moe_combine(ps.data(), slot_loc.data_ptr<int>(), w, out.data_ptr(), r, pf.data(), (int)out.size(0), (int)topk,
                                  (int)out.size(1), (int)peer_src.size(), (int)rank, (uint32_t)epoch, dtype_code(out), (int)num_ctas,
                                  cur_stream()));
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "paddlefleetx_b200 sm_90a kernel library";
  m.def("gemm", &gemm, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("out") = py::none(), py::arg("a_kmajor") = true,
        py::arg("b_kmajor") = true, py::arg("epilogue") = 0, py::arg("out_mode") = 0, py::arg("config") = 0);
  m.def("gemm_rs_scatter", &gemm_rs_scatter);
  m.def("slot_reduce", &slot_reduce);
  m.def("gemm_ag", &gemm_ag);
  m.def("quantize_rows", &quantize_rows);
  m.def("gemm_lowp", &gemm_lowp, py::arg("a"), py::arg("b"), py::arg("row_scale") = py::none(), py::arg("col_scale") = py::none(),
        py::arg("bias") = py::none(), py::arg("config") = 0, py::arg("out_dtype") = py::none());
  m.def("norm_fwd", &norm_fwd);
  m.def("norm_bwd", &norm_bwd, py::arg("dy"), py::arg("x"), py::arg("w"), py::arg("mean"), py::arg("rstd"), py::arg("rms"), py::arg("has_bias"),
        py::arg("dres") = py::none());
  m.def("bias_gelu_fwd", &bias_gelu_fwd);
  m.def("bias_gelu_bwd", &bias_gelu_bwd);
  m.def("bias_swiglu_fwd", &bias_swiglu_fwd);
  m.def("bias_swiglu_bwd", &bias_swiglu_bwd);
  m.def("bias_dropout_add_fwd", &bias_dropout_add_fwd);
  m.def("dropout_bwd", &dropout_bwd);
  m.def("colsum", &colsum);
  m.def("ce_stats", &ce_stats);
  m.def("ce_bwd_", &ce_bwd_);
  m.def("sumsq_", &sumsq_);
  m.def("clip_coef_", &clip_coef_);
  m.def("adamw_flat_", &adamw_flat_, py::arg("p_lp"), py::arg("master"), py::arg("grad"), py::arg("m"), py::arg("v"), py::arg("lr"), py::arg("beta1"),
        py::arg("beta2"), py::arg("eps"), py::arg("wd"), py::arg("step"), py::arg("gscale") = py::none(), py::arg("found_inf") = py::none(),
        py::arg("cta_budget") = 0);
  m.def("accumulate_f32_", &accumulate_f32_);
  m.def("topp_sampling", &topp_sampling);
  m.def("rope", &rope);
  m.def("causal_softmax_fwd", &causal_softmax_fwd);
  m.def("causal_softmax_bwd", &causal_softmax_bwd);
  m.def("ipc_alloc", &ipc_alloc);
  m.def("ipc_open", &ipc_open);
  m.def("ipc_close", &ipc_close);
  m.def("ipc_free", &ipc_free);
  m.def("tensor_from_ptr", &tensor_from_ptr);
  m.def("p2p_barrier", &p2p_barrier);
  m.def("p2p_reduce_scatter", &p2p_reduce_scatter);
  m.def("p2p_all_gather", &p2p_all_gather);
  m.def("attention_fwd", &attention_fwd);
  m.def("moe_tile_table", &moe_tile_table);
  m.def("quantize_mxfp8", &quantize_mxfp8);
  m.def("gemm_mxfp8", &gemm_mxfp8, py::arg("a"), py::arg("sfa"), py::arg("b"), py::arg("sfb"), py::arg("bias") = py::none());
  m.def("evoformer_attention_fwd", &evoformer_attention_fwd);
  m.def("evoformer_attention_bwd", &evoformer_attention_bwd);
  m.def("gemm_grouped", &gemm_grouped, py::arg("a"), py::arg("b"), py::arg("bias"), py::arg("tile_group"), py::arg("out"), py::arg("b_kmajor") = true,
        py::arg("epilogue") = 0, py::arg("out2") = py::none(), py::arg("aux") = py::none(), py::arg("row_align") = 128);
  m.def("gemm_grouped_wgrad", &gemm_grouped_wgrad);
  m.def("grouped_colsum", &grouped_colsum);
  m.def("tmap_cache_stats", []() { uint64_t h = 0, ms = 0; pfx::tmap_cache_stats(&h, &ms); return std::make_pair((int64_t)h, (int64_t)ms); });
  m.def("embedding_fwd", &embedding_fwd);
  m.def("embedding_bwd_", &embedding_bwd_);
  m.def("embedding_bwd_max_tokens", &embedding_bwd_max_tokens);
  m.def("attention_fwd_v2", &attention_fwd_v2);
  m.def("attention_bwd", &attention_bwd);
  m.def("attention_doc_bounds", &attention_doc_bounds);
  m.def("attention_fwd_doc", &attention_fwd_doc);
  m.def("attention_bwd_doc", &attention_bwd_doc);
  m.def("attention_decode", &attention_decode);
  m.def("attention_decode_packed", &attention_decode_packed);
  m.def("gemm_bias_gelu_dual", &gemm_bias_gelu_dual);
  m.def("gemm_dgelu", &gemm_dgelu, py::arg("dy"), py::arg("w"), py::arg("z"), py::arg("config") = 0);
  m.def("gemv_skinny", &gemv_skinny);
  m.def("gemm_smallm", &gemm_smallm);
  m.def("gemv_w8a8", &gemv_w8a8, py::arg("xq"), py::arg("wq"), py::arg("xs"), py::arg("ws"), py::arg("bias") = py::none(),
        py::arg("out_dtype") = py::none());
  m.def("gemv_fused", &gemv_fused);
  m.def("gemv_set_tuning", [](int64_t cols, int64_t split) { pfx::gemv_set_tuning((int)cols, (int)split); });
  m.def("moe_route", &moe_route);
  m.def("moe_dispatch", &moe_dispatch);
  m.def("moe_combine", &moe_combine);
  m.def("adamw_p2p_broadcast_", &adamw_p2p_broadcast_);
  m.def("vmm_caps", &vmm_caps);
  m.def("vmm_mc_granularity", &vmm_mc_granularity);
  m.def("vmm_arena_alloc", &vmm_arena_alloc);
  m.def("vmm_arena_import", &vmm_arena_import);
  m.def("vmm_mc_create", &vmm_mc_create);
  m.def("vmm_mc_import", &vmm_mc_import);
  m.def("vmm_mc_add_device", &vmm_mc_add_device);
  m.def("vmm_mc_bind_and_map", &vmm_mc_bind_and_map);
  m.def("vmm_unmap", &vmm_unmap);
  m.def("nvls_barrier", &nvls_barrier);
  m.def("p2p_flag_barrier", &p2p_flag_barrier);
  m.def("symm_reduce_scatter", &symm_reduce_scatter);
  m.def("symm_all_gather", &symm_all_gather);
  m.def("adamw_symm_broadcast_", &adamw_symm_broadcast_);
}
