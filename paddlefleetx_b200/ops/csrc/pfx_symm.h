// Symmetric-memory runtime (symm_vmm.cpp) and the NVLS / peer-memory collective kernels built on it (comm_nvls.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <string>

namespace pfx {
namespace vmm {

struct Caps {
  bool vmm = false;          // cuMem* virtual memory management
  bool fd_export = false;    // POSIX file-descriptor shareable handles
  bool multicast = false;    // NVLink-SHARP multicast objects (multimem.* instructions)
  size_t granularity = 0;    // recommended physical allocation granularity
};
Caps query_caps();
size_t multicast_granularity(int world, size_t bytes, bool recommended);

// Physical allocation of `bytes` (a multiple of the granularity) on the current device, mapped read/write, zero-filled;
// returns its base address and an exportable file descriptor (caller closes it after the peers imported it).
bool arena_alloc(size_t bytes, int64_t* ptr, int* fd, std::string* err);
// Map a peer's allocation (received fd) into this process.
bool arena_import(int fd, size_t bytes, int64_t* ptr, std::string* err);
// Multicast object life cycle: create (one rank) / import (the others) -> add_device (all) -> [group barrier] ->
// bind_and_map (all; binds the local arena at offset 0 and maps the multicast address range).
bool mc_create(size_t bytes, int world, int64_t* mc_id, int* fd, std::string* err);
bool mc_import(int fd, int64_t* mc_id, std::string* err);
bool mc_add_device(int64_t mc_id, std::string* err);
bool mc_bind_and_map(int64_t mc_id, int64_t local_arena_ptr, size_t bytes, int64_t* mc_ptr, std::string* err);
void unmap(int64_t ptr);

}  // namespace vmm

// ---- comm_nvls.cu: collectives over multicast (NVLS) and unicast peer addresses; dtype codes 0 = fp16, 1 = bf16, 3 = fp32.
// All kernels use <= 64 registers / thread, 256 threads and no shared memory beyond a few words to stay small; beside
// the wgmma GEMM CTA (288 threads x 168 registers) they do not fit on the same SM any more (see comm_nvls.cu).

// Barrier over the group on the stream: one multimem.red (+1 on every rank's flag) and a local spin until `target` arrivals.
cudaError_t nvls_barrier(uint32_t* mc_flag, uint32_t* local_flag, uint32_t target, cudaStream_t st);
// Unicast fallback: store `epoch` into slot [rank] of every peer's flag row, wait until all slots of the local row reach it.
cudaError_t p2p_flag_barrier(uint32_t** peer_flags, int rank, int world, uint32_t epoch, cudaStream_t st);

// out[i] = scale * sum_r buf_r[shard_offset + i]  for the calling rank's shard; in-switch reduction when `mc_src` is set
// (multimem.ld_reduce, fp32 accumulation), pull over unicast peer pointers otherwise.  Optionally accumulates the sum of
// squares of the (scaled) result into `sumsq` (grad-norm without another pass) and/or adds into `out` (gradient accumulation).
cudaError_t symm_reduce_scatter(const void* mc_src, void* const* peer_src, size_t shard_offset_elems, void* out, size_t n, int rank, int world,
                                int in_dtype, int out_dtype, float scale, bool accumulate, float* sumsq, int num_ctas, cudaStream_t st);
// dst_r[dst_offset + i] = src[i] on every rank r (multimem.st when `mc_dst` is set, posted unicast stores otherwise).
cudaError_t symm_all_gather(void* mc_dst, void* const* peer_dst, size_t dst_offset_bytes, const void* src, size_t bytes, int rank, int world,
                            int num_ctas, cudaStream_t st);
// AdamW on the owner's fp32 master shard; the new low-precision weights are stored ONCE to the multicast address (the
// switch replicates them into every rank's parameter buffer) or to each peer (unicast fallback): update + all-gather in
// one kernel.
cudaError_t adamw_symm_broadcast(void* mc_params, void* const* peer_params, size_t shard_offset_elems, float* master, const void* grad, float* m,
                                 float* v, size_t n, float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2,
                                 const float* gscale, const float* found_inf, int grad_dtype, int lp_dtype, int rank, int world, int num_ctas,
                                 cudaStream_t st);

}  // namespace pfx
