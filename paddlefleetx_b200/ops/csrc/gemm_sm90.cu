// Persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] (+)= A[M,K] * B[N,K]^T  (+ bias[N]) (-> GELU)
//
//   * operands bf16 (or fp16), fp32 accumulation in registers, output bf16 (TMA store) or fp32 (direct,
//     optionally accumulating into the destination = fused main-grad accumulation for wgrad).
//   * A and B may each be K-major (row-major [rows, K]) or MN-major (row-major [K, rows]) so the
//     forward (X W^T), dgrad (dY W) and wgrad (dY^T X) GEMMs of a Linear layer all run without a
//     transpose pass (wgmma reads 16-bit operands of either major from 128-byte-swizzled shared memory).
//   * warp roles: warp 8 = TMA producer (mbarrier ring of 128 x 64 / BLOCK_N x 64 stages), warps 0-7 = two consumer
//     warpgroups, each wgmma m64 x BLOCK_N x 16 over its 64 rows of the 128 x BLOCK_N tile, then the epilogue from its
//     accumulator fragment (registers -> swizzled smem -> TMA store).  One k-block of wgmma stays in flight while the next
//     is issued; the producer runs ahead into the next tile during the epilogue.
//
// Fused compute+collective modes (tensor/sequence parallel linears, see parallel/fused_tp.py):
//   * kOutMode = 3  "GEMM -> reduce-scatter": the epilogue stores each finished tile straight into the DESTINATION
//     rank's staging buffer through its NVLink-mapped (CUDA IPC) address — slot [src_rank][row_in_shard][N] — tile
//     by tile while the mainloop keeps the tensor cores busy; tiles for remote ranks are scheduled first.  A small
//     reduce kernel (comm_p2p.cu) then sums the world slots.
//   * comm.ag_world > 1  "all-gather -> GEMM": extra CTAs of the SAME kernel push this rank's A shard into every
//     peer's gathered buffer (posted P2P stores) and raise per-chunk flags; the TMA producer of each GEMM CTA
//     waits on the flag of the chunk it is about to load.  Local-shard tiles are issued first so the mainloop
//     starts immediately and the transfer hides behind it.
//
// This is the kernel every Linear layer of the framework runs on (reference call sites L1-L5 in
// SURVEY §2.6: QKV / out-proj / FFN1 / FFN2 / LM head use cuBLAS(Lt) in the reference).
#include "pfx_ptx.cuh"
#include "pfx_gemm.h"
#include <cudaTypedefs.h>
#include <cstdio>

namespace pfx {

constexpr int kBlockM = 128;   // rows of A per CTA: two consumer warpgroups of 64 rows each
constexpr int kBlockK = 64;    // 64 x 2 B = one 128-byte swizzle span
constexpr int kMmaK = 16;
constexpr int kNumConsumerWarps = 8;
constexpr int kNumThreads = 288;   // warps 0-7 = two consumer warpgroups, warp 8 = TMA producer (ptxas allots 168 registers per thread)
constexpr int kGroupM = 16;    // tile-raster group height (L2 reuse)
constexpr int kStoreCols = 64; // columns per TMA-store box (128 B of bf16)

template <int kBlockN>
struct GemmSmem {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = kBlockN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = kBlockM * kStoreCols * 2;   // one store box
  static constexpr int kNumEpiBufs = 2;
  static constexpr int kBarrierBytes = 1024;
  // 12 KB of the SM's 228 KB stay free: a co-resident communication / optimizer CTA needs its own 1 KB system reservation (plus any static
  // shared memory), and a GEMM that fills the SM to the last kilobyte serialises with every kernel on the side streams instead of sharing it.
  static constexpr int kHeadroom = 12 * 1024;
  static constexpr int kBudget = 227 * 1024 - kHeadroom - 1024 /*align slack*/ - kBarrierBytes - kNumEpiBufs * kEpiBytes;
  static constexpr int kStages = (kBudget / kStageBytes) > 8 ? 8 : (kBudget / kStageBytes);
  static constexpr int kTotal = 1024 + kStages * kStageBytes + kNumEpiBufs * kEpiBytes + kBarrierBytes;
};

struct TileCoord { int m_blk, n_blk; };
struct alignas(64) PeerMaps { CUtensorMap m[8]; };   // per-destination-rank staging tensor maps (GEMM -> reduce-scatter)

__device__ __forceinline__ TileCoord tile_coord(int tile, int num_m_blocks, int num_n_blocks, int m_rotate = 0) {
  const int tiles_per_group = kGroupM * num_n_blocks;
  const int group = tile / tiles_per_group;
  const int first_m = group * kGroupM;
  const int group_m = min(kGroupM, num_m_blocks - first_m);
  const int in_group = tile - group * tiles_per_group;
  int m = first_m + in_group % group_m;
  if (m_rotate) { m += m_rotate; if (m >= num_m_blocks) m -= num_m_blocks; }
  return {m, in_group / group_m};
}

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Communication role of the all-gather->GEMM mode: push rows [my_rank*rows_per_rank, +rows_per_rank) of A (local
// shard, row stride K elements) into every peer's gathered buffer, chunk by chunk, then publish the chunk flag.
__device__ void ag_push_role(const GemmComm& c, int comm_cta, int num_comm_ctas, int K) {
  const int chunk_rows = c.chunk_rows;
  const int chunks = c.rows_per_rank / chunk_rows;
  const size_t vec_per_row = (size_t)K * 2 / 16;
  const uint4* src = reinterpret_cast<const uint4*>(c.a_local);
  // work item = (chunk, peer): with W ranks a shard has only rows/chunk chunks but (W - 1) destinations each, so the items —
  // not the chunks — are spread over the communication CTAs (at W = 8 a chunk-per-CTA split left 12 of 16 CTAs idle and
  // serialised seven 2 MB pushes on each of the others)
  const int peers = c.ag_world - 1;
  for (int item = comm_cta; item < chunks * peers; item += num_comm_ctas) {
    const int ch = item / peers;
    const int dst = (c.my_rank + 1 + item % peers) % c.ag_world;
    const size_t v0 = (size_t)ch * chunk_rows * vec_per_row, nv = (size_t)chunk_rows * vec_per_row;
    uint4* out = reinterpret_cast<uint4*>(c.peer_gather[dst]) + (size_t)c.my_rank * c.rows_per_rank * vec_per_row + v0;
    for (size_t i = threadIdx.x; i < nv; i += 4 * blockDim.x) {
      uint4 r[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) if (i + u * blockDim.x < nv) r[u] = __ldg(src + v0 + i + u * blockDim.x);
#pragma unroll
      for (int u = 0; u < 4; ++u) if (i + u * blockDim.x < nv) out[i + u * blockDim.x] = r[u];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(c.peer_flags[dst] + c.my_rank * chunks + ch, c.epoch);
    __syncthreads();
  }
}

// kOutMode: 0 = bf16/fp16 via TMA store, 1 = fp32 direct store, 2 = fp32 direct accumulate (D += acc),
//           3 = bf16 scatter into the destination rank's staging buffer over NVLink (GEMM -> reduce-scatter)
template <int kBlockN, bool kAK, bool kBK, int kOutMode>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_a_local,
                  float* __restrict__ out_f32, const __nv_bfloat16* __restrict__ bias,
                  int M, int N, int K, int ldd, int epilogue, uint32_t ab_format, const __grid_constant__ GemmComm comm,
                  const __grid_constant__ PeerMaps peer_maps, const __grid_constant__ CUtensorMap tmap_d2,
                  const __nv_bfloat16* __restrict__ aux, int ld_aux, const __grid_constant__ GemmGroup grp) {
  using S = GemmSmem<kBlockN>;
  constexpr int kStages = S::kStages;
  static_assert(kStages >= 2, "pipeline needs at least two stages");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_ab = smem_base;
  const uint32_t smem_epi = smem_base + kStages * S::kStageBytes;
  const uint32_t smem_bar = smem_epi + S::kNumEpiBufs * S::kEpiBytes;
  auto full_bar = [&](int s) { return smem_bar + 8u * s; };
  auto empty_bar = [&](int s) { return smem_bar + 8u * (kStages + s); };

  const uint32_t warp = warp_id();
  const uint32_t lane = lane_id();

  const int num_m_blocks = (M + kBlockM - 1) / kBlockM;
  const int num_n_blocks = (N + kBlockN - 1) / kBlockN;
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int num_k_blocks = (K + kBlockK - 1) / kBlockK;
  const int num_comm_ctas = comm.ag_world > 1 ? comm.num_comm_ctas : 0;
  const int num_ctas = (int)gridDim.x - num_comm_ctas;
  const int cta_id = blockIdx.x;
  if (cta_id >= num_ctas) {   // ---- communication CTAs (all-gather -> GEMM mode): no barriers
    ag_push_role(comm, cta_id - num_ctas, num_comm_ctas, K);
    return;
  }
  int m_rotate = 0;
  if (comm.rows_per_rank > 0 && comm.world > 1) {   // start one rank "after" ourselves: remote tiles first (RS) /
    const int blocks_per_rank = comm.rows_per_rank / kBlockM;                 // local tiles first (AG)
    m_rotate = ((comm.my_rank + (kOutMode == 3 ? 1 : 0)) % comm.world) * blocks_per_rank;
  }

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (kOutMode == 0) tma_prefetch_desc(&tmap_d);
    if (kOutMode == 3) { for (int i = 0; i < comm.world; ++i) tma_prefetch_desc(&peer_maps.m[i]); }
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kNumConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== TMA producer
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = cta_id; tile < num_tiles; tile += num_ctas) {
        const TileCoord tc = tile_coord(tile, num_m_blocks, num_n_blocks, m_rotate);
        int m_idx = tc.m_blk * kBlockM;
        const int n_idx = tc.n_blk * kBlockN;
        int tile_k_blocks = num_k_blocks, k_base = 0, b_row_off = 0;
        if (grp.mode == 1) {          // the expert that owns this row block selects the slice of the stacked B operand
          const int g = __ldg(grp.tile_group + tc.m_blk);
          if (g < 0) continue;
          b_row_off = g * grp.b_group_stride;
        } else if (grp.mode == 2) {   // the tile's expert selects the K (token-row) range; A is addressed inside the expert's [rows, m_per_group]
          const int g = (tc.m_blk * kBlockM) / grp.m_per_group;
          k_base = __ldg(grp.seg + 2 * g);
          tile_k_blocks = __ldg(grp.seg + 2 * g + 1) / kBlockK;
          m_idx -= g * grp.m_per_group;
        }
        for (int kb = 0; kb < tile_k_blocks; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_ab + stage * S::kStageBytes;
          const uint32_t sb = sa + S::kABytes;
          const uint32_t fb = full_bar(stage);
          const int k_idx = k_base + kb * kBlockK;
          mbar_arrive_expect_tx(fb, S::kStageBytes);
          if constexpr (kAK) {
            if (comm.ag_world > 1) {
              const int src_rank = m_idx / comm.rows_per_rank;
              if (src_rank == comm.my_rank) {
                tma_load_2d(&tmap_a_local, fb, sa, k_idx, m_idx - src_rank * comm.rows_per_rank);
              } else {
                if (kb == 0) {   // first touch of this m-block: wait until the owner has pushed the chunk
                  const int chunks = comm.rows_per_rank / comm.chunk_rows;
                  const uint32_t* fl = comm.my_flags + src_rank * chunks + (m_idx - src_rank * comm.rows_per_rank) / comm.chunk_rows;
                  const long long t0 = clock64();
                  while ((int32_t)(ld_acquire_sys(fl) - comm.epoch) < 0) {   // epochs only grow
                    if (clock64() - t0 > 20000000000ll) __trap();   // all-gather flag timeout (no printf: see mbar_wait)
                  }
                }
                tma_load_2d(&tmap_a, fb, sa, k_idx, m_idx);
              }
            } else {
              tma_load_2d(&tmap_a, fb, sa, k_idx, m_idx);
            }
          } else {
#pragma unroll
            for (int j = 0; j < kBlockM / 64; ++j) tma_load_2d(&tmap_a, fb, sa + j * 8192, m_idx + j * 64, k_idx);
          }
          if constexpr (kBK) {
            tma_load_2d(&tmap_b, fb, sb, k_idx, n_idx + b_row_off);
          } else {
#pragma unroll
            for (int j = 0; j < kBlockN / 64; ++j) tma_load_2d(&tmap_b, fb, sb + j * 8192, n_idx + j * 64, k_idx + b_row_off);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================================================================== consumers: mainloop (wgmma) + epilogue, 64 rows per warpgroup
    const uint32_t wg = warp >> 2;
    const uint32_t row_lo = wg * 64u + (warp & 3u) * 16u + (lane >> 2);   // this thread's rows inside the CTA tile: row_lo and row_lo + 8
    const uint32_t col_in8 = (lane & 3u) * 2u;                            // ... and its column pair inside every 8-column group
    const bool is_store_thread = threadIdx.x == 0;
    // K-major SW128: 8-row groups 1024 B apart.  MN-major SW128: 8-k groups 1024 B apart, 64-element
    // MN chunks (one TMA box of 64 k-rows x 128 B) 8192 B apart.
    constexpr uint64_t kDescA = kAK ? wgmma_desc_hi_lo(16, 1024) : wgmma_desc_hi_lo(8192, 1024);
    constexpr uint64_t kDescB = kBK ? wgmma_desc_hi_lo(16, 1024) : wgmma_desc_hi_lo(8192, 1024);
    constexpr uint32_t kAdvA = kAK ? (kMmaK * 2) : (kMmaK * 128);   // bytes per K = 16 step
    constexpr uint32_t kAdvB = kBK ? (kMmaK * 2) : (kMmaK * 128);
    int stage = 0; uint32_t phase = 0;
    uint32_t store_iter = 0;
    float acc[kBlockN / 2];
    for (int tile = cta_id; tile < num_tiles; tile += num_ctas) {
      const TileCoord tc = tile_coord(tile, num_m_blocks, num_n_blocks, m_rotate);
      const int row0 = tc.m_blk * kBlockM;
      const int col_tile = tc.n_blk * kBlockN;
      const __nv_bfloat16* tile_bias = bias;
      int tile_k_blocks = num_k_blocks;
      if (grp.mode == 1) {
        const int g = __ldg(grp.tile_group + tc.m_blk);
        if (g < 0) continue;
        if (bias != nullptr) tile_bias = bias + (size_t)g * N;
      } else if (grp.mode == 2) {
        tile_k_blocks = __ldg(grp.seg + 2 * ((tc.m_blk * kBlockM) / grp.m_per_group) + 1) / kBlockK;
      }
      const bool empty_k = tile_k_blocks == 0;   // K-grouped tile of an expert without tokens: the accumulator was never written, the result is zero
      int prev_stage = -1;
      for (int kb = 0; kb < tile_k_blocks; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa = smem_ab + stage * S::kStageBytes + wg * 8192u;   // this warpgroup's 64 rows (K-major) / 64-row chunk (MN-major)
        const uint32_t sb = smem_ab + stage * S::kStageBytes + S::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
          const uint64_t da = wgmma_desc(sa + k * kAdvA, kDescA);
          const uint64_t db = wgmma_desc(sb + k * kAdvB, kDescB);
          if (ab_format == 1) WgmmaSS<kBlockN, true, !kAK, !kBK>::mma(acc, da, db, (kb | k) != 0 ? 1u : 0u);
          else WgmmaSS<kBlockN, false, !kAK, !kBK>::mma(acc, da, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (prev_stage >= 0) {   // one k-block stays in flight: the previous one has retired, hand its stage back to the producer
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(empty_bar(prev_stage));
        }
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));

#pragma unroll
      for (int c = 0; c < kBlockN / kStoreCols; ++c) {
        const int col0 = col_tile + c * kStoreCols;
        const int cb = col0 + (int)col_in8;       // column of v[4 j] / v[4 j + 2]; v[4 j + 1] / v[4 j + 3] are one to the right
        float v[32];                              // v[4 j + e]: row row_lo + 8 (e / 2), column cb + 8 j + (e % 2)
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = empty_k ? 0.f : acc[c * 32 + i];
        if (epilogue == EPI_BIAS || epilogue == EPI_BIAS_GELU || epilogue == EPI_BIAS_GELU_DUAL) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (cb + 8 * j < N) {   // N % 8 == 0 is required by the host wrapper
              const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(tile_bias + cb + 8 * j));
              v[4 * j] += f.x; v[4 * j + 1] += f.y; v[4 * j + 2] += f.x; v[4 * j + 3] += f.y;
            }
          }
        }
        if (epilogue == EPI_BIAS_GELU || epilogue == EPI_GELU) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = gelu_tanh(v[i]);
        }
        if (epilogue == EPI_DGELU) {      // acc * gelu'(saved pre-activation)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int grow_aux = row0 + (int)row_lo + 8 * hh;
            if (grow_aux < M) {
              const __nv_bfloat16* ap = aux + (size_t)grow_aux * ld_aux + cb;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                if (cb + 8 * j < N) {
                  const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ap + 8 * j));
                  v[4 * j + 2 * hh] *= gelu_tanh_grad(f.x); v[4 * j + 2 * hh + 1] *= gelu_tanh_grad(f.y);
                }
              }
            }
          }
        }
        if constexpr (kOutMode == 0 || kOutMode == 3) {
          // pack v[] into the swizzled staging buffer and TMA-store it; called twice per chunk by the dual-output epilogue
          auto store_chunk = [&](const CUtensorMap* map_d) {
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
            for (int j = 0; j < 8; ++j) {
              uint32_t p;
              if (ab_format == 1) {
                p = pack_bf16x2(v[4 * j + 2 * hh], v[4 * j + 2 * hh + 1]);
              } else {
                __half2 h2 = __floats2half2_rn(v[4 * j + 2 * hh], v[4 * j + 2 * hh + 1]);
                p = *reinterpret_cast<uint32_t*>(&h2);
              }
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + (((uint32_t)j ^ (r & 7u)) << 4)), "r"(p) : "memory");
            }
          }
          fence_proxy_async_smem();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (is_store_thread) {
            if (col0 < N && row0 < M) {
              if constexpr (kOutMode == 3) {
                // tile -> owner rank's staging slot [my_rank] through its NVLink-mapped address (TMA store to peer memory)
                const int dst_rank = row0 / comm.rows_per_rank;
                tma_store_2d(&peer_maps.m[dst_rank], smem_epi + buf * S::kEpiBytes, col0,
                             comm.my_rank * comm.rows_per_rank + (row0 - dst_rank * comm.rows_per_rank));
              } else {
                tma_store_2d(map_d, smem_epi + buf * S::kEpiBytes, col0, row0);
              }
            }
            tma_store_commit();
          }
          ++store_iter;
          };
          store_chunk(&tmap_d);
          if (epilogue == EPI_BIAS_GELU_DUAL) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = gelu_tanh(v[i]);
            store_chunk(&tmap_d2);
          }
        } else {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int grow = row0 + (int)row_lo + 8 * hh;
            if (grow < M) {
              float* dst = out_f32 + (size_t)grow * ldd + cb;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                if (cb + 8 * j < N) {   // N % 4 == 0 required
                  float2 o = make_float2(v[4 * j + 2 * hh], v[4 * j + 2 * hh + 1]);
                  if constexpr (kOutMode == 2) {
                    const float2 old = *reinterpret_cast<const float2*>(dst + 8 * j);
                    o.x += old.x; o.y += old.y;
                  }
                  *reinterpret_cast<float2*>(dst + 8 * j) = o;
                }
              }
            }
          }
        }
      }
    }
    if ((kOutMode == 0 || kOutMode == 3) && is_store_thread) tma_store_wait<0>();
  }
}

// ============================================================================ host side
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult qres;
    void* p = nullptr;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || p == nullptr) return nullptr;
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// A tensor map is a pure function of (address, dtype, dims, strides, box, swizzle): it does not reference the allocation, so a descriptor
// encoded for one tensor is valid for any later tensor at the same address with the same geometry.  Training re-launches the same few
// hundred GEMM / attention shapes on allocator-recycled addresses every step, so a small direct-mapped, per-thread cache removes the
// 3-12 driver encode calls per launch (1-2 us each: invisible at 6.7B, a visible host cost on 345M / ViT / decode).
namespace {
struct TmapKey {
  uint64_t ptr, d0, d1, d2, s0, s1;
  uint32_t b0, b1, b2, kind;            // kind: dtype | swizzle << 8 | rank << 16
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && s0 == o.s0 && s1 == o.s1 && b0 == o.b0 && b1 == o.b1 && b2 == o.b2 && kind == o.kind;
  }
};
struct TmapSlot { TmapKey key; CUtensorMap map; bool valid; };
constexpr int kTmapCacheSlots = 2048;
uint64_t g_tmap_hits = 0, g_tmap_misses = 0;

inline uint64_t tmap_hash(const TmapKey& k) {
  uint64_t h = k.ptr * 0x9E3779B97F4A7C15ull;
  auto mix = [&](uint64_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); };
  mix(k.d0); mix(k.d1); mix(k.d2); mix(k.s0); mix(k.s1); mix(((uint64_t)k.b0 << 32) | k.b1); mix(((uint64_t)k.b2 << 32) | k.kind);
  return h ^ (h >> 29);
}

template <typename Encode>
inline bool tmap_cached(CUtensorMap* out, const TmapKey& key, Encode&& encode) {
  // cuTensorMapEncodeTiled is a DRIVER call: it fails with CUDA_ERROR_INVALID_CONTEXT on a thread that has not touched the runtime yet
  // (autograd's backward threads, when the caching allocator served every tensor without a runtime call).  Bind the primary context once.
  thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  thread_local TmapSlot* slots = new TmapSlot[kTmapCacheSlots]();
  TmapSlot& s = slots[tmap_hash(key) & (kTmapCacheSlots - 1)];
  if (s.valid && s.key == key) { *out = s.map; ++g_tmap_hits; return true; }
  if (!encode(&s.map)) { s.valid = false; return false; }
  s.key = key; s.valid = true; ++g_tmap_misses;
  *out = s.map;
  return true;
}
}  // namespace

void tmap_cache_stats(uint64_t* hits, uint64_t* misses) { *hits = g_tmap_hits; *misses = g_tmap_misses; }

// 2-D row-major tensor [outer, inner] (inner contiguous), 128-byte swizzle, box = [box_outer, box_inner].
bool make_tmap_2d(CUtensorMap* map, const void* ptr, int elem_bytes, int dtype_code, uint64_t inner, uint64_t outer,
                  uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer) {
  auto fn = get_encode_fn();
  if (!fn) return false;
  CUtensorMapDataType dt;
  switch (dtype_code) {
    case 0: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16; break;
    case 1: dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; break;
    case 2: dt = CU_TENSOR_MAP_DATA_TYPE_UINT8; break;
    default: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; break;
  }
  (void)elem_bytes;
  const TmapKey key{(uint64_t)ptr, inner, outer, 0, row_stride_bytes, 0, box_inner, box_outer, 0, (uint32_t)dtype_code | (1u << 8) | (2u << 16)};
  return tmap_cached(map, key, [&](CUtensorMap* m) {
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
      fprintf(stderr, "pfx: cuTensorMapEncodeTiled failed (%d): ptr %p dims {%llu, %llu} stride %llu box {%u, %u} dtype %d\n", (int)r, ptr,
              (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_stride_bytes, box_inner, box_outer, dtype_code);
    return r == CUDA_SUCCESS;
  });
}

bool make_tmap_2d_plain(CUtensorMap* map, const void* ptr, int dtype_code, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                        uint32_t box_inner, uint32_t box_outer) {
  auto fn = get_encode_fn();
  if (!fn) return false;
  const CUtensorMapDataType dt = dtype_code == 3 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : (dtype_code == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  const TmapKey key{(uint64_t)ptr, inner, outer, 0, row_stride_bytes, 0, box_inner, box_outer, 0, (uint32_t)dtype_code | (0u << 8) | (2u << 16)};
  return tmap_cached(map, key, [&](CUtensorMap* m) {
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    return fn(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  });
}

bool make_tmap_bshd(CUtensorMap* map, const void* ptr, int dtype_code, uint64_t inner, uint64_t S, uint64_t B, uint64_t s_stride_bytes,
                    uint64_t b_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool* swapped) {
  auto fn = get_encode_fn();
  if (!fn) return false;
  const CUtensorMapDataType dt = dtype_code == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const bool sw = B > 1 && b_stride_bytes < s_stride_bytes;
  if (swapped) *swapped = sw;
  const TmapKey key{(uint64_t)ptr, inner, S, B, s_stride_bytes, b_stride_bytes, box_cols, box_rows, 0, (uint32_t)dtype_code | (1u << 8) | (3u << 16)};
  return tmap_cached(map, key, [&](CUtensorMap* m) {
    cuuint64_t dims[3] = {inner, sw ? B : S, sw ? S : B};
    cuuint64_t strides[2] = {sw ? b_stride_bytes : s_stride_bytes, sw ? s_stride_bytes : b_stride_bytes};
    if (B == 1) strides[1] = strides[0] * dims[1];      // a unit dimension: any legal stride
    cuuint32_t box[3] = {box_cols, sw ? 1u : box_rows, sw ? box_rows : 1u};
    cuuint32_t estr[3] = {1, 1, 1};
    return fn(m, dt, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  });
}

// An argument combination the kernel family cannot run is a programming error upstream: say which check refused it (the bare
// "invalid argument" of the CUDA error string does not).
static cudaError_t gemm_reject(const GemmArgs& g, int block_n, int line) {
  fprintf(stderr, "pfx gemm: rejected at gemm_sm90.cu:%d  (M %d N %d K %d lda %d ldb %d ldd %d a_k %d b_k %d out_mode %d epilogue %d cfg 128x%d group mode %d "
                  "groups %d b_stride %d m_per_group %d row_align %d comm rows %d)\n", line, g.M, g.N, g.K, g.lda, g.ldb, g.ldd, (int)g.a_kmajor, (int)g.b_kmajor,
          g.out_mode, g.epilogue, block_n, g.group.mode, g.group.groups, g.group.b_group_stride, g.group.m_per_group, g.group.row_align, g.comm.rows_per_rank);
  return cudaErrorInvalidValue;
}

template <int kBlockN, bool kAK, bool kBK, int kOutMode>
static cudaError_t launch_cfg(const GemmArgs& g, cudaStream_t stream) {
  using S = GemmSmem<kBlockN>;
  CUtensorMap ta, tb, td;
  const int dt = g.ab_format;  // 0 = fp16, 1 = bf16
  bool ok = true;
  const GemmGroup& gg = g.group;
  if (gg.mode == 1) {
    if (gg.tile_group == nullptr || gg.groups < 1 || gg.row_align % kBlockM != 0 || g.comm.rows_per_rank > 0) return gemm_reject(g, kBlockN, __LINE__);
    if (gg.b_group_stride != (kBK ? g.N : g.K) || g.K % kBlockK != 0) return gemm_reject(g, kBlockN, __LINE__);
  } else if (gg.mode == 2) {
    if (kAK || kBK || gg.seg == nullptr || gg.groups < 1 || gg.m_per_group % kBlockM != 0 || g.M != gg.groups * gg.m_per_group ||
        g.comm.rows_per_rank > 0 || g.epilogue != EPI_NONE) return gemm_reject(g, kBlockN, __LINE__);
  }
  // grouped operands: B stacks the experts along its outer dimension (mode 1); A spans one expert's m_per_group columns (mode 2)
  const uint64_t a_mn = gg.mode == 2 ? (uint64_t)gg.m_per_group : (uint64_t)g.M;
  const uint64_t b_outer_k = gg.mode == 1 ? (uint64_t)gg.groups * g.N : (uint64_t)g.N;     // K-major B: rows
  const uint64_t b_outer_mn = gg.mode == 1 ? (uint64_t)gg.groups * g.K : (uint64_t)g.K;   // MN-major B: k rows
  if (kAK) ok &= make_tmap_2d(&ta, g.a, 2, dt, g.K, g.M, (uint64_t)g.lda * 2, kBlockK, kBlockM);
  else     ok &= make_tmap_2d(&ta, g.a, 2, dt, a_mn, g.K, (uint64_t)g.lda * 2, 64, kBlockK);
  if (kBK) ok &= make_tmap_2d(&tb, g.b, 2, dt, g.K, b_outer_k, (uint64_t)g.ldb * 2, kBlockK, kBlockN);
  else     ok &= make_tmap_2d(&tb, g.b, 2, dt, g.N, b_outer_mn, (uint64_t)g.ldb * 2, 64, kBlockK);
  if (kOutMode == 0) ok &= make_tmap_2d(&td, g.d, 2, dt, g.N, g.M, (uint64_t)g.ldd * 2, kStoreCols, kBlockM);
  else td = ta;
  CUtensorMap td2 = td;
  if (g.epilogue == EPI_BIAS_GELU_DUAL) {
    if (kOutMode != 0 || g.d2 == nullptr || g.bias == nullptr) return gemm_reject(g, kBlockN, __LINE__);
    ok &= make_tmap_2d(&td2, g.d2, 2, dt, g.N, g.M, (uint64_t)g.ldd * 2, kStoreCols, kBlockM);
  }
  if (g.epilogue == EPI_DGELU && (g.aux == nullptr || g.ld_aux % 8 || (reinterpret_cast<uintptr_t>(g.aux) & 15) || dt != 1)) return gemm_reject(g, kBlockN, __LINE__);
  PeerMaps pm;
  for (int i = 0; i < 8; ++i) pm.m[i] = ta;
  if (kOutMode == 3) {
    for (int i = 0; i < g.comm.world; ++i)
      ok &= make_tmap_2d(&pm.m[i], g.comm.peer_out[i], 2, dt, g.N, (uint64_t)g.comm.world * g.comm.rows_per_rank, (uint64_t)g.ldd * 2,
                         kStoreCols, kBlockM);
  }
  CUtensorMap tal = ta;
  if (g.comm.ag_world > 1) {
    if (!kAK) return gemm_reject(g, kBlockN, __LINE__);
    ok &= make_tmap_2d(&tal, g.comm.a_local, 2, dt, g.K, g.comm.rows_per_rank, (uint64_t)g.K * 2, kBlockK, kBlockM);
  }
  if (!ok) return gemm_reject(g, kBlockN, __LINE__);
  if (g.comm.rows_per_rank > 0 && (g.comm.rows_per_rank % kBlockM) != 0) return gemm_reject(g, kBlockN, __LINE__);

  auto kern = gemm_wgmma_kernel<kBlockN, kAK, kBK, kOutMode>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int num_m_blocks = (g.M + kBlockM - 1) / kBlockM;
  const int num_n_blocks = (g.N + kBlockN - 1) / kBlockN;
  const int tiles = num_m_blocks * num_n_blocks;
  const int comm_ctas = g.comm.ag_world > 1 ? g.comm.num_comm_ctas : 0;
  int ctas = g.num_sms - comm_ctas;
  if (ctas > tiles) ctas = tiles;
  if (ctas < 1) ctas = 1;
  ctas += comm_ctas;

  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(ctas);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = S::kTotal;
  cfg.stream = stream;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, kern, ta, tb, td, tal, reinterpret_cast<float*>(g.d), reinterpret_cast<const __nv_bfloat16*>(g.bias),
                            g.M, g.N, g.K, g.ldd, g.epilogue, (uint32_t)g.ab_format, g.comm, pm, td2,
                            reinterpret_cast<const __nv_bfloat16*>(g.aux), g.ld_aux, g.group);
  if (le != cudaSuccess) {
    fprintf(stderr, "pfx gemm: launch failed (%s): grid %d, smem %d B\n", cudaGetErrorString(le), ctas, S::kTotal);
    return gemm_reject(g, kBlockN, __LINE__);
  }
  return le;
}

template <int kBlockN, int kOutMode>
static cudaError_t launch_major(const GemmArgs& g, cudaStream_t s) {
  if (g.a_kmajor && g.b_kmajor) return launch_cfg<kBlockN, true, true, kOutMode>(g, s);
  if (g.a_kmajor && !g.b_kmajor) return launch_cfg<kBlockN, true, false, kOutMode>(g, s);
  if (!g.a_kmajor && g.b_kmajor) return launch_cfg<kBlockN, false, true, kOutMode>(g, s);
  return launch_cfg<kBlockN, false, false, kOutMode>(g, s);
}

template <int kBlockN>
static cudaError_t launch_out(const GemmArgs& g, cudaStream_t s) {
  switch (g.out_mode) {
    case 0: return launch_major<kBlockN, 0>(g, s);
    case 1: return launch_major<kBlockN, 1>(g, s);
    case 2: return launch_major<kBlockN, 2>(g, s);
    default: return launch_major<kBlockN, 3>(g, s);
  }
}

cudaError_t gemm_wgmma(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return cudaSuccess;
  return launch_out<128>(g, stream);   // 128 x 128 tiles: 64 accumulator registers per consumer thread (161-168 registers in all; four variants spill 32 bytes)
}

}  // namespace pfx
