// Host-side helpers shared by the C-ABI launchers: error reporting, device queries, TMA descriptors.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>

#include "../../include/hpc_b200.h"

namespace b200 {

void set_last_error(const char* fmt, ...);

#define HPC_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      b200::set_last_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,          \
                           cudaGetErrorString(_e));                                       \
      return HPC_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define HPC_REQUIRE(cond, ...)             \
  do {                                     \
    if (!(cond)) {                         \
      b200::set_last_error(__VA_ARGS__);   \
      return HPC_ERR_UNSUPPORTED;          \
    }                                      \
  } while (0)

int sm_count();
// HPC_B200_PDL=0 turns programmatic dependent launch off (plain stream order), default on.
bool pdl_enabled();
// Two zeroed int32 (work counter, finished-CTA counter) for kernels that re-arm their scheduler
// themselves (the last CTA resets both): no memset between launches, so PDL chains and graph
// replays are unaffected. Outside a capture there is one pair per (device, stream) for the life of
// the process, and one per host thread for cudaStreamPerThread, whose handle value every thread
// shares. Launches on one stream are serialised (a PDL successor claims work only after its
// pdl_wait()), so the pair is never used by two running kernels. A stream handle that CUDA reuses
// after cudaStreamDestroy inherits the pair, which is safe once the old stream's work has finished.
// A launch being captured into a CUDA graph gets a pair of its own, which the graph keeps; graphs
// may then be replayed on any streams at once. Safe to call during a capture, including a
// process's first call.
int* scheduler_counter(cudaStream_t stream);
// Sixteen zeroed bytes (two pairs, 8-byte aligned) handed out exactly as scheduler_counter, from a
// table of their own, for state a kernel keeps across launches on one stream. `*serial` (if not
// null) receives the block's number, unique in the process and the same on every call for a stream.
int* stream_state(cudaStream_t stream, uint64_t* serial);

// Encode a tiled TMA descriptor (uint8 elements). dims/strides innermost-first; strides in bytes for
// dims 1..rank-1. Returns 0 on success.
int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle,
                   CUtensorMapL2promotion promo = CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
// Same for 2-byte and 4-byte element types.
int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes, const void* base,
                int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                CUtensorMapSwizzle swizzle,
                CUtensorMapL2promotion promo = CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
// TMA descriptor of one paged K or V cache with a head dim of 128: `num_blocks` pages of `page`
// tokens x `heads` heads, strides in elements. A box is one head's `page` token rows of 128 bytes
// (the whole head dim for fp8, one half of it for bf16), 128B swizzle. The dimension order follows
// the strides, which TMA wants ascending: (d, head, token, blk) for token-major (NHD) caches, with
// *head_first = 1, and (d, token, head, blk) for head-major (HND) ones; the smem image is the same.
int encode_paged_kv_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes,
                         const void* base, int heads, int page, int num_blocks, int64_t blk_stride,
                         int64_t tok_stride, int64_t head_stride, int* head_first);

// Makes sure `kern` may use `bytes` of dynamic shared memory on the current device: calls
// cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) only when no call
// for this (kernel, device) has set at least `bytes` yet. Keyed by the kernel's address, so every
// template instantiation is set on its own.
cudaError_t set_max_dynamic_smem(const void* kern, int bytes);

// Launch `kern` so that it may start before the previous kernel in `stream` has finished
// (programmatic dependent launch; the kernel calls pdl_wait() before touching global memory).
// `cluster_x` > 1 additionally launches thread-block clusters of that size.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    n++;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = static_cast<unsigned>(cluster_x);
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    n++;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace b200
