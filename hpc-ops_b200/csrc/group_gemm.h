// Internal C++ interface of the grouped FP8 and bf16 GEMMs (used by the FusedMoE pipeline launchers).
#pragma once
#include <cuda_runtime.h>

namespace b200 {
namespace ggemm {
// mode bits: 1 = blockwise scales, 2 = fused SiLU*mul + quant epilogue
int run(int mode, const void* x, const void* w, const int* seqlens, const int* cu_seqlens,
        const float* xscale_t, const float* wscale, const float* act_scale, void* y, void* q_out,
        float* q_scale_t, int num_group, int m, int n, int k, int m_pad, int kpad4, int scale_tile,
        int use_bf16_mul, cudaStream_t stream);
int scale_tile_from_avg(int avg);
// bf16 X [m, k] . W[g]^T (W [num_group, n, k]) -> bf16 y [m, n]; fused: n = 2*I gate then up rows,
// y = bf16(silu(bf16(gate)) * bf16(up)) [m, I] (group_gemm_bf16.cu)
int run_bf16(bool fused, const void* x, const void* w, const int* seqlens, const int* cu_seqlens,
             void* y, int num_group, int m, int n, int k, cudaStream_t stream);
}  // namespace ggemm
}  // namespace b200
