// Fused RMSNorm -> FP8 (H100 / sm_90a): the prologue that produces the e4m3 activations of the
// per-tensor FP8 GEMMs and the per-tensor FusedMoE. HBM-streaming: every row is read once with
// 16-byte loads and kept in registers.
//
//   fused_rmsnorm_with_scale : x bf16 [T, H], w bf16 [H], scale f32 [1] (or [2] with is_moe)
//     r  = rsqrtf(sum(x^2) / H + eps)          (fp32 sum of squares)
//     y  = (x * w) * r                          (fp32)
//     q0 = e4m3_rn_satfinite(y * (1 / scale[0]))
//     is_moe: also y as fp32 and q1 = e4m3_rn_satfinite(y * (1 / scale[1]))
//   (reference src/normalization/fused_rmsnorm_with_scale.cu, which supports H 320 / 4096 / 5120
//   only and folds 1/scale into r; the order here is fixed so that q0 is the same byte whether or
//   not is_moe is set.)
//
// Layout: 256 threads per CTA, `kWpr` warps per row, 8 / kWpr rows per CTA, each thread holding
// `kIter` 16-byte vectors (8 elements) of its row. kWpr is the smallest of 1, 2, 4, 8 that keeps
// kIter <= 4 (kIter reaches 8 only at H > 8192 with 8 warps), so short rows pack many rows into a
// CTA and long rows spread over more warps instead of more registers.
#include <cuda_bf16.h>

#include "common.cuh"
#include "host_utils.h"

namespace b200 {
namespace norm {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxHidden = 16384;

template <int kIter, int kWpr, bool kMoe>
__global__ void __launch_bounds__(kThreads)
    rmsnorm_quant_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                         uint8_t* __restrict__ q0, float* __restrict__ y32, uint8_t* __restrict__ q1,
                         const float* __restrict__ scale, float eps, int rows, int hidden) {
  constexpr int kRowThreads = kWpr * 32;
  __shared__ float red[kWarps];
  const int warp = threadIdx.x >> 5;
  const int sub = threadIdx.x % kRowThreads;  // thread index within its row
  const long long row = static_cast<long long>(blockIdx.x) * (kWarps / kWpr) + warp / kWpr;
  const int nvec = hidden >> 3;
  const bool live = row < rows;
  const __nv_bfloat16* xr = x + row * hidden;

  uint4 xv[kIter], wv[kIter];
#pragma unroll
  for (int i = 0; i < kIter; i++) {
    const int v = sub + i * kRowThreads;
    xv[i] = make_uint4(0, 0, 0, 0);
    wv[i] = make_uint4(0, 0, 0, 0);
    if (live && v < nvec) {
      xv[i] = ld_nc_v4(xr + v * 8);
      wv[i] = *reinterpret_cast<const uint4*>(w + v * 8);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kIter; i++) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&xv[i]);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __bfloat1622float2(h[j]);
      ss = __fmaf_rn(f.x, f.x, ss);
      ss = __fmaf_rn(f.y, f.y, ss);
    }
  }
  // warp sum, then (rows spanning warps) the row's warp partials in warp order, as stem.cu's
  // block_sum_256 does for a whole CTA: every thread of a row ends with the same bits
  ss = warp_sum_f32(ss);
  if constexpr (kWpr > 1) {
    if ((threadIdx.x & 31) == 0) red[warp] = ss;
    __syncthreads();
    const int first = warp - warp % kWpr;
    ss = 0.f;
#pragma unroll
    for (int k = 0; k < kWpr; k++) ss += red[first + k];
  }
  if (!live) return;
  const float r = rsqrtf(ss / static_cast<float>(hidden) + eps);
  const float inv0 = 1.0f / __ldg(scale);
  const float inv1 = kMoe ? 1.0f / __ldg(scale + 1) : 0.f;

#pragma unroll
  for (int i = 0; i < kIter; i++) {
    const int v = sub + i * kRowThreads;
    if (v >= nvec) break;
    const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xv[i]);
    const __nv_bfloat162* wh = reinterpret_cast<const __nv_bfloat162*>(&wv[i]);
    float y[8];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 xf = __bfloat1622float2(xh[j]);
      const float2 wf = __bfloat1622float2(wh[j]);
      y[2 * j] = __fmul_rn(__fmul_rn(xf.x, wf.x), r);
      y[2 * j + 1] = __fmul_rn(__fmul_rn(xf.y, wf.y), r);
    }
    const long long off = row * hidden + v * 8;
    uint2 o;
    o.x = cvt_e4m3x4(y[0] * inv0, y[1] * inv0, y[2] * inv0, y[3] * inv0);
    o.y = cvt_e4m3x4(y[4] * inv0, y[5] * inv0, y[6] * inv0, y[7] * inv0);
    *reinterpret_cast<uint2*>(q0 + off) = o;
    if constexpr (kMoe) {
      float4* yp = reinterpret_cast<float4*>(y32 + off);
      yp[0] = make_float4(y[0], y[1], y[2], y[3]);
      yp[1] = make_float4(y[4], y[5], y[6], y[7]);
      o.x = cvt_e4m3x4(y[0] * inv1, y[1] * inv1, y[2] * inv1, y[3] * inv1);
      o.y = cvt_e4m3x4(y[4] * inv1, y[5] * inv1, y[6] * inv1, y[7] * inv1);
      *reinterpret_cast<uint2*>(q1 + off) = o;
    }
  }
}

// warps per row for a hidden size: the smallest of 1, 2, 4, 8 with at most 4 vectors per thread
static int warps_per_row(int hidden) {
  const int nvec = hidden / 8;
  for (int wpr = 1; wpr < kWarps; wpr *= 2)
    if (nvec <= wpr * 32 * 4) return wpr;
  return kWarps;
}

template <int kIter, int kWpr>
static void launch(bool is_moe, int grid, cudaStream_t stream, const __nv_bfloat16* x,
                   const __nv_bfloat16* w, uint8_t* q0, float* y32, uint8_t* q1, const float* scale,
                   float eps, int rows, int hidden) {
  if (is_moe)
    rmsnorm_quant_kernel<kIter, kWpr, true>
        <<<grid, kThreads, 0, stream>>>(x, w, q0, y32, q1, scale, eps, rows, hidden);
  else
    rmsnorm_quant_kernel<kIter, kWpr, false>
        <<<grid, kThreads, 0, stream>>>(x, w, q0, y32, q1, scale, eps, rows, hidden);
}

}  // namespace norm
}  // namespace b200

using namespace b200;  // NOLINT

// replaces reference src/normalization/fused_rmsnorm_with_scale.h (fused_rmsnorm_with_scale_async).
// output_fp32 / output_fp8_scale2 are written (and required) only with is_moe.
extern "C" int hpc_fused_rmsnorm_with_scale_async(const void* input_ptr, const void* weight_ptr,
                                                  void* output_ptr, void* output_fp32_ptr,
                                                  void* output_fp8_scale2_ptr, const void* scale_ptr,
                                                  float eps, int batch_size, int hidden_state,
                                                  int is_moe, cudaStream_t stream) {
  HPC_REQUIRE(hidden_state >= 8 && hidden_state % 8 == 0,
              "fused_rmsnorm_with_scale: hidden size %d must be a positive multiple of 8",
              hidden_state);
  HPC_REQUIRE(hidden_state <= norm::kMaxHidden,
              "fused_rmsnorm_with_scale: hidden size %d exceeds the supported maximum of %d",
              hidden_state, norm::kMaxHidden);
  HPC_REQUIRE(batch_size >= 0, "fused_rmsnorm_with_scale: negative batch size %d", batch_size);
  HPC_REQUIRE(!is_moe || (output_fp32_ptr != nullptr && output_fp8_scale2_ptr != nullptr),
              "fused_rmsnorm_with_scale: is_moe needs the fp32 and second fp8 outputs");
  auto al = [](const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
  HPC_REQUIRE(al(input_ptr, 16) && al(weight_ptr, 16) && al(output_ptr, 8) &&
                  (!is_moe || (al(output_fp32_ptr, 16) && al(output_fp8_scale2_ptr, 8))),
              "fused_rmsnorm_with_scale: input and weight must be 16-byte aligned, fp8 outputs "
              "8-byte and the fp32 output 16-byte aligned");
  if (batch_size == 0) return HPC_OK;
  const int wpr = norm::warps_per_row(hidden_state);
  const int iters = (hidden_state / 8 + wpr * 32 - 1) / (wpr * 32);
  const int grid = (batch_size + (norm::kWarps / wpr) - 1) / (norm::kWarps / wpr);
  const auto* x = static_cast<const __nv_bfloat16*>(input_ptr);
  const auto* w = static_cast<const __nv_bfloat16*>(weight_ptr);
  auto* q0 = static_cast<uint8_t*>(output_ptr);
  auto* y32 = static_cast<float*>(output_fp32_ptr);
  auto* q1 = static_cast<uint8_t*>(output_fp8_scale2_ptr);
  const auto* sc = static_cast<const float*>(scale_ptr);
  const bool moe = is_moe != 0;
#define HPC_NORM_LAUNCH(I, W) norm::launch<I, W>(moe, grid, stream, x, w, q0, y32, q1, sc, eps, batch_size, hidden_state)
  switch (wpr * 16 + iters) {
    case 1 * 16 + 1: HPC_NORM_LAUNCH(1, 1); break;
    case 1 * 16 + 2: HPC_NORM_LAUNCH(2, 1); break;
    case 1 * 16 + 3: HPC_NORM_LAUNCH(3, 1); break;
    case 1 * 16 + 4: HPC_NORM_LAUNCH(4, 1); break;
    case 2 * 16 + 3: HPC_NORM_LAUNCH(3, 2); break;
    case 2 * 16 + 4: HPC_NORM_LAUNCH(4, 2); break;
    case 4 * 16 + 3: HPC_NORM_LAUNCH(3, 4); break;
    case 4 * 16 + 4: HPC_NORM_LAUNCH(4, 4); break;
    case 8 * 16 + 3: HPC_NORM_LAUNCH(3, 8); break;
    case 8 * 16 + 4: HPC_NORM_LAUNCH(4, 8); break;
    case 8 * 16 + 5: HPC_NORM_LAUNCH(5, 8); break;
    case 8 * 16 + 6: HPC_NORM_LAUNCH(6, 8); break;
    case 8 * 16 + 7: HPC_NORM_LAUNCH(7, 8); break;
    case 8 * 16 + 8: HPC_NORM_LAUNCH(8, 8); break;
    default:
      HPC_REQUIRE(false, "fused_rmsnorm_with_scale: no kernel for hidden size %d", hidden_state);
  }
#undef HPC_NORM_LAUNCH
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}
