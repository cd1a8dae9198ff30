// Stand-alone activation / quantisation helpers of the MoE path (H100 / sm_90a) — pure HBM-bound
// streaming kernels, 16-byte vector loads, grid = multiple of the SM count.
//
//   act_mul_and_quant : out[r, c] = e4m3( silu(gate[r, c]) * up[r, c] * scale )      gate_up bf16 [R, 2C]
//                       (reference src/activation/activation.cu:19-136, launcher :528-625; in the
//                       fused MoE pipeline this work is the epilogue of the Gate-Up GEMM instead)
//   scaled_fp8_quant  : out[i] = e4m3( in[i] * (1 / scale) )                          in f32 / f16 / bf16
//                       (reference src/activation/activation.cu:461-500, launcher :783-804)
//   masked_act_mul_and_quant / masked_act_mul_and_blockwise_quant : the same silu(gate) * up over
//                       the per-expert padded (DeepEP low-latency) layout [E * T_max, 2C], valid rows
//                       only, per-tensor or 1x128 blockwise e4m3 (reference activation.cu:203-280 and
//                       :358-433; there every thread visits every padded row)
//   blockwise_fp8_quant : bf16 [M, K] -> e4m3 [M, K] and 1x128 scales f32 [M, K / 128], the
//                       blockwise arithmetic above without the SiLU * mul (no reference counterpart:
//                       the activation side of the blockwise FP8 GEMMs)
//   gather_rows       : dst[i, :] = src[row_indices[i], :]   (the A-operand gather of the reference's
//                       scatter grouped GEMM, src/group_gemm/cp_async/group_gemm_fp8_scatter.cu:20-46,
//                       done here as a streaming pre-pass in front of the TMA-fed grouped GEMM)
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "group_gemm.h"
#include "host_utils.h"

namespace b200 {
namespace act {

constexpr int kThreads = 256;

__device__ __forceinline__ float silu_exact(float x) { return x / (1.f + expf(-x)); }

// silu(gate) * up for the 8 columns at `g` (gate) and `g + half_col` (up) of one row: 16 B of
// gate + 16 B of up in. With `use_bf16_mul` the product is formed in bf16 as the reference kernel
// and its test do; otherwise in fp32.
__device__ __forceinline__ void silu_mul8(const __nv_bfloat16* g, int half_col, int use_bf16_mul,
                                          float (&m)[8]) {
  const uint4 gv = ld_nc_v4(g);
  const uint4 uv = ld_nc_v4(g + half_col);
  const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(&gv);
  const __nv_bfloat162* u2 = reinterpret_cast<const __nv_bfloat162*>(&uv);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float2 gf = __bfloat1622float2(g2[i]);
    const float s0 = silu_exact(gf.x), s1 = silu_exact(gf.y);
    if (use_bf16_mul) {
      const __nv_bfloat162 p = __hmul2(__floats2bfloat162_rn(s0, s1), u2[i]);
      const float2 pf = __bfloat1622float2(p);
      m[2 * i] = pf.x;
      m[2 * i + 1] = pf.y;
    } else {
      const float2 uf = __bfloat1622float2(u2[i]);
      m[2 * i] = s0 * uf.x;
      m[2 * i + 1] = s1 * uf.y;
    }
  }
}

// 8 values times `scale` -> 8 e4m3 bytes
__device__ __forceinline__ uint2 quant8(const float (&m)[8], float scale) {
  uint2 w;
  w.x = cvt_e4m3x4(m[0] * scale, m[1] * scale, m[2] * scale, m[3] * scale);
  w.y = cvt_e4m3x4(m[4] * scale, m[5] * scale, m[6] * scale, m[7] * scale);
  return w;
}

// one thread = 8 output columns of one row: 16 B of gate + 16 B of up in, 8 B out
__global__ void __launch_bounds__(kThreads)
    act_mul_and_quant_kernel(uint8_t* __restrict__ out, const __nv_bfloat16* __restrict__ in,
                             const float* __restrict__ scale_ptr, long long num_row, int half_col,
                             int use_bf16_mul) {
  const float scale = __ldg(scale_ptr);
  const int vec_per_row = half_col >> 3;
  const long long total = num_row * vec_per_row;
  for (long long v = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; v < total;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    const long long r = v / vec_per_row;
    const int c = static_cast<int>(v - r * vec_per_row) << 3;
    float m[8];
    silu_mul8(in + r * (2LL * half_col) + c, half_col, use_bf16_mul, m);
    *reinterpret_cast<uint2*>(out + r * half_col + c) = quant8(m, scale);
  }
}

// ---- masked (per-expert padded) layout ---------------------------------------------------------
// Row e * T_max + t of [E * T_max, 2C] is valid when t < clamp(num_per_expert[e], 0, T_max). Each
// CTA reads the E counts once into an exclusive prefix sum in shared memory (warp 0, 32 experts per
// step), then strides over the (valid row, 8 columns) items only: item i is the (i / vpr)-th valid
// row, whose expert is found by binary search in the prefix. Invalid rows are neither read nor
// written, and the work follows the number of valid rows, not E * T_max.
__device__ __forceinline__ void expert_prefix(const int* __restrict__ num_per_expert, int num_expert,
                                              int t_max, int* prefix) {
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int carry = 0;
    if (lane == 0) prefix[0] = 0;
    for (int base = 0; base < num_expert; base += 32) {
      int c = base + lane < num_expert ? __ldg(num_per_expert + base + lane) : 0;
      c = min(max(c, 0), t_max);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, c, o);
        if (lane >= o) c += n;
      }
      if (base + lane < num_expert) prefix[base + lane + 1] = carry + c;
      carry += __shfl_sync(0xffffffffu, c, 31);
    }
  }
  __syncthreads();
}

// the padded row of the k-th valid row: the expert e with prefix[e] <= k < prefix[e + 1]
__device__ __forceinline__ long long valid_row(const int* prefix, int num_expert, int t_max, int k) {
  int lo = 0, hi = num_expert;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (prefix[mid + 1] <= k) lo = mid + 1;
    else hi = mid;
  }
  return static_cast<long long>(lo) * t_max + (k - prefix[lo]);
}

// per-tensor: out = e4m3(silu(gate) * up * scale[0]), the row body of act_mul_and_quant
// (use_bf16_mul = 0)
__global__ void __launch_bounds__(kThreads)
    masked_act_mul_and_quant_kernel(uint8_t* __restrict__ out, const __nv_bfloat16* __restrict__ in,
                                    const float* __restrict__ scale_ptr,
                                    const int* __restrict__ num_per_expert, int num_expert,
                                    int t_max, int half_col) {
  extern __shared__ int prefix[];
  expert_prefix(num_per_expert, num_expert, t_max, prefix);
  const float scale = __ldg(scale_ptr);
  const int vpr = half_col >> 3;
  const int total = prefix[num_expert] * vpr;  // < 2^31, checked by the launcher
  for (int v = blockIdx.x * kThreads + threadIdx.x; v < total; v += gridDim.x * kThreads) {
    const int k = v / vpr;
    const int c = (v - k * vpr) << 3;
    const long long r = valid_row(prefix, num_expert, t_max, k);
    float m[8];
    silu_mul8(in + r * (2LL * half_col) + c, half_col, 0, m);
    *reinterpret_cast<uint2*>(out + r * half_col + c) = quant8(m, scale);
  }
}

// One 1x128 block held as 8 values by each of the 16 lanes of a half-warp (`half_mask`): sc =
// amax / 448 over the block, returns the lane's 8 codes e4m3(v * (1 / (sc + 1e-8))).
__device__ __forceinline__ uint2 blockwise_quant8(const float (&m)[8], unsigned half_mask,
                                                  float& sc) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(m[i]));
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(half_mask, amax, o));
  sc = amax / 448.0f;
  const float inv = 1.0f / (sc + 1e-8f);
  return quant8(m, inv);
}

// blockwise: per (row, 128 columns) = 16 lanes x 8 columns, sc = amax / 448,
// out = e4m3(v * (1 / (sc + 1e-8))), out_scale[row, block] = sc (row-major [E * T_max, C / 128]).
// vpr is a multiple of 16 and so is every item index a half-warp starts at, so the 16 lanes of a
// 128-column block are always the 16 lanes of one half-warp and reach the loop test together.
__global__ void __launch_bounds__(kThreads)
    masked_act_mul_and_blockwise_quant_kernel(uint8_t* __restrict__ out,
                                              float* __restrict__ out_scale,
                                              const __nv_bfloat16* __restrict__ in,
                                              const int* __restrict__ num_per_expert,
                                              int num_expert, int t_max, int half_col) {
  extern __shared__ int prefix[];
  expert_prefix(num_per_expert, num_expert, t_max, prefix);
  const int vpr = half_col >> 3;
  const int total = prefix[num_expert] * vpr;
  const int lane = threadIdx.x & 31;
  const unsigned half_mask = 0xffffu << (lane & 16);
  for (int v = blockIdx.x * kThreads + threadIdx.x; v < total; v += gridDim.x * kThreads) {
    const int k = v / vpr;
    const int c = (v - k * vpr) << 3;
    const long long r = valid_row(prefix, num_expert, t_max, k);
    float m[8];
    silu_mul8(in + r * (2LL * half_col) + c, half_col, 0, m);
    float sc;
    *reinterpret_cast<uint2*>(out + r * half_col + c) = blockwise_quant8(m, half_mask, sc);
    if ((lane & 15) == 0) out_scale[r * (half_col >> 7) + (c >> 7)] = sc;
  }
}

// bf16 [M, K] (row stride `ld` elements) -> e4m3 [M, K] and sc f32 [M, K / 128], the arithmetic of
// masked_act_mul_and_blockwise_quant_kernel without the SiLU * mul. vpr = K / 8 is a multiple of 16,
// so the 16 lanes of a 128-column block are again the 16 lanes of one half-warp.
__global__ void __launch_bounds__(kThreads)
    blockwise_fp8_quant_kernel(uint8_t* __restrict__ out, float* __restrict__ out_scale,
                               const __nv_bfloat16* __restrict__ in, long long num_row, int num_col,
                               long long ld) {
  pdl_launch_dependents();
  pdl_wait();
  const int vpr = num_col >> 3;
  const long long total = num_row * vpr;
  const int lane = threadIdx.x & 31;
  const unsigned half_mask = 0xffffu << (lane & 16);
  for (long long v = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; v < total;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    const long long r = v / vpr;
    const int c = static_cast<int>(v - r * vpr) << 3;
    const uint4 raw = ld_nc_v4(in + r * ld + c);
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
    float m[8];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float2 f = __bfloat1622float2(h2[i]);
      m[2 * i] = f.x;
      m[2 * i + 1] = f.y;
    }
    float sc;
    *reinterpret_cast<uint2*>(out + r * num_col + c) = blockwise_quant8(m, half_mask, sc);
    if ((lane & 15) == 0) out_scale[r * (num_col >> 7) + (c >> 7)] = sc;
  }
}

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// one thread = one 16-byte input vector (4 floats or 8 halves)
template <typename T>
__global__ void __launch_bounds__(kThreads)
    scaled_fp8_quant_kernel(uint8_t* __restrict__ out, const T* __restrict__ in,
                            const float* __restrict__ scale_ptr, long long numel) {
  constexpr int kVec = 16 / sizeof(T);
  const float inv = 1.0f / __ldg(scale_ptr);
  const long long nvec = numel / kVec;
  for (long long v = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    const uint4 raw = ld_nc_v4(in + v * kVec);
    const T* e = reinterpret_cast<const T*>(&raw);
    float f[kVec];
#pragma unroll
    for (int i = 0; i < kVec; i++) f[i] = to_f32<T>(e[i]) * inv;
    uint32_t w[kVec / 4];
#pragma unroll
    for (int i = 0; i < kVec / 4; i++) w[i] = cvt_e4m3x4(f[4 * i], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
    if constexpr (kVec == 4) {
      *reinterpret_cast<uint32_t*>(out + v * 4) = w[0];
    } else {
      *reinterpret_cast<uint2*>(out + v * 8) = make_uint2(w[0], w[1]);
    }
  }
  // ragged tail (numel not a multiple of the vector width)
  if (blockIdx.x == 0) {
    for (long long i = nvec * kVec + threadIdx.x; i < numel; i += kThreads) {
      const float f = to_f32<T>(in[i]) * inv;
      out[i] = static_cast<uint8_t>(cvt_e4m3x4(f, 0.f, 0.f, 0.f) & 0xffu);
    }
  }
}

// one warp per destination row, 16-byte copies
__global__ void __launch_bounds__(kThreads)
    gather_rows_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src,
                       const int* __restrict__ row_indices, int num_rows, int src_rows,
                       int vec_per_row) {
  const int warps_per_block = kThreads / 32;
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < num_rows;
       r += gridDim.x * warps_per_block) {
    int s = __ldg(row_indices + r);
    s = s < 0 ? 0 : (s >= src_rows ? src_rows - 1 : s);  // never read outside the pool
    const uint4* sp = src + static_cast<long long>(s) * vec_per_row;
    uint4* dp = dst + static_cast<long long>(r) * vec_per_row;
    for (int c = lane; c < vec_per_row; c += 32) dp[c] = ld_nc_v4(sp + c);
  }
}

static int stream_grid(long long work_items) {
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  long long blocks = (work_items + kThreads - 1) / kThreads;
  const long long cap = static_cast<long long>(sms) * 8;  // 8 resident blocks of 256 threads per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

}  // namespace act
}  // namespace b200

using namespace b200;  // NOLINT

// replaces reference src/activation/activation.h:15-17 (act_mul_and_quant_async, bf16 in, e4m3 out).
// num_col = 2 * C (gate columns then up columns).
extern "C" int hpc_act_mul_and_quant_async(void* y_ptr, const void* x_ptr, const float* scale_ptr,
                                           int num_row, int num_col, int use_bf16_mul,
                                           cudaStream_t stream) {
  HPC_REQUIRE(num_col > 0 && num_col % 16 == 0,
              "act_mul_and_quant: last dim (%d) must be a multiple of 16", num_col);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x_ptr) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(y_ptr) & 7) == 0,
              "act_mul_and_quant: input must be 16-byte and output 8-byte aligned");
  if (num_row <= 0) return HPC_OK;
  const int half = num_col / 2;
  const long long items = static_cast<long long>(num_row) * (half / 8);
  act::act_mul_and_quant_kernel<<<act::stream_grid(items), act::kThreads, 0, stream>>>(
      static_cast<uint8_t*>(y_ptr), static_cast<const __nv_bfloat16*>(x_ptr), scale_ptr, num_row,
      half, use_bf16_mul);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// Shared argument checks of the two masked launchers; sets *items and *smem.
static int masked_setup(const char* what, const void* y_ptr, const void* x_ptr,
                        const void* num_per_expert_ptr, int num_total_tokens,
                        int num_intermediate_size, int num_tokens_per_expert, int col_multiple,
                        int* items_out, size_t* smem) {
  HPC_REQUIRE(num_intermediate_size > 0 && num_intermediate_size % col_multiple == 0,
              "%s: intermediate size (%d) must be a positive multiple of %d", what,
              num_intermediate_size, col_multiple);
  HPC_REQUIRE(num_tokens_per_expert > 0 && num_total_tokens >= 0 &&
                  num_total_tokens % num_tokens_per_expert == 0,
              "%s: rows (%d) must be a multiple of the tokens per expert (%d)", what,
              num_total_tokens, num_tokens_per_expert);
  const int num_expert = num_total_tokens / num_tokens_per_expert;
  HPC_REQUIRE(num_expert <= 8192, "%s: %d experts exceed the supported 8192", what, num_expert);
  HPC_REQUIRE(num_expert == 0 || num_per_expert_ptr != nullptr, "%s: num_per_expert missing", what);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x_ptr) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(y_ptr) & 7) == 0,
              "%s: input must be 16-byte and output 8-byte aligned", what);
  // the kernels index items in 32 bits: items plus one grid stride (<= 8 * 256 per SM) must fit
  const long long items = static_cast<long long>(num_total_tokens) * (num_intermediate_size / 8);
  HPC_REQUIRE(items <= (1LL << 30), "%s: %lld 8-column items exceed the supported 2^30", what,
              items);
  *items_out = static_cast<int>(items);
  *smem = static_cast<size_t>(num_expert + 1) * sizeof(int);
  return HPC_OK;
}

// replaces reference src/activation/activation.h (masked_act_mul_and_quant_async).
// input bf16 [num_total_tokens, 2 * num_intermediate_size], rows grouped per expert in blocks of
// num_tokens_per_expert; only the first clamp(num_per_expert[e], 0, T_max) rows of expert e are
// read and written.
extern "C" int hpc_masked_act_mul_and_quant_async(void* output_ptr, const void* input_ptr,
                                                  const float* scale_ptr,
                                                  const int* num_per_expert_ptr,
                                                  int num_total_tokens, int num_intermediate_size,
                                                  int num_tokens_per_expert, cudaStream_t stream) {
  int items = 0;
  size_t smem = 0;
  const int rc = masked_setup("masked_act_mul_and_quant", output_ptr, input_ptr, num_per_expert_ptr,
                              num_total_tokens, num_intermediate_size, num_tokens_per_expert, 8,
                              &items, &smem);
  if (rc != HPC_OK) return rc;
  if (num_total_tokens == 0) return HPC_OK;
  const int grid = act::stream_grid(items);
  act::masked_act_mul_and_quant_kernel<<<grid, act::kThreads, smem, stream>>>(
      static_cast<uint8_t*>(output_ptr), static_cast<const __nv_bfloat16*>(input_ptr), scale_ptr,
      num_per_expert_ptr, num_total_tokens / num_tokens_per_expert, num_tokens_per_expert,
      num_intermediate_size);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// replaces reference src/activation/activation.h (masked_act_mul_and_blockwise_quant_async).
// output_scale f32 row-major [num_total_tokens, num_intermediate_size / 128].
extern "C" int hpc_masked_act_mul_and_blockwise_quant_async(
    void* output_ptr, float* output_scale_ptr, const void* input_ptr, const int* num_per_expert_ptr,
    int num_total_tokens, int num_intermediate_size, int num_tokens_per_expert,
    cudaStream_t stream) {
  int items = 0;
  size_t smem = 0;
  const int rc = masked_setup("masked_act_mul_and_blockwise_quant", output_ptr, input_ptr,
                              num_per_expert_ptr, num_total_tokens, num_intermediate_size,
                              num_tokens_per_expert, 128, &items, &smem);
  if (rc != HPC_OK) return rc;
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(output_scale_ptr) & 3) == 0,
              "masked_act_mul_and_blockwise_quant: output_scale must be 4-byte aligned");
  if (num_total_tokens == 0) return HPC_OK;
  const int grid = act::stream_grid(items);
  act::masked_act_mul_and_blockwise_quant_kernel<<<grid, act::kThreads, smem, stream>>>(
      static_cast<uint8_t*>(output_ptr), output_scale_ptr,
      static_cast<const __nv_bfloat16*>(input_ptr), num_per_expert_ptr,
      num_total_tokens / num_tokens_per_expert, num_tokens_per_expert, num_intermediate_size);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// No reference counterpart: the 1x128 activation quantiser in front of the blockwise FP8 GEMMs.
// input bf16 [num_row, num_col] with row stride input_ld elements; output e4m3 [num_row, num_col]
// and output_scale f32 [num_row, num_col / 128], both contiguous.
extern "C" int hpc_blockwise_fp8_quant_async(void* output_ptr, float* output_scale_ptr,
                                             const void* input_ptr, int num_row, int num_col,
                                             int64_t input_ld, cudaStream_t stream) {
  HPC_REQUIRE(num_row >= 0 && num_col > 0 && num_col % 128 == 0,
              "blockwise_fp8_quant: shape [%d, %d] needs rows >= 0 and columns a positive multiple "
              "of 128", num_row, num_col);
  HPC_REQUIRE(input_ld >= num_col && input_ld % 8 == 0,
              "blockwise_fp8_quant: row stride %lld must be >= %d and a multiple of 8 elements",
              static_cast<long long>(input_ld), num_col);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(input_ptr) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(output_ptr) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(output_scale_ptr) & 3) == 0,
              "blockwise_fp8_quant: input must be 16-byte, output 8-byte and output_scale 4-byte "
              "aligned");
  if (num_row == 0) return HPC_OK;
  const long long items = static_cast<long long>(num_row) * (num_col / 8);
  HPC_CUDA_CHECK(launch_pdl(act::blockwise_fp8_quant_kernel, dim3(act::stream_grid(items)),
                            dim3(act::kThreads), 0, stream, 1, static_cast<uint8_t*>(output_ptr),
                            output_scale_ptr, static_cast<const __nv_bfloat16*>(input_ptr),
                            static_cast<long long>(num_row), num_col,
                            static_cast<long long>(input_ld)));
  return HPC_OK;
}

// replaces reference src/activation/activation.h:46-53 (scaled_fp8_quant_async overloads).
// in_dtype: 0 = float32, 1 = float16, 2 = bfloat16.
extern "C" int hpc_scaled_fp8_quant_async(void* y_ptr, const void* x_ptr, const float* scale_ptr,
                                          int64_t numel, int in_dtype, cudaStream_t stream) {
  HPC_REQUIRE(in_dtype >= 0 && in_dtype <= 2, "scaled_fp8_quant: bad input dtype code %d", in_dtype);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x_ptr) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(y_ptr) & 7) == 0,
              "scaled_fp8_quant: input must be 16-byte and output 8-byte aligned");
  if (numel <= 0) return HPC_OK;
  uint8_t* y = static_cast<uint8_t*>(y_ptr);
  if (in_dtype == 0) {
    act::scaled_fp8_quant_kernel<float><<<act::stream_grid(numel / 4), act::kThreads, 0, stream>>>(
        y, static_cast<const float*>(x_ptr), scale_ptr, numel);
  } else if (in_dtype == 1) {
    act::scaled_fp8_quant_kernel<__half><<<act::stream_grid(numel / 8), act::kThreads, 0, stream>>>(
        y, static_cast<const __half*>(x_ptr), scale_ptr, numel);
  } else {
    act::scaled_fp8_quant_kernel<__nv_bfloat16>
        <<<act::stream_grid(numel / 8), act::kThreads, 0, stream>>>(
            y, static_cast<const __nv_bfloat16*>(x_ptr), scale_ptr, numel);
  }
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// replaces reference src/group_gemm/cp_async/group_gemm.h:11-16 (group_gemm_fp8_multistage_async):
// the small-M cp.async kernel of the reference is served by the same wgmma grouped GEMM
// (per-group scalar y_scale). tiles / cu_tiles / task_map: accepted, ignored.
extern "C" int hpc_group_gemm_fp8_multistage_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* y_scale_ptr,
    const void* seqlens_ptr, const void* cu_seqlens_ptr, const void* tiles_ptr,
    const void* cu_tiles_ptr, const void* task_map_ptr, int task_map_len, int m, int n, int k,
    int num_group, int num_seq_per_group_avg, int use_pdl, cudaStream_t stream) {
  (void)tiles_ptr; (void)cu_tiles_ptr; (void)task_map_ptr; (void)task_map_len; (void)use_pdl;
  return ggemm::run(0, x_ptr, w_ptr, static_cast<const int*>(seqlens_ptr),
                    static_cast<const int*>(cu_seqlens_ptr), nullptr,
                    static_cast<const float*>(y_scale_ptr), nullptr, y_ptr, nullptr, nullptr,
                    num_group, m, n, k, 0, 0, ggemm::scale_tile_from_avg(num_seq_per_group_avg), 0,
                    stream);
}

// replaces reference src/group_gemm/cp_async/group_gemm.h:18-24 (group_gemm_fp8_scatter_async):
// row i of the compact problem is row row_indices[i] of the pool x [pool_rows, k]. `gather_ptr`
// is an e4m3 scratch of m * k bytes (extra argument: the reference gathers inside its kernel).
extern "C" int hpc_group_gemm_fp8_scatter_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* y_scale_ptr,
    const void* row_indices_ptr, const void* seqlens_ptr, const void* cu_seqlens_ptr,
    const void* tiles_ptr, const void* cu_tiles_ptr, const void* task_map_ptr, int task_map_len,
    int m, int n, int k, int num_group, int num_seq_per_group_avg, int use_pdl, void* gather_ptr,
    int pool_rows, cudaStream_t stream) {
  HPC_REQUIRE(k > 0 && k % 16 == 0, "scatter group gemm: k (%d) must be a multiple of 16", k);
  HPC_REQUIRE(gather_ptr != nullptr && pool_rows > 0, "scatter group gemm: gather scratch / pool rows missing");
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x_ptr) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(gather_ptr) & 15) == 0,
              "scatter group gemm: x and scratch must be 16-byte aligned");
  if (m <= 0) return HPC_OK;
  const int warps_per_block = act::kThreads / 32;
  int blocks = (m + warps_per_block - 1) / warps_per_block;
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  if (blocks > sms * 8) blocks = sms * 8;
  act::gather_rows_kernel<<<blocks, act::kThreads, 0, stream>>>(
      static_cast<uint4*>(gather_ptr), static_cast<const uint4*>(x_ptr),
      static_cast<const int*>(row_indices_ptr), m, pool_rows, k / 16);
  HPC_CUDA_CHECK(cudaGetLastError());
  return hpc_group_gemm_fp8_multistage_async(y_ptr, gather_ptr, w_ptr, y_scale_ptr, seqlens_ptr,
                                             cu_seqlens_ptr, tiles_ptr, cu_tiles_ptr, task_map_ptr,
                                             task_map_len, m, n, k, num_group,
                                             num_seq_per_group_avg, use_pdl, stream);
}
