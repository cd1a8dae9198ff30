// FusedMoE FP8 pipeline (H100 / sm_90a): routing, Gate-Up GEMM (+ fused SiLU*mul + quant),
// Down GEMM, top-k weighted reduce.
//
// Replaces reference src/fuse_moe/fuse_moe.cu:14-116 (fuse_moe_async / fuse_moe_blockwise_async),
// src/fuse_moe/count_and_gather*.cu and src/fuse_moe/reduce.cu:17-142.
//
// Differences from the reference:
//   * routing is deterministic: one block per local expert walks topk_ids in token order, so the row
//     order inside an expert is reproducible (the reference claims slots with atomics,
//     count_and_gather_for_blockwise.cu:204-231). Counts / cumsums are identical.
//   * the activation (SiLU*mul + FP8 re-quant) is the epilogue of the Gate-Up GEMM: the bf16
//     Gate-Up matrix (1.88 GB at T=4096,k=8,I=14336) is never written to or read from HBM.
#include "common.cuh"
#include "group_gemm.h"
#include "host_utils.h"

namespace b200 {
namespace moe {

constexpr int kRouteThreads = 1024;
constexpr int kMaxExperts = 512;

// ---- kernel A: histogram of local experts, topk_pos := -1 -------------------------------------
__global__ void __launch_bounds__(256)
    moe_count_kernel(const int* __restrict__ topk_ids, int* __restrict__ topk_pos,
                     int* __restrict__ counts, int total, int num_expert_local, int expert_base) {
  __shared__ int hist[kMaxExperts];
  for (int i = threadIdx.x; i < num_expert_local; i += blockDim.x) hist[i] = 0;
  pdl_wait();  // PDL: whatever ran before on the stream may still be producing topk_ids
  pdl_launch_dependents();
  __syncthreads();
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int e = topk_ids[idx] - expert_base;
    topk_pos[idx] = -1;
    if (e >= 0 && e < num_expert_local) atomicAdd(&hist[e], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < num_expert_local; i += blockDim.x) {
    if (hist[i]) atomicAdd(&counts[i], hist[i]);
  }
}

// ---- kernel B: one block per local expert: cumsums, positions (token order), row gather -------
__global__ void __launch_bounds__(kRouteThreads)
    moe_route_gather_kernel(const uint8_t* __restrict__ x, const float* __restrict__ x_scale,
                            const int* __restrict__ topk_ids, const int* __restrict__ counts,
                            uint8_t* __restrict__ gathered, float* __restrict__ xs_t,
                            int* __restrict__ topk_pos, int* __restrict__ cu_tokens,
                            int* __restrict__ tiles, int* __restrict__ cu_tiles, int num_tokens,
                            int num_topk, int hidden, int num_expert_local, int expert_base,
                            int scale_tile, int m_pad) {
  __shared__ int s_warp[kRouteThreads / 32];
  __shared__ int s_base[2];  // cu_tokens[e], pad_base[e]
  const int e = blockIdx.x;
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int nwarps = kRouteThreads / 32;

  pdl_wait();  // the histogram is complete
  pdl_launch_dependents();
  if (warp == 0) {
    // exclusive scans over the experts: rows and scale columns (padded to scale_tile)
    int carry = 0, carry_pad = 0, carry_tiles = 0;
    for (int g0 = 0; g0 < num_expert_local; g0 += 32) {
      const int g = g0 + lane;
      const int c = g < num_expert_local ? counts[g] : 0;
      const int tl = (c + scale_tile - 1) / scale_tile;
      int ic = c, it = tl;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, ic, o);
        const int b = __shfl_up_sync(0xffffffffu, it, o);
        if (lane >= o) {
          ic += a;
          it += b;
        }
      }
      if (g < num_expert_local) {
        if (g == e) {
          s_base[0] = carry + ic - c;
          s_base[1] = (carry_tiles + it - tl) * scale_tile;
        }
        if (e == 0) {
          cu_tokens[g] = carry + ic - c;
          tiles[g] = tl;
          cu_tiles[g] = carry_tiles + it - tl;
        }
      }
      carry += __shfl_sync(0xffffffffu, ic, 31);
      carry_tiles += __shfl_sync(0xffffffffu, it, 31);
    }
    if (e == 0 && lane == 0) {
      cu_tokens[num_expert_local] = carry;
      cu_tiles[num_expert_local] = carry_tiles;
    }
    (void)carry_pad;
  }
  __syncthreads();
  const int row_base = s_base[0];
  const int col_base = s_base[1];
  const int my_expert = e + expert_base;
  const int total = num_tokens * num_topk;
  if (counts[e] == 0) return;

  // each warp owns a contiguous, ordered segment of the flattened (token, k) list
  const int seg = ((total + nwarps - 1) / nwarps + 31) / 32 * 32;
  const int beg = warp * seg;
  const int end = beg + seg < total ? beg + seg : total;
  int cnt = 0;
  for (int i = beg + lane; i < end; i += 32) {
    cnt += (__ldg(topk_ids + i) == my_expert) ? 1 : 0;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) s_warp[warp] = cnt;
  __syncthreads();
  int off = 0;
  for (int w = 0; w < warp; w++) off += s_warp[w];

  const int kb_count = hidden / 128;
  for (int i0 = beg; i0 < end; i0 += 32) {
    const int i = i0 + lane;
    const bool hit = (i < end) && (__ldg(topk_ids + i) == my_expert);
    unsigned mask = __ballot_sync(0xffffffffu, hit);
    while (mask) {
      const int src_lane = __ffs(mask) - 1;
      mask &= mask - 1;
      const int idx = i0 + src_lane;
      const int token = idx / num_topk;
      const int local = off++;
      const int row = row_base + local;
      if (lane == 0) topk_pos[idx] = row;
      const uint4* src = reinterpret_cast<const uint4*>(x + static_cast<long long>(token) * hidden);
      uint4* dst = reinterpret_cast<uint4*>(gathered + static_cast<long long>(row) * hidden);
      for (int v = lane; v < hidden / 16; v += 32) dst[v] = ld_nc_v4(src + v);
      if (xs_t != nullptr) {
        for (int kb = lane; kb < kb_count; kb += 32) {
          xs_t[static_cast<long long>(kb) * m_pad + col_base + local] =
              __ldg(x_scale + static_cast<long long>(token) * kb_count + kb);
        }
      }
    }
  }
}

// ---- reduce: y[t] = sum_k down_out[pos[t,k]] * w[t,k] (+ shared) ------------------------------
// (reference src/fuse_moe/reduce.cu:17-83: fp32 accumulate in k order, skip pos < 0)
__global__ void __launch_bounds__(256)
    moe_reduce_kernel(__nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ x,
                      const int* __restrict__ topk_pos, const float* __restrict__ topk_scale,
                      const __nv_bfloat16* __restrict__ shared, int num_tokens, int hidden,
                      int num_topk) {
  const int vec_per_row = hidden / 8;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  pdl_wait();  // the Down GEMM's rows are complete
  pdl_launch_dependents();
  if (gid >= static_cast<long long>(num_tokens) * vec_per_row) return;
  const int t = static_cast<int>(gid / vec_per_row);
  const int v = static_cast<int>(gid % vec_per_row);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = 0.f;
  for (int k = 0; k < num_topk; k++) {
    const int pos = __ldg(topk_pos + t * num_topk + k);
    if (pos < 0) continue;
    const float w = __ldg(topk_scale + t * num_topk + k);
    const uint4 raw = ld_nc_v4(x + static_cast<long long>(pos) * hidden + v * 8);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float2 f = __bfloat1622float2(h[i]);
      acc[2 * i] += f.x * w;
      acc[2 * i + 1] += f.y * w;
    }
  }
  if (shared != nullptr) {
    const uint4 raw = ld_nc_v4(shared + static_cast<long long>(t) * hidden + v * 8);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float2 f = __bfloat1622float2(h[i]);
      acc[2 * i] += f.x;
      acc[2 * i + 1] += f.y;
    }
  }
  uint4 out;
  __nv_bfloat162 o0 = __floats2bfloat162_rn(acc[0], acc[1]);
  __nv_bfloat162 o1 = __floats2bfloat162_rn(acc[2], acc[3]);
  __nv_bfloat162 o2 = __floats2bfloat162_rn(acc[4], acc[5]);
  __nv_bfloat162 o3 = __floats2bfloat162_rn(acc[6], acc[7]);
  out.x = *reinterpret_cast<uint32_t*>(&o0);
  out.y = *reinterpret_cast<uint32_t*>(&o1);
  out.z = *reinterpret_cast<uint32_t*>(&o2);
  out.w = *reinterpret_cast<uint32_t*>(&o3);
  *reinterpret_cast<uint4*>(y + static_cast<long long>(t) * hidden + v * 8) = out;
}

static int route(const void* x, const float* x_scale, void* gathered, float* xs_t,
                 const int* topk_ids, int* topk_pos, int* counts, int* cu_tokens, int* tiles,
                 int* cu_tiles, int num_tokens, int num_topk, int hidden, int num_expert_local,
                 int rank_ep, int scale_tile, int m_pad, cudaStream_t stream) {
  HPC_REQUIRE(num_expert_local > 0 && num_expert_local <= kMaxExperts,
              "fuse_moe: local experts %d not in (0, %d]", num_expert_local, kMaxExperts);
  HPC_REQUIRE(hidden % 16 == 0 && (x_scale == nullptr || hidden % 128 == 0),
              "fuse_moe: hidden (%d) must be a multiple of 16 (128 for blockwise scales)", hidden);
  const int total = num_tokens * num_topk;
  HPC_CUDA_CHECK(cudaMemsetAsync(counts, 0, sizeof(int) * num_expert_local, stream));
  if (total == 0) return HPC_OK;
  const int expert_base = rank_ep * num_expert_local;
  int grid = (total + 1023) / 1024;
  grid = grid > 592 ? 592 : grid;
  moe_count_kernel<<<grid, 256, 0, stream>>>(topk_ids, topk_pos, counts, total, num_expert_local,
                                             expert_base);
  HPC_CUDA_CHECK(cudaGetLastError());
  // from here on the pipeline is a PDL chain (as the reference chains its MoE stages,
  // src/fuse_moe/fuse_moe.cu:71-116): route/gather -> Gate-Up GEMM -> Down GEMM -> reduce
  HPC_CUDA_CHECK(launch_pdl(moe_route_gather_kernel, dim3(num_expert_local), dim3(kRouteThreads), 0,
                            stream, 1, static_cast<const uint8_t*>(x), x_scale, topk_ids,
                            static_cast<const int*>(counts), static_cast<uint8_t*>(gathered), xs_t,
                            topk_pos, cu_tokens, tiles, cu_tiles, num_tokens, num_topk, hidden,
                            num_expert_local, expert_base, scale_tile, m_pad));
  return HPC_OK;
}

static int reduce(void* y, const void* x, const int* topk_pos, const float* topk_scale,
                  const void* shared, int num_tokens, int hidden, int num_topk,
                  cudaStream_t stream) {
  HPC_REQUIRE(hidden % 8 == 0, "reduce: hidden (%d) must be a multiple of 8", hidden);
  const long long work = static_cast<long long>(num_tokens) * (hidden / 8);
  if (work == 0) return HPC_OK;
  const int grid = static_cast<int>((work + 255) / 256);
  HPC_CUDA_CHECK(launch_pdl(moe_reduce_kernel, dim3(grid), dim3(256), 0, stream, 1,
                            static_cast<__nv_bfloat16*>(y), static_cast<const __nv_bfloat16*>(x),
                            topk_pos, topk_scale, static_cast<const __nv_bfloat16*>(shared),
                            num_tokens, hidden, num_topk));
  return HPC_OK;
}

// row-major scales [m rows (group-padded), n] -> transposed [n, m] with each group's columns
// compacted to tilem-multiples (reference src/group_gemm/group_gemm_blockwise_fp8.cu:19-86)
__global__ void __launch_bounds__(256)
    reformat_x_scale_kernel(float* __restrict__ out, const float* __restrict__ in,
                            const int* __restrict__ seqlens, const int* __restrict__ cu_seqlens,
                            int num_group, int m, int n, int tilem) {
  __shared__ int s_base;
  const int g = blockIdx.x;
  if (threadIdx.x < 32) {
    int acc = 0;
    for (int j = threadIdx.x; j < g; j += 32) acc += (seqlens[j] + tilem - 1) / tilem * tilem;
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (threadIdx.x == 0) s_base = acc;
  }
  __syncthreads();
  const int rows = seqlens[g];
  const int src0 = cu_seqlens[g];
  const int dst0 = s_base;
  for (int i = threadIdx.x; i < rows * n; i += blockDim.x) {
    const int r = i / n, c = i - r * n;
    out[static_cast<long long>(c) * m + dst0 + r] = in[static_cast<long long>(src0 + r) * n + c];
  }
}

}  // namespace moe
}  // namespace b200

using namespace b200;  // NOLINT

extern "C" int hpc_reformat_x_scale_async(void* output_ptr, const void* xscale_ptr,
                                          const void* seqlens_ptr, const void* cu_seqlens_ptr,
                                          int num_group, int m, int n, int tilem,
                                          cudaStream_t stream) {
  HPC_REQUIRE(num_group > 0 && tilem > 0, "reformat_x_scale: bad arguments");
  moe::reformat_x_scale_kernel<<<num_group, 256, 0, stream>>>(
      static_cast<float*>(output_ptr), static_cast<const float*>(xscale_ptr),
      static_cast<const int*>(seqlens_ptr), static_cast<const int*>(cu_seqlens_ptr), num_group, m,
      n, tilem);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// replaces reference src/fuse_moe/fuse_moe.h:24-32 (blockwise_count_and_gather_async)
extern "C" int hpc_blockwise_count_and_gather_async(
    const void* input_ptr, const void* input_scale_ptr, void* gate_up_input_ptr,
    void* gate_up_output_ptr, void* gate_up_input_scale_ptr, void* down_input_ptr,
    void* down_output_ptr, const void* topk_ids_ptr, void* topk_pos_ptr,
    void* num_tokens_per_group_ptr, void* cu_num_tokens_per_group_ptr, void* gate_up_tmas_ptr,
    void* down_tmas_ptr, void* tiles_ptr, void* cu_tiles_ptr, void* gateup_task_map_ptr,
    void* down_task_map_ptr, int num_tokens, int num_padded_tokens, int hidden_size,
    int intermediate_size, int num_topk, int num_expert_local, int eprank,
    int num_tokens_per_group_avg, int use_pdl, cudaStream_t stream) {
  (void)gate_up_output_ptr; (void)down_input_ptr; (void)down_output_ptr; (void)gate_up_tmas_ptr;
  (void)down_tmas_ptr; (void)gateup_task_map_ptr; (void)down_task_map_ptr; (void)intermediate_size;
  (void)use_pdl;
  return moe::route(input_ptr, static_cast<const float*>(input_scale_ptr), gate_up_input_ptr,
                    static_cast<float*>(gate_up_input_scale_ptr),
                    static_cast<const int*>(topk_ids_ptr), static_cast<int*>(topk_pos_ptr),
                    static_cast<int*>(num_tokens_per_group_ptr),
                    static_cast<int*>(cu_num_tokens_per_group_ptr), static_cast<int*>(tiles_ptr),
                    static_cast<int*>(cu_tiles_ptr), num_tokens, num_topk, hidden_size,
                    num_expert_local, eprank, ggemm::scale_tile_from_avg(num_tokens_per_group_avg),
                    num_padded_tokens, stream);
}

// replaces reference src/fuse_moe/fuse_moe.h:15-22 (count_and_gather_async)
extern "C" int hpc_count_and_gather_async(
    void* gate_up_input_ptr, void* gate_up_output_ptr, void* down_input_ptr, void* down_output_ptr,
    const void* x_ptr, const void* topk_ids_ptr, void* topk_pos_ptr, void* seqlens_ptr,
    void* cu_seqlens_ptr, void* gate_up_tmas_ptr, void* down_tmas_ptr, void* tiles_ptr,
    void* cu_tiles_ptr, void* gateup_task_map_ptr, void* down_task_map_ptr, int num_seq,
    int hidden_size, int intermediate_size, int num_topk, int num_expert, int eprank,
    int num_seq_per_group_avg, cudaStream_t stream) {
  (void)gate_up_output_ptr; (void)down_input_ptr; (void)down_output_ptr; (void)gate_up_tmas_ptr;
  (void)down_tmas_ptr; (void)gateup_task_map_ptr; (void)down_task_map_ptr; (void)intermediate_size;
  return moe::route(x_ptr, nullptr, gate_up_input_ptr, nullptr,
                    static_cast<const int*>(topk_ids_ptr), static_cast<int*>(topk_pos_ptr),
                    static_cast<int*>(seqlens_ptr), static_cast<int*>(cu_seqlens_ptr),
                    static_cast<int*>(tiles_ptr), static_cast<int*>(cu_tiles_ptr), num_seq, num_topk,
                    hidden_size, num_expert, eprank,
                    ggemm::scale_tile_from_avg(num_seq_per_group_avg), 0, stream);
}

// replaces reference src/fuse_moe/fuse_moe.h:34-36 (reduce_async)
extern "C" int hpc_reduce_async(void* y_ptr, const void* x_ptr, const void* topk_pos_ptr,
                                const void* topk_scale_ptr, const void* shared_output_ptr,
                                int total_num_seq, int num_seq, int hidden_size, int num_topk,
                                int use_pdl, cudaStream_t stream) {
  (void)total_num_seq; (void)use_pdl;
  return moe::reduce(y_ptr, x_ptr, static_cast<const int*>(topk_pos_ptr),
                     static_cast<const float*>(topk_scale_ptr), shared_output_ptr, num_seq,
                     hidden_size, num_topk, stream);
}

// replaces reference src/fuse_moe/fuse_moe.h:50-62 (fuse_moe_blockwise_async).
// `intermediate_size` is gate_up_weight.size(1) = 2*I, as in the reference entry.
// `gate_up_output_ptr` is unused (may be NULL): the activation is fused into the Gate-Up GEMM.
extern "C" int hpc_fuse_moe_blockwise_async(
    void* output_ptr, const void* input_ptr, const void* input_scale_ptr, void* gate_up_input_ptr,
    void* gate_up_input_scale_ptr, void* gate_up_output_ptr, const void* gate_up_weight_ptr,
    const void* gate_up_weight_scale_ptr, void* gate_up_tmas_ptr, void* down_input_ptr,
    void* down_input_scale_ptr, void* down_output_ptr, const void* down_weight_ptr,
    const void* down_weight_scale_ptr, void* down_tmas_ptr, const void* topk_ids_ptr,
    const void* topk_scale_ptr, void* topk_pos_ptr, void* num_tokens_per_group_ptr,
    void* cu_num_tokens_per_group_ptr, void* tiles_ptr, void* cu_tiles_ptr,
    const void* shared_output_ptr, void* gateup_task_map_ptr, void* down_task_map_ptr,
    int num_gateup_waves, int num_down_waves, int num_tokens, int num_padded_tokens,
    int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int gate_up_weight_scale_lastdim_pad4, int down_weight_scale_lastdim_pad4,
    int rank_ep, cudaStream_t stream) {
  (void)gate_up_output_ptr; (void)gate_up_tmas_ptr; (void)down_tmas_ptr; (void)gateup_task_map_ptr;
  (void)down_task_map_ptr; (void)num_gateup_waves; (void)num_down_waves;
  HPC_REQUIRE(num_expert_total > 0, "fuse_moe_blockwise: num_expert_total must be positive");
  HPC_REQUIRE(intermediate_size % 256 == 0,
              "fuse_moe_blockwise: gate_up rows (%d) must be a multiple of 256", intermediate_size);
  const int avg = num_tokens * num_topk / num_expert_total;
  const int st = ggemm::scale_tile_from_avg(avg);
  const int rows = num_tokens * num_topk;
  const int inter = intermediate_size / 2;
  int rc = moe::route(input_ptr, static_cast<const float*>(input_scale_ptr), gate_up_input_ptr,
                      static_cast<float*>(gate_up_input_scale_ptr),
                      static_cast<const int*>(topk_ids_ptr), static_cast<int*>(topk_pos_ptr),
                      static_cast<int*>(num_tokens_per_group_ptr),
                      static_cast<int*>(cu_num_tokens_per_group_ptr), static_cast<int*>(tiles_ptr),
                      static_cast<int*>(cu_tiles_ptr), num_tokens, num_topk, hidden_size,
                      num_expert_local, rank_ep, st, num_padded_tokens, stream);
  if (rc) return rc;
  // Gate-Up GEMM + SiLU*mul + 128-block quant -> down_input (fp8) + down_input_scale
  rc = ggemm::run(3, gate_up_input_ptr, gate_up_weight_ptr,
                  static_cast<const int*>(num_tokens_per_group_ptr),
                  static_cast<const int*>(cu_num_tokens_per_group_ptr),
                  static_cast<const float*>(gate_up_input_scale_ptr),
                  static_cast<const float*>(gate_up_weight_scale_ptr), nullptr, nullptr,
                  down_input_ptr, static_cast<float*>(down_input_scale_ptr), num_expert_local, rows,
                  intermediate_size, hidden_size, num_padded_tokens,
                  gate_up_weight_scale_lastdim_pad4, st, 0, stream);
  if (rc) return rc;
  // Down GEMM -> bf16 down_output
  rc = ggemm::run(1, down_input_ptr, down_weight_ptr,
                  static_cast<const int*>(num_tokens_per_group_ptr),
                  static_cast<const int*>(cu_num_tokens_per_group_ptr),
                  static_cast<const float*>(down_input_scale_ptr),
                  static_cast<const float*>(down_weight_scale_ptr), nullptr, down_output_ptr,
                  nullptr, nullptr, num_expert_local, rows, hidden_size, inter, num_padded_tokens,
                  down_weight_scale_lastdim_pad4, st, 0, stream);
  if (rc) return rc;
  return moe::reduce(output_ptr, down_output_ptr, static_cast<const int*>(topk_pos_ptr),
                     static_cast<const float*>(topk_scale_ptr), shared_output_ptr, num_tokens,
                     hidden_size, num_topk, stream);
}

// replaces reference src/fuse_moe/fuse_moe.h:38-48 (fuse_moe_async, per-tensor scales) and the
// cp.async low-latency variant src/fuse_moe/cp_async/fuse_moe_cp_async.h:23-33 (same math).
extern "C" int hpc_fuse_moe_async(
    void* output_ptr, const void* input_ptr, void* gate_up_input_ptr, void* gate_up_output_ptr,
    const void* gate_up_weight_ptr, const void* gate_up_scale_ptr, void* gate_up_tmas_ptr,
    const void* act_and_mul_scale_ptr, void* down_input_ptr, void* down_output_ptr,
    const void* down_weight_ptr, const void* down_scale_ptr, void* down_tmas_ptr,
    const void* topk_ids_ptr, const void* topk_scale_ptr, void* topk_pos_ptr, void* seqlens_ptr,
    void* cu_seqlens_ptr, void* tiles_ptr, void* cu_tiles_ptr, const void* shared_output_ptr,
    void* gateup_task_map_ptr, void* down_task_map_ptr, int num_gateup_waves, int num_down_waves,
    int num_seq, int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int rank_ep, int use_bf16_mul, cudaStream_t stream) {
  (void)gate_up_output_ptr; (void)gate_up_tmas_ptr; (void)down_tmas_ptr; (void)gateup_task_map_ptr;
  (void)down_task_map_ptr; (void)num_gateup_waves; (void)num_down_waves;
  HPC_REQUIRE(num_expert_total > 0, "fuse_moe: num_expert_total must be positive");
  HPC_REQUIRE(intermediate_size % 128 == 0 && hidden_size % 64 == 0,
              "fuse_moe: gate_up rows (%d) must be a multiple of 128 and hidden (%d) of 64",
              intermediate_size, hidden_size);
  const int avg = num_seq * num_topk / num_expert_total;
  const int st = ggemm::scale_tile_from_avg(avg);
  const int rows = num_seq * num_topk;
  const int inter = intermediate_size / 2;
  int rc = moe::route(input_ptr, nullptr, gate_up_input_ptr, nullptr,
                      static_cast<const int*>(topk_ids_ptr), static_cast<int*>(topk_pos_ptr),
                      static_cast<int*>(seqlens_ptr), static_cast<int*>(cu_seqlens_ptr),
                      static_cast<int*>(tiles_ptr), static_cast<int*>(cu_tiles_ptr), num_seq,
                      num_topk, hidden_size, num_expert_local, rank_ep, st, 0, stream);
  if (rc) return rc;
  rc = ggemm::run(2, gate_up_input_ptr, gate_up_weight_ptr, static_cast<const int*>(seqlens_ptr),
                  static_cast<const int*>(cu_seqlens_ptr), nullptr,
                  static_cast<const float*>(gate_up_scale_ptr),
                  static_cast<const float*>(act_and_mul_scale_ptr), nullptr, down_input_ptr,
                  nullptr, num_expert_local, rows, intermediate_size, hidden_size, 0, 0, st,
                  use_bf16_mul, stream);
  if (rc) return rc;
  rc = ggemm::run(0, down_input_ptr, down_weight_ptr, static_cast<const int*>(seqlens_ptr),
                  static_cast<const int*>(cu_seqlens_ptr), nullptr,
                  static_cast<const float*>(down_scale_ptr), nullptr, down_output_ptr, nullptr,
                  nullptr, num_expert_local, rows, hidden_size, inter, 0, 0, st, 0, stream);
  if (rc) return rc;
  return moe::reduce(output_ptr, down_output_ptr, static_cast<const int*>(topk_pos_ptr),
                     static_cast<const float*>(topk_scale_ptr), shared_output_ptr, num_seq,
                     hidden_size, num_topk, stream);
}

// bf16 FusedMoE (no reference counterpart): route -> fused Gate-Up GEMM (SiLU*mul epilogue) ->
// Down GEMM -> reduce, one PDL chain on `stream`, no allocation and no host synchronisation.
// `intermediate_size` is I (gate_up_weight.size(1) / 2). Every limit is checked before the first
// launch.
extern "C" int hpc_fuse_moe_bf16_async(
    void* output_ptr, const void* input_ptr, void* gate_up_input_ptr, const void* gate_up_weight_ptr,
    void* down_input_ptr, void* down_output_ptr, const void* down_weight_ptr,
    const void* topk_ids_ptr, const void* topk_scale_ptr, void* topk_pos_ptr, void* counts_ptr,
    void* cu_counts_ptr, void* tiles_ptr, void* cu_tiles_ptr, const void* shared_output_ptr,
    int num_tokens, int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int rank_ep, cudaStream_t stream) {
  HPC_REQUIRE(num_tokens >= 0, "fuse_moe_bf16: negative num_tokens %d", num_tokens);
  HPC_REQUIRE(num_expert_local > 0 && num_expert_local <= moe::kMaxExperts,
              "fuse_moe_bf16: local experts %d not in (0, %d]", num_expert_local, moe::kMaxExperts);
  HPC_REQUIRE(num_expert_total >= num_expert_local,
              "fuse_moe_bf16: num_expert_total %d below the %d local experts", num_expert_total,
              num_expert_local);
  HPC_REQUIRE(num_topk > 0 && num_topk <= 128, "fuse_moe_bf16: num_topk %d not in (0, 128]", num_topk);
  HPC_REQUIRE(hidden_size > 0 && hidden_size % 128 == 0,
              "fuse_moe_bf16: hidden (%d) must be a positive multiple of 128", hidden_size);
  HPC_REQUIRE(intermediate_size > 0 && intermediate_size % 128 == 0,
              "fuse_moe_bf16: intermediate (%d) must be a positive multiple of 128", intermediate_size);
  const void* ptrs[] = {output_ptr, input_ptr, gate_up_input_ptr, gate_up_weight_ptr, down_input_ptr,
                        down_output_ptr, down_weight_ptr, shared_output_ptr};
  for (const void* q : ptrs) {
    HPC_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0, "fuse_moe_bf16: tensors must be 16-byte aligned");
  }
  if (num_tokens == 0) return HPC_OK;
  const int rows = num_tokens * num_topk;
  const int* counts = static_cast<const int*>(counts_ptr);
  const int* cu_counts = static_cast<const int*>(cu_counts_ptr);
  // a bf16 row is 2*H bytes for the route kernel's byte copy; the tile counts it writes are in
  // 128-row m-tiles of the bf16 GEMM
  int rc = moe::route(input_ptr, nullptr, gate_up_input_ptr, nullptr,
                      static_cast<const int*>(topk_ids_ptr), static_cast<int*>(topk_pos_ptr),
                      static_cast<int*>(counts_ptr), static_cast<int*>(cu_counts_ptr),
                      static_cast<int*>(tiles_ptr), static_cast<int*>(cu_tiles_ptr), num_tokens,
                      num_topk, 2 * hidden_size, num_expert_local, rank_ep, 128, 0, stream);
  if (rc) return rc;
  rc = ggemm::run_bf16(true, gate_up_input_ptr, gate_up_weight_ptr, counts, cu_counts,
                       down_input_ptr, num_expert_local, rows, 2 * intermediate_size, hidden_size,
                       stream);
  if (rc) return rc;
  rc = ggemm::run_bf16(false, down_input_ptr, down_weight_ptr, counts, cu_counts, down_output_ptr,
                       num_expert_local, rows, hidden_size, intermediate_size, stream);
  if (rc) return rc;
  return moe::reduce(output_ptr, down_output_ptr, static_cast<const int*>(topk_pos_ptr),
                     static_cast<const float*>(topk_scale_ptr), shared_output_ptr, num_tokens,
                     hidden_size, num_topk, stream);
}
