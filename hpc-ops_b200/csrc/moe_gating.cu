// Fused MoE top-k gating (H100 / sm_90a): router logits [T, E] -> topk_ids int32 [T, k] and
// topk_weights f32 [T, k], the input fuse_moe* consumes. Per token row, in fp32:
//
//   s_e  = softmax over all E (expf(x_e - max) / sum)   or   sigmoid 1 / (1 + expf(-x_e))
//   c_e  = x_e (softmax without bias: the same order as s_e, exactly)   else   s_e + bias_e
//   groups (G > 1): group score = max key, or the sum of its top-2 keys with a bias; the
//          topk_group best groups (score desc, group id asc) stay eligible
//   ids  = k rounds of arg-max over eligible keys in the order (key desc, id asc), NaN lowest
//   w_i  = s_{id_i}; renormalize: w_i / sum_i w_i (rank order); then w_i * routed_scaling_factor
//
// Layout: one warp per token, 8 tokens per 256-thread CTA. Lane l loads 16-byte vectors
// l, l + 32, ... of its row with ld.global.nc and keeps the (at most 16) values in registers; no
// shared or global scratch. Every key is packed with its id into one u64,
//   (order-preserving int of the key) << 32 | (0xFFFF - id),
// so that the u64 maximum is the (key desc, id asc) winner: an arg-max is a per-lane maximum over
// the slots followed by a 5-step __shfl_xor_sync butterfly, and every lane ends with the same
// winner. The value 0 sits below every key (NaN included) and marks a slot that is padding, not
// eligible or already chosen.
#include <cuda_bf16.h>

#include <climits>

#include "common.cuh"
#include "host_utils.h"

namespace b200 {
namespace gating {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kSlots = 16;  // values per lane at E = 512
constexpr int kMaxExperts = 32 * kSlots;
constexpr int kMaxTopk = 16;

// Total order on fp32 keys as int32: -0 equals +0, NaN sits below -inf.
__device__ __forceinline__ int ord_key(float f) {
  if (f != f) return INT_MIN + 1;
  int b = __float_as_int(f);
  if (b == INT_MIN) b = 0;
  return b >= 0 ? b : b ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float key_value(int o) {
  return __int_as_float(o >= 0 ? o : o ^ 0x7FFFFFFF);
}
__device__ __forceinline__ uint64_t pack(int o, int id) {
  return (static_cast<uint64_t>(static_cast<uint32_t>(o) ^ 0x80000000u) << 32) |
         static_cast<uint32_t>(0xFFFF - id);
}
__device__ __forceinline__ int packed_id(uint64_t p) {
  return 0xFFFF - static_cast<int>(static_cast<uint32_t>(p) & 0xFFFFu);
}
__device__ __forceinline__ int packed_ord(uint64_t p) {
  return static_cast<int>(static_cast<uint32_t>(p >> 32) ^ 0x80000000u);
}
__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint64_t w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}
template <int N>
__device__ __forceinline__ uint64_t argmax(const uint64_t (&p)[N]) {
  uint64_t m = p[0];
#pragma unroll
  for (int j = 1; j < N; j++) m = p[j] > m ? p[j] : m;
  return warp_max_u64(m);
}

__device__ __forceinline__ float sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

template <typename T>
struct Vec;
template <>
struct Vec<float> {
  static constexpr int kWidth = 4;
  __device__ __forceinline__ static void unpack(uint4 r, float* x) {
    x[0] = __uint_as_float(r.x);
    x[1] = __uint_as_float(r.y);
    x[2] = __uint_as_float(r.z);
    x[3] = __uint_as_float(r.w);
  }
};
template <>
struct Vec<__nv_bfloat16> {
  static constexpr int kWidth = 8;
  __device__ __forceinline__ static void unpack(uint4 r, float* x) {
    pair(r.x, x);
    pair(r.y, x + 2);
    pair(r.z, x + 4);
    pair(r.w, x + 6);
  }
  __device__ __forceinline__ static void pair(uint32_t w, float* x) {
    x[0] = __uint_as_float(w << 16);
    x[1] = __uint_as_float(w & 0xFFFF0000u);
  }
};

// Slot j = i * kW + c of lane l holds expert (l + 32 i) * kW + c.
template <typename T, bool kSigmoid, bool kBias, bool kGrouped>
__global__ void __launch_bounds__(kThreads, 2)
    moe_topk_gating_kernel(const T* __restrict__ logits, long long ld,
                           const float* __restrict__ bias, int* __restrict__ topk_ids,
                           float* __restrict__ topk_weights, int rows, int E, int topk, int G,
                           int topk_group, int renormalize, float scaling) {
  constexpr int kW = Vec<T>::kWidth;
  constexpr int kVec = kSlots / kW;
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long t = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (t >= rows) return;  // the whole warp leaves together
  const T* row = logits + t * ld;
  const int nvec = (E + kW - 1) / kW;

  float x[kSlots];
#pragma unroll
  for (int i = 0; i < kVec; i++) {
    const int v = lane + 32 * i;
    if (v < nvec) {
      Vec<T>::unpack(ld_nc_v4(row + static_cast<long long>(v) * kW), x + i * kW);
    } else {
#pragma unroll
      for (int c = 0; c < kW; c++) x[i * kW + c] = 0.f;
    }
  }
  auto expert = [&](int j) { return (lane + 32 * (j / kW)) * kW + j % kW; };

  // softmax statistics over all E: fmaxf skips NaN; each lane sums its slots in order, then the
  // butterfly adds the lanes (every lane ends with the same bits)
  float mx = -INFINITY, sum_e = 0.f;
  if constexpr (!kSigmoid) {
#pragma unroll
    for (int j = 0; j < kSlots; j++)
      if (expert(j) < E) mx = fmaxf(mx, x[j]);
    mx = warp_max_f32(mx);
#pragma unroll
    for (int j = 0; j < kSlots; j++)
      if (expert(j) < E) sum_e += expf(x[j] - mx);
    sum_e = warp_sum_f32(sum_e);
  }
  auto score = [&](float v) { return kSigmoid ? sigmoid(v) : expf(v - mx) / sum_e; };

  uint64_t p[kSlots];
#pragma unroll
  for (int j = 0; j < kSlots; j++) {
    const int e = expert(j);
    p[j] = 0;
    if (e < E) {
      float c = x[j];
      if constexpr (kSigmoid || kBias) c = score(x[j]);
      if constexpr (kBias) c = c + __ldg(bias + e);
      p[j] = pack(ord_key(c), e);
    }
  }

  if constexpr (kGrouped) {
    // group g's score lives in slot g / 32 of lane g % 32
    const int gsize = E / G;
    uint64_t gp[kSlots];
#pragma unroll
    for (int jj = 0; jj < kSlots; jj++) {
      gp[jj] = 0;
      for (int q = 0; q < 32; q++) {
        const int g = 32 * jj + q;
        if (g >= G) break;
        const unsigned lo = static_cast<unsigned>(g * gsize);
        int a1 = INT_MIN, a2 = INT_MIN;  // the lane's two largest keys of group g
#pragma unroll
        for (int j = 0; j < kSlots; j++) {
          if (static_cast<unsigned>(expert(j)) - lo < static_cast<unsigned>(gsize)) {
            const int k = packed_ord(p[j]);
            if (k > a1) {
              a2 = a1;
              a1 = k;
            } else if (k > a2) {
              a2 = k;
            }
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const int b1 = __shfl_xor_sync(0xffffffffu, a1, o);
          const int b2 = __shfl_xor_sync(0xffffffffu, a2, o);
          a2 = max(min(a1, b1), max(a2, b2));
          a1 = max(a1, b1);
        }
        const int gs = kBias ? ord_key(key_value(a1) + key_value(a2)) : a1;
        if (lane == q) gp[jj] = pack(gs, g);
      }
    }
    uint32_t keep = 0;  // the lane's slots in a chosen group
    for (int r = 0; r < topk_group; r++) {
      const uint64_t win = argmax(gp);
      const unsigned lo = static_cast<unsigned>(packed_id(win) * gsize);
#pragma unroll
      for (int jj = 0; jj < kSlots; jj++)
        if (gp[jj] == win) gp[jj] = 0;
#pragma unroll
      for (int j = 0; j < kSlots; j++)
        if (static_cast<unsigned>(expert(j)) - lo < static_cast<unsigned>(gsize)) keep |= 1u << j;
    }
#pragma unroll
    for (int j = 0; j < kSlots; j++)
      if (!((keep >> j) & 1u)) p[j] = 0;
  }

  // k rounds of arg-max; the winner's owner lane hands its logit to every lane, which all compute
  // its score with the same instructions that made the key
  float wsum = 0.f, my_w = 0.f;
  int my_id = 0;
  for (int r = 0; r < topk; r++) {
    const uint64_t win = argmax(p);
    const int id = packed_id(win);
    float xo = 0.f;
#pragma unroll
    for (int j = 0; j < kSlots; j++) {
      if (p[j] == win) {
        xo = x[j];
        p[j] = 0;
      }
    }
    const float s = score(__shfl_sync(0xffffffffu, xo, (id / kW) & 31));
    wsum += s;
    if (lane == r) {
      my_id = id;
      my_w = s;
    }
  }
  if (lane < topk) {
    float w = my_w;
    if (renormalize) w = w / wsum;
    w = w * scaling;
    topk_ids[t * topk + lane] = my_id;
    topk_weights[t * topk + lane] = w;
  }
}

template <typename T, bool kSigmoid, bool kBias>
static cudaError_t launch(bool grouped, int grid, cudaStream_t stream, const void* logits,
                          long long ld, const float* bias, int* ids, float* w, int rows, int E,
                          int topk, int G, int topk_group, int renormalize, float scaling) {
  const T* x = static_cast<const T*>(logits);
  if (grouped)
    return launch_pdl(moe_topk_gating_kernel<T, kSigmoid, kBias, true>, dim3(grid), dim3(kThreads),
                      0, stream, 1, x, ld, bias, ids, w, rows, E, topk, G, topk_group, renormalize,
                      scaling);
  return launch_pdl(moe_topk_gating_kernel<T, kSigmoid, kBias, false>, dim3(grid), dim3(kThreads),
                    0, stream, 1, x, ld, bias, ids, w, rows, E, topk, G, topk_group, renormalize,
                    scaling);
}

template <typename T>
static cudaError_t launch_dtype(int scoring, bool has_bias, bool grouped, int grid,
                                cudaStream_t stream, const void* logits, long long ld,
                                const float* bias, int* ids, float* w, int rows, int E, int topk,
                                int G, int topk_group, int renormalize, float scaling) {
#define HPC_GATING_LAUNCH(S, B)                                                                 \
  return launch<T, S, B>(grouped, grid, stream, logits, ld, bias, ids, w, rows, E, topk, G,    \
                         topk_group, renormalize, scaling)
  if (scoring == 1) {
    if (has_bias) HPC_GATING_LAUNCH(true, true);
    HPC_GATING_LAUNCH(true, false);
  }
  if (has_bias) HPC_GATING_LAUNCH(false, true);
  HPC_GATING_LAUNCH(false, false);
#undef HPC_GATING_LAUNCH
}

}  // namespace gating
}  // namespace b200

using namespace b200;  // NOLINT

extern "C" int hpc_moe_topk_gating_async(const void* router_logits_ptr,
                                         const float* correction_bias_ptr, int* topk_ids_ptr,
                                         float* topk_weights_ptr, int num_tokens, int num_experts,
                                         int logits_dtype, int topk, int scoring, int renormalize,
                                         int num_expert_group, int topk_group, int64_t row_stride,
                                         float routed_scaling_factor, cudaStream_t stream) {
  const int E = num_experts, G = num_expert_group;
  HPC_REQUIRE(num_tokens >= 0, "moe_topk_gating: negative number of tokens %d", num_tokens);
  HPC_REQUIRE(E >= 1 && E <= gating::kMaxExperts,
              "moe_topk_gating: number of experts %d outside [1, %d]", E, gating::kMaxExperts);
  HPC_REQUIRE(topk >= 1 && topk <= gating::kMaxTopk && topk <= E,
              "moe_topk_gating: topk %d outside [1, min(%d, number of experts %d)]", topk,
              gating::kMaxTopk, E);
  HPC_REQUIRE(logits_dtype == 0 || logits_dtype == 1,
              "moe_topk_gating: logits dtype code %d is neither 0 (float32) nor 1 (bfloat16)",
              logits_dtype);
  HPC_REQUIRE(scoring == 0 || scoring == 1,
              "moe_topk_gating: scoring %d is neither 0 (softmax) nor 1 (sigmoid)", scoring);
  HPC_REQUIRE(G >= 1 && E % G == 0,
              "moe_topk_gating: num_expert_group %d must be positive and divide the %d experts", G,
              E);
  HPC_REQUIRE(topk_group >= 1 && topk_group <= G,
              "moe_topk_gating: topk_group %d outside [1, num_expert_group %d]", topk_group, G);
  HPC_REQUIRE(topk <= topk_group * (E / G),
              "moe_topk_gating: topk %d exceeds the %d experts of topk_group %d groups", topk,
              topk_group * (E / G), topk_group);
  HPC_REQUIRE(G == 1 || correction_bias_ptr == nullptr || E / G >= 2,
              "moe_topk_gating: a correction bias with groups needs at least 2 experts per group "
              "(the group score is the sum of its top-2 keys), got %d", E / G);
  const int esize = logits_dtype == 0 ? 4 : 2;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  // the stride between rows matters only when there are two or more of them
  HPC_REQUIRE(num_tokens <= 1 || (row_stride >= E && (row_stride * esize) % 16 == 0),
              "moe_topk_gating: row stride %lld elements must be at least the %d experts and a "
              "multiple of 16 bytes", static_cast<long long>(row_stride), E);
  if (num_tokens == 0) return HPC_OK;
  HPC_REQUIRE(router_logits_ptr != nullptr && topk_ids_ptr != nullptr &&
                  topk_weights_ptr != nullptr,
              "moe_topk_gating: router_logits, topk_ids and topk_weights must not be null");
  HPC_REQUIRE(al16(router_logits_ptr), "moe_topk_gating: router_logits must be 16-byte aligned");
  const int grid = (num_tokens + gating::kWarps - 1) / gating::kWarps;
  const bool has_bias = correction_bias_ptr != nullptr;
  const bool grouped = G > 1;
  cudaError_t err;
  if (logits_dtype == 0)
    err = gating::launch_dtype<float>(scoring, has_bias, grouped, grid, stream, router_logits_ptr,
                                      row_stride, correction_bias_ptr, topk_ids_ptr,
                                      topk_weights_ptr, num_tokens, E, topk, G, topk_group,
                                      renormalize, routed_scaling_factor);
  else
    err = gating::launch_dtype<__nv_bfloat16>(scoring, has_bias, grouped, grid, stream,
                                              router_logits_ptr, row_stride, correction_bias_ptr,
                                              topk_ids_ptr, topk_weights_ptr, num_tokens, E, topk,
                                              G, topk_group, renormalize, routed_scaling_factor);
  HPC_CUDA_CHECK(err);
  return HPC_OK;
}
