// Fused token sampler: repetition penalty -> temperature -> [softmax] -> top-k -> [softmax] ->
// top-p -> Gumbel-max, and the penalty-mask write-back, in one launch (DESIGN.md §3.10).
//
// A row is split into `S` slices (S in {1, 2, 4, 8}, as many CTAs as the SMs up to that cap),
// one CTA per slice, and the S CTAs of a row form a thread-block cluster: each CTA reduces its slice
// and the rank-0 CTA merges the slices through distributed shared memory. Selection works on the
// tempered logits x for every softmax policy (exp is monotonic), so the chosen candidates and their
// order are exact; only p = softmax(x) and log p carry rounding.
//
// Internal noise is Philox4x32-10 keyed by the seed; counter = (token / 4, row, launch offset). The
// launch offset is `rng_base + *rng_word`; the last CTA of the launch advances *rng_word.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include <climits>

#include "sampler_common.cuh"

namespace cg = cooperative_groups;

namespace b200 {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr unsigned kFull = 0xffffffffu;

struct SamplerParams {
  const void* logits;
  int64_t row_stride;  // elements
  int batch, vocab;
  uint8_t* mask;  // [MAX_BS, mask_stride] bit per token, or null
  int64_t mask_stride;
  const int* slot;
  const float* rp;
  float rp_val;
  const float* temp;
  float temp_val;
  int policy;  // 0 NONE, 1 BEFORE_TOPK, 2 AFTER_TOPK
  const void* topk;
  int topk_is64;
  int topk_val;
  const float* topp;
  float topp_val;
  const float* noise;  // [B, V] fp32 Gumbel noise, or null for Philox
  const int64_t* draft;
  uint64_t seed;
  unsigned long long* rng_word;  // [0] launch counter, [1] low half: finished-CTA counter
  uint64_t rng_base;
  int* out;
  int chunks_per_slice;  // 8-token chunks
};

__device__ __forceinline__ float noise_at(const SamplerParams& p, int row, int tok, uint64_t offset) {
  if (p.noise != nullptr) return p.noise[static_cast<int64_t>(row) * p.vocab + tok];
  const float4 g = philox_gumbel4(p.seed, static_cast<uint32_t>(tok) >> 2, row, offset);
  const int j = tok & 3;
  return j == 0 ? g.x : j == 1 ? g.y : j == 2 ? g.z : g.w;
}

struct RowScalars {
  float rp, inv_rp, temp;
  const uint8_t* mask_row;
};

__device__ __forceinline__ RowScalars row_scalars(const SamplerParams& p, int b) {
  RowScalars s;
  s.rp = p.rp != nullptr ? p.rp[b] : p.rp_val;
  s.inv_rp = __fdiv_rn(1.0f, s.rp);
  s.temp = p.temp != nullptr ? p.temp[b] : p.temp_val;
  s.mask_row = (p.mask != nullptr && s.rp > 0.f) ? p.mask + p.slot[b] * p.mask_stride : nullptr;
  return s;
}

// steps 1-3 on the chunk of tokens 8c .. 8c+7
__device__ __forceinline__ void penalise_and_temper(const RowScalars& s, int c, float (&x)[8]) {
  if (s.mask_row != nullptr) {
    const uint32_t bits = s.mask_row[c];
#pragma unroll
    for (int j = 0; j < 8; j++)
      if ((bits >> j) & 1u) x[j] = x[j] > 0.f ? __fmul_rn(x[j], s.inv_rp) : __fmul_rn(x[j], s.rp);
  }
  if (s.temp > 0.f) {
#pragma unroll
    for (int j = 0; j < 8; j++) x[j] = __fdiv_rn(x[j], s.temp);
  }
}

// ================================ temperature-only fast path ======================================
__device__ __forceinline__ void argmax_step(float s, int id, float& best, int& best_id) {
  if (better(s, id, best, best_id)) best = s, best_id = id;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) sampler_temperature_kernel(const SamplerParams p) {
  __shared__ float red_v[kWarps];
  __shared__ int red_i[kWarps];
  cg::cluster_group cluster = cg::this_cluster();
  const int b = blockIdx.y;
  const int slice = static_cast<int>(cluster.block_rank());
  pdl_wait();
  const uint64_t offset = launch_offset(p.rng_word, p.rng_base);
  const T* row = static_cast<const T*>(p.logits) + b * p.row_stride;
  const float temp = p.temp != nullptr ? p.temp[b] : p.temp_val;
  const bool sample = temp > 0.f;  // false for t <= 0 and NaN: plain argmax
  const int64_t d = p.draft != nullptr ? p.draft[b] : -1;
  const int c0 = slice * p.chunks_per_slice;
  const int c1 = min(c0 + p.chunks_per_slice, p.vocab / 8);
  const float* noise_row = p.noise != nullptr ? p.noise + static_cast<int64_t>(b) * p.vocab : nullptr;

  float best = -INFINITY;
  int best_id = INT_MAX;
  for (int c = c0 + threadIdx.x; c < c1; c += kThreads) {
    float x[8];
    load8(row, c, x);
    if (sample) {
#pragma unroll
      for (int j = 0; j < 8; j++) x[j] = __fdiv_rn(x[j], temp);
      float g[8];
      if (noise_row != nullptr) {
        const float4 a = ld_nc_f4(noise_row + 8 * c), e = ld_nc_f4(noise_row + 8 * c + 4);
        g[0] = a.x, g[1] = a.y, g[2] = a.z, g[3] = a.w, g[4] = e.x, g[5] = e.y, g[6] = e.z, g[7] = e.w;
      } else {
        const float4 a = philox_gumbel4(p.seed, 2 * c, b, offset), e = philox_gumbel4(p.seed, 2 * c + 1, b, offset);
        g[0] = a.x, g[1] = a.y, g[2] = a.z, g[3] = a.w, g[4] = e.x, g[5] = e.y, g[6] = e.z, g[7] = e.w;
      }
#pragma unroll
      for (int j = 0; j < 8; j++) x[j] = __fadd_rn(x[j], g[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) argmax_step(8 * c + j == d ? -INFINITY : x[j], 8 * c + j, best, best_id);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(kFull, best, o);
    const int i = __shfl_xor_sync(kFull, best_id, o);
    argmax_step(v, i, best, best_id);
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) red_v[warp] = best, red_i[warp] = best_id;
  __syncthreads();
  if (warp == 0) {
    best = lane < kWarps ? red_v[lane] : -INFINITY;
    best_id = lane < kWarps ? red_i[lane] : INT_MAX;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(kFull, best, o);
      const int i = __shfl_xor_sync(kFull, best_id, o);
      argmax_step(v, i, best, best_id);
    }
    if (lane == 0) red_v[0] = best, red_i[0] = best_id;
  }
  cluster.sync();
  if (slice == 0 && warp == 0) {
    const int n = static_cast<int>(cluster.num_blocks());
    best = -INFINITY, best_id = INT_MAX;
    if (lane < n) {
      best = *cluster.map_shared_rank(&red_v[0], lane);
      best_id = *cluster.map_shared_rank(&red_i[0], lane);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(kFull, best, o);
      const int i = __shfl_xor_sync(kFull, best_id, o);
      argmax_step(v, i, best, best_id);
    }
    if (lane == 0) p.out[b] = best_id;
  }
  cluster.sync();  // keep every CTA's shared memory alive until rank 0 has read it
  advance_rng(p.rng_word);
}

// ===================================== full path ==================================================
// A sorted top-KMAX list held by one warp: lane l keeps ranks l, l + 32, ...
template <int KMAX>
struct WarpTopK {
  static constexpr int R = KMAX / 32;
  float v[R];
  int id[R];
  float thr_v;  // rank KMAX - 1: a candidate must beat it to enter
  int thr_id;

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int r = 0; r < R; r++) v[r] = -INFINITY, id[r] = INT_MAX;
    thr_v = -INFINITY, thr_id = INT_MAX;
  }

  __device__ __forceinline__ void insert(float cv, int ci, int lane) {
    int pos = 0;
#pragma unroll
    for (int r = 0; r < R; r++) pos += __popc(__ballot_sync(kFull, better(v[r], id[r], cv, ci)));
#pragma unroll
    for (int r = R - 1; r >= 0; r--) {
      float up_v = __shfl_up_sync(kFull, v[r], 1);
      int up_i = __shfl_up_sync(kFull, id[r], 1);
      if (r > 0) {
        const float carry_v = __shfl_sync(kFull, v[r > 0 ? r - 1 : 0], 31);
        const int carry_i = __shfl_sync(kFull, id[r > 0 ? r - 1 : 0], 31);
        if (lane == 0) up_v = carry_v, up_i = carry_i;
      }
      const int g = lane + 32 * r;
      if (g > pos) {
        v[r] = up_v, id[r] = up_i;
      } else if (g == pos) {
        v[r] = cv, id[r] = ci;
      }
    }
    thr_v = __shfl_sync(kFull, v[R - 1], 31);
    thr_id = __shfl_sync(kFull, id[R - 1], 31);
  }

  // every lane offers one candidate; most fail the threshold test and cost one compare
  __device__ __forceinline__ void offer(float x, int i, int lane) {
    unsigned m = __ballot_sync(kFull, better(x, i, thr_v, thr_id));
    while (m != 0) {
      const int src = __ffs(m) - 1;
      m &= m - 1;
      const float cv = __shfl_sync(kFull, x, src);
      const int ci = __shfl_sync(kFull, i, src);
      if (better(cv, ci, thr_v, thr_id)) insert(cv, ci, lane);
    }
  }
};

// Merge sorted lists pairwise in shared memory until one is left in list 0. Entries are distinct
// (token ids are), so each entry's rank in the merged list is its index plus the number of entries
// of the other list that are better.
template <int KMAX>
__device__ void merge_lists(float* val, int* ids, float* tv, int* ti, int n) {
  for (; n > 1; n = (n + 1) / 2) {
    const int pairs = n / 2;
    for (int e = threadIdx.x; e < pairs * 2 * KMAX; e += kThreads) {
      const int pr = e / (2 * KMAX), side = (e / KMAX) & 1, i = e % KMAX;
      const int self = (2 * pr + side) * KMAX, other = (2 * pr + 1 - side) * KMAX;
      const float x = val[self + i];
      const int xi = ids[self + i];
      int lo = 0, hi = KMAX;  // count of entries in `other` better than (x, xi)
      while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (better(val[other + mid], ids[other + mid], x, xi)) lo = mid + 1; else hi = mid;
      }
      const int rank = i + lo;
      if (rank < KMAX) tv[pr * KMAX + rank] = x, ti[pr * KMAX + rank] = xi;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < pairs * KMAX; e += kThreads) val[e] = tv[e], ids[e] = ti[e];
    if (n & 1)  // odd list out moves down to slot `pairs`
      for (int e = threadIdx.x; e < KMAX; e += kThreads)
        val[pairs * KMAX + e] = val[(n - 1) * KMAX + e], ids[pairs * KMAX + e] = ids[(n - 1) * KMAX + e];
    __syncthreads();
  }
}

template <typename T, int KMAX>
__global__ void __launch_bounds__(kThreads, 1) sampler_full_kernel(const SamplerParams p) {
  constexpr int kLists = kWarps > kSamplerMaxSlices ? kWarps : kSamplerMaxSlices;
  __shared__ float lv[kLists * KMAX];
  __shared__ int li[kLists * KMAX];
  __shared__ float tv[kLists / 2 * KMAX];
  __shared__ int ti[kLists / 2 * KMAX];
  __shared__ float red_m[kWarps], red_s[kWarps];
  cg::cluster_group cluster = cg::this_cluster();
  const int b = blockIdx.y;
  const int slice = static_cast<int>(cluster.block_rank());
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  pdl_wait();
  const uint64_t offset = launch_offset(p.rng_word, p.rng_base);
  const T* row = static_cast<const T*>(p.logits) + b * p.row_stride;
  const RowScalars rs = row_scalars(p, b);
  const bool before = p.policy == 1;
  const int c0 = slice * p.chunks_per_slice;
  const int c1 = min(c0 + p.chunks_per_slice, p.vocab / 8);

  WarpTopK<KMAX> top;
  top.init();
  float m = -INFINITY, s = 0.f;
  // one chunk of 8 consecutive tokens per lane per step; the trip count is warp-uniform
  const int steps = (c1 - c0 + kThreads - 1) / kThreads;
  for (int k = 0; k < steps; k++) {
    const int c = c0 + k * kThreads + threadIdx.x;
    const bool valid = c < c1;
    float x[8];
    if (valid) {
      load8(row, c, x);
      penalise_and_temper(rs, c, x);
    } else {
#pragma unroll
      for (int j = 0; j < 8; j++) x[j] = -INFINITY;
    }
    if (before && valid) {
#pragma unroll
      for (int j = 0; j < 8; j++) online_add(x[j], m, s);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) top.offer(x[j], valid ? 8 * c + j : INT_MAX, lane);
  }
#pragma unroll
  for (int r = 0; r < WarpTopK<KMAX>::R; r++)
    lv[warp * KMAX + lane + 32 * r] = top.v[r], li[warp * KMAX + lane + 32 * r] = top.id[r];
  if (before) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(kFull, m, o), s2 = __shfl_xor_sync(kFull, s, o);
      online_merge(m2, s2, m, s);
    }
    if (lane == 0) red_m[warp] = m, red_s[warp] = s;
  }
  __syncthreads();
  merge_lists<KMAX>(lv, li, tv, ti, kWarps);
  if (before && threadIdx.x == 0) {
    for (int w = 1; w < kWarps; w++) online_merge(red_m[w], red_s[w], red_m[0], red_s[0]);
  }
  cluster.sync();
  const int n = static_cast<int>(cluster.num_blocks());
  if (slice == 0) {
    if (n > 1) {
      // the other slices' lists go after our own, then merge again
      for (int e = threadIdx.x; e < (n - 1) * KMAX; e += kThreads) {
        const int src = 1 + e / KMAX, i = e % KMAX;
        lv[src * KMAX + i] = *cluster.map_shared_rank(&lv[i], src);
        li[src * KMAX + i] = *cluster.map_shared_rank(&li[i], src);
      }
      if (before && threadIdx.x == 0) {
        for (int r = 1; r < n; r++)
          online_merge(*cluster.map_shared_rank(&red_m[0], r), *cluster.map_shared_rank(&red_s[0], r),
                       red_m[0], red_s[0]);
      }
    }
  }
  cluster.sync();  // remote reads done: the other CTAs may leave
  if (slice != 0) {
    advance_rng(p.rng_word);
    return;
  }
  if (n > 1) merge_lists<KMAX>(lv, li, tv, ti, n);

  if (warp == 0) {
    constexpr int R = KMAX / 32;
    int64_t kb64 = p.topk_val;
    if (p.topk != nullptr)
      kb64 = p.topk_is64 ? static_cast<const int64_t*>(p.topk)[b] : static_cast<const int*>(p.topk)[b];
    const int kb = (kb64 >= 1 && kb64 <= KMAX) ? static_cast<int>(kb64) : KMAX;
    const float topp = p.topp != nullptr ? p.topp[b] : p.topp_val;
    float x[R], pr[R];
    int tok[R];
#pragma unroll
    for (int r = 0; r < R; r++) x[r] = lv[lane + 32 * r], tok[r] = li[lane + 32 * r];
    if (p.policy != 0) {
      // p = exp(x - M) / S, and 0 wherever exp(x - M) is 0 (the -inf logits, ranks >= K_b)
      const float top_x = lv[0];
      float e_sum = 0.f;
#pragma unroll
      for (int r = 0; r < R; r++) {
        pr[r] = (lane + 32 * r < kb && x[r] != -INFINITY) ? expf(x[r] - top_x) : 0.f;
        e_sum += pr[r];
      }
      const float denom = before ? red_s[0] : warp_sum_f32(e_sum);
#pragma unroll
      for (int r = 0; r < R; r++) pr[r] = pr[r] > 0.f ? __fdiv_rn(pr[r], denom) : 0.f;
    }
    // top-p: keep rank 0 and every rank whose exclusive prefix sum of p is below topp
    bool keep[R];
    float carry = 0.f;
#pragma unroll
    for (int r = 0; r < R; r++) {
      float inc = p.policy != 0 ? pr[r] : 0.f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(kFull, inc, o);
        if (lane >= o) inc = __fadd_rn(inc, t);
      }
      const float prev = __shfl_up_sync(kFull, inc, 1);
      const float excl = lane > 0 ? __fadd_rn(carry, prev) : carry;
      const int rank = lane + 32 * r;
      keep[r] = rank < kb && (rank == 0 || !(topp > 0.f) || excl < topp);
      carry = __fadd_rn(carry, __shfl_sync(kFull, inc, 31));
    }
    float best = -INFINITY;
    int best_id = INT_MAX;
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (lane + 32 * r >= kb) continue;
      float key = -INFINITY;
      if (keep[r]) {
        const float val = p.policy == 0 ? x[r] : (pr[r] > 0.f ? logf(pr[r]) : -INFINITY);
        key = __fadd_rn(val, noise_at(p, b, tok[r], offset));
      }
      argmax_step(key, tok[r], best, best_id);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(kFull, best, o);
      const int i = __shfl_xor_sync(kFull, best_id, o);
      argmax_step(v, i, best, best_id);
    }
    if (lane == 0) {
      p.out[b] = best_id;
      if (p.mask != nullptr) {
        uint8_t* byte = p.mask + p.slot[b] * p.mask_stride + best_id / 8;
        const uintptr_t a = reinterpret_cast<uintptr_t>(byte);
        unsigned int* word = reinterpret_cast<unsigned int*>(a & ~uintptr_t(3));
        atomicOr(word, (1u << (best_id % 8)) << (8 * (a & 3)));
      }
    }
  }
  advance_rng(p.rng_word);
}

template <typename T>
int launch(const SamplerParams& p0, bool full, int max_topk, cudaStream_t stream) {
  SamplerParams p = p0;
  const int s = pick_slices(p.batch, p.vocab);
  p.chunks_per_slice = (p.vocab / 8 + s - 1) / s;
  const dim3 grid(s, p.batch);
  if (!full) {
    HPC_CUDA_CHECK(launch_pdl(sampler_temperature_kernel<T>, grid, dim3(kThreads), 0, stream, s, p));
  } else if (max_topk == 32) {
    HPC_CUDA_CHECK(launch_pdl(sampler_full_kernel<T, 32>, grid, dim3(kThreads), 0, stream, s, p));
  } else {
    HPC_CUDA_CHECK(launch_pdl(sampler_full_kernel<T, 64>, grid, dim3(kThreads), 0, stream, s, p));
  }
  return HPC_OK;
}

int dispatch(SamplerParams& p, int dtype, bool full, int max_topk, cudaStream_t stream) {
  if (p.batch == 0) return HPC_OK;
  if (p.noise == nullptr) {
    RngState st;
    const int rc = rng_state(stream, &st);
    if (rc != HPC_OK) return rc;
    p.rng_word = st.word;
    p.rng_base = st.base;
  }
  return dtype == 0 ? launch<float>(p, full, max_topk, stream)
                    : launch<__nv_bfloat16>(p, full, max_topk, stream);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int hpc_fused_sampler_async(
    int* out, const void* logits, int64_t row_stride, int dtype, int batch, int vocab,
    uint8_t* penalty_mask, int64_t mask_stride, const int* slot_id, const float* repetition_penalty,
    float repetition_penalty_val, const float* temperature, float temperature_val, int softmax_policy,
    const void* topk, int topk_is_int64, int topk_val, const float* topp, float topp_val,
    int max_topk, const float* gumbel_noise, uint64_t seed, cudaStream_t stream) {
  const char* who = "fused_sampler";
  HPC_REQUIRE(max_topk == 32 || max_topk == 64, "%s: max_topk %d is not one of the built sizes 32, 64", who, max_topk);
  const int rc = check_common(logits, row_stride, dtype, batch, vocab, max_topk, who);
  if (rc != HPC_OK) return rc;
  HPC_REQUIRE(softmax_policy >= 0 && softmax_policy <= 2, "%s: softmax_policy %d is not 0, 1 or 2", who, softmax_policy);
  HPC_REQUIRE((penalty_mask == nullptr) == (slot_id == nullptr),
              "%s: penalty_mask and slot_id go together: pass both or neither", who);
  HPC_REQUIRE(penalty_mask == nullptr ||
                  (mask_stride >= vocab / 8 && reinterpret_cast<uintptr_t>(penalty_mask) % 4 == 0),
              "%s: penalty_mask must be 4-byte aligned with rows of at least V/8 bytes", who);
  HPC_REQUIRE(gumbel_noise != nullptr || seed > 0, "%s: the kernel's own noise needs a seed >= 1", who);
  HPC_REQUIRE(reinterpret_cast<uintptr_t>(gumbel_noise) % 16 == 0, "%s: gumbel_noise must be 16-byte aligned", who);
  SamplerParams p = {};
  p.logits = logits, p.row_stride = row_stride, p.batch = batch, p.vocab = vocab;
  p.mask = penalty_mask, p.mask_stride = mask_stride, p.slot = slot_id;
  p.rp = repetition_penalty, p.rp_val = repetition_penalty_val;
  p.temp = temperature, p.temp_val = temperature_val;
  p.policy = softmax_policy;
  p.topk = topk, p.topk_is64 = topk_is_int64, p.topk_val = topk_val;
  p.topp = topp, p.topp_val = topp_val;
  p.noise = gumbel_noise, p.seed = seed, p.out = out;
  return dispatch(p, dtype, true, max_topk, stream);
}

extern "C" int hpc_fused_sampler_temperature_sample_async(
    int* out, const void* logits, int64_t row_stride, int dtype, int batch, int vocab,
    const float* temperature, float temperature_val, const float* gumbel_noise,
    const int64_t* draft_token_ids, uint64_t seed, cudaStream_t stream) {
  const char* who = "fused_sampler_temperature_sample";
  const int rc = check_common(logits, row_stride, dtype, batch, vocab, 1, who);
  if (rc != HPC_OK) return rc;
  HPC_REQUIRE(gumbel_noise != nullptr || seed > 0, "%s: the kernel's own noise needs a seed >= 1", who);
  HPC_REQUIRE(reinterpret_cast<uintptr_t>(gumbel_noise) % 16 == 0, "%s: gumbel_noise must be 16-byte aligned", who);
  SamplerParams p = {};
  p.logits = logits, p.row_stride = row_stride, p.batch = batch, p.vocab = vocab;
  p.temp = temperature, p.temp_val = temperature_val;
  p.noise = gumbel_noise, p.draft = draft_token_ids, p.seed = seed, p.out = out;
  return dispatch(p, dtype, false, 32, stream);
}

extern "C" int hpc_sampler_rng_offset(cudaStream_t stream, uint64_t* offset) {
  RngState st;
  const int rc = rng_state(stream, &st);
  if (rc != HPC_OK) return rc;
  unsigned long long w = 0;
  HPC_CUDA_CHECK(cudaMemcpyAsync(&w, st.word, sizeof(w), cudaMemcpyDeviceToHost, stream));
  HPC_CUDA_CHECK(cudaStreamSynchronize(stream));
  *offset = st.base + w;
  return HPC_OK;
}
