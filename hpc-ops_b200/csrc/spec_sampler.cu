// Fused speculative sampling (DESIGN.md §3.15): accept or reject the K draft tokens of each
// request against the target model's logits and draw the recovered or bonus token, in two launches
// chained by programmatic dependent launch, with no host synchronisation and no allocation.
//
// 1. spec_row_stats_kernel streams every row r = b (K + 1) + i of the logits once and writes a
//    32-byte record: for sampling requests (t > 0) the softmax statistics (m, Z) of x / t, p(d_i)
//    and q_i(d_i); for greedy requests the argmax of x. No noise is drawn here.
// 2. spec_sample_kernel runs one cluster per request. Every CTA decides the request's acceptances
//    from its K records (cheap), then the cluster streams only the emitting row, draws noise there
//    and merges the winner; rank 0 writes the request's tokens and count. Greedy requests stream
//    nothing.
// Both use the fused sampler's row split (pick_slices, S-CTA clusters merged through distributed
// shared memory in rank 0), 16-byte loads and Philox mapping (sampler_common.cuh).
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
constexpr int kMaxDraft = 8;
constexpr unsigned kFull = 0xffffffffu;

// Per-row result of pass 1, 32 bytes (the Python layer allocates [rows, 8] int32)
struct RowRecord {
  float m;   // max of x / t (sampling requests)
  float z;   // sum of expf(x / t - m)
  float pd;  // p(d_i) for i < K and d_i in [0, V), else 0
  float qd;  // q_i(d_i) (1 for one-hot drafts) for i < K and d_i in [0, V), else 0
  int amax;  // argmax of x in [0, V), ties to the smaller id (greedy requests)
  int pad[3];
};

struct SpecParams {
  const void* logits;
  int64_t row_stride;  // elements
  int batch, ndraft, vocab;
  const void* draft;  // [B, K] int32 or int64
  int draft_is64;
  const float* draft_probs;  // [B, K, V] fp32, or null: one-hot drafts
  const float* temp;
  float temp_val;
  const float* uniform;  // [B, K] fp32, or null: Philox
  const float* noise;    // [B (K + 1), V] fp32 Gumbel noise, or null: Philox
  uint64_t seed;
  unsigned long long* rng_word;
  uint64_t rng_base;
  RowRecord* rec;     // [B (K + 1)]
  int* out;           // [B, K + 1]
  int* num_accepted;  // [B]
  int chunks_per_slice;
};

__device__ __forceinline__ float temp_of(const SpecParams& p, int b) {
  return p.temp != nullptr ? p.temp[b] : p.temp_val;
}

__device__ __forceinline__ int64_t draft_of(const SpecParams& p, int b, int i) {
  const int64_t k = static_cast<int64_t>(b) * p.ndraft + i;
  return p.draft_is64 ? static_cast<const int64_t*>(p.draft)[k] : static_cast<const int*>(p.draft)[k];
}

__device__ __forceinline__ void argmax_step(float s, int id, float& best, int& best_id) {
  if (better(s, id, best, best_id)) best = s, best_id = id;
}

template <int WIDTH>
__device__ __forceinline__ void shfl_argmax(float& best, int& best_id) {
#pragma unroll
  for (int o = WIDTH / 2; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(kFull, best, o);
    const int i = __shfl_xor_sync(kFull, best_id, o);
    argmax_step(v, i, best, best_id);
  }
}

// CTA arg-max of (best, best_id) into red_v[0], red_i[0]
__device__ __forceinline__ void cta_argmax(float best, int best_id, float* red_v, int* red_i) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  shfl_argmax<32>(best, best_id);
  if (lane == 0) red_v[warp] = best, red_i[warp] = best_id;
  __syncthreads();
  if (warp == 0) {
    best = lane < kWarps ? red_v[lane] : -INFINITY;
    best_id = lane < kWarps ? red_i[lane] : INT_MAX;
    shfl_argmax<kWarps>(best, best_id);
    if (lane == 0) red_v[0] = best, red_i[0] = best_id;
  }
}

// Cluster arg-max of every CTA's red_v[0], red_i[0], valid in warp 0 of rank 0 (after a
// cluster.sync that follows cta_argmax)
__device__ __forceinline__ void cluster_argmax(cg::cluster_group& cluster, float* red_v, int* red_i,
                                               float& best, int& best_id) {
  const int lane = threadIdx.x % 32;
  const int n = static_cast<int>(cluster.num_blocks());
  best = -INFINITY, best_id = INT_MAX;
  if (lane < n) {
    best = *cluster.map_shared_rank(&red_v[0], lane);
    best_id = *cluster.map_shared_rank(&red_i[0], lane);
  }
  shfl_argmax<kSamplerMaxSlices>(best, best_id);
}

// (max of x, sum of expf((x - max) / t)) of two partials, in units of x; rt = 1 / t
__device__ __forceinline__ void stats_merge(float m2, float s2, float rt, float& m, float& s) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) {
    m = m2, s = s2;
  } else if (m2 > m) {
    s = s * expf((m - m2) * rt) + s2;
    m = m2;
  } else {
    s += s2 * expf((m2 - m) * rt);
  }
}

__device__ __forceinline__ float load1(const float* row, int64_t v) { return row[v]; }
__device__ __forceinline__ float load1(const __nv_bfloat16* row, int64_t v) {
  return __bfloat162float(row[v]);
}

// ======================================== pass 1 ===================================================
template <typename T>
__global__ void __launch_bounds__(kThreads, 4) spec_row_stats_kernel(const SpecParams p) {
  __shared__ float red_a[kWarps], red_b[kWarps];
  __shared__ int red_i[kWarps];
  cg::cluster_group cluster = cg::this_cluster();
  const int r = blockIdx.y;
  const int b = r / (p.ndraft + 1), i = r - b * (p.ndraft + 1);
  const int slice = static_cast<int>(cluster.block_rank());
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  pdl_wait();
  const T* row = static_cast<const T*>(p.logits) + static_cast<int64_t>(r) * p.row_stride;
  const float t = temp_of(p, b);
  const int c0 = slice * p.chunks_per_slice;
  const int c1 = min(c0 + p.chunks_per_slice, p.vocab / 8);

  if (!(t > 0.f)) {  // greedy request (t <= 0 or NaN): argmax of x
    float best = -INFINITY;
    int best_id = INT_MAX;
    for (int c = c0 + threadIdx.x; c < c1; c += kThreads) {
      float x[8];
      load8(row, c, x);
#pragma unroll
      for (int j = 0; j < 8; j++) argmax_step(x[j], 8 * c + j, best, best_id);
    }
    cta_argmax(best, best_id, red_a, red_i);
    cluster.sync();
    if (slice == 0 && warp == 0) {
      cluster_argmax(cluster, red_a, red_i, best, best_id);
      if (lane == 0) {
        RowRecord rec = {};
        rec.amax = best_id == INT_MAX ? 0 : best_id;  // a row of NaN
        p.rec[r] = rec;
      }
    }
    cluster.sync();  // keep every CTA's shared memory alive until rank 0 has read it
    return;
  }

  // sampling request: the max mx of x and s = sum expf((x - mx) * (1 / t)), so m = fl(mx / t) and
  // Z = s (dividing by t > 0 and rounding are monotonic) without a division per token
  const float rt = __frcp_rn(t);
  float mx = -INFINITY, s = 0.f;
  for (int c = c0 + threadIdx.x; c < c1; c += kThreads) {
    float x[8];
    load8(row, c, x);
    float cm = x[0];
#pragma unroll
    for (int j = 1; j < 8; j++) cm = fmaxf(cm, x[j]);
    if (cm > mx) {
      s = s * expf((mx - cm) * rt);
      mx = cm;
    }
    if (mx != -INFINITY) {
#pragma unroll
      for (int j = 0; j < 8; j++) s += expf((x[j] - mx) * rt);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(kFull, mx, o), s2 = __shfl_xor_sync(kFull, s, o);
    stats_merge(m2, s2, rt, mx, s);
  }
  if (lane == 0) red_a[warp] = mx, red_b[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kWarps; w++) stats_merge(red_a[w], red_b[w], rt, red_a[0], red_b[0]);
  }
  cluster.sync();
  if (slice == 0 && threadIdx.x == 0) {
    float m = red_a[0], z = red_b[0];
    const int n = static_cast<int>(cluster.num_blocks());
    for (int q = 1; q < n; q++)
      stats_merge(*cluster.map_shared_rank(&red_a[0], q), *cluster.map_shared_rank(&red_b[0], q), rt, m, z);
    RowRecord rec = {};
    rec.m = __fdiv_rn(m, t);
    rec.z = z;
    if (i < p.ndraft) {
      const int64_t d = draft_of(p, b, i);
      if (d >= 0 && d < p.vocab) {
        const float xt = __fdiv_rn(load1(row, d), t);
        rec.pd = __fdiv_rn(expf(__fsub_rn(xt, rec.m)), rec.z);
        rec.qd = p.draft_probs != nullptr
                     ? p.draft_probs[(static_cast<int64_t>(b) * p.ndraft + i) * p.vocab + d]
                     : 1.f;
      }
    }
    p.rec[r] = rec;
  }
  cluster.sync();
}

// ======================================== pass 2 ===================================================
template <typename T>
__global__ void __launch_bounds__(kThreads) spec_sample_kernel(const SpecParams p) {
  __shared__ float red_v[2][kWarps];
  __shared__ int red_i[2][kWarps];
  __shared__ int s_accepted;
  cg::cluster_group cluster = cg::this_cluster();
  const int b = blockIdx.y;
  const int K = p.ndraft;
  const int slice = static_cast<int>(cluster.block_rank());
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  pdl_wait();
  const uint64_t offset = launch_offset(p.rng_word, p.rng_base);
  const float t = temp_of(p, b);
  const bool sample = t > 0.f;  // false for t <= 0 and NaN: greedy

  // every CTA decides the request: lane i < K judges draft i, the first rejection ends the run
  if (warp == 0) {
    bool accept = false;
    if (lane < K) {
      const int r = b * (K + 1) + lane;
      const int64_t d = draft_of(p, b, lane);
      if (!sample) {
        accept = d == p.rec[r].amax;
      } else if (d >= 0 && d < p.vocab) {
        const float u = p.uniform != nullptr ? p.uniform[b * K + lane]
                                             : uniform_of(philox_at(p.seed, 0xFFFFFFFFu, r, offset).x);
        accept = __fmul_rn(u, p.rec[r].qd) < p.rec[r].pd;
      }
    }
    const unsigned rejected = __ballot_sync(kFull, lane < K && !accept);
    if (lane == 0) s_accepted = rejected != 0 ? __ffs(rejected) - 1 : K;
  }
  __syncthreads();
  const int n = s_accepted;
  const int r = b * (K + 1) + n;  // the row that emits the recovered or bonus token

  int token = 0;
  if (sample) {
    const T* row = static_cast<const T*>(p.logits) + static_cast<int64_t>(r) * p.row_stride;
    const float* noise_row = p.noise != nullptr ? p.noise + static_cast<int64_t>(r) * p.vocab : nullptr;
    // residual max(0, p - q) at a rejected draft with draft_probs; otherwise x / t + g, with a
    // rejected one-hot draft's token excluded as the temperature sampler excludes it
    const bool residual = p.draft_probs != nullptr && n < K;
    const float* q_row =
        residual ? p.draft_probs + (static_cast<int64_t>(b) * K + n) * p.vocab : nullptr;
    const int64_t d = (!residual && n < K) ? draft_of(p, b, n) : -1;
    const float m = p.rec[r].m, z = p.rec[r].z;
    const int c0 = slice * p.chunks_per_slice;
    const int c1 = min(c0 + p.chunks_per_slice, p.vocab / 8);
    float best = -INFINITY, plain = -INFINITY;  // residual key (or the only key), x / t + g
    int best_id = INT_MAX, plain_id = INT_MAX;
    for (int c = c0 + threadIdx.x; c < c1; c += kThreads) {
      float x[8], g[8];
      load8(row, c, x);
#pragma unroll
      for (int j = 0; j < 8; j++) x[j] = __fdiv_rn(x[j], t);
      if (noise_row != nullptr) {
        load8(noise_row, c, g);
      } else {
        const float4 a = philox_gumbel4(p.seed, 2 * c, r, offset), e = philox_gumbel4(p.seed, 2 * c + 1, r, offset);
        g[0] = a.x, g[1] = a.y, g[2] = a.z, g[3] = a.w, g[4] = e.x, g[5] = e.y, g[6] = e.z, g[7] = e.w;
      }
      if (residual) {
        float q[8];
        load8(q_row, c, q);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float pv = __fdiv_rn(expf(__fsub_rn(x[j], m)), z);
          if (pv > q[j]) argmax_step(__fadd_rn(logf(__fsub_rn(pv, q[j])), g[j]), 8 * c + j, best, best_id);
          argmax_step(__fadd_rn(x[j], g[j]), 8 * c + j, plain, plain_id);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float key = __fadd_rn(x[j], g[j]);
          argmax_step(8 * c + j == d ? -INFINITY : key, 8 * c + j, best, best_id);
        }
      }
    }
    cta_argmax(best, best_id, red_v[0], red_i[0]);
    if (residual) cta_argmax(plain, plain_id, red_v[1], red_i[1]);
    cluster.sync();
    if (slice == 0 && warp == 0) {
      cluster_argmax(cluster, red_v[0], red_i[0], best, best_id);
      if (residual) {
        cluster_argmax(cluster, red_v[1], red_i[1], plain, plain_id);
        if (best_id == INT_MAX) best_id = plain_id;  // empty residual: sample from p
      }
      token = __shfl_sync(kFull, best_id, 0);  // the merge leaves it in lanes 0 .. 7 only
    }
    cluster.sync();  // keep every CTA's shared memory alive until rank 0 has read it
  } else if (slice == 0) {
    token = p.rec[r].amax;
  }
  if (slice == 0 && threadIdx.x <= K) {  // warp 0, where every lane holds the token
    const int k = threadIdx.x;
    int v = -1;
    if (k < n) v = static_cast<int>(draft_of(p, b, k));
    else if (k == n) v = token == INT_MAX ? 0 : token;  // no key that is not NaN
    p.out[b * (K + 1) + k] = v;
    if (k == 0) p.num_accepted[b] = n;
  }
  advance_rng(p.rng_word);
}

template <typename T>
int launch(const SpecParams& p0, cudaStream_t stream) {
  SpecParams p = p0;
  const int rows = p.batch * (p.ndraft + 1);
  const int s1 = pick_slices(rows, p.vocab);
  p.chunks_per_slice = (p.vocab / 8 + s1 - 1) / s1;
  HPC_CUDA_CHECK(launch_pdl(spec_row_stats_kernel<T>, dim3(s1, rows), dim3(kThreads), 0, stream, s1, p));
  const int s2 = pick_slices(p.batch, p.vocab);
  p.chunks_per_slice = (p.vocab / 8 + s2 - 1) / s2;
  HPC_CUDA_CHECK(launch_pdl(spec_sample_kernel<T>, dim3(s2, p.batch), dim3(kThreads), 0, stream, s2, p));
  return HPC_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int hpc_fused_speculative_sampler_async(
    int* output_token_ids, int* num_accepted, void* row_records, const void* target_logits,
    int64_t row_stride, int dtype, int batch, int num_draft, int vocab, const void* draft_token_ids,
    int draft_is_int64, const float* draft_probs, const float* temperature, float temperature_val,
    const float* uniform, const float* gumbel_noise, uint64_t seed, cudaStream_t stream) {
  const char* who = "fused_speculative_sampler";
  HPC_REQUIRE(num_draft >= 1 && num_draft <= kMaxDraft, "%s: %d draft tokens per request; 1 to %d are supported",
              who, num_draft, kMaxDraft);
  HPC_REQUIRE(batch >= 0 && batch <= 65535 / (num_draft + 1),
              "%s: batch %d x (K + 1) = %d rows exceeds 65535", who, batch, batch * (num_draft + 1));
  const int rc = check_common(target_logits, row_stride, dtype, batch * (num_draft + 1), vocab, 1, who);
  if (rc != HPC_OK) return rc;
  HPC_REQUIRE((uniform == nullptr) == (gumbel_noise == nullptr),
              "%s: uniform and gumbel_noise go together: pass both or neither", who);
  const bool sampling = temperature != nullptr || temperature_val > 0.f;
  HPC_REQUIRE(gumbel_noise != nullptr || !sampling || seed > 0,
              "%s: the kernel's own noise needs a seed >= 1", who);
  HPC_REQUIRE(reinterpret_cast<uintptr_t>(gumbel_noise) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(draft_probs) % 16 == 0,
              "%s: gumbel_noise and draft_probs must be 16-byte aligned", who);
  HPC_REQUIRE(batch == 0 || (output_token_ids != nullptr && num_accepted != nullptr &&
                             draft_token_ids != nullptr && row_records != nullptr &&
                             reinterpret_cast<uintptr_t>(row_records) % 16 == 0),
              "%s: outputs, draft_token_ids and a 16-byte aligned row-record scratch are required", who);
  if (batch == 0) return HPC_OK;
  SpecParams p = {};
  p.logits = target_logits, p.row_stride = row_stride;
  p.batch = batch, p.ndraft = num_draft, p.vocab = vocab;
  p.draft = draft_token_ids, p.draft_is64 = draft_is_int64, p.draft_probs = draft_probs;
  p.temp = temperature, p.temp_val = temperature_val;
  p.uniform = uniform, p.noise = gumbel_noise, p.seed = seed;
  p.rec = static_cast<RowRecord*>(row_records);
  p.out = output_token_ids, p.num_accepted = num_accepted;
  if (gumbel_noise == nullptr && sampling) {
    RngState st;
    const int rs = rng_state(stream, &st);
    if (rs != HPC_OK) return rs;
    p.rng_word = st.word;
    p.rng_base = st.base;
  }
  return dtype == 0 ? launch<float>(p, stream) : launch<__nv_bfloat16>(p, stream);
}
