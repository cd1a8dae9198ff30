// Stem block-mask generation for block-sparse FP8 prefill (DESIGN.md §3.12): four stages, each one
// C-ABI entry, that turn a paged FP8 KV cache and packed FP8 Q into the u8 block mask
// attention_with_kvcache_blocksparse_prefill_fp8 takes.
//
//   prep_paged_kv  kflat[b, hkv, kb, 16 x 128] bf16: per 128-key block, group g in [0, 16) is the sum
//                  of the dequantised K rows g + 16 r (r < 8), stored in segment 15 - g;
//                  vbias[b, hkv, kb] fp32 from the log-normalised maxima of ||v|| over 16 rows
//                  (a second, one-CTA-per-head kernel: its statistics span the whole request).
//   prep_varlen_q  qflat[b, hq, qb, 16 x 128] bf16, the same group sums of qscale * q, natural order.
//   oam_gemm       logits[b, hq, qb, kb] = qflat . kflat^T / 64 + vbias[hkv], -inf outside the
//                  request and (causal) above the block diagonal. bf16 wgmma, K = 2048.
//   tpd            mask[b, hq, qb, kb] u8: the exact top-`budget` threshold of each row's ordered bf16
//                  keys, or-ed with the sink, the recent window and the diagonal.
//
// The prep kernels stream the cache and Q once with 16-byte loads and are bound by HBM. The GEMM and
// the TPD kernel read only what the previous stage wrote, never synchronise the host and keep no
// state between launches, so they can be captured in a CUDA graph.
#include <cuda_bf16.h>
#include <stdint.h>

#include "common.cuh"
#include "host_utils.h"

namespace b200 {
namespace stem {

constexpr int kBlock = 128;           // stem block: tokens per Q / KV block
constexpr int kStride = 16;           // groups per block
constexpr int kSamples = kBlock / kStride;  // rows summed per group (8)
constexpr int kDim = 128;             // head dim
constexpr int kFlat = kStride * kDim;  // 2048: flattened block vector
constexpr int kPrepThreads = 128;     // 16 groups x 8 sixteen-byte chunks of a 128-byte row
constexpr unsigned kFull = 0xffffffffu;

__host__ __device__ __forceinline__ int cdiv(int a, int b) { return (a + b - 1) / b; }

// 16 fp8 e4m3 values -> fp32 (exact)
__device__ __forceinline__ void e4m3x16_to_f32(uint4 v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const uint32_t lo = e4m3x2_to_f16x2(static_cast<uint16_t>(w[i] & 0xffffu));
    const uint32_t hi = e4m3x2_to_f16x2(static_cast<uint16_t>(w[i] >> 16));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&lo));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    f[4 * i] = a.x;
    f[4 * i + 1] = a.y;
    f[4 * i + 2] = b.x;
    f[4 * i + 3] = b.y;
  }
}

// 16 fp32 -> 16 bf16 (round to nearest even), 32 bytes at `dst` (16-byte aligned)
__device__ __forceinline__ void store_bf16x16(__nv_bfloat16* dst, const float* f) {
  uint4 a, b;
  a.x = pack_bf16x2(f[0], f[1]);
  a.y = pack_bf16x2(f[2], f[3]);
  a.z = pack_bf16x2(f[4], f[5]);
  a.w = pack_bf16x2(f[6], f[7]);
  b.x = pack_bf16x2(f[8], f[9]);
  b.y = pack_bf16x2(f[10], f[11]);
  b.z = pack_bf16x2(f[12], f[13]);
  b.w = pack_bf16x2(f[14], f[15]);
  st_v4(dst, a);
  st_v4(dst + 8, b);
}

// ---------------------------------------------------------------------------------------------
// prep_paged_kv
// ---------------------------------------------------------------------------------------------
struct PrepKvParams {
  const uint8_t* k;
  const uint8_t* v;
  const float* kscale;  // [1] (per tensor) or per token: [page, page / 32, hkv, 32] via ks_* strides
  const float* vscale;  // [1] or [hkv]
  const int* block_ids;
  const int* kv_seq_lens;
  __nv_bfloat16* kflat;
  float* vbias;
  float* v_norm_down;  // [b, hkv, max_down] scratch
  int num_head_kv, max_blocks, max_kb, max_down;
  int64_t k_blk, k_tok, k_head, v_blk, v_tok, v_head;  // cache strides, elements
  int64_t ks_blk, ks_chunk, ks_head;                   // per-token kscale strides, fp32 elements
  float lambda;
};

// grid (max_kb, B * Hkv), 128 threads. Thread t owns 16-byte chunk t % 8 of a row; for K it sums
// group t / 8, for V it takes rows t / 8 + 16 i. Rows at or past kv_len are never read.
template <int kPage, bool kPerTokenK>
__global__ void __launch_bounds__(kPrepThreads)
    prep_paged_kv_kernel(const PrepKvParams p) {
  __shared__ int s_page[kBlock / kPage];
  __shared__ float s_ks[kBlock];
  __shared__ float s_norm[kBlock];
  pdl_wait();
  const int sb = blockIdx.x;
  const int b = blockIdx.y / p.num_head_kv;
  const int h = blockIdx.y % p.num_head_kv;
  const int kv_len = __ldg(p.kv_seq_lens + b);
  if (sb >= cdiv(kv_len, kBlock)) return;
  const int t = threadIdx.x;
  const int row0 = sb * kBlock;
  const int valid = min(kv_len - row0, kBlock);  // rows of this block inside the request
  if (t < kBlock / kPage) {
    const int pg = row0 / kPage + t;
    s_page[t] = t * kPage < valid ? __ldg(p.block_ids + static_cast<int64_t>(b) * p.max_blocks + pg) : 0;
  }
  __syncthreads();
  if constexpr (kPerTokenK) {
    // row r of the block: kscale[page, (r % kPage) / 32, h, r % 32]
    const int r = t;
    float s = 0.f;
    if (r < valid) {
      const int rp = r % kPage;
      s = __ldg(p.kscale + s_page[r / kPage] * p.ks_blk + (rp >> 5) * p.ks_chunk + h * p.ks_head +
                (rp & 31));
    }
    s_ks[r] = s;
    __syncthreads();
  }
  const int c = t & 7;
  const int g = t >> 3;
  // ---- K: group g = rows g + 16 r ----
  {
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; j++) acc[j] = 0.f;
    uint4 raw[kSamples];
#pragma unroll
    for (int r = 0; r < kSamples; r++) {
      const int row = g + kStride * r;
      raw[r] = make_uint4(0, 0, 0, 0);
      if (row < valid) {
        const uint8_t* src = p.k + s_page[row / kPage] * p.k_blk + (row % kPage) * p.k_tok +
                             h * p.k_head + c * 16;
        raw[r] = ld_nc_v4(src);
      }
    }
#pragma unroll
    for (int r = 0; r < kSamples; r++) {
      const int row = g + kStride * r;
      if (row < valid) {
        float f[16];
        e4m3x16_to_f32(raw[r], f);
        if constexpr (kPerTokenK) {
          const float s = s_ks[row];
#pragma unroll
          for (int j = 0; j < 16; j++) acc[j] = __fmaf_rn(s, f[j], acc[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 16; j++) acc[j] += f[j];  // exact: 8 e4m3 terms fit in 24 bits
        }
      }
    }
    if constexpr (!kPerTokenK) {
      const float s = __ldg(p.kscale);
#pragma unroll
      for (int j = 0; j < 16; j++) acc[j] *= s;
    }
    __nv_bfloat16* dst = p.kflat +
                         ((static_cast<int64_t>(b) * p.num_head_kv + h) * p.max_kb + sb) * kFlat +
                         (kStride - 1 - g) * kDim + c * 16;
    store_bf16x16(dst, acc);
  }
  // ---- V: ||v * vscale|| of every row (0 past kv_len), then the max over 16 rows ----
  {
    const float vs = __ldg(p.vscale + (kPerTokenK ? h : 0));
#pragma unroll 2
    for (int i = 0; i < kBlock / 16; i++) {
      const int row = g + 16 * i;
      float ss = 0.f;
      if (row < valid) {
        const uint8_t* src = p.v + s_page[row / kPage] * p.v_blk + (row % kPage) * p.v_tok +
                             h * p.v_head + c * 16;
        float f[16];
        e4m3x16_to_f32(ld_nc_v4(src), f);
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const float x = f[j] * vs;
          ss = __fmaf_rn(x, x, ss);
        }
      }
      ss += __shfl_xor_sync(kFull, ss, 1);
      ss += __shfl_xor_sync(kFull, ss, 2);
      ss += __shfl_xor_sync(kFull, ss, 4);
      if (c == 0) s_norm[row] = sqrtf(ss);
    }
    __syncthreads();
    if (t < kSamples) {
      float m = 0.f;
#pragma unroll
      for (int j = 0; j < 16; j++) m = fmaxf(m, s_norm[16 * t + j]);
      p.v_norm_down[(static_cast<int64_t>(b) * p.num_head_kv + h) * p.max_down + sb * kSamples + t] = m;
    }
  }
  pdl_launch_dependents();
}

// grid B * Hkv, 256 threads: log(x + 1e-6) of the request's ceil(kv / 128) * 8 maxima, their mean
// and unbiased std, then vbias[kb] = mean over the block's 8 of lambda * relu((log - mean) / (std +
// 1e-6)).
constexpr int kVbiasThreads = 256;
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum_f32(v);
  __syncthreads();  // `red` free from any earlier use
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < kVbiasThreads / 32; w++) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kVbiasThreads) vbias_kernel(const PrepKvParams p) {
  __shared__ float red[kVbiasThreads / 32];
  pdl_wait();
  const int b = blockIdx.x / p.num_head_kv;
  const int h = blockIdx.x % p.num_head_kv;
  const int nkb = min(cdiv(__ldg(p.kv_seq_lens + b), kBlock), p.max_kb);
  const int n = nkb * kSamples;
  if (n == 0) return;
  const float* x = p.v_norm_down + (static_cast<int64_t>(b) * p.num_head_kv + h) * p.max_down;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kVbiasThreads) s += logf(x[i] + 1e-6f);
  const float mean = block_sum_256(s, red) / static_cast<float>(n);
  float q = 0.f;
  for (int i = threadIdx.x; i < n; i += kVbiasThreads) {
    const float d = logf(x[i] + 1e-6f) - mean;
    q = __fmaf_rn(d, d, q);
  }
  const float var = block_sum_256(q, red);
  const float sd = n > 1 ? sqrtf(var / static_cast<float>(n - 1)) : 0.f;
  const float inv = 1.f / (sd + 1e-6f);
  float* out = p.vbias + (static_cast<int64_t>(b) * p.num_head_kv + h) * p.max_kb;
  for (int kb = threadIdx.x; kb < nkb; kb += kVbiasThreads) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < kSamples; j++) {
      const float z = (logf(x[kb * kSamples + j] + 1e-6f) - mean) * inv;
      acc += p.lambda * fmaxf(z, 0.f);
    }
    out[kb] = acc / static_cast<float>(kSamples);
  }
}

// ---------------------------------------------------------------------------------------------
// prep_varlen_q
// ---------------------------------------------------------------------------------------------
struct PrepQParams {
  const uint8_t* q;
  const float* qscale;
  const int* q_seq_lens;
  const int* cu_seqlens_q;
  __nv_bfloat16* qflat;
  int num_head_q, max_qb;
  int64_t ld_q;                     // elements between tokens
  int64_t qs_b, qs_h, qs_t;         // qscale strides, elements
};

// grid (max_qb, B * Hq), 128 threads; thread t sums group t / 8 of chunk t % 8
__global__ void __launch_bounds__(kPrepThreads) prep_varlen_q_kernel(const PrepQParams p) {
  __shared__ float s_qs[kBlock];
  pdl_wait();
  const int qb = blockIdx.x;
  const int b = blockIdx.y / p.num_head_q;
  const int h = blockIdx.y % p.num_head_q;
  const int q_len = __ldg(p.q_seq_lens + b);
  if (qb >= cdiv(q_len, kBlock)) return;
  const int t = threadIdx.x;
  const int tok0 = qb * kBlock;
  const int valid = min(q_len - tok0, kBlock);
  s_qs[t] = t < valid ? __ldg(p.qscale + b * p.qs_b + h * p.qs_h + (tok0 + t) * p.qs_t) : 0.f;
  __syncthreads();
  const int c = t & 7;
  const int g = t >> 3;
  const int64_t base = static_cast<int64_t>(__ldg(p.cu_seqlens_q + b)) + tok0;
  uint4 raw[kSamples];
#pragma unroll
  for (int r = 0; r < kSamples; r++) {
    const int row = g + kStride * r;
    raw[r] = row < valid ? ld_nc_v4(p.q + (base + row) * p.ld_q + h * kDim + c * 16)
                         : make_uint4(0, 0, 0, 0);
  }
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; j++) acc[j] = 0.f;
#pragma unroll
  for (int r = 0; r < kSamples; r++) {
    const int row = g + kStride * r;
    if (row < valid) {
      float f[16];
      e4m3x16_to_f32(raw[r], f);
      const float s = s_qs[row];
#pragma unroll
      for (int j = 0; j < 16; j++) acc[j] = __fmaf_rn(s, f[j], acc[j]);
    }
  }
  store_bf16x16(p.qflat + ((static_cast<int64_t>(b) * p.num_head_q + h) * p.max_qb + qb) * kFlat +
                    g * kDim + c * 16,
                acc);
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------------------------
// oam_gemm
// ---------------------------------------------------------------------------------------------
// A CTA computes a 128 x 128 tile of logits: 128 key blocks, and `heads` query heads of one GQA
// group stacked along M with `rows` query blocks each (rows = 8 * (16 / heads), so every head's
// slice starts on a 1024-byte swizzle atom), so one kflat tile serves the whole group. K = 2048 is
// walked in 64-element (128-byte) chunks through a 4-stage TMA ring: one producer warp, two
// consumer warpgroups of 64 rows each.
constexpr int kGemmStages = 4;
constexpr int kChunk = 64;
constexpr int kChunks = kFlat / kChunk;  // 32
constexpr int kTileBytes = 128 * kChunk * 2;  // 16 KB: one operand, one chunk
constexpr int kGemmThreads = 288;        // 2 consumer warpgroups + 1 producer warp
constexpr int kGemmSmem = 2 * kGemmStages * kTileBytes + 2 * kGemmStages * 8;

struct GemmParams {
  const float* vbias;
  const int* q_seq_lens;
  const int* kv_seq_lens;
  __nv_bfloat16* logits;
  int num_head_q, num_head_kv, group;  // group = Hq / Hkv
  int heads, rows, head_chunks;        // heads stacked per tile, q blocks per head, chunks per group
  int max_qb, max_kb, n_qt, n_kt;
  int causal;
};

__global__ void __launch_bounds__(kGemmThreads, 1)
    oam_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q,
                    const __grid_constant__ CUtensorMap tmap_k, const GemmParams p) {
  using MMA = WgmmaBF16<128, 0, 0>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* q_smem = smem;
  uint8_t* k_smem = smem + kGemmStages * kTileBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * kGemmStages * kTileBytes);
  uint64_t* empty = full + kGemmStages;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int qt = blockIdx.x / p.n_kt;
  const int kt = blockIdx.x % p.n_kt;
  const int hc = blockIdx.y % p.head_chunks;
  const int bh = blockIdx.y / p.head_chunks;
  const int b = bh / p.num_head_kv;
  const int hkv = bh % p.num_head_kv;
  const int hq0 = hkv * p.group + hc * p.heads;
  const int nheads = min(p.heads, p.group - hc * p.heads);

  if (warp == 8 && lane == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_k);
    for (int i = 0; i < kGemmStages; i++) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    fence_barrier_init();
  }
  pdl_wait();
  __syncthreads();

  const int q_len = __ldg(p.q_seq_lens + b);
  const int kv_len = __ldg(p.kv_seq_lens + b);
  // (clamped to the output: lengths past it address no column, and vbias has max_kb entries)
  const int num_qb = min(cdiv(q_len, kBlock), p.max_qb);
  const int num_kb = min(cdiv(kv_len, kBlock), p.max_kb);
  const int off = (kv_len - q_len + kBlock - 1) / kBlock;  // causal block offset (C division)
  const int qb_lo = qt * p.rows;
  const int kb_lo = kt * 128;
  const bool dead = qb_lo >= num_qb || kb_lo >= num_kb ||
                    (p.causal && min(qb_lo + p.rows, num_qb) - 1 + off < kb_lo);
  const __nv_bfloat16 ninf = __float2bfloat16(-INFINITY);

  if (dead) {  // every element of the tile is -inf: no loads, no MMA
    if (warp == 8) return;
    const int n_cols = min(128, p.max_kb - kb_lo);
    const int n_rows = min(p.rows, p.max_qb - qb_lo);
    for (int e = tid; e < nheads * n_rows * 128; e += 256) {
      const int col = e & 127;
      const int rr = e >> 7;
      if (col >= n_cols) continue;
      const int hq = hq0 + rr / n_rows;
      const int qb = qb_lo + rr % n_rows;
      p.logits[((static_cast<int64_t>(b) * p.num_head_q + hq) * p.max_qb + qb) * p.max_kb + kb_lo +
               col] = ninf;
    }
    return;
  }

  if (warp == 8) {
    // ---- producer ----
    const uint32_t bytes = static_cast<uint32_t>(nheads * p.rows * kChunk * 2 + kTileBytes);
    for (int kc = 0; kc < kChunks; kc++) {
      const int st = kc % kGemmStages;
      const uint32_t ph = ((kc / kGemmStages) & 1) ^ 1;
      mbar_wait_nocall(&empty[st], ph);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full[st], bytes);
        for (int g = 0; g < nheads; g++) {
          tma_load_4d(q_smem + st * kTileBytes + g * p.rows * 128, &tmap_q, &full[st], kc * kChunk,
                      qb_lo, hq0 + g, b);
        }
        tma_load_4d(k_smem + st * kTileBytes, &tmap_k, &full[st], kc * kChunk, kb_lo, hkv, b);
      }
      __syncwarp();
    }
    return;
  }

  // ---- consumers: warpgroup wg computes rows 64 wg .. 64 wg + 63 ----
  const int wg = warp >> 2;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.f;
  // K-major 128B-swizzled tiles: 8-row groups 1024 B apart, one k16 step = 32 B of a row
  const uint64_t qdesc = make_smem_desc(smem_u32(q_smem) + wg * 8192, 16, 1024, kLayoutSW128);
  const uint64_t kdesc = make_smem_desc(smem_u32(k_smem), 16, 1024, kLayoutSW128);
  for (int kc = 0; kc < kChunks; kc++) {
    const int st = kc % kGemmStages;
    mbar_wait_nocall(&full[st], (kc / kGemmStages) & 1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      MMA::ss(acc, qdesc + static_cast<uint64_t>(st * (kTileBytes >> 4)) + kk * 2,
              kdesc + static_cast<uint64_t>(st * (kTileBytes >> 4)) + kk * 2, (kc | kk) > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_anchor<64>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
  }

  // ---- epilogue: scale, bias, mask, bf16 ----
  const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c_base = 2 * (lane & 3);
  const float* vb = p.vbias + (static_cast<int64_t>(b) * p.num_head_kv + hkv) * p.max_kb;
  const bool pair_ok = (p.max_kb & 1) == 0;
#pragma unroll
  for (int hr = 0; hr < 2; hr++) {
    const int r = r_base + 8 * hr;
    const int g = r / p.rows;
    const int qb = qb_lo + r % p.rows;
    if (g >= nheads || qb >= p.max_qb) continue;
    __nv_bfloat16* dst =
        p.logits + ((static_cast<int64_t>(b) * p.num_head_q + hq0 + g) * p.max_qb + qb) * p.max_kb;
    const bool row_ok = qb < num_qb;
#pragma unroll
    for (int j = 0; j < 16; j++) {
      float v2[2];
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int kb = kb_lo + 8 * j + c_base + e;
        const bool ok = row_ok && kb < num_kb && !(p.causal && qb + off < kb);
        v2[e] = ok ? __fmaf_rn(acc[4 * j + 2 * hr + e], 1.f / 64.f, __ldg(vb + kb)) : -INFINITY;
      }
      const int kb0 = kb_lo + 8 * j + c_base;
      if (pair_ok && kb0 + 1 < p.max_kb) {
        *reinterpret_cast<uint32_t*>(dst + kb0) = pack_bf16x2(v2[0], v2[1]);
      } else {
        if (kb0 < p.max_kb) dst[kb0] = __float2bfloat16_rn(v2[0]);
        if (kb0 + 1 < p.max_kb) dst[kb0 + 1] = __float2bfloat16_rn(v2[1]);
      }
    }
  }
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------------------------
// tpd
// ---------------------------------------------------------------------------------------------
struct TpdParams {
  const __nv_bfloat16* logits;
  uint8_t* mask;
  const int* q_seq_lens;
  const int* kv_seq_lens;
  const int* num_prompt_tokens;
  int num_heads, max_qb, max_kb;
  float alpha;
  int initial_blocks, window_size;
  float rate_m;
  int bias_m;
  float rate_l;
  int bias_l;
};

constexpr int kTpdThreads = 256;
constexpr int kTpdWarpKb = 1024;  // rows up to this many blocks: one warp per row, 8 rows per CTA
constexpr uint16_t kNonFinite = 0x007F;  // below every finite key

// bf16 bits -> 16-bit key whose unsigned order is the float order; non-finite -> kNonFinite
__device__ __forceinline__ uint16_t ordered_key(uint16_t bits) {
  if ((bits & 0x7F80u) == 0x7F80u) return kNonFinite;
  return (bits & 0x8000u) ? static_cast<uint16_t>(~bits) : static_cast<uint16_t>(bits ^ 0x8000u);
}

// Budget of query block `q_pos` (absolute: q row + causal offset): the 3-regime schedule on the
// prompt's block count, then the linear decay toward k * alpha. Every step is one IEEE-rounded
// fp32 operation (the decay a single fma) so the result is reproducible bit for bit.
__device__ __forceinline__ int tpd_budget(const TpdParams& p, int q_pos, int prompt_blocks) {
  int k;
  if (prompt_blocks < 56) {
    k = prompt_blocks;
  } else if (prompt_blocks < 160) {
    k = static_cast<int>(__fmul_rn(static_cast<float>(prompt_blocks), p.rate_m)) + p.bias_m;
  } else {
    k = static_cast<int>(__fmul_rn(static_cast<float>(prompt_blocks), p.rate_l)) + p.bias_l;
  }
  const int decay_len = prompt_blocks - k;
  if (q_pos < k || decay_len <= 1) return k;
  const float kf = static_cast<float>(k);
  const float k_end = __fmul_rn(kf, p.alpha);
  const float t = __fdiv_rn(static_cast<float>(q_pos - k), static_cast<float>(decay_len - 1));
  const int budget = static_cast<int>(floorf(__fmaf_rn(t, __fsub_rn(k_end, kf), kf)));
  return budget < 1 ? 1 : (budget > k ? k : budget);
}

template <int kN>
__device__ __forceinline__ void group_sync() {
  if constexpr (kN == 32) {
    __syncwarp();
  } else {
    __syncthreads();
  }
}

// Within one 256-bin histogram (bins ordered by value), find the largest bin `bin` with
// count(>= bin) >= need; returns it and count(> bin) through `above`. Run by one whole warp.
__device__ __forceinline__ int hist_select(const int* hist, int need, int* above) {
  const int lane = threadIdx.x & 31;
  int cnt[8];
  int s = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {  // lane 0 owns the 8 highest bins
    cnt[j] = hist[255 - 8 * lane - j];
    s += cnt[j];
  }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += y;
  }
  const int excl = incl - s;
  const unsigned who = __ballot_sync(kFull, excl < need && need <= incl);
  const int src = __ffs(who) - 1;
  int bin = 0, a = 0;
  if (lane == src) {
    int cum = excl;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      if (cum + cnt[j] >= need) {
        bin = 255 - 8 * lane - j;
        a = cum;
        break;
      }
      cum += cnt[j];
    }
  }
  *above = __shfl_sync(kFull, a, src);
  return __shfl_sync(kFull, bin, src);
}

// One mask row by kN threads (a warp, or the whole CTA): keys to shared memory, total finite count
// and the high-byte histogram, the byte holding the threshold, the low-byte histogram of the keys
// sharing it; T is the largest key with count(key >= T) >= budget.
template <int kN>
__device__ __forceinline__ void tpd_row(const TpdParams& p, int b, int h, int qr, uint16_t* keys,
                                        int* hist, int* s_sel, int tid) {
  const int q_len = __ldg(p.q_seq_lens + b);
  const int kv_len = __ldg(p.kv_seq_lens + b);
  const int qi = cdiv(q_len, kBlock);
  const int ki = min(cdiv(kv_len, kBlock), p.max_kb);  // keys[] holds max_kb entries
  const int64_t row = ((static_cast<int64_t>(b) * p.num_heads + h) * p.max_qb + qr) * p.max_kb;
  uint8_t* out = p.mask + row;
  if (qi == 0 || ki == 0 || qr >= qi) {
    for (int c = tid; c < p.max_kb; c += kN) out[c] = 0;
    return;
  }
  const int prompt_blocks = cdiv(__ldg(p.num_prompt_tokens + b), kBlock);
  const int off = (kv_len - q_len + kBlock - 1) / kBlock;
  const int budget = tpd_budget(p, qr + off, prompt_blocks);
  const uint16_t* src = reinterpret_cast<const uint16_t*>(p.logits + row);

  for (int i = tid; i < 256; i += kN) hist[i] = 0;
  group_sync<kN>();
  for (int c = tid; c < ki; c += kN) {
    const uint16_t key = ordered_key(__ldg(src + c));
    keys[c] = key;
    if (key != kNonFinite) atomicAdd(&hist[key >> 8], 1);
  }
  group_sync<kN>();
  const int lane = tid & 31;
  // s_sel: [0] threshold, [1] high byte still to resolve (-1: threshold final), [2] count above
  if (tid < 32) {
    int total = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) total += hist[8 * lane + j];
    total = __reduce_add_sync(kFull, total);
    if (budget <= 0) {
      if (lane == 0) s_sel[0] = 0xFFFF, s_sel[1] = -1;  // no finite key reaches 0xFFFF
    } else if (budget >= total) {
      if (lane == 0) s_sel[0] = kNonFinite + 1, s_sel[1] = -1;  // every finite key
    } else {
      int above;
      const int hi = hist_select(hist, budget, &above);
      if (lane == 0) s_sel[1] = hi, s_sel[2] = above;
    }
  }
  group_sync<kN>();
  const int hi = s_sel[1];
  if (hi >= 0) {
    for (int i = tid; i < 256; i += kN) hist[i] = 0;
    group_sync<kN>();
    for (int c = tid; c < ki; c += kN) {
      const uint16_t key = keys[c];
      if (key != kNonFinite && (key >> 8) == hi) atomicAdd(&hist[key & 255], 1);
    }
    group_sync<kN>();
    if (tid < 32) {
      int dummy;
      const int lo = hist_select(hist, budget - s_sel[2], &dummy);
      __syncwarp();
      if (lane == 0) s_sel[0] = (hi << 8) | lo;
    }
    group_sync<kN>();
  }
  const int thr = s_sel[0];
  const int diag = min(qr + off, ki - 1);
  for (int c = tid; c < p.max_kb; c += kN) {
    bool sel = false;
    if (c < ki) {
      sel = keys[c] >= thr || c < p.initial_blocks || (c <= diag && c > diag - p.window_size) ||
            c == diag;
    }
    out[c] = sel ? 1 : 0;
  }
}

// narrow rows: grid (ceil(max_qb / 8), Hq, B), warp w of a CTA takes q row 8 x + w
__global__ void __launch_bounds__(kTpdThreads) tpd_warp_kernel(const TpdParams p) {
  __shared__ uint16_t keys[kTpdThreads / 32][kTpdWarpKb];
  __shared__ int hist[kTpdThreads / 32][256];
  __shared__ int sel[kTpdThreads / 32][4];
  pdl_wait();
  const int w = threadIdx.x >> 5;
  const int qr = blockIdx.x * (kTpdThreads / 32) + w;
  if (qr < p.max_qb) tpd_row<32>(p, blockIdx.z, blockIdx.y, qr, keys[w], hist[w], sel[w], threadIdx.x & 31);
  pdl_launch_dependents();
}

// wide rows (up to 32768 blocks): grid (max_qb, Hq, B), the CTA takes one row; keys in dynamic smem
__global__ void __launch_bounds__(kTpdThreads) tpd_cta_kernel(const TpdParams p) {
  extern __shared__ __align__(16) uint8_t dyn[];
  __shared__ int hist[256];
  __shared__ int sel[4];
  pdl_wait();
  tpd_row<kTpdThreads>(p, blockIdx.z, blockIdx.y, blockIdx.x, reinterpret_cast<uint16_t*>(dyn), hist,
                       sel, threadIdx.x);
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
int prep_kv_launch(const char* who, bool per_token, void* kflat, void* vbias, const void* kcache,
                   const void* vcache, const void* kscale, const void* vscale, const void* block_ids,
                   const void* kv_seq_lens, int num_batch, int num_dim_qk, int num_dim_v,
                   int num_head_kv, int block_size, int scale_block_size, int max_blocks,
                   int stem_block_size, int stem_stride, float lambda, int max_kb, int max_down,
                   int64_t ldK, int64_t ldV, int64_t ldKS, int64_t ldKS1, int64_t ldKS2,
                   int64_t ldK1, int64_t ldK2, int64_t ldV1, int64_t ldV2, void* v_norm_down,
                   cudaStream_t stream) {
  HPC_REQUIRE(stem_block_size == kBlock && stem_stride == kStride,
              "%s: only stem_block_size=128, stem_stride=16 is supported (got %d, %d)", who,
              stem_block_size, stem_stride);
  HPC_REQUIRE(num_dim_qk == kDim && num_dim_v == kDim,
              "%s: unsupported dim_qk=%d dim_v=%d (expected 128, 128)", who, num_dim_qk, num_dim_v);
  HPC_REQUIRE(block_size == 32 || block_size == 64, "%s: kv_block_size must be 32 or 64, got %d",
              who, block_size);
  HPC_REQUIRE(!per_token || scale_block_size == block_size / 32,
              "%s: per-token kscale must hold %d rows of 32 scales per page (got %d)", who,
              block_size / 32, scale_block_size);
  HPC_REQUIRE(num_batch >= 0 && num_head_kv > 0 && max_kb >= 0 && max_down == max_kb * kSamples,
              "%s: bad num_batch / num_head_kv / max_num_stem_blocks / max_k_down_len (%d, %d, %d, "
              "%d)", who, num_batch, num_head_kv, max_kb, max_down);
  const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  HPC_REQUIRE(al16(kcache) && al16(vcache) && al16(kflat),
              "%s: kcache, vcache and kflat must be 16-byte aligned", who);
  HPC_REQUIRE(ldK % 16 == 0 && ldK1 % 16 == 0 && ldK2 % 16 == 0 && ldV % 16 == 0 &&
                  ldV1 % 16 == 0 && ldV2 % 16 == 0,
              "%s: cache block, token and head strides must be multiples of 16 bytes", who);
  if (num_batch == 0 || max_kb == 0) return HPC_OK;
  PrepKvParams p = {};
  p.k = static_cast<const uint8_t*>(kcache);
  p.v = static_cast<const uint8_t*>(vcache);
  p.kscale = static_cast<const float*>(kscale);
  p.vscale = static_cast<const float*>(vscale);
  p.block_ids = static_cast<const int*>(block_ids);
  p.kv_seq_lens = static_cast<const int*>(kv_seq_lens);
  p.kflat = static_cast<__nv_bfloat16*>(kflat);
  p.vbias = static_cast<float*>(vbias);
  p.v_norm_down = static_cast<float*>(v_norm_down);
  p.num_head_kv = num_head_kv;
  p.max_blocks = max_blocks;
  p.max_kb = max_kb;
  p.max_down = max_down;
  p.k_blk = ldK, p.k_tok = ldK1, p.k_head = ldK2;
  p.v_blk = ldV, p.v_tok = ldV1, p.v_head = ldV2;
  p.ks_blk = ldKS, p.ks_chunk = ldKS1, p.ks_head = ldKS2;
  p.lambda = lambda;
  const dim3 grid(max_kb, num_batch * num_head_kv);
  void (*kern)(PrepKvParams);
  if (per_token) {
    kern = block_size == 32 ? prep_paged_kv_kernel<32, true> : prep_paged_kv_kernel<64, true>;
  } else {
    kern = block_size == 32 ? prep_paged_kv_kernel<32, false> : prep_paged_kv_kernel<64, false>;
  }
  HPC_CUDA_CHECK(launch_pdl(kern, grid, dim3(kPrepThreads), 0, stream, 1, p));
  HPC_CUDA_CHECK(launch_pdl(vbias_kernel, dim3(num_batch * num_head_kv), dim3(kVbiasThreads), 0,
                            stream, 1, p));
  return HPC_OK;
}

}  // namespace stem
}  // namespace b200

using namespace b200;         // NOLINT
using namespace b200::stem;   // NOLINT

// replaces reference src/stem/stem_oam_prep_paged_kv_dim128.h (kv per tensor); the cache's token
// and head strides (elements) follow ldK / ldV, so NHD and HND caches both work
extern "C" int hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(
    void* kflat_ptr, void* vbias_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const void* kscale_ptr, const void* vscale_ptr, const void* block_ids_ptr,
    const void* kv_seq_lens_ptr, int num_batch, int num_dim_qk, int num_dim_v, int num_head_kv,
    int num_kvcache_blocks, int block_size, int num_seq_max_blocks, int stem_block_size,
    int stem_stride, float lambda_mag, int max_num_stem_blocks, int max_k_down_len, int64_t ldK,
    int64_t ldV, int64_t ldK1, int64_t ldK2, int64_t ldV1, int64_t ldV2, void* v_norm_down_ptr,
    cudaStream_t stream) {
  (void)num_kvcache_blocks;
  return prep_kv_launch("stem_oam_prep_paged_kv", false, kflat_ptr, vbias_ptr, kcache_ptr,
                        vcache_ptr, kscale_ptr, vscale_ptr, block_ids_ptr, kv_seq_lens_ptr,
                        num_batch, num_dim_qk, num_dim_v, num_head_kv, block_size, 0,
                        num_seq_max_blocks, stem_block_size, stem_stride, lambda_mag,
                        max_num_stem_blocks, max_k_down_len, ldK, ldV, 0, 0, 0, ldK1, ldK2, ldV1,
                        ldV2, v_norm_down_ptr, stream);
}

// replaces reference src/stem/stem_oam_prep_paged_kv_dim128.h (k per token, v per head)
extern "C" int hpc_stem_oam_prep_paged_kv_qkpertoken_perhead_vperhead_dim128_async(
    void* kflat_ptr, void* vbias_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const void* kscale_ptr, const void* vscale_ptr, const void* block_ids_ptr,
    const void* kv_seq_lens_ptr, int num_batch, int num_dim_qk, int num_dim_v, int num_head_kv,
    int num_kvcache_blocks, int block_size, int scale_block_size, int num_seq_max_blocks,
    int stem_block_size, int stem_stride, float lambda_mag, int max_num_stem_blocks,
    int max_k_down_len, int64_t ldK, int64_t ldV, int64_t ldKS, int64_t ldKS1, int64_t ldKS2,
    int64_t ldK1, int64_t ldK2, int64_t ldV1, int64_t ldV2, void* v_norm_down_ptr,
    cudaStream_t stream) {
  (void)num_kvcache_blocks;
  return prep_kv_launch("stem_oam_prep_paged_kv", true, kflat_ptr, vbias_ptr, kcache_ptr,
                        vcache_ptr, kscale_ptr, vscale_ptr, block_ids_ptr, kv_seq_lens_ptr,
                        num_batch, num_dim_qk, num_dim_v, num_head_kv, block_size,
                        scale_block_size, num_seq_max_blocks, stem_block_size, stem_stride,
                        lambda_mag, max_num_stem_blocks, max_k_down_len, ldK, ldV, ldKS, ldKS1,
                        ldKS2, ldK1, ldK2, ldV1, ldV2, v_norm_down_ptr, stream);
}

// replaces reference src/stem/stem_oam_prep_varlen_q_dim128.h; qscale is read through its strides
// (elements), so a qscale padded past max_num_q_blocks * 128 tokens is read correctly
extern "C" int hpc_stem_oam_prep_varlen_q_dim128_async(
    void* qflat_ptr, const void* q_fp8_ptr, const void* qscale_ptr, const void* q_seq_lens_ptr,
    const void* cu_seqlens_q_ptr, int num_batch, int num_head_q, int ldQ, int stem_block_size,
    int stem_stride, int max_num_q_blocks, int64_t ldQS, int64_t ldQS1, int64_t ldQS2,
    cudaStream_t stream) {
  HPC_REQUIRE(stem_block_size == kBlock && stem_stride == kStride,
              "stem_oam_prep_varlen_q: only stem_block_size=128, stem_stride=16 is supported (got "
              "%d, %d)", stem_block_size, stem_stride);
  HPC_REQUIRE(num_batch >= 0 && num_head_q > 0 && max_num_q_blocks >= 0,
              "stem_oam_prep_varlen_q: bad num_batch / num_head_q / max_num_q_blocks (%d, %d, %d)",
              num_batch, num_head_q, max_num_q_blocks);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(q_fp8_ptr) & 15) == 0 && ldQ % 16 == 0 &&
                  (reinterpret_cast<uintptr_t>(qflat_ptr) & 15) == 0,
              "stem_oam_prep_varlen_q: q_fp8 and qflat must be 16-byte aligned and the q token "
              "stride a multiple of 16 bytes");
  if (num_batch == 0 || max_num_q_blocks == 0) return HPC_OK;
  PrepQParams p = {};
  p.q = static_cast<const uint8_t*>(q_fp8_ptr);
  p.qscale = static_cast<const float*>(qscale_ptr);
  p.q_seq_lens = static_cast<const int*>(q_seq_lens_ptr);
  p.cu_seqlens_q = static_cast<const int*>(cu_seqlens_q_ptr);
  p.qflat = static_cast<__nv_bfloat16*>(qflat_ptr);
  p.num_head_q = num_head_q;
  p.max_qb = max_num_q_blocks;
  p.ld_q = ldQ;
  p.qs_b = ldQS, p.qs_h = ldQS1, p.qs_t = ldQS2;
  HPC_CUDA_CHECK(launch_pdl(prep_varlen_q_kernel, dim3(max_num_q_blocks, num_batch * num_head_q),
                            dim3(kPrepThreads), 0, stream, 1, p));
  return HPC_OK;
}

// replaces reference src/stem/stem_oam_gemm_dim128.h; writes every element of block_logits
// [num_batch, num_head_q, max_num_qb, max_num_kb] (contiguous), so it needs no prior fill
extern "C" int hpc_stem_oam_gemm_dim128_async(
    void* block_logits_ptr, const void* qflat_ptr, const void* kflat_ptr, const void* vbias_ptr,
    const void* q_seq_lens_ptr, const void* kv_seq_lens_ptr, int num_batch, int num_head_q,
    int num_head_kv, int max_num_qb, int max_num_kb, int stem_block_size, int stem_stride,
    int causal, cudaStream_t stream) {
  HPC_REQUIRE(stem_block_size == kBlock && stem_stride == kStride,
              "stem_oam_gemm: only stem_block_size=128, stem_stride=16 is supported (got %d, %d)",
              stem_block_size, stem_stride);
  HPC_REQUIRE(num_head_q > 0 && num_head_kv > 0 && num_head_q % num_head_kv == 0,
              "stem_oam_gemm: num_head_q (%d) must be a multiple of num_head_kv (%d)", num_head_q,
              num_head_kv);
  HPC_REQUIRE(num_batch >= 0 && max_num_qb >= 0 && max_num_kb >= 0,
              "stem_oam_gemm: bad num_batch / max_num_qb / max_num_kb (%d, %d, %d)", num_batch,
              max_num_qb, max_num_kb);
  const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  HPC_REQUIRE(al16(qflat_ptr) && al16(kflat_ptr) && al16(block_logits_ptr),
              "stem_oam_gemm: qflat, kflat and block_logits must be 16-byte aligned");
  if (num_batch == 0 || max_num_qb == 0 || max_num_kb == 0) return HPC_OK;

  GemmParams p = {};
  p.vbias = static_cast<const float*>(vbias_ptr);
  p.q_seq_lens = static_cast<const int*>(q_seq_lens_ptr);
  p.kv_seq_lens = static_cast<const int*>(kv_seq_lens_ptr);
  p.logits = static_cast<__nv_bfloat16*>(block_logits_ptr);
  p.num_head_q = num_head_q;
  p.num_head_kv = num_head_kv;
  p.group = num_head_q / num_head_kv;
  p.heads = p.group < 16 ? p.group : 16;
  p.rows = 8 * (16 / p.heads);
  p.head_chunks = cdiv(p.group, p.heads);
  p.max_qb = max_num_qb;
  p.max_kb = max_num_kb;
  p.n_qt = cdiv(max_num_qb, p.rows);
  p.n_kt = cdiv(max_num_kb, 128);
  p.causal = causal ? 1 : 0;

  const CUtensorMapDataType bf16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap tq, tk;
  {
    uint64_t dims[4] = {kFlat, static_cast<uint64_t>(max_num_qb), static_cast<uint64_t>(num_head_q),
                        static_cast<uint64_t>(num_batch)};
    uint64_t strides[3] = {kFlat * 2ull, kFlat * 2ull * max_num_qb,
                           kFlat * 2ull * max_num_qb * num_head_q};
    uint32_t box[4] = {kChunk, static_cast<uint32_t>(p.rows), 1, 1};
    if (int rc = encode_tmap(&tq, bf16, 2, qflat_ptr, 4, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)) {
      return rc;
    }
  }
  {
    uint64_t dims[4] = {kFlat, static_cast<uint64_t>(max_num_kb), static_cast<uint64_t>(num_head_kv),
                        static_cast<uint64_t>(num_batch)};
    uint64_t strides[3] = {kFlat * 2ull, kFlat * 2ull * max_num_kb,
                           kFlat * 2ull * max_num_kb * num_head_kv};
    uint32_t box[4] = {kChunk, 128, 1, 1};
    if (int rc = encode_tmap(&tk, bf16, 2, kflat_ptr, 4, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)) {
      return rc;
    }
  }
  HPC_REQUIRE(static_cast<int64_t>(num_batch) * num_head_kv * p.head_chunks <= 65535,
              "stem_oam_gemm: num_batch * num_head_kv too large (%d x %d)", num_batch, num_head_kv);
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(oam_gemm_kernel), kGemmSmem));
  const dim3 grid(p.n_qt * p.n_kt, num_batch * num_head_kv * p.head_chunks);
  HPC_CUDA_CHECK(launch_pdl(oam_gemm_kernel, grid, dim3(kGemmThreads), kGemmSmem, stream, 1, tq, tk, p));
  return HPC_OK;
}

// replaces reference src/stem/stem_tpd.h; writes every byte of mask [num_batch, num_heads, max_Qb,
// max_Kb], so it needs no prior fill
extern "C" int hpc_stem_tpd_async(
    void* mask_ptr, const void* block_logits_ptr, const void* q_seq_lens_ptr,
    const void* kv_seq_lens_ptr, const void* num_prompt_tokens_ptr, int num_batch, int num_heads,
    int max_Qb, int max_Kb, int block_size, float alpha, int initial_blocks, int window_size,
    float k_block_num_rate_medium, int k_block_num_bias_medium, float k_block_num_rate_large,
    int k_block_num_bias_large, cudaStream_t stream) {
  HPC_REQUIRE(block_size == kBlock, "stem_tpd: block_size must be 128 (got %d)", block_size);
  HPC_REQUIRE(max_Kb <= 32768, "stem_tpd: max_Kb=%d exceeds 32768 limit", max_Kb);
  HPC_REQUIRE(num_batch >= 0 && num_heads > 0 && max_Qb >= 0 && max_Kb >= 0,
              "stem_tpd: bad num_batch / num_heads / max_Qb / max_Kb (%d, %d, %d, %d)", num_batch,
              num_heads, max_Qb, max_Kb);
  HPC_REQUIRE(num_batch <= 65535 && num_heads <= 65535, "stem_tpd: too many requests or heads");
  if (num_batch == 0 || max_Qb == 0 || max_Kb == 0) return HPC_OK;
  TpdParams p = {};
  p.logits = static_cast<const __nv_bfloat16*>(block_logits_ptr);
  p.mask = static_cast<uint8_t*>(mask_ptr);
  p.q_seq_lens = static_cast<const int*>(q_seq_lens_ptr);
  p.kv_seq_lens = static_cast<const int*>(kv_seq_lens_ptr);
  p.num_prompt_tokens = static_cast<const int*>(num_prompt_tokens_ptr);
  p.num_heads = num_heads;
  p.max_qb = max_Qb;
  p.max_kb = max_Kb;
  p.alpha = alpha;
  p.initial_blocks = initial_blocks;
  p.window_size = window_size;
  p.rate_m = k_block_num_rate_medium;
  p.bias_m = k_block_num_bias_medium;
  p.rate_l = k_block_num_rate_large;
  p.bias_l = k_block_num_bias_large;
  if (max_Kb <= kTpdWarpKb) {
    const dim3 grid(cdiv(max_Qb, kTpdThreads / 32), num_heads, num_batch);
    HPC_CUDA_CHECK(launch_pdl(tpd_warp_kernel, grid, dim3(kTpdThreads), 0, stream, 1, p));
  } else {
    const int smem = max_Kb * 2;
    HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(tpd_cta_kernel), smem));
    const dim3 grid(max_Qb, num_heads, num_batch);
    HPC_CUDA_CHECK(launch_pdl(tpd_cta_kernel, grid, dim3(kTpdThreads), smem, stream, 1, p));
  }
  return HPC_OK;
}
