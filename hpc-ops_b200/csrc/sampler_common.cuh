// Pieces shared by the token samplers (sampler.cu, spec_sampler.cu): Philox4x32-10 and the
// uniform / Gumbel mapping of the internal noise, the per-stream launch offset, the
// (value desc, id asc) order, the 8-token row loaders, online softmax statistics, the row split
// and the logits checks of the launchers.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include "common.cuh"
#include "host_utils.h"

namespace b200 {

constexpr int kSamplerMaxSlices = 8;

// ---- Philox4x32-10 (Salmon et al., SC'11) --------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ uint4 philox_at(uint64_t seed, uint32_t c0, uint32_t c1, uint64_t offset) {
  return philox4x32_10(
      make_uint4(c0, c1, static_cast<uint32_t>(offset), static_cast<uint32_t>(offset >> 32)),
      make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
}

// 23 random bits -> u in [2^-24, 1 - 2^-24], every value exact in fp32
__device__ __forceinline__ float uniform_of(uint32_t x) {
  return __fmaf_rn(static_cast<float>(x >> 9), 1.1920928955078125e-7f, 5.9604644775390625e-8f);
}

// g = -log(-log u) is finite
__device__ __forceinline__ float gumbel_of(uint32_t x) { return -logf(-logf(uniform_of(x))); }

// Gumbel noise of tokens 4q .. 4q+3 of `row`
__device__ __forceinline__ float4 philox_gumbel4(uint64_t seed, uint32_t q, int row, uint64_t offset) {
  const uint4 r = philox_at(seed, q, static_cast<uint32_t>(row), offset);
  return make_float4(gumbel_of(r.x), gumbel_of(r.y), gumbel_of(r.z), gumbel_of(r.w));
}

// The last CTA of the launch to get here advances the launch counter: every CTA has read the
// offset before it arrives. rng_word[0] is the launch counter, the low half of rng_word[1] the
// finished-CTA counter.
__device__ __forceinline__ void advance_rng(unsigned long long* rng_word) {
  if (rng_word == nullptr || threadIdx.x != 0) return;
  __threadfence();
  unsigned int* done = reinterpret_cast<unsigned int*>(rng_word + 1);
  const unsigned int total = gridDim.x * gridDim.y;
  if (atomicAdd(done, 1u) == total - 1) {
    rng_word[0] += 1;
    *done = 0;
    __threadfence();
  }
}

__device__ __forceinline__ uint64_t launch_offset(unsigned long long* rng_word, uint64_t rng_base) {
  return rng_word != nullptr ? rng_base + *reinterpret_cast<volatile unsigned long long*>(rng_word) : 0;
}

// (value descending, token id ascending); NaN is never better
__device__ __forceinline__ bool better(float a, int ia, float b, int ib) {
  return a > b || (a == b && ia < ib);
}

// tokens 8c .. 8c+7 of a row as fp32 (16-byte loads: two for fp32, one for bf16)
template <typename T>
__device__ __forceinline__ void load8(const T* row, int c, float (&x)[8]);
template <>
__device__ __forceinline__ void load8<float>(const float* row, int c, float (&x)[8]) {
  const float4 a = ld_nc_f4(row + 8 * c), b = ld_nc_f4(row + 8 * c + 4);
  x[0] = a.x, x[1] = a.y, x[2] = a.z, x[3] = a.w, x[4] = b.x, x[5] = b.y, x[6] = b.z, x[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* row, int c, float (&x)[8]) {
  const uint4 v = ld_nc_v4(row + 8 * c);
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    x[2 * i] = __uint_as_float(w[i] << 16);
    x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

// online softmax statistics: running max m and sum s of exp(x - m)
__device__ __forceinline__ void online_add(float x, float& m, float& s) {
  if (x == -INFINITY) return;
  if (x > m) {
    s = s * expf(m - x) + 1.f;
    m = x;
  } else {
    s += expf(x - m);
  }
}

__device__ __forceinline__ void online_merge(float m2, float s2, float& m, float& s) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) {
    m = m2, s = s2;
  } else if (m2 > m) {
    s = s * expf(m - m2) + s2;
    m = m2;
  } else {
    s += s2 * expf(m2 - m);
  }
}

// Smallest power-of-two slice count with slices * rows >= SMs, capped at the portable cluster
// size 8 (so fewer than 17 rows leave SMs idle), and no slice under 16 chunks.
inline int pick_slices(int rows, int vocab) {
  const int sms = sm_count() > 0 ? sm_count() : 132;
  int s = 1;
  while (s < kSamplerMaxSlices && s * rows < sms && vocab / 8 / (2 * s) >= 16) s *= 2;
  return s;
}

struct RngState {
  unsigned long long* word;
  uint64_t base;
};

// Launch-offset word of `stream` (of its own for a captured launch); the base makes offsets of
// different words disjoint, so two graphs or streams sampling with one seed draw different noise.
inline int rng_state(cudaStream_t stream, RngState* st) {
  uint64_t serial = 0;
  int* w = stream_state(stream, &serial);
  if (w == nullptr) return HPC_ERR_CUDA;
  st->word = reinterpret_cast<unsigned long long*>(w);
  st->base = serial << 40;
  return HPC_OK;
}

inline int check_common(const void* logits, int64_t row_stride, int dtype, int batch, int vocab,
                        int max_topk, const char* who) {
  HPC_REQUIRE(dtype == 0 || dtype == 1, "%s: logits dtype must be float32 or bfloat16", who);
  HPC_REQUIRE(batch >= 0 && batch <= 65535, "%s: batch %d out of range [0, 65535]", who, batch);
  HPC_REQUIRE(vocab % 8 == 0 && vocab >= max_topk && vocab <= 262144,
              "%s: vocab size %d must be a multiple of 8 in [%d, 262144]", who, vocab, max_topk);
  const int elem = dtype == 0 ? 4 : 2;
  HPC_REQUIRE(row_stride >= vocab && (row_stride * elem) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(logits) % 16 == 0,
              "%s: logits rows must be 16-byte aligned (row stride %lld elements)", who,
              static_cast<long long>(row_stride));
  return HPC_OK;
}

}  // namespace b200
