// Definitions shared by the block-sparse prefill kernels (prefill_blocksparse_fp8*.cu): work-item
// decoding, launch parameters, tile constants, the FMA-pipe exp2.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace b200 {
namespace prefill {

constexpr int kTile = 128;
constexpr int kPage = 64;
constexpr int kD = 128;
constexpr int kTileBytes = kTile * kD;  // 16 KB fp8
constexpr int kStages = 2;
constexpr int kMaxKvTiles = 1024;  // seq_kv <= 128 K

struct Params {
  const int* cu_seqlens_q;
  const int* seqlens_kv;
  const int* block_ids;
  const uint8_t* block_mask;  // [B, Hq, mask_mq, mask_kb] or NULL
  const float* qscale;        // [B, Hq, qscale_ld]
  const float* kscale;        // [1] or per-token [blocks, 2, Hkv, 32]
  const float* vscale;        // [1] or [Hkv]
  __nv_bfloat16* out;
  int* work_counter;
  long long ks_stride_blk, ks_stride_grp, ks_stride_head;  // per-token k-scale strides (floats)
  int num_batch, num_head_q, num_head_kv, group;
  int max_q_tiles;
  int mask_mq, mask_kb;
  int max_blocks;
  int qscale_ld;  // padded q length of qscale
  int ld_out;     // elements between tokens of out
  int k_head_first, v_head_first;
  float softmax_scale_log2;
};

struct Work {
  int b, hq, mq;
  int q0;        // first token row (global) of the tile
  int rows;      // valid rows
  int seq_q, seq_kv;
  int num_tile_kv;  // causal extent of this Q tile in KV tiles
};

// kKvOffsets: p.seqlens_kv holds B + 1 key offsets (cu_seqlens_kv), not B lengths.
template <bool kKvOffsets = false>
__device__ __forceinline__ bool decode_work(const Params& p, int w, Work& k) {
  const int per_level = p.num_batch * p.num_head_q;
  if (w >= p.max_q_tiles * per_level) return false;
  const int level = w / per_level;
  const int rem = w - level * per_level;
  k.mq = p.max_q_tiles - 1 - level;  // heaviest first
  k.b = rem / p.num_head_q;
  k.hq = rem - k.b * p.num_head_q;
  const int s0 = p.cu_seqlens_q[k.b];
  k.seq_q = p.cu_seqlens_q[k.b + 1] - s0;
  k.seq_kv = kKvOffsets ? p.seqlens_kv[k.b + 1] - p.seqlens_kv[k.b] : p.seqlens_kv[k.b];
  k.q0 = s0 + k.mq * kTile;
  const int left = k.seq_q - k.mq * kTile;
  k.rows = left < kTile ? left : kTile;
  if (k.rows <= 0) {
    k.rows = 0;
    k.num_tile_kv = 0;
    return true;  // not an item of this request; caller skips it
  }
  long long lim = static_cast<long long>(k.seq_kv) - k.seq_q + (k.mq + 1) * kTile;  // exclusive
  if (lim > k.seq_kv) lim = k.seq_kv;
  if (lim < 0) lim = 0;
  k.num_tile_kv = static_cast<int>((lim + kTile - 1) / kTile);
  return true;
}

constexpr int kKsBufs = 4;  // k-scale buffers: one more than the K ring needs (see producer)

// 2^x for a pair of scores on the FMA / ALU pipes (Cody-Waite split + degree-3 polynomial on
// [-0.5, 0.5], relative error 7.5e-5): the MUFU unit (4 lanes per scheduler) is the busiest pipe of
// the softmax pass, so a fixed share of the exponentials is computed this way instead.
__device__ __forceinline__ void exp2_poly_pair(const uint64_t x2, float& e0, float& e1) {
  float x0, x1;
  unpack_f2(x2, x0, x1);
  x0 = fmaxf(x0, -120.f);  // keeps 2^n a normal number; P below 2^-10 rounds to 0 anyway
  x1 = fmaxf(x1, -120.f);
  const uint64_t x = pack_f2(x0, x1);
  const uint64_t t = fadd2(x, pack_f2(12582912.f, 12582912.f));  // 1.5 * 2^23: low bits = round(x)
  const uint64_t r = fadd2(t, pack_f2(-12582912.f, -12582912.f));
  const uint64_t f = ffma2(r, pack_f2(-1.f, -1.f), x);
  uint64_t q = ffma2(f, pack_f2(0.0551716685f, 0.0551716685f), pack_f2(0.2426111251f, 0.2426111251f));
  q = ffma2(q, f, pack_f2(0.6932609677f, 0.6932609677f));
  q = ffma2(q, f, pack_f2(0.9999280572f, 0.9999280572f));
  float q0, q1, t0, t1;
  unpack_f2(q, q0, q1);
  unpack_f2(t, t0, t1);
  e0 = __uint_as_float(__float_as_uint(q0) + (__float_as_uint(t0) << 23));
  e1 = __uint_as_float(__float_as_uint(q1) + (__float_as_uint(t1) << 23));
}

}  // namespace prefill
}  // namespace b200
