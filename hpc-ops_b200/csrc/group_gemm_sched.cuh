// Tile scheduling and epilogue arithmetic shared by the persistent grouped GEMMs (group_gemm_fp8.cu,
// group_gemm_bf16.cu).
//
// Every CTA derives the same tile list from seqlens in its prologue (one warp scans <= 512 groups
// into shared memory); a tile id maps to (group, n-tile, m-tile) with the m-tiles of one
// (group, n-tile) adjacent, so the CTAs that share a weight tile run at about the same time. Tile ids
// are claimed from a self-resetting global counter pair (host_utils.h scheduler_counter): [0] is
// the next tile, [1] counts the CTAs that are done, and the last CTA out zeroes both.
#pragma once
#include "common.cuh"

namespace b200 {
namespace ggemm {

__device__ __forceinline__ float silu_f(float x) {
  // x / (1 + exp(-x)) with ex2.approx / approximate division (relative error ~1e-6, far below
  // the bf16 / e4m3 granularity around it; reference src/utils/utils.cuh:300-330 does the same).
  // An IEEE expf + division here costs ~35 % of a Gate-Up tile's MMA time in the epilogue.
  return __fdividef(x, 1.f + __expf(-x));
}

__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

struct TileInfo {
  int g, mt, nt;
  int row0;    // first row (global) of the tile
  int nvalid;  // valid rows in the tile
  int scol0;   // first activation-scale column of the tile
};

// smem-resident schedule: cu_tiles (prefix of m-tiles*NT), pad_base (scale column base) per group
struct Sched {
  int* cu_tiles;   // [G+1]
  int* pad_base;   // [G]
  int* rows;       // [G]
  int* row_start;  // [G]
  int num_group;
  int nt_count;
};

// Prologue scan, run by one whole warp of every CTA: per group its first tile id, its first
// activation-scale column (rows padded to p.scale_tile), its row count and its first row. `p` is the
// kernel's parameter block (fields seqlens, cu_seqlens, num_group, scale_tile). A macro, not an
// inline function: inlining a function here moves the basic blocks of the FP8 kernels, whose machine
// code this header must leave exactly as it was.
#define GGEMM_SCHEDULE_SCAN(p, BM, nt_count, s_cu_tiles, s_pad_base, s_rows, s_row_start, lane) \
{                                                                              \
  int carry_tiles = 0, carry_pad = 0;                                          \
  for (int g0 = 0; g0 < (p).num_group; g0 += 32) {                             \
    const int g = g0 + (lane);                                                 \
    const int r = g < (p).num_group ? (p).seqlens[g] : 0;                      \
    const int mt = (r + (BM) - 1) / (BM);                                      \
    const int pd = (r + (p).scale_tile - 1) / (p).scale_tile * (p).scale_tile; \
    int it = mt * (nt_count), ip = pd;                                         \
    _Pragma("unroll")                                                          \
    for (int o = 1; o < 32; o <<= 1) {                                         \
      const int a = __shfl_up_sync(0xffffffffu, it, o);                        \
      const int b = __shfl_up_sync(0xffffffffu, ip, o);                        \
      if ((lane) >= o) {                                                       \
        it += a;                                                               \
        ip += b;                                                               \
      }                                                                        \
    }                                                                          \
    if (g < (p).num_group) {                                                   \
      (s_cu_tiles)[g] = carry_tiles + it - mt * (nt_count);                    \
      (s_pad_base)[g] = carry_pad + ip - pd;                                   \
      (s_rows)[g] = r;                                                         \
      (s_row_start)[g] = (p).cu_seqlens[g];                                    \
    }                                                                          \
    carry_tiles += __shfl_sync(0xffffffffu, it, 31);                           \
    carry_pad += __shfl_sync(0xffffffffu, ip, 31);                             \
  }                                                                            \
  if ((lane) == 0) (s_cu_tiles)[(p).num_group] = carry_tiles;                  \
}

template <int kBM>
__device__ __forceinline__ bool decode_tile(const Sched& s, int tile, TileInfo& t) {
  if (tile >= s.cu_tiles[s.num_group]) return false;
  int lo = 0, hi = s.num_group - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (s.cu_tiles[mid] <= tile) {
      lo = mid;
    } else {
      hi = mid - 1;
    }
  }
  const int g = lo;
  const int local = tile - s.cu_tiles[g];
  const int mtiles = (s.rows[g] + kBM - 1) / kBM;
  t.g = g;
  t.nt = local / mtiles;
  t.mt = local - t.nt * mtiles;
  t.row0 = s.row_start[g] + t.mt * kBM;
  const int left = s.rows[g] - t.mt * kBM;
  t.nvalid = left < kBM ? left : kBM;
  t.scol0 = s.pad_base[g] + t.mt * kBM;
  return true;
}

// The next tile id, claimed by lane 0 of the producer warp and broadcast to the warp.
__device__ __forceinline__ int claim_tile(int* tile_counter, int lane) {
  int v = 0;
  if (lane == 0) v = atomicAdd(tile_counter, 1);
  return __shfl_sync(0xffffffffu, v, 0);
}

// Called by one thread per CTA once the CTA claims no more tiles: the last CTA out re-arms the
// scheduler for the next launch (no memset between launches: a memset node would break a PDL
// chain, and a graph replay needs nothing else).
__device__ __forceinline__ void release_scheduler(int* tile_counter) {
  __threadfence();
  if (atomicAdd(tile_counter + 1, 1) == static_cast<int>(gridDim.x) - 1) {
    tile_counter[0] = 0;
    tile_counter[1] = 0;
    __threadfence();
  }
}

}  // namespace ggemm
}  // namespace b200
