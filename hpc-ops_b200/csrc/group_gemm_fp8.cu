// Grouped FP8 GEMM for MoE (H100 / sm_90a), written from scratch.
//
//   Y[rows of group g, :] = X[rows of group g, :] . W[g]^T        X: [M, K] e4m3, W: [G, N, K] e4m3
//
// scale modes
//   blockwise : per 128-wide K block kb   acc += (X_kb . W_kb^T) * xscale[kb, row] * wscale[g, n/128, kb]
//               (reference src/group_gemm/kernels.cuh:532-892, semantics of
//                tests/test_fuse_moe_blockwise.py:84-138)
//   per-tensor: acc = (X . W^T) * yscale[g]   (reference src/group_gemm/kernels.cuh:215-530)
// epilogues
//   plain     : bf16 Y[M, N]
//   fused act : N = 2*I (gate rows then up rows of W): q = silu(bf16(gate)) * bf16(up), then either
//               128-column block quant (scale = amax/448, q/(scale+1e-8) -> e4m3, scales transposed)
//               (reference src/activation/activation.cu:282-356) or per-tensor quant q / act_scale
//               (reference src/activation/activation.cu:19-136). The bf16 Gate-Up matrix never
//               goes to HBM.
//
// Kernel: persistent, one CTA per SM, 160 threads:
//   warp 4      TMA producer: A tile 64 rows x 128 B, B tile 256 rows x 128 B per K block
//               (3 stages x 40 KB, 128B swizzle), tile ids claimed from a global counter
//   warps 0-3   one consumer warpgroup: every K block is converted to fp16 in shared memory (see
//               convert_stage) and multiplied with wgmma (K-major A and B) for the 64 x 256 tile.
//               Per-tensor: one m64n256 accumulator over all K blocks.
//               Blockwise: per K block two m64n128 products (one per 128-column half), each
//               promoted with the block scales into the running accumulator. The running
//               accumulator and a product take 192 registers per thread: with a single consumer
//               warpgroup the CTA may use up to 255 (two warpgroups would be capped at 168).
//               The epilogue works on the accumulator fragment: the gate and
//               up values of one output column are in the same thread, the amax of a row over its
//               128 quantised columns is a reduction over the 4 threads of a quad.
#include "common.cuh"
#include "group_gemm_sched.cuh"
#include "host_utils.h"

namespace b200 {
namespace ggemm {

constexpr int kBM = 64;
constexpr int kBN = 256;
constexpr int kBK = 128;
constexpr int kStages = 3;
constexpr int kABytes = kBM * kBK;
constexpr int kBBytes = kBN * kBK;
constexpr int kStageBytes = kABytes + kBBytes;
// fused Gate-Up: fp16 copy of a K block, each operand as two 64-element K halves of 128-B rows
constexpr int kA16Half = kBM * 128;
constexpr int kB16Half = kBN * 128;
constexpr int kF16Bytes = 2 * (kA16Half + kB16Half);
constexpr int kConvBar = 1;  // named barrier of the consumer warpgroup
constexpr int kConsumerWarps = 4;  // one warpgroup
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kMaxGroups = 512;
constexpr int kTileQ = 4;
constexpr int kXsSlots = kStages + 2;  // activation-scale ring (see the producer)
constexpr int kMaxKB = 128;            // K blocks per tile whose weight scales are staged (K <= 16384)

struct Params {
  const int* seqlens;      // [G] rows per group
  const int* cu_seqlens;   // [G+1] first row of each group in X / Y
  const float* xscale_t;   // blockwise: [K/128, m_pad] (column of (g, i) = pad_base[g] + i)
  const float* wscale;     // blockwise: [G, N/128, kpad4]; per-tensor: yscale [G]
  const float* act_scale;  // per-tensor fused: [1]
  __nv_bfloat16* y;        // plain: [M, N]
  uint8_t* q_out;          // fused: e4m3 [M, N/2]
  float* q_scale_t;        // fused blockwise: [N/2/128, m_pad]
  int num_group;
  int m_total;
  int n;       // rows of W per group
  int k;
  int m_pad;
  int kpad4;
  int scale_tile;  // column padding granule of the transposed activation-scale layout
  int use_bf16_mul;
  int* tile_counter;  // dynamic tile scheduler: [0] next tile, [1] CTAs done (self-resetting)
};

// dynamic shared memory: operand stages, fp16 operand copy, schedule arrays, scale rings, barriers,
// tile queue
constexpr int kSmemBytes = kStages * kStageBytes + kF16Bytes + (kMaxGroups + 4 + 3 * kMaxGroups) * 4 +
                           kXsSlots * kBM * 4 + kTileQ * 2 * kMaxKB * 4 +
                           (2 * kStages + 2 * kTileQ) * 8 + kTileQ * 4;
static_assert(kSmemBytes <= 227 * 1024, "grouped GEMM smem exceeds the sm_90 per-block limit");

template <bool kBlockwise, bool kFused>
__global__ void __launch_bounds__(kThreads, 1)
    group_gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a,
                          const __grid_constant__ CUtensorMap tmap_b, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stages = smem;
  uint8_t* f16_smem = smem + kStages * kStageBytes;
  int* s_cu_tiles = reinterpret_cast<int*>(f16_smem + kF16Bytes);
  int* s_pad_base = s_cu_tiles + (kMaxGroups + 4);  // keeps everything after 16-B aligned
  int* s_rows = s_pad_base + kMaxGroups;
  int* s_row_start = s_rows + kMaxGroups;
  float* s_xs = reinterpret_cast<float*>(s_row_start + kMaxGroups);  // [kXsSlots][128] activation scales
  float* s_ws = s_xs + kXsSlots * kBM;               // [kTileQ][2][kMaxKB] weight scales of a tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_ws + kTileQ * 2 * kMaxKB);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  uint64_t* tq_full = bars + 2 * kStages;   // tile-id queue (kTileQ slots): producer -> consumers
  uint64_t* tq_empty = tq_full + kTileQ;
  int* s_tileq = reinterpret_cast<int*>(tq_empty + kTileQ);

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int KB = (p.k + kBK - 1) / kBK;  // a ragged last K block is zero-filled by TMA
  const int nt_count = kFused ? (p.n / 2 + 127) / 128 : (p.n + kBN - 1) / kBN;
  const int nblk_per_group = p.n / 128;

  // ---- set-up that touches no global memory (overlaps the previous kernel under PDL) ----
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
    for (int i = 0; i < kStages; i++) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConsumerWarps);
    }
    for (int i = 0; i < kTileQ; i++) {
      mbar_init(&tq_full[i], 1);
      mbar_init(&tq_empty[i], kConsumerWarps);
    }
    fence_barrier_init();
  }
  pdl_launch_dependents();
  pdl_wait();  // routing (seqlens, gathered rows, scales) / the previous GEMM's output are complete

  // ---- schedule prologue: every CTA derives the same tile list from seqlens ----
  if (warp == 2) {
    // one warp scans <= 512 groups
    GGEMM_SCHEDULE_SCAN(p, kBM, nt_count, s_cu_tiles, s_pad_base, s_rows, s_row_start, lane);
  }
  __syncthreads();

  Sched sched{s_cu_tiles, s_pad_base, s_rows, s_row_start, p.num_group, nt_count};

  if (warp == kProducerWarp) {
    {
      // =========================== TMA producer ==========================================
      // The whole warp runs this loop with warp-uniform values (tile fields are broadcast with
      // shfl) and ONE elected lane issues: TMA / mbarrier instructions take their operands from
      // uniform registers, and for values the compiler cannot prove uniform it wraps every such
      // instruction in an elect + broadcast loop.
      // A rows of a group are re-read by every n-tile -> keep them in L2. Weight tiles are shared
      // by the 2-3 m-tiles of the same (group, n-tile), which run on neighbouring CTAs at about
      // the same time -> default policy.
      const uint64_t pol_a = make_policy_evict_last();
      uint32_t it = 0;
      uint32_t xsl = 0;  // it % kXsSlots
      uint32_t tq = 0;
      TileInfo t;
      // Dynamic scheduler: tiles are claimed from a global counter, so tiles with neighbouring ids
      // (the m-tiles sharing one weight tile) start within a short window on different CTAs and
      // share that weight tile through L2. The id of the next tile is claimed one tile ahead.
      int next_tile = claim_tile(p.tile_counter, lane);
      while (true) {
        const int tile = next_tile;
        bool valid = decode_tile<kBM>(sched, tile, t);
        valid = __shfl_sync(0xffffffffu, static_cast<int>(valid), 0) != 0;
        t.g = __shfl_sync(0xffffffffu, t.g, 0);
        t.nt = __shfl_sync(0xffffffffu, t.nt, 0);
        t.row0 = __shfl_sync(0xffffffffu, t.row0, 0);
        t.nvalid = __shfl_sync(0xffffffffu, t.nvalid, 0);
        t.scol0 = __shfl_sync(0xffffffffu, t.scol0, 0);
        const uint32_t qs = tq % kTileQ;
        mbar_wait(&tq_empty[qs], ((tq / kTileQ) & 1) ^ 1);
        const int nb0 = kFused ? t.nt : t.nt * 2;
        int nb1 = kFused ? nblk_per_group / 2 + t.nt : t.nt * 2 + 1;
        if (nb1 >= nblk_per_group) nb1 = nb0;
        if (elect_one()) {
          s_tileq[qs] = valid ? tile : -1;
          if (kBlockwise && valid) {
            // the tile's weight scales (KB floats for each 128-column half) travel with its queue slot
            const uint32_t bytes = static_cast<uint32_t>(p.kpad4) * 4u;
            mbar_arrive_expect_tx(&tq_full[qs], 2 * bytes);
            const float* ws = p.wscale + static_cast<long long>(t.g) * nblk_per_group * p.kpad4;
            bulk_load_1d(s_ws + (qs * 2 + 0) * kMaxKB, ws + static_cast<long long>(nb0) * p.kpad4, bytes, &tq_full[qs]);
            bulk_load_1d(s_ws + (qs * 2 + 1) * kMaxKB, ws + static_cast<long long>(nb1) * p.kpad4, bytes, &tq_full[qs]);
          } else {
            mbar_arrive(&tq_full[qs]);
          }
        }
        __syncwarp();
        tq++;
        if (!valid) break;
        next_tile = claim_tile(p.tile_counter, lane);
        const int nrow0 = kFused ? t.nt * 128 : t.nt * kBN;
        const int nrow1 = kFused ? p.n / 2 + t.nt * 128 : t.nt * kBN + 128;
        // activation scales of the tile's rows: 16-byte granules covering the valid rows
        const uint32_t xs_bytes = static_cast<uint32_t>((t.nvalid + 3) / 4) * 16u;
        for (int kb = 0; kb < KB; kb++, it++) {
          const uint32_t s = it % kStages;
          uint8_t* a_dst = stages + s * kStageBytes;
          uint8_t* b_dst = a_dst + kABytes;
          mbar_wait(&empty[s], ((it / kStages) & 1) ^ 1);
          if (elect_one()) {
            uint32_t extra = 0;
            if constexpr (kBlockwise) {
              // The K block's 128 activation scales ride on the stage's barrier. Ring of kStages + 2
              // slots with no "empty" barrier: K block `it` is loaded once stage s is free, i.e.
              // every consumer has released K block it - kStages, and a consumer reads the scales
              // of a K block before it releases that block's stage -- so the previous user of this
              // slot, K block it - kStages - 2, has been read by all of them.
              extra = xs_bytes;
            }
            mbar_arrive_expect_tx(&full[s], kStageBytes + extra);
            if constexpr (kBlockwise) {
              bulk_load_1d(s_xs + xsl * kBM, p.xscale_t + static_cast<long long>(kb) * p.m_pad + t.scol0,
                           xs_bytes, &full[s]);
            }
            tma_load_2d_hint(a_dst, &tmap_a, &full[s], kb * kBK, t.row0, pol_a);
            tma_load_3d(b_dst, &tmap_b, &full[s], kb * kBK, nrow0, t.g);
            tma_load_3d(b_dst + kBBytes / 2, &tmap_b, &full[s], kb * kBK, nrow1, t.g);
          }
          if (++xsl == kXsSlots) xsl = 0;
          __syncwarp();
        }
      }
      if (lane == 0) release_scheduler(p.tile_counter);
    }
  } else {
    // =========================== consumer warpgroups: wgmma + epilogue ====================
    const int g8 = lane >> 2;
    const int t4 = lane & 3;
    // fragment rows of this thread within the tile: r_lo (registers with (i / 2) even), r_lo + 8
    const int r_lo = warp * 16 + g8;
    const int r_hi = r_lo + 8;

    uint32_t it = 0;   // K-block counter (smem ring)
    uint32_t xsl = 0;  // it % kXsSlots (blockwise)
    uint32_t tq = 0;
    TileInfo t;
    while (true) {
      const uint32_t qs = tq % kTileQ;
      mbar_wait(&tq_full[qs], (tq / kTileQ) & 1);
      const int tile = s_tileq[qs];
      tq++;
      if (tile < 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&tq_empty[qs]);
        break;
      }
      decode_tile<kBM>(sched, tile, t);

      // acc[h * 64 + i]: 128-column half h, register i of the m64n128 fragment (the m64n256
      // fragment has the same order: its columns 128..255 are registers 64..127)
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; i++) acc[i] = 0.f;

      // Every K block is converted to fp16 (exact for e4m3) and multiplied with fp16 wgmma, which
      // accumulates in fp32. fp8 wgmma keeps fewer accumulator bits: its rounding differences flip
      // e4m3 codes of the re-quantised Gate-Up activation and, where the partial sums of a K block
      // cancel, move long-K (Down GEMM) outputs by more than the blockwise tolerance. Returns once
      // the fp8 stage has been released.
      auto convert_stage = [&](uint32_t s) {
        const uint8_t* src = stages + s * kStageBytes;
        // the fp16 copy is rewritten only once every warp's slice of the previous wgmma (run on
        // that warp's own tensor core, and reading all of B) has completed
        named_bar_sync(kConvBar, kConsumerWarps * 32);
        for (int q = tid; q < (kBM + kBN) * 8; q += kConsumerWarps * 32) {
          const int row = q >> 3, c = q & 7;
          const bool is_a = row < kBM;
          const int rr = is_a ? row : row - kBM;
          const uint4 v = *reinterpret_cast<const uint4*>(src + (is_a ? 0 : kABytes) + sw128_offset(rr, c));
          uint8_t* dst = f16_smem + (is_a ? 0 : 2 * kA16Half) + (c >> 2) * (is_a ? kA16Half : kB16Half);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
          uint32_t h[8];
#pragma unroll
          for (int i = 0; i < 4; i++) {
            h[2 * i] = e4m3x2_to_f16x2(static_cast<uint16_t>(w[i] & 0xffffu));
            h[2 * i + 1] = e4m3x2_to_f16x2(static_cast<uint16_t>(w[i] >> 16));
          }
          *reinterpret_cast<uint4*>(dst + sw128_offset(rr, 2 * (c & 3))) = make_uint4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<uint4*>(dst + sw128_offset(rr, 2 * (c & 3) + 1)) = make_uint4(h[4], h[5], h[6], h[7]);
        }
        fence_proxy_async_smem();
        named_bar_sync(kConvBar, kConsumerWarps * 32);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      };
      const uint64_t a16 = make_smem_desc(smem_u32(f16_smem), 16, 1024, kLayoutSW128);
      const uint64_t b16 = make_smem_desc(smem_u32(f16_smem) + 2 * kA16Half, 16, 1024, kLayoutSW128);

      if constexpr (kBlockwise) {
        const float* ws0 = s_ws + (qs * 2 + 0) * kMaxKB;
        const float* ws1 = s_ws + (qs * 2 + 1) * kMaxKB;
        for (int kb = 0; kb < KB; kb++, it++) {
          const uint32_t s = it % kStages;
          mbar_wait(&full[s], (it / kStages) & 1);
          // block scales from shared memory, staged by the producer with the operands of this
          // K block; rows past the tile's end have no scale loaded
          const float xs_lo = r_lo < t.nvalid ? s_xs[xsl * kBM + r_lo] : 0.f;
          const float xs_hi = r_hi < t.nvalid ? s_xs[xsl * kBM + r_hi] : 0.f;
          if (++xsl == kXsSlots) xsl = 0;
          const float w0 = ws0[kb], w1 = ws1[kb];
          convert_stage(s);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            float part[64];  // overwritten: the first wgmma of the block does not read D
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; k++) {  // K halves of 64, 16 per wgmma
              WgmmaF16<128, 0, 0>::ss(part, a16 + (k >> 2) * (kA16Half >> 4) + (k & 3) * 2,
                                      b16 + (k >> 2) * (kB16Half >> 4) + h * (128 * 128 >> 4) + (k & 3) * 2,
                                      k > 0);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_anchor<64>(part);
            const float w = h ? w1 : w0;
            const float f_lo = xs_lo * w, f_hi = xs_hi * w;
#pragma unroll
            for (int i = 0; i < 64; i++) {
              acc[64 * h + i] = __fmaf_rn(part[i], ((i >> 1) & 1) ? f_hi : f_lo, acc[64 * h + i]);
            }
          }
        }
      } else {
        for (int kb = 0; kb < KB; kb++, it++) {
          const uint32_t s = it % kStages;
          mbar_wait(&full[s], (it / kStages) & 1);
          convert_stage(s);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 8; k++) {
            WgmmaF16<256, 0, 0>::ss(acc, a16 + (k >> 2) * (kA16Half >> 4) + (k & 3) * 2,
                                    b16 + (k >> 2) * (kB16Half >> 4) + (k & 3) * 2, (kb | k) > 0);
          }
          wgmma_commit();
          wgmma_wait<0>();
        }
        wgmma_anchor<128>(acc);
        const float ys = __ldg(p.wscale + t.g);
#pragma unroll
        for (int i = 0; i < 128; i++) acc[i] *= ys;
      }
      // the queue slot (tile id + its weight scales) is free once the K loop is through
      __syncwarp();
      if (lane == 0) mbar_arrive(&tq_empty[qs]);

      // ---------------- tile epilogue ----------------
      const bool ok_lo = r_lo < t.nvalid, ok_hi = r_hi < t.nvalid;
      const long long grow_lo = static_cast<long long>(t.row0) + r_lo;
      const long long grow_hi = grow_lo + 8;
      if constexpr (!kFused) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
          for (int j = 0; j < 16; j++) {
            const int col = t.nt * kBN + h * 128 + 8 * j + 2 * t4;
            if (col >= p.n) continue;
            const float* v = acc + h * 64 + 4 * j;
            __nv_bfloat162 b_lo = __floats2bfloat162_rn(v[0], v[1]);
            __nv_bfloat162 b_hi = __floats2bfloat162_rn(v[2], v[3]);
            if (ok_lo) *reinterpret_cast<__nv_bfloat162*>(p.y + grow_lo * p.n + col) = b_lo;
            if (ok_hi) *reinterpret_cast<__nv_bfloat162*>(p.y + grow_hi * p.n + col) = b_hi;
          }
        }
      } else {
        // silu(gate) * up on the bf16-rounded Gate-Up values (the reference materialises the
        // Gate-Up output as bf16 before the activation: src/fuse_moe/entry.cc:565-566); gate in
        // half 0, up in half 1 at the same register index
        float amax_lo = 0.f, amax_hi = 0.f;
#pragma unroll
        for (int i = 0; i < 64; i++) {
          const float g = bf16_round(acc[i]), u = bf16_round(acc[64 + i]);
          float a = silu_f(g);
          if (!kBlockwise && p.use_bf16_mul) {
            a = bf16_round(bf16_round(a) * u);
          } else {
            a *= u;
          }
          acc[i] = a;
          if ((i >> 1) & 1) {
            amax_hi = fmaxf(amax_hi, fabsf(a));
          } else {
            amax_lo = fmaxf(amax_lo, fabsf(a));
          }
        }
        float inv_lo, inv_hi;
        if constexpr (kBlockwise) {
          // a row's 128 columns are spread over the 4 threads of a quad
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            amax_lo = fmaxf(amax_lo, __shfl_xor_sync(0xffffffffu, amax_lo, o));
            amax_hi = fmaxf(amax_hi, __shfl_xor_sync(0xffffffffu, amax_hi, o));
          }
          const float sc_lo = amax_lo / 448.f, sc_hi = amax_hi / 448.f;
          inv_lo = 1.f / (sc_lo + 1e-8f);
          inv_hi = 1.f / (sc_hi + 1e-8f);
          if (t4 == 0) {
            float* qs_col = p.q_scale_t + static_cast<long long>(t.nt) * p.m_pad + t.scol0;
            if (ok_lo) qs_col[r_lo] = sc_lo;
            if (ok_hi) qs_col[r_hi] = sc_hi;
          }
        } else {
          inv_lo = inv_hi = __ldg(p.act_scale);  // per-tensor: the scale is a multiplier (activation.cu:19-136)
        }
        const int ncols = p.n / 2;
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const int col = t.nt * 128 + 8 * j + 2 * t4;
          if (col >= ncols) continue;
          const float* v = acc + 4 * j;
          if (ok_lo) {
            *reinterpret_cast<uint16_t*>(p.q_out + grow_lo * ncols + col) =
                cvt_e4m3x2(v[0] * inv_lo, v[1] * inv_lo);
          }
          if (ok_hi) {
            *reinterpret_cast<uint16_t*>(p.q_out + grow_hi * ncols + col) =
                cvt_e4m3x2(v[2] * inv_hi, v[3] * inv_hi);
          }
        }
      }
    }
  }
}

template <bool kBlockwise, bool kFused>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Params& p, cudaStream_t stream) {
  auto kern = group_gemm_fp8_kernel<kBlockwise, kFused>;
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(kern), kSmemBytes));
  Params pp = p;
  pp.tile_counter = scheduler_counter(stream);  // self-resetting pair: per stream, or per captured launch
  if (pp.tile_counter == nullptr) return HPC_ERR_CUDA;
  HPC_CUDA_CHECK(launch_pdl(kern, dim3(sm_count()), dim3(kThreads), kSmemBytes, stream, 1, ta, tb, pp));
  return HPC_OK;
}

// Common launcher. mode bits: 1 = blockwise scales, 2 = fused activation epilogue.
int run(int mode, const void* x, const void* w, const int* seqlens, const int* cu_seqlens,
        const float* xscale_t, const float* wscale, const float* act_scale, void* y, void* q_out,
        float* q_scale_t, int num_group, int m, int n, int k, int m_pad, int kpad4, int scale_tile,
        int use_bf16_mul, cudaStream_t stream) {
  HPC_REQUIRE(num_group > 0 && num_group <= kMaxGroups, "group gemm: num_group %d not in (0, %d]",
              num_group, kMaxGroups);
  if (mode & 1) {
    HPC_REQUIRE(k % 128 == 0 && k >= 128, "group gemm: k (%d) must be a multiple of 128", k);
    HPC_REQUIRE(n % 128 == 0, "group gemm: n (%d) must be a multiple of 128", n);
    if (mode & 2) HPC_REQUIRE(n % 256 == 0, "fused act: gate_up rows (%d) must be a multiple of 256", n);
    HPC_REQUIRE(kpad4 % 4 == 0 && kpad4 * 128 >= k && kpad4 <= kMaxKB,
                "group gemm: weight-scale row length %d must be a multiple of 4 covering k/128 (<= %d)",
                kpad4, kMaxKB);
    HPC_REQUIRE(m_pad % 4 == 0 && scale_tile % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(xscale_t) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(wscale) & 15) == 0,
                "group gemm: activation-scale columns (%d, tile %d) must be multiples of 4 and the "
                "scale tensors 16-byte aligned", m_pad, scale_tile);
  } else {
    HPC_REQUIRE(k % 16 == 0 && k >= 16, "group gemm: k (%d) must be a multiple of 16", k);
    HPC_REQUIRE(n % 64 == 0, "group gemm: n (%d) must be a multiple of 64", n);
    if (mode & 2) HPC_REQUIRE(n % 32 == 0, "fused act: gate_up rows (%d) must be a multiple of 32", n);
  }
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
              "group gemm: x and weight must be 16-byte aligned");
  if (m <= 0) return HPC_OK;
  HPC_REQUIRE(scale_tile > 0, "group gemm: scale_tile must be positive");

  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(m)};
    uint64_t strides[1] = {static_cast<uint64_t>(k)};
    uint32_t box[2] = {128, static_cast<uint32_t>(kBM)};
    int rc = encode_tmap_u8(&ta, x, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {static_cast<uint64_t>(k), static_cast<uint64_t>(n),
                        static_cast<uint64_t>(num_group)};
    uint64_t strides[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(k) * n};
    uint32_t box[3] = {128, 128, 1};
    int rc = encode_tmap_u8(&tb, w, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  Params p;
  p.seqlens = seqlens;
  p.cu_seqlens = cu_seqlens;
  p.xscale_t = xscale_t;
  p.wscale = wscale;
  p.act_scale = act_scale;
  p.y = static_cast<__nv_bfloat16*>(y);
  p.q_out = static_cast<uint8_t*>(q_out);
  p.q_scale_t = q_scale_t;
  p.num_group = num_group;
  p.m_total = m;
  p.n = n;
  p.k = k;
  p.m_pad = m_pad;
  p.kpad4 = kpad4;
  p.scale_tile = scale_tile;
  p.use_bf16_mul = use_bf16_mul;
  switch (mode & 3) {
    case 0: return launch<false, false>(ta, tb, p, stream);
    case 1: return launch<true, false>(ta, tb, p, stream);
    case 2: return launch<false, true>(ta, tb, p, stream);
    default: return launch<true, true>(ta, tb, p, stream);
  }
}

// Activation-scale column granule from the average rows per group (reference
// src/fuse_moe/entry.cc:525-543). The one rule of the library: the grouped GEMMs, the FusedMoE route
// and, through hpc_scale_tile_from_avg, reformat_x_scale and the Python host code all take it from
// here, so a layout written by one is the layout read by the other.
int scale_tile_from_avg(int avg) {
  if (avg <= 8) return 8;
  if (avg <= 16) return 16;
  if (avg <= 32) return 32;
  if (avg <= 48) return 48;
  if (avg <= 64) return 64;
  if (avg <= 96) return 48;
  if (avg <= 128) return 32;
  if (avg <= 144) return 48;
  return 64;
}

}  // namespace ggemm
}  // namespace b200

using namespace b200;  // NOLINT

extern "C" int hpc_scale_tile_from_avg(int num_seq_per_group_avg) {
  return ggemm::scale_tile_from_avg(num_seq_per_group_avg);
}

// replaces reference src/group_gemm/group_gemm.h:22-29 (group_gemm_blockwise_fp8_async). The
// tmas / tiles / cu_tiles / task_map / num_waves / update_tma / use_pdl arguments are accepted for
// signature compatibility; this build derives its tile schedule inside the kernel.
extern "C" int hpc_group_gemm_blockwise_fp8_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* seqlens_ptr,
    const void* cu_seqlens_ptr, const void* xscale_ptr, const void* wscale_ptr, void* tmas_ptr,
    void* tiles_ptr, void* cu_tiles_ptr, void* task_map_ptr, int num_waves, int num_group, int m,
    int n, int k, int m_pad, int num_block_k_pad4, int num_seq_per_group_avg, int update_tma,
    int use_pdl, cudaStream_t stream) {
  (void)tmas_ptr; (void)tiles_ptr; (void)cu_tiles_ptr; (void)task_map_ptr; (void)num_waves;
  (void)update_tma; (void)use_pdl;
  return ggemm::run(1, x_ptr, w_ptr, static_cast<const int*>(seqlens_ptr),
                    static_cast<const int*>(cu_seqlens_ptr), static_cast<const float*>(xscale_ptr),
                    static_cast<const float*>(wscale_ptr), nullptr, y_ptr, nullptr, nullptr,
                    num_group, m, n, k, m_pad, num_block_k_pad4,
                    ggemm::scale_tile_from_avg(num_seq_per_group_avg), 0, stream);
}

// replaces reference src/group_gemm/group_gemm.h:12-20 (group_gemm_fp8_async, per-group y_scale)
extern "C" int hpc_group_gemm_fp8_async(void* y_ptr, const void* x_ptr, const void* w_ptr,
                                        const void* seqlens_ptr, const void* cu_seqlens_ptr,
                                        const void* y_scale, void* tmas_ptr, void* tiles_ptr,
                                        void* cu_tiles_ptr, void* task_map_ptr, int num_waves,
                                        int num_group, int m, int n, int k,
                                        int num_seq_per_group_avg, int update_tma, int use_pdl,
                                        cudaStream_t stream) {
  (void)tmas_ptr; (void)tiles_ptr; (void)cu_tiles_ptr; (void)task_map_ptr; (void)num_waves;
  (void)update_tma; (void)use_pdl; (void)num_seq_per_group_avg;
  return ggemm::run(0, x_ptr, w_ptr, static_cast<const int*>(seqlens_ptr),
                    static_cast<const int*>(cu_seqlens_ptr), nullptr,
                    static_cast<const float*>(y_scale), nullptr, y_ptr, nullptr, nullptr, num_group,
                    m, n, k, 0, 0, 64, 0, stream);
}
