// MLA decode attention (absorbed multi-head latent attention) over a paged bf16 latent cache.
//
// With weight absorption every query head is 576 wide ([q_nope . W_UK (512) | q_pe (64)]) and
// every cached token is one 576-wide row ([kv_c (512) | k_pe (64)]) shared by all heads; V is
// columns 0..511 of the same row. So this is multi-query attention with one latent kv head:
//
//   * query tile : 64 rows of one request in q's (sq, h) order; T = ceil(H (mtp+1) / 64) tiles.
//                  The split-k task map (decode_taskmap.cu) is built with num_head_kv = T, so a
//                  "kv head" of the map is a query tile; every tile streams the same pages.
//   * persistent grid = num_total_ctas; each CTA walks its bin (128-key tiles = two 64-token pages).
//                  With T >= 2 the walk is rotated (decode_common.cuh) so that CTAs that stream
//                  the same page do so at the same step and the later tiles can hit L2.
//   * warpgroup 2 : TMA producer (one warp, setmaxnreg 40). Q tile: nine [64 rows x 64 dims]
//                  128B-swizzled boxes (72 KB). A page: nine [64 keys x 64 dims] boxes (72 KB),
//                  2 stages.
//   * warpgroup 0 : S[64, 64] = Q . K^T (36 x m64n64k16, both K-major), zeroes the V rows past
//                  the task's last key, base-2 online softmax on the fragment, P -> bf16 smem
//                  (8 KB, 128B swizzle) with the per-row rescale factor; then O[:, 0:256] += P . V.
//   * warpgroup 1 : O[:, 256:512] += P . V (m64n256k16, V MN-major straight from the K tile).
//   * single-chunk (request, tile) pairs write bf16 y; split chunks write an fp32 partial + LSE
//                  into one of two slots of the bin that ran them; mla_combine_kernel merges them.
#include "decode_common.cuh"

#ifndef HPC_DECODE_MLA_PROBE
#define HPC_DECODE_MLA_PROBE 0  // 1: consumers only wait for the pages; 2: no loads (tools/)
#endif

namespace b200 {
namespace decode_mla {

using decode::BinWalk;
using decode::kTaskStride;
using decode::load_task;
using decode::Segment;
using decode::Task;

constexpr int kDqk = 576;
constexpr int kDv = 512;
constexpr int kPage = 64;
constexpr int kRows = 64;                 // query rows per tile
constexpr int kBoxBytes = 64 * 128;       // [64 rows x 64 bf16]
constexpr int kBoxes = kDqk / 64;         // 9
constexpr int kTileBytes = kBoxes * kBoxBytes;  // 72 KB: a Q tile or a page
constexpr int kStages = 2;
constexpr int kThreads = 384;
constexpr int kProducerWarp = 8;
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kCarryFloats = 256 * 128 + 128 * 4;  // per CTA: both O halves + WG 0's m, l
static_assert(kProducerRegs * 128 + kConsumerRegs * 256 <= 65536,
              "setmaxnreg split exceeds the register file");

constexpr int kOffQ = 0;
constexpr int kOffStages = kOffQ + kTileBytes;
constexpr int kOffP = kOffStages + kStages * kTileBytes;
constexpr int kOffAlpha = kOffP + kBoxBytes;      // float[64]: rescale of this page
constexpr int kOffInv = kOffAlpha + kRows * 4;    // float[64]: 1 / row sum at a segment's end
constexpr int kOffBar = kOffInv + kRows * 4;
constexpr int kNumBars = 2 * kStages + 4;
constexpr int kSmemBytes = kOffBar + kNumBars * 8;
static_assert(kSmemBytes <= 227 * 1024, "decode MLA smem exceeds the sm_90 per-block limit");

struct Params {
  const int* task_map;
  const int* block_ids;
  __nv_bfloat16* y;
  float* partial;     // [2 * num_total_ctas slots][64 rows][512]
  float* lse;         // [2 * num_total_ctas slots][64 rows], base 2
  int* chunk_base;    // [B * T]: bin of chunk 0 of each split pair
  float* carry;       // [num_total_ctas][kCarryFloats]: state of the task a rotated walk splits
  int ld_y;
  int num_batch;
  int num_seq_q;
  int num_head_q;
  int head_log2;
  int num_tiles;      // T
  int num_seq_max_blocks;
  int rotate;
  float scale_log2;   // softmax_scale * log2(e)
};

// Split chunk `c` of a pair whose chunk 0 ran in bin `base`: chunk c > 0 starts its bin, chunk 0
// ends its bin, and a bin holds at most one of each, so two slots per bin never collide.
__device__ __forceinline__ long long chunk_slot(int base, int c) {
  return c == 0 ? 2LL * base + 1 : 2LL * (base + c);
}

__device__ __forceinline__ void page_range(const Segment& sg, const Task& t, int& pb, int& pe) {
  const int npages = (t.num_seqkv + kPage - 1) / kPage;
  const int te = sg.te < 0 ? t.num_tile_kv : sg.te;
  pb = 2 * sg.tb;
  pe = 2 * te < npages ? 2 * te : npages;
}

__global__ void __launch_bounds__(kThreads, 1)
    decode_attn_mla_kernel(const __grid_constant__ CUtensorMap tmap_q,
                           const __grid_constant__ CUtensorMap tmap_kv, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* q_smem = smem + kOffQ;
  uint8_t* stages = smem + kOffStages;
  uint8_t* p_smem = smem + kOffP;
  float* s_alpha = reinterpret_cast<float*>(smem + kOffAlpha);
  float* s_inv = reinterpret_cast<float*>(smem + kOffInv);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  uint64_t* q_full = bars + 2 * kStages;
  uint64_t* q_empty = q_full + 1;
  uint64_t* p_full = q_full + 2;
  uint64_t* p_free = q_full + 3;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_kv);
    for (int i = 0; i < kStages; i++) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // one arrival per consumer warp
    }
    mbar_init(q_full, 1);
    mbar_init(q_empty, 4);    // warps of warpgroup 0, after the segment's last QK
    mbar_init(p_full, 128);   // warpgroup 0's threads, each after its P / alpha stores and fence
    mbar_init(p_free, 128);   // warpgroup 1's threads, after the PV that read P
    fence_barrier_init();
  }
  __syncthreads();

  pdl_launch_dependents();
  pdl_wait();

  const int ntpc1 = p.task_map[0];
  const int* bin = p.task_map + (1 + static_cast<long long>(blockIdx.x) * ntpc1) * kTaskStride;
  const int u0 = p.rotate ? decode::walk_start(p.task_map, blockIdx.x) : 0;
  const BinWalk walk = decode::scan_bin(bin, ntpc1 - 1, u0, lane);
  const int nseg = decode::num_segments(walk);

  if (warp >= kProducerWarp) {
    // =========================== TMA producer ===============================================
    setmaxnreg_dec<kProducerRegs>();
    if (warp != kProducerWarp) return;
    // a page is read by the T tiles of its request: keep it for the CTAs that follow under the
    // rotated walk; streamed once otherwise
    const uint64_t pol = p.rotate ? make_policy_evict_normal() : make_policy_evict_first();
    const int heads_per_box = p.num_head_q < kRows ? p.num_head_q : kRows;
    const int tiles_per_tok = p.num_head_q / heads_per_box;  // H >= 64: H / 64, else 1
    const int toks_per_tile = kRows / heads_per_box;          // H < 64: 64 / H, else 1
    uint32_t n = 0;
    Task t;
    for (int j = 0; j < nseg; j++) {
      const Segment sg = decode::segment_of(walk, j);
      if (!load_task(bin + static_cast<long long>(sg.row) * kTaskStride, t)) break;
      t.ihead_kv = __shfl_sync(0xffffffffu, t.ihead_kv, 0);
      t.ibatch = __shfl_sync(0xffffffffu, t.ibatch, 0);
      int pb, pe;
      page_range(sg, t, pb, pe);
      pb = __shfl_sync(0xffffffffu, pb, 0);
      pe = __shfl_sync(0xffffffffu, pe, 0);
      mbar_wait_nocall(q_empty, (j & 1) ^ 1);
#if HPC_DECODE_MLA_PROBE != 2
      if (elect_one()) {
        mbar_arrive_expect_tx(q_full, kTileBytes);
        const int tok = t.ibatch * p.num_seq_q + (t.ihead_kv / tiles_per_tok) * toks_per_tile;
        const int head0 = (t.ihead_kv % tiles_per_tok) * kRows;
        for (int bx = 0; bx < kBoxes; bx++) {
          tma_load_3d(q_smem + bx * kBoxBytes, &tmap_q, q_full, bx * 64, head0, tok);
        }
      }
#else
      if (elect_one()) mbar_arrive(q_full);
#endif
      __syncwarp();
      const int* ids = p.block_ids + static_cast<long long>(t.ibatch) * p.num_seq_max_blocks +
                       t.iseq_start / kPage;
      for (int g0 = pb; g0 < pe; g0 += 32) {
        const int bi = g0 + lane < pe ? g0 + lane : pe - 1;
        const int my_id = __ldg(ids + bi);
        const int gn = pe - g0 < 32 ? pe - g0 : 32;
        for (int k = 0; k < gn; k++, n++) {
          const int id = __shfl_sync(0xffffffffu, my_id, k);
          const uint32_t st = n % kStages;
          mbar_wait_nocall(&empty[st], ((n / kStages) & 1) ^ 1);
#if HPC_DECODE_MLA_PROBE != 2
          if (elect_one()) {
            mbar_arrive_expect_tx(&full[st], kTileBytes);
            uint8_t* dst = stages + st * kTileBytes;
            for (int bx = 0; bx < kBoxes; bx++) {
              tma_load_3d_hint(dst + bx * kBoxBytes, &tmap_kv, &full[st], bx * 64, 0, id, pol);
            }
          }
#else
          (void)id;
          if (elect_one()) mbar_arrive(&full[st]);
#endif
          __syncwarp();
        }
      }
    }
    return;
  }

  // =========================== consumers ===================================================
  setmaxnreg_inc<kConsumerRegs>();
  // 0: QK + softmax + O[:, 0:256]; 1: O[:, 256:512] (broadcast so that it is warp-uniform)
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
  const int wtid = tid & 127;
  const int g8 = lane >> 2;
  const int t4 = lane & 3;
  const int r0 = (warp & 3) * 16 + g8;  // fragment rows r0 and r0 + 8 of the tile
  const int* chunk_table = p.task_map + kTaskStride * (ntpc1 * p.task_map[1] + 1);
  float* carry = p.carry + static_cast<long long>(blockIdx.x) * kCarryFloats;

  //  Q / K / P : K-major, 128B swizzle, 8-row groups 1024 B apart; 16 dims = +32 B, box = +8 KB
  //  V half    : MN-major, 128B swizzle: 64-column boxes 8 KB apart (LBO), 8-key groups 1 KB
  //              apart (SBO); 16 keys = +2 KB
  const uint64_t qdesc = make_smem_desc(smem_u32(q_smem), 16, 1024, kLayoutSW128);
  const uint64_t kdesc0 = make_smem_desc(smem_u32(stages), 16, 1024, kLayoutSW128);
  const uint64_t vdesc0 =
      make_smem_desc(smem_u32(stages) + wg * 4 * kBoxBytes, kBoxBytes, 1024, kLayoutSW128);
  const uint64_t pdesc = make_smem_desc(smem_u32(p_smem), 16, 1024, kLayoutSW128);

  uint32_t n = 0;
  Task t;
  for (int j = 0; j < nseg; j++) {
    const Segment sg = decode::segment_of(walk, j);
    if (!load_task(bin + static_cast<long long>(sg.row) * kTaskStride, t)) break;
    int pb, pe;
    page_range(sg, t, pb, pe);
    const int tile = t.ihead_kv;
    const int lim_len = t.num_seqkv;
    const int lim_causal = t.num_seqkvcache;
    // query token of fragment rows r0 and r0 + 8 (rows past the request's last token see more
    // keys; they are never written)
    const int sq0 = (tile * kRows + r0) >> p.head_log2;
    const int sq1 = (tile * kRows + r0 + 8) >> p.head_log2;

    float o[128];
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    if (sg.restore) {
#pragma unroll
      for (int i = 0; i < 128; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(carry + (i / 4) * 1024 + tid * 4);
        o[i] = v.x;
        o[i + 1] = v.y;
        o[i + 2] = v.z;
        o[i + 3] = v.w;
      }
      if (wg == 0) {
        const float4 v = *reinterpret_cast<const float4*>(carry + 256 * 128 + wtid * 4);
        m0 = v.x;
        m1 = v.y;
        l0 = v.z;
        l1 = v.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 128; i++) o[i] = 0.f;
    }
#if HPC_DECODE_MLA_PROBE == 1
    if (wg == 0) mbar_wait_nocall(q_full, j & 1);
    for (int pg = pb; pg < pe; pg++, n++) {
      const uint32_t st = n % kStages;
      mbar_wait_nocall(&full[st], (n / kStages) & 1);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
    }
    if (wg == 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(q_empty);
    }
    continue;
#endif
    if (wg == 0) mbar_wait_nocall(q_full, j & 1);

    float inv0 = 0.f, inv1 = 0.f;  // warpgroup 1: 1 / row sum, published with the last P
    for (int pg = pb; pg < pe; pg++, n++) {
      const uint32_t st = n % kStages;
      const uint32_t ph = (n / kStages) & 1;
      float a0 = 1.f, a1 = 1.f;
      if (wg == 0) {
        // ---- S = Q . K^T over 576 dims ----
        mbar_wait_nocall(&full[st], ph);
        float s[32];
        {
          const uint64_t kd = kdesc0 + static_cast<uint64_t>(st * (kTileBytes >> 4));
          wgmma_fence();
#pragma unroll
          for (int bx = 0; bx < kBoxes; bx++) {
#pragma unroll
            for (int k = 0; k < 4; k++) {
              const uint64_t off = static_cast<uint64_t>((bx * kBoxBytes + k * 32) >> 4);
              WgmmaBF16<64, 0, 0>::ss(s, qdesc + off, kd + off, (bx | k) > 0);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_anchor<32>(s);
        }
        if (pg == pe - 1) {  // the segment's last QK has completed: the Q tile may be replaced
          __syncwarp();
          if (lane == 0) mbar_arrive(q_empty);
        }
        const int key0 = pg * kPage;
        // keys past the task's last one: V rows of the page may hold anything (NaN included) and
        // 0 * NaN would reach O, so they are zeroed in all eight V boxes
        const int valid = lim_len - key0;
        if (valid < kPage) {
          uint8_t* base = stages + st * kTileBytes;
          const int nz = (kPage - valid) * 8 * 8;  // 16-byte chunks: rows x boxes x chunks
          for (int i = wtid; i < nz; i += 128) {
            const int row = valid + i / 64;
            const int bx = (i / 8) & 7;
            const int c = i & 7;
            *reinterpret_cast<uint4*>(base + bx * kBoxBytes + row * 128 + c * 16) =
                make_uint4(0, 0, 0, 0);
          }
          fence_proxy_async_smem();
        }
        // ---- base-2 online softmax on the fragment ----
        const int lim_min = lim_len < lim_causal ? lim_len : lim_causal;
        const bool need_mask = key0 + kPage > lim_min;
        const float c = p.scale_log2;
        float tm0 = -INFINITY, tm1 = -INFINITY;
#pragma unroll
        for (int i = 0; i < 32; i++) {
          float v = s[i] * c;
          if (need_mask) {
            const int key = key0 + 8 * (i >> 2) + 2 * t4 + (i & 1);
            const int sq = (i & 2) ? sq1 : sq0;
            v = (key >= lim_len || key > lim_causal + sq) ? -INFINITY : v;
          }
          s[i] = v;
          if (i & 2) {
            tm1 = fmaxf(tm1, v);
          } else {
            tm0 = fmaxf(tm0, v);
          }
        }
        tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 1));
        tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 2));
        tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 1));
        tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 2));
        const float mn0 = fmaxf(m0, tm0);
        const float mn1 = fmaxf(m1, tm1);
        const float ms0 = mn0 == -INFINITY ? 0.f : mn0;  // all keys so far masked: P = 0, alpha = 1
        const float ms1 = mn1 == -INFINITY ? 0.f : mn1;
        a0 = m0 == -INFINITY ? 1.f : exp2_approx(m0 - ms0);
        a1 = m1 == -INFINITY ? 1.f : exp2_approx(m1 - ms1);
        m0 = mn0;
        m1 = mn1;
        float ps0 = 0.f, ps1 = 0.f;
        // P (bf16) into the 128B-swizzled [64 rows x 64 keys] tile; free once warpgroup 1's
        // previous PV has completed (warpgroup 0's own PV precedes this in program order)
        mbar_wait_nocall(p_free, (n & 1) ^ 1);
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
          const float e0 = exp2_approx(s[4 * jj] - ms0);
          const float e1 = exp2_approx(s[4 * jj + 1] - ms0);
          const float e2 = exp2_approx(s[4 * jj + 2] - ms1);
          const float e3 = exp2_approx(s[4 * jj + 3] - ms1);
          ps0 += e0 + e1;
          ps1 += e2 + e3;
          *reinterpret_cast<uint32_t*>(p_smem + sw128_offset(r0, jj) + t4 * 4) = pack_bf16x2(e0, e1);
          *reinterpret_cast<uint32_t*>(p_smem + sw128_offset(r0 + 8, jj) + t4 * 4) =
              pack_bf16x2(e2, e3);
        }
        l0 = l0 * a0 + ps0;
        l1 = l1 * a1 + ps1;
        if (t4 == 0) {
          s_alpha[r0] = a0;
          s_alpha[r0 + 8] = a1;
        }
        if (pg == pe - 1) {  // row sums of the segment, for warpgroup 1's epilogue
          float lt0 = l0 + __shfl_xor_sync(0xffffffffu, l0, 1);
          lt0 += __shfl_xor_sync(0xffffffffu, lt0, 2);
          float lt1 = l1 + __shfl_xor_sync(0xffffffffu, l1, 1);
          lt1 += __shfl_xor_sync(0xffffffffu, lt1, 2);
          if (t4 == 0) {
            s_inv[r0] = lt0 > 0.f ? 1.f / lt0 : 0.f;
            s_inv[r0 + 8] = lt1 > 0.f ? 1.f / lt1 : 0.f;
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(p_full);
        named_bar_sync(decode::kSoftmaxBar, 128);  // P and the zeroed V rows are complete
      } else {
        mbar_wait_nocall(p_full, n & 1);
        a0 = s_alpha[r0];
        a1 = s_alpha[r0 + 8];
      }
      // ---- O_half = alpha O_half + P . V_half ----
#pragma unroll
      for (int i = 0; i < 128; i++) o[i] *= (i & 2) ? a1 : a0;
      {
        const uint64_t vd = vdesc0 + static_cast<uint64_t>(st * (kTileBytes >> 4));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) {
          WgmmaBF16<256, 0, 1>::ss(o, pdesc + ((k * 32) >> 4), vd + ((k * 2048) >> 4), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<128>(o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      if (wg == 1) {
        if (pg == pe - 1) {
          inv0 = s_inv[r0];  // read before p_free lets warpgroup 0 overwrite it
          inv1 = s_inv[r0 + 8];
        }
        mbar_arrive(p_free);
      }
    }

    // ---- segment epilogue ----
    if (sg.save) {  // first part of a split task: keep the state for the walk's last segment
#pragma unroll
      for (int i = 0; i < 128; i += 4) {
        *reinterpret_cast<float4*>(carry + (i / 4) * 1024 + tid * 4) =
            make_float4(o[i], o[i + 1], o[i + 2], o[i + 3]);
      }
      if (wg == 0) {
        *reinterpret_cast<float4*>(carry + 256 * 128 + wtid * 4) = make_float4(m0, m1, l0, l1);
      }
      continue;
    }
    if (wg == 0) {
      float lt0 = l0 + __shfl_xor_sync(0xffffffffu, l0, 1);
      lt0 += __shfl_xor_sync(0xffffffffu, lt0, 2);
      float lt1 = l1 + __shfl_xor_sync(0xffffffffu, l1, 1);
      lt1 += __shfl_xor_sync(0xffffffffu, lt1, 2);
      inv0 = lt0 > 0.f ? 1.f / lt0 : 0.f;
      inv1 = lt1 > 0.f ? 1.f / lt1 : 0.f;
      l0 = lt0;
      l1 = lt1;
    }
    const int rows = p.num_head_q * p.num_seq_q;
    const int ri0 = tile * kRows + r0;
    const int ri1 = ri0 + 8;
    const int col0 = wg * 256 + 2 * t4;
    const bool single = __ldg(chunk_table + tile * p.num_batch + t.ibatch) == 1;
    if (single) {
      const int hm = p.num_head_q - 1;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int ri = h ? ri1 : ri0;
        if (ri >= rows) continue;
        const float inv = h ? inv1 : inv0;
        __nv_bfloat16* dst = p.y +
                             (static_cast<long long>(t.ibatch) * p.num_seq_q + (ri >> p.head_log2)) *
                                 p.ld_y +
                             (ri & hm) * kDv + col0;
#pragma unroll
        for (int jj = 0; jj < 32; jj++) {
          *reinterpret_cast<uint32_t*>(dst + 8 * jj) =
              pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        }
      }
    } else {
      const int base = static_cast<int>(blockIdx.x) - t.ichunk;
      const long long slot = chunk_slot(base, t.ichunk);
      if (t.ichunk == 0 && tid == 0) p.chunk_base[t.ibatch * p.num_tiles + tile] = base;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r = r0 + 8 * h;
        const float inv = h ? inv1 : inv0;
        float* dst = p.partial + (slot * kRows + r) * kDv + col0;
#pragma unroll
        for (int jj = 0; jj < 32; jj++) {
          *reinterpret_cast<float2*>(dst + 8 * jj) =
              make_float2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        }
        if (wg == 0 && t4 == 0) {
          const float m = h ? m1 : m0;
          const float l = h ? l1 : l0;
          p.lse[slot * kRows + r] = (m == -INFINITY || l <= 0.f) ? -INFINITY : m + log2_approx(l);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// split-k combine over 512-wide rows: y = sum_c 2^(lse_c - m) O_c / sum_c 2^(lse_c - m) -> bf16.
// Block (pair, g) merges rows 8g..8g+7 of the pair's query tile; thread = 4 columns.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
    mla_combine_kernel(__nv_bfloat16* __restrict__ y, const float* __restrict__ partial,
                       const float* __restrict__ lse, const int* __restrict__ chunk_base,
                       const int* __restrict__ task_map, int num_batch, int num_seq_q,
                       int num_head_q, int head_log2, int num_tiles, int ldY) {
  const int pair = blockIdx.x;  // b * T + tile
  const int b = pair / num_tiles;
  const int tile = pair - b * num_tiles;

  pdl_wait();
  pdl_launch_dependents();

  const int* chunk_table = task_map + kTaskStride * (task_map[0] * task_map[1] + 1);
  const int nch = chunk_table[tile * num_batch + b];
  if (nch <= 1) return;  // written by the attention kernel itself
  const int base = chunk_base[pair];
  const int rows = num_head_q * num_seq_q;
  for (int r = blockIdx.y * 8; r < blockIdx.y * 8 + 8; r++) {
    const int ri = tile * kRows + r;
    if (ri >= rows) break;
    float m = -INFINITY;
    for (int c = 0; c < nch; c++) m = fmaxf(m, __ldg(lse + chunk_slot(base, c) * kRows + r));
    float l = 0.f;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m != -INFINITY) {
      for (int c = 0; c < nch; c++) {
        const long long slot = chunk_slot(base, c);
        const float lc = __ldg(lse + slot * kRows + r);
        if (lc == -INFINITY) continue;
        const float w = exp2_approx(lc - m);
        const float4 v = ld_nc_f4(partial + (slot * kRows + r) * kDv + threadIdx.x * 4);
        acc.x += w * v.x;
        acc.y += w * v.y;
        acc.z += w * v.z;
        acc.w += w * v.w;
        l += w;
      }
    }
    const float inv = l > 0.f ? 1.f / l : 0.f;
    uint2 pk;
    pk.x = pack_bf16x2(acc.x * inv, acc.y * inv);
    pk.y = pack_bf16x2(acc.z * inv, acc.w * inv);
    __nv_bfloat16* dst = y + (static_cast<long long>(b) * num_seq_q + (ri >> head_log2)) * ldY +
                         (ri & (num_head_q - 1)) * kDv + threadIdx.x * 4;
    *reinterpret_cast<uint2*>(dst) = pk;
  }
}

}  // namespace decode_mla
}  // namespace b200

using namespace b200;  // NOLINT

extern "C" int hpc_attention_decode_mla_bf16_async(
    void* y_ptr, void* workspace_ptr, int* chunk_base_ptr, const int* task_map_ptr,
    const void* q_ptr, const void* kv_ptr, const int* block_ids_ptr, int num_batch,
    int num_seq_q, int num_head_q, int num_dim_qk, int num_kvcache_blocks, int block_size,
    int num_seq_max_blocks, int ldY, int ldQ, int64_t kv_block_stride, int64_t kv_token_stride,
    float softmax_scale, int num_total_ctas, cudaStream_t stream) {
  using namespace decode_mla;
  HPC_REQUIRE(task_map_ptr != nullptr && workspace_ptr != nullptr && chunk_base_ptr != nullptr &&
                  y_ptr != nullptr && q_ptr != nullptr && kv_ptr != nullptr &&
                  block_ids_ptr != nullptr,
              "attention_decode_mla_bf16: null pointer argument");
  HPC_REQUIRE(num_head_q == 8 || num_head_q == 16 || num_head_q == 32 || num_head_q == 64 ||
                  num_head_q == 128,
              "attention_decode_mla_bf16: num_head_q must be 8, 16, 32, 64 or 128, got %d",
              num_head_q);
  HPC_REQUIRE(num_seq_q >= 1 && num_seq_q <= 4,
              "attention_decode_mla_bf16: num_seq_q (mtp + 1) must be 1..4, got %d", num_seq_q);
  HPC_REQUIRE(num_dim_qk == kDqk, "attention_decode_mla_bf16: head dim must be 576, got %d",
              num_dim_qk);
  HPC_REQUIRE(block_size == kPage, "attention_decode_mla_bf16: page size must be 64, got %d",
              block_size);
  HPC_REQUIRE(num_batch >= 1 && num_batch <= 2048,
              "attention_decode_mla_bf16: batch must be 1..2048, got %d", num_batch);
  HPC_REQUIRE(num_total_ctas >= 1 && num_kvcache_blocks >= 1 && num_seq_max_blocks >= 1,
              "attention_decode_mla_bf16: bad geometry");
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(q_ptr) & 15) == 0 && (ldQ % 8) == 0,
              "attention_decode_mla_bf16: q and its row stride must be 16-byte aligned");
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(kv_ptr) & 15) == 0 && (kv_block_stride % 8) == 0 &&
                  (kv_token_stride % 8) == 0 && kv_token_stride >= kDqk,
              "attention_decode_mla_bf16: kv cache base and strides must be multiples of 16 bytes");
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(y_ptr) & 15) == 0 && (ldY % 8) == 0,
              "attention_decode_mla_bf16: output and its row stride must be 16-byte aligned");

  const int rows = num_head_q * num_seq_q;
  Params p{};
  p.task_map = task_map_ptr;
  p.block_ids = block_ids_ptr;
  p.y = static_cast<__nv_bfloat16*>(y_ptr);
  float* ws = static_cast<float*>(workspace_ptr);
  p.partial = ws;
  p.lse = ws + 2LL * num_total_ctas * kRows * kDv;
  p.carry = p.lse + 2LL * num_total_ctas * kRows;
  p.chunk_base = chunk_base_ptr;
  p.ld_y = ldY;
  p.num_batch = num_batch;
  p.num_seq_q = num_seq_q;
  p.num_head_q = num_head_q;
  p.head_log2 = __builtin_ctz(static_cast<unsigned>(num_head_q));
  p.num_tiles = (rows + kRows - 1) / kRows;
  p.num_seq_max_blocks = num_seq_max_blocks;
  p.rotate = p.num_tiles >= 2 ? 1 : 0;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;

  CUtensorMap tq, tkv;
  {
    const uint32_t hb = num_head_q < kRows ? num_head_q : kRows;
    uint64_t dims[3] = {kDqk, static_cast<uint64_t>(num_head_q),
                        static_cast<uint64_t>(num_batch) * num_seq_q};
    uint64_t strides[2] = {kDqk * 2, static_cast<uint64_t>(ldQ) * 2};
    uint32_t box[3] = {64, hb, kRows / hb};
    if (int rc = encode_tmap(&tq, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, q_ptr, 3, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B)) {
      return rc;
    }
  }
  {
    uint64_t dims[3] = {kDqk, kPage, static_cast<uint64_t>(num_kvcache_blocks)};
    uint64_t strides[2] = {static_cast<uint64_t>(kv_token_stride) * 2,
                           static_cast<uint64_t>(kv_block_stride) * 2};
    uint32_t box[3] = {64, kPage, 1};
    if (int rc = encode_tmap(&tkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, kv_ptr, 3, dims, strides,
                             box, CU_TENSOR_MAP_SWIZZLE_128B)) {
      return rc;
    }
  }
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(decode_attn_mla_kernel),
                                      kSmemBytes));
  HPC_CUDA_CHECK(launch_pdl(decode_attn_mla_kernel, dim3(num_total_ctas), dim3(kThreads),
                            kSmemBytes, stream, 1, tq, tkv, p));
  HPC_CUDA_CHECK(launch_pdl(mla_combine_kernel, dim3(num_batch * p.num_tiles, kRows / 8),
                            dim3(128), 0, stream, 1, p.y, p.partial, p.lse, p.chunk_base,
                            p.task_map, num_batch, num_seq_q, num_head_q, p.head_log2,
                            p.num_tiles, ldY));
  return HPC_OK;
}
