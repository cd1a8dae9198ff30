// BF16 causal prefill attention (H100 / sm_90a): varlen self-attention on contiguous q/k/v, and
// prefill (including chunked prefill) over a paged bf16 KV cache.
//
// Replaces reference src/attention/prefill/prefill.cc:20-71 (attention_prefill_bf16_async and
// attention_with_kvcache_prefill_bf16_async, each a multi-stage / warp-specialised kernel pair
// chosen by problem size) with one kernel template and one launch path; the two ops differ only in
// how the producer addresses K and V.
//
// Work item = (batch, q head, 128-row Q tile), handed out heaviest-first (largest Q tile index
// first) by the self-re-arming counter pair of scheduler_counter (prefill_common.cuh decode_work).
// An item visits the 128-key tiles inside its causal extent, nothing else.
//
// CTA = 288 threads, one CTA per SM:
//   warp 8     : TMA producer. Q tile, then K tiles into a 2-slot ring and V tiles into another.
//                A tile is two [128 rows x 64 dims] halves with 128-byte swizzled rows.
//                Paged: a page of 16 / 32 / 64 tokens lands as a [page x 64] box per half at row
//                offset page_index * page (as in decode_attn_bf16.cu). Dense: one [128 x 64] box
//                per half from a (d, head, token) descriptor; rows past total_seq are zero-filled.
//   warps 0-7  : two warpgroups, warpgroup w owns query rows [64w, 64w+64) of the tile.
//                S[64 q, 128 keys] = Q . K^T with m64n128k16 wgmma (both operands K-major in smem);
//                causal / length mask and base-2 online softmax on the fragment (a row's 128
//                scores are spread over the 4 threads of a quad); P -> bf16 in registers, which
//                are the A operand of O[64 q, 128 d] += P . V (wgmma "rs"; V is the MN-major B
//                operand as TMA stored it). O stays in fp32 registers across the item's tiles.
#include "common.cuh"
#include "host_utils.h"
#include "prefill_common.cuh"

namespace b200 {
namespace prefill_bf16 {

using prefill::decode_work;
using prefill::kD;
using prefill::kTile;
using prefill::Params;
using prefill::Work;

constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kGroupBar0 = 1;                // named barriers 1, 2: one per consumer warpgroup
constexpr int kHalfBytes = kTile * 128;      // [128 rows x 64 bf16]: 16 KB
constexpr int kTileBytes = 2 * kHalfBytes;   // a Q, K or V tile: 32 KB
constexpr int kStages = 2;

struct Smem {
  static constexpr int kOffK = 0;                             // kStages x 32 KB
  static constexpr int kOffV = kOffK + kStages * kTileBytes;  // kStages x 32 KB
  static constexpr int kOffQ = kOffV + kStages * kTileBytes;  // 32 KB
  static constexpr int kOffBar = kOffQ + kTileBytes;
  static constexpr int kNumBars = 4 * kStages + 2;
  static constexpr int kOffWork = kOffBar + kNumBars * 8;
  static constexpr int kTotal = kOffWork + 16;
  static_assert(kTotal <= 227 * 1024, "bf16 prefill smem exceeds the sm_90 per-block limit");
};

// Protocol (mbarriers; "phase" = use-count parity), n = running KV-tile counter of the CTA:
//   q_full      producer: item published (work id in smem, Q tile landed)
//   q_empty     the 8 consumer warps finished the item's last QK (Q tile and work slot reusable)
//   k_full/k_empty[slot]   K ring; a warp releases the slot once its QK(n) wgmma has completed
//   v_full/v_empty[slot]   V ring; released once the warp's PV(n) wgmma has completed
// The V slot of the tile that holds a request's last key has its rows past that key zeroed by each
// warpgroup before its PV (both write the same zeros): P is 0 there, but whatever the cache or the
// next request holds in those rows (NaN included) must not reach O through 0 * v.
template <bool kPaged>
__global__ void __launch_bounds__(kThreads, 1)
    prefill_bf16_kernel(const __grid_constant__ CUtensorMap tmap_q,
                        const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const Params p,
                        const int page_log2) {
  using L = Smem;
  using MMA = WgmmaBF16<128, 0, 0>;   // S = Q . K^T
  using MMA_PV = WgmmaBF16<128, 0, 1>;  // O += P . V, V MN-major
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* k_smem = smem + L::kOffK;
  uint8_t* v_smem = smem + L::kOffV;
  uint8_t* q_smem = smem + L::kOffQ;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  int* s_work = reinterpret_cast<int*>(smem + L::kOffWork);

  uint64_t* k_full = bars;
  uint64_t* k_empty = bars + kStages;
  uint64_t* v_full = bars + 2 * kStages;
  uint64_t* v_empty = bars + 3 * kStages;
  uint64_t* q_full = bars + 4 * kStages;
  uint64_t* q_empty = q_full + 1;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_k);
    prefetch_tensormap(&tmap_v);
    for (int i = 0; i < kStages; i++) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], kConsumerWarps);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], kConsumerWarps);
    }
    mbar_init(q_full, 1);
    mbar_init(q_empty, kConsumerWarps);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // =========================== producer ==============================================
    const uint64_t pol_kv = make_policy_evict_last();  // K/V of a request is re-read by its q heads
    const int page = 1 << page_log2;
    const int ppt = kTile >> page_log2;                // pages per 128-key tile: 8, 4 or 2
    const uint32_t page_bytes = static_cast<uint32_t>(page) * 128u;
    uint32_t n = 0;     // kv tile counter (rings)
    uint32_t item = 0;  // item counter
    while (true) {
      int w = 0;
      if (lane == 0) w = atomicAdd(p.work_counter, 1);
      w = __shfl_sync(0xffffffffu, w, 0);
      Work k;
      const bool alive = decode_work(p, w, k);
      if (alive && k.rows == 0) continue;  // Q tile beyond this request
      mbar_wait_nocall(q_empty, (item & 1) ^ 1);
      // warp-uniform copies of what the elected lane's TMA instructions take as operands
      const int u_hq = __shfl_sync(0xffffffffu, k.hq, 0);
      const int u_q0 = __shfl_sync(0xffffffffu, k.q0, 0);
      const int u_ntile = __shfl_sync(0xffffffffu, k.num_tile_kv, 0);
      if (elect_one()) {
        s_work[0] = alive ? w : -1;
        if (alive) {
          mbar_arrive_expect_tx(q_full, kTileBytes);
          tma_load_3d(q_smem, &tmap_q, q_full, 0, u_hq, u_q0);
          tma_load_3d(q_smem + kHalfBytes, &tmap_q, q_full, 64, u_hq, u_q0);
        } else {
          mbar_arrive(q_full);
        }
      }
      __syncwarp();
      item++;
      if (!alive) {
        // the last CTA out re-arms the work counter for the next launch (see host_utils.h
        // scheduler_counter)
        if (lane == 0) {
          __threadfence();
          if (atomicAdd(p.work_counter + 1, 1) == static_cast<int>(gridDim.x) - 1) {
            p.work_counter[0] = 0;
            p.work_counter[1] = 0;
            __threadfence();
          }
        }
        break;
      }
      const int hkv = u_hq / p.group;
      const int kc1 = p.k_head_first ? hkv : 0, kc2 = p.k_head_first ? 0 : hkv;
      const int vc1 = p.v_head_first ? hkv : 0, vc2 = p.v_head_first ? 0 : hkv;
      if constexpr (kPaged) {
        const int nblk = (k.seq_kv + page - 1) >> page_log2;
        const int* ids = p.block_ids + static_cast<long long>(k.b) * p.max_blocks;
        const int tiles_per_group = 32 / ppt;  // page ids fetched 32 at a time, one per lane
        for (int g0 = 0; g0 < u_ntile; g0 += tiles_per_group) {
          int bi = g0 * ppt + lane;
          bi = bi < nblk ? bi : nblk - 1;  // pages past the last one re-read it (keys masked)
          const int my_id = __ldg(ids + bi);
          const int gt = (u_ntile - g0) < tiles_per_group ? (u_ntile - g0) : tiles_per_group;
          for (int tt = 0; tt < gt; tt++) {
            const uint32_t st = n % kStages;
            const uint32_t ph = ((n / kStages) & 1) ^ 1;
            mbar_wait_nocall(&k_empty[st], ph);  // QK(n - kStages) finished
            if (elect_one()) mbar_arrive_expect_tx(&k_full[st], kTileBytes);
            __syncwarp();
            for (int j = 0; j < ppt; j++) {
              const int id = __shfl_sync(0xffffffffu, my_id, tt * ppt + j);
              if (elect_one()) {
                uint8_t* d = k_smem + st * kTileBytes + j * page_bytes;
                tma_load_4d_hint(d, &tmap_k, &k_full[st], 0, kc1, kc2, id, pol_kv);
                tma_load_4d_hint(d + kHalfBytes, &tmap_k, &k_full[st], 64, kc1, kc2, id, pol_kv);
              }
              __syncwarp();
            }
            mbar_wait_nocall(&v_empty[st], ph);  // PV(n - kStages) finished
            if (elect_one()) mbar_arrive_expect_tx(&v_full[st], kTileBytes);
            __syncwarp();
            for (int j = 0; j < ppt; j++) {
              const int id = __shfl_sync(0xffffffffu, my_id, tt * ppt + j);
              if (elect_one()) {
                uint8_t* d = v_smem + st * kTileBytes + j * page_bytes;
                tma_load_4d_hint(d, &tmap_v, &v_full[st], 0, vc1, vc2, id, pol_kv);
                tma_load_4d_hint(d + kHalfBytes, &tmap_v, &v_full[st], 64, vc1, vc2, id, pol_kv);
              }
              __syncwarp();
            }
            n++;
          }
        }
      } else {
        const int u_s0 = __shfl_sync(0xffffffffu, k.q0 - k.mq * kTile, 0);  // request's first row
        for (int j = 0; j < u_ntile; j++) {
          const int row = u_s0 + j * kTile;
          const uint32_t st = n % kStages;
          const uint32_t ph = ((n / kStages) & 1) ^ 1;
          mbar_wait_nocall(&k_empty[st], ph);
          if (elect_one()) {
            uint8_t* d = k_smem + st * kTileBytes;
            mbar_arrive_expect_tx(&k_full[st], kTileBytes);
            tma_load_3d_hint(d, &tmap_k, &k_full[st], 0, hkv, row, pol_kv);
            tma_load_3d_hint(d + kHalfBytes, &tmap_k, &k_full[st], 64, hkv, row, pol_kv);
          }
          __syncwarp();
          mbar_wait_nocall(&v_empty[st], ph);
          if (elect_one()) {
            uint8_t* d = v_smem + st * kTileBytes;
            mbar_arrive_expect_tx(&v_full[st], kTileBytes);
            tma_load_3d_hint(d, &tmap_v, &v_full[st], 0, hkv, row, pol_kv);
            tma_load_3d_hint(d + kHalfBytes, &tmap_v, &v_full[st], 64, hkv, row, pol_kv);
          }
          __syncwarp();
          n++;
        }
      }
    }
  } else {
    // =========================== consumer warpgroups =======================================
    const int wg = warp >> 2;
    const int wtid = tid & 127;
    const int g8 = lane >> 2;
    const int t4 = lane & 3;
    // fragment rows of this thread (query rows of the tile): registers with (i / 2) odd -> r[1]
    const int r[2] = {wg * 64 + (warp & 3) * 16 + g8, wg * 64 + (warp & 3) * 16 + g8 + 8};
    const float c = p.softmax_scale_log2;
    //  Q rows, K tile : K-major, 128B swizzle, 8-row groups 1024 B apart; one k16 step consumes
    //                   32 B of a row; dims 64..127 are the second half (+16 KB)
    //  V tile         : MN-major B (d contiguous as stored): the two 64-dim halves are 16 KB apart
    //                   (LBO), 8-key groups 1024 B apart (SBO); one k16 step consumes 2048 B
    const uint64_t qdesc = make_smem_desc(smem_u32(q_smem) + wg * 8192, 16, 1024, kLayoutSW128);
    const uint64_t kdesc0 = make_smem_desc(smem_u32(k_smem), 16, 1024, kLayoutSW128);
    const uint64_t vdesc0 = make_smem_desc(smem_u32(v_smem), kHalfBytes, 1024, kLayoutSW128);

    uint32_t n = 0;
    uint32_t item = 0;
    while (true) {
      mbar_wait_nocall(q_full, item & 1);
      const int w = s_work[0];
      if (w < 0) break;
      Work k;
      decode_work(p, w, k);
      const int ntile = k.num_tile_kv;
      bool row_ok[2];
      int row_lim[2];
      float mrun[2], lrun[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        row_ok[h] = r[h] < k.rows;
        // kv positions visible to this row: pos <= row_lim and pos < seq_kv
        row_lim[h] = k.seq_kv - k.seq_q + k.mq * kTile + r[h];
        mrun[h] = -INFINITY;  // running maximum of the row, log2 units
        lrun[h] = 0.f;        // this thread's share of the row sum (its 32 columns)
      }
      const int tile_lim_min = k.seq_kv - k.seq_q + k.mq * kTile;  // row 0
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; i++) o[i] = 0.f;
      if (ntile == 0) {  // no visible key: Q is not read
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty);
      }

      for (int j = 0; j < ntile; j++) {
        const uint32_t st = n % kStages;
        const uint32_t ph = (n / kStages) & 1;
        // ---- S = Q . K^T for this warpgroup's 64 rows ----
        mbar_wait_nocall(&k_full[st], ph);
        float sv[64];  // overwritten: the first wgmma does not read D
        wgmma_fence();
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
#pragma unroll
          for (int kk = 0; kk < 4; kk++) {
            MMA::ss(sv, qdesc + h2 * (kHalfBytes >> 4) + kk * 2,
                    kdesc0 + static_cast<uint64_t>(st * (kTileBytes >> 4)) + h2 * (kHalfBytes >> 4) +
                        kk * 2,
                    (h2 | kk) > 0);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(sv);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&k_empty[st]);
          if (j == ntile - 1) mbar_arrive(q_empty);  // the item's last QK: Q tile reusable
        }

        // ---- mask, row maxima ----
        const int key0 = j * kTile;
        const bool need_mask = (key0 + kTile - 1 > tile_lim_min) || (key0 + kTile > k.seq_kv);
        float vmax[2] = {-INFINITY, -INFINITY};
        if (need_mask) {
#pragma unroll
          for (int i = 0; i < 64; i++) {
            const int h = (i >> 1) & 1;
            const int pos = key0 + 8 * (i >> 2) + 2 * t4 + (i & 1);
            sv[i] = (pos > row_lim[h] || pos >= k.seq_kv) ? -INFINITY : sv[i];
            vmax[h] = fmaxf(vmax[h], sv[i]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 64; i++) vmax[(i >> 1) & 1] = fmaxf(vmax[(i >> 1) & 1], sv[i]);
        }
        float alpha[2], bias[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          vmax[h] = fmaxf(vmax[h], __shfl_xor_sync(0xffffffffu, vmax[h], 1));
          vmax[h] = fmaxf(vmax[h], __shfl_xor_sync(0xffffffffu, vmax[h], 2));
          const float mnew = fmaxf(mrun[h], vmax[h] * c);
          const bool dead = (mnew == -INFINITY);  // no visible key in this row so far
          alpha[h] = dead ? 1.f : exp2_approx(mrun[h] - mnew);
          bias[h] = dead ? 0.f : -mnew;
          mrun[h] = mnew;
        }
        if (__any_sync(0xffffffffu, alpha[0] != 1.f || alpha[1] != 1.f)) {
#pragma unroll
          for (int i = 0; i < 64; i++) o[i] *= alpha[(i >> 1) & 1];
        }
        // ---- P = 2^(s c - m) -> bf16 pairs: the A fragment of the PV wgmma ----
        uint32_t pa[32];
        float psum[2] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 32; q++) {  // registers 2q, 2q + 1: one row, adjacent columns
          const int h = q & 1;
          const float e0 = exp2_approx(__fmaf_rn(sv[2 * q], c, bias[h]));
          const float e1 = exp2_approx(__fmaf_rn(sv[2 * q + 1], c, bias[h]));
          psum[h] += e0 + e1;
          pa[q] = pack_bf16x2(e0, e1);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) lrun[h] = lrun[h] * alpha[h] + psum[h];

        // ---- O += P . V ----
        mbar_wait_nocall(&v_full[st], ph);
        if (key0 + kTile > k.seq_kv) {
          // rows of keys >= seq_kv -> 0 (see the protocol comment)
          uint8_t* vs = v_smem + st * kTileBytes;
          const int r0 = k.seq_kv - key0;
          for (int e = r0 * 16 + wtid; e < kTile * 16; e += 128) {
            const int row = e >> 4, part = e & 15;
            *reinterpret_cast<uint4*>(vs + (part >> 3) * kHalfBytes + row * 128 + (part & 7) * 16) =
                make_uint4(0, 0, 0, 0);
          }
          fence_proxy_async_smem();
          named_bar_sync(kGroupBar0 + wg, 128);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; kk++) {
          MMA_PV::rs(o, pa + 4 * kk,
                     vdesc0 + static_cast<uint64_t>(st * (kTileBytes >> 4)) + kk * (2048 >> 4), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);
        n++;
      }

      // ---- epilogue: O / row sum -> bf16 rows ----
      float inv[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float l = lrun[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[h] = 1.f / l;  // a row that sees no key has sum 0 -> NaN
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (!row_ok[h]) continue;
        __nv_bfloat16* dst = p.out + static_cast<long long>(k.q0 + r[h]) * p.ld_out + k.hq * kD;
#pragma unroll
        for (int jj = 0; jj < 16; jj++) {
          const int col = 8 * jj + 2 * t4;
          *reinterpret_cast<uint32_t*>(dst + col) =
              pack_bf16x2(o[4 * jj + 2 * h] * inv[h], o[4 * jj + 2 * h + 1] * inv[h]);
        }
      }
      item++;
    }
  }
}

}  // namespace prefill_bf16
}  // namespace b200

using namespace b200;  // NOLINT

// Common launcher of the two ops. Strides in elements; k_* / v_* are (blk, tok, head) for the
// paged op and (-, tok, -) for the dense one, whose heads are 128 elements apart.
static int prefill_bf16_launch(const char* who, bool paged, void* y_ptr, const void* q_ptr,
                               const void* k_ptr, const void* v_ptr, const int* cu_seqlens_q_ptr,
                               const int* seqlens_kv_ptr, const int* block_ids_ptr, int num_batch,
                               int total_seq_q, int max_seq_q, int num_dim_qk, int num_dim_v,
                               int num_head_q, int num_head_kv, int num_kvcache_blocks,
                               int block_size, int max_blocks, int ldY, int ldQ, int64_t k_blk,
                               int64_t k_tok, int64_t k_head, int64_t v_blk, int64_t v_tok,
                               int64_t v_head, cudaStream_t stream) {
  HPC_REQUIRE(num_dim_qk == 128 && num_dim_v == 128,
              "%s: head dim must be 128 for qk and v (got %d and %d)", who, num_dim_qk, num_dim_v);
  HPC_REQUIRE(num_head_q > 0 && num_head_kv > 0 && num_head_q % num_head_kv == 0,
              "%s: num_head_q (%d) must be a positive multiple of num_head_kv (%d)", who, num_head_q,
              num_head_kv);
  HPC_REQUIRE(num_batch > 0 && total_seq_q >= 0 && max_seq_q >= 0,
              "%s: bad num_batch / total_seq_q / max_seqlens_q (%d, %d, %d)", who, num_batch,
              total_seq_q, max_seq_q);
  if (paged) {
    HPC_REQUIRE(block_size == 16 || block_size == 32 || block_size == 64,
                "%s: kvcache paged blocksize must be 16, 32 or 64 (got %d)", who, block_size);
    HPC_REQUIRE(num_kvcache_blocks > 0 && max_blocks > 0, "%s: empty kv cache or block table", who);
  }
  const auto al16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  HPC_REQUIRE(al16(q_ptr) && al16(k_ptr) && al16(v_ptr) && al16(y_ptr),
              "%s: q, k, v and output must be 16-byte aligned", who);
  HPC_REQUIRE(ldQ % 8 == 0 && ldY % 2 == 0 && k_blk % 8 == 0 && k_tok % 8 == 0 &&
                  k_head % 8 == 0 && v_blk % 8 == 0 && v_tok % 8 == 0 && v_head % 8 == 0,
              "%s: token, head and block strides must be multiples of 16 bytes", who);
  if (total_seq_q == 0 || max_seq_q == 0) return HPC_OK;

  const CUtensorMapDataType bf16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  // (d, head, token) rows of 64 dims: a [128 tokens x 64] box per half-tile
  const auto rows_tmap = [&](CUtensorMap* t, const void* base, int heads, int64_t tok) {
    uint64_t dims[3] = {128, static_cast<uint64_t>(heads), static_cast<uint64_t>(total_seq_q)};
    uint64_t strides[2] = {256, static_cast<uint64_t>(tok) * 2};
    uint32_t box[3] = {64, 1, static_cast<uint32_t>(prefill::kTile)};
    return encode_tmap(t, bf16, 2, base, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  };
  CUtensorMap tq, tk, tv;
  int khf = 1, vhf = 1;
  if (int rc = rows_tmap(&tq, q_ptr, num_head_q, ldQ)) return rc;
  if (paged) {
    if (int rc = encode_paged_kv_tmap(&tk, bf16, 2, k_ptr, num_head_kv, block_size,
                                      num_kvcache_blocks, k_blk, k_tok, k_head, &khf)) {
      return rc;
    }
    if (int rc = encode_paged_kv_tmap(&tv, bf16, 2, v_ptr, num_head_kv, block_size,
                                      num_kvcache_blocks, v_blk, v_tok, v_head, &vhf)) {
      return rc;
    }
  } else {
    if (int rc = rows_tmap(&tk, k_ptr, num_head_kv, k_tok)) return rc;
    if (int rc = rows_tmap(&tv, v_ptr, num_head_kv, v_tok)) return rc;
  }

  int* counter = scheduler_counter(stream);  // work-item counter {next item, CTAs done}, self-resetting
  if (counter == nullptr) return HPC_ERR_CUDA;

  prefill::Params p = {};
  p.cu_seqlens_q = cu_seqlens_q_ptr;
  p.seqlens_kv = seqlens_kv_ptr;
  p.block_ids = block_ids_ptr;
  p.out = static_cast<__nv_bfloat16*>(y_ptr);
  p.work_counter = counter;
  p.num_batch = num_batch;
  p.num_head_q = num_head_q;
  p.num_head_kv = num_head_kv;
  p.group = num_head_q / num_head_kv;
  p.max_q_tiles = (max_seq_q + prefill::kTile - 1) / prefill::kTile;
  p.max_blocks = max_blocks;
  p.ld_out = ldY;
  p.k_head_first = khf;
  p.v_head_first = vhf;
  p.softmax_scale_log2 = 1.4426950408889634f / sqrtf(128.f);
  const int page_log2 = block_size == 16 ? 4 : block_size == 32 ? 5 : 6;

  const int grid = sm_count();  // one resident CTA per SM
  const auto kern =
      paged ? prefill_bf16::prefill_bf16_kernel<true> : prefill_bf16::prefill_bf16_kernel<false>;
  constexpr int smem_bytes = prefill_bf16::Smem::kTotal;
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(kern), smem_bytes));
  kern<<<grid, prefill_bf16::kThreads, smem_bytes, stream>>>(tq, tk, tv, p, page_log2);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

// replaces reference src/attention/prefill/prefill.h:12-17 (attention_prefill_bf16_async)
extern "C" int hpc_attention_prefill_bf16_async(
    void* y_ptr, const void* q_ptr, const void* k_ptr, const void* v_ptr, const int* seqlens_q_ptr,
    const int* cu_seqlens_q_ptr, int num_batch, int total_seq_q, int max_seq_q, int num_dim_qk,
    int num_dim_v, int num_head_q, int num_head_kv, int ldY, int ldQ, int ldK, int ldV,
    cudaStream_t stream) {
  // request b attends to itself: its kv length is its q length and its k/v rows are its q rows
  return prefill_bf16_launch("attention_prefill_bf16", false, y_ptr, q_ptr, k_ptr, v_ptr,
                             cu_seqlens_q_ptr, seqlens_q_ptr, nullptr, num_batch, total_seq_q,
                             max_seq_q, num_dim_qk, num_dim_v, num_head_q, num_head_kv, 0, 64, 0,
                             ldY, ldQ, 0, ldK, 128, 0, ldV, 128, stream);
}

// replaces reference src/attention/prefill/prefill.h:19-25 (attention_with_kvcache_prefill_bf16_async)
extern "C" int hpc_attention_with_kvcache_prefill_bf16_async(
    void* y_ptr, const void* q_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const int* cu_seqlens_q_ptr, const int* block_ids_ptr, const int* seqlens_kvcache_ptr,
    int num_batch, int total_seq_q, int max_seq_q, int num_dim_qk, int num_dim_v, int num_head_q,
    int num_head_kv, int num_kvcache_blocks, int block_size, int num_seq_max_blocks, int ldY,
    int ldQ, int64_t ldK, int64_t ldK1, int64_t ldK2, int64_t ldV, int64_t ldV1, int64_t ldV2,
    cudaStream_t stream) {
  return prefill_bf16_launch("attention_with_kvcache_prefill_bf16", true, y_ptr, q_ptr, kcache_ptr,
                             vcache_ptr, cu_seqlens_q_ptr, seqlens_kvcache_ptr, block_ids_ptr,
                             num_batch, total_seq_q, max_seq_q, num_dim_qk, num_dim_v, num_head_q,
                             num_head_kv, num_kvcache_blocks, block_size, num_seq_max_blocks, ldY,
                             ldQ, ldK, ldK1, ldK2, ldV, ldV1, ldV2, stream);
}
