// MLA prefill attention (H100 / sm_90a): varlen causal attention in the un-absorbed form
// DeepSeek-V2/V3-style models run at prefill. Per head, the 192-wide query is [q_nope (128) |
// q_pe (64)], the 192-wide key is [k_nope (128, per head) | k_pe (64, one row shared by all heads)]
// and the value is 128 wide. Keys are dense, request b's at rows cu_seqlens_kv[b] .., and the mask
// is bottom-right causal: query i of a request with nq queries and nk keys sees keys
// j <= nk - nq + i.
//
// The structure is that of prefill_bf16.cu (one persistent CTA per SM, work item = (request, head,
// 128-row Q tile), heaviest first through prefill_common.cuh decode_work and a scheduler_counter
// pair). What differs in every role:
//   warp 8     : TMA producer. Q tile = three [128 rows x 64 dims] 128B-swizzled boxes (48 KB);
//                K tile = two boxes of k_nope from a (d, head, token) descriptor and one of k_pe
//                from a (d, token) descriptor (48 KB, 2-slot ring); V tile = two boxes (32 KB,
//                2-slot ring). k_pe is re-read by every head's items, so it is loaded evict_last,
//                as K and V are. Rows past the last key token are zero-filled by TMA.
//   warps 0-7  : S[64 q, 128 keys] = Q . K^T as one chain of 12 m64n128k16 steps over the 192
//                dims; mask, base-2 online softmax, P -> bf16 in registers as the A operand of
//                O[64 q, 128 d] += P . V (wgmma "rs", V MN-major as stored). A row that sees no
//                key writes zeros.
#include <cmath>

#include "common.cuh"
#include "host_utils.h"
#include "prefill_common.cuh"

namespace b200 {
namespace prefill_mla {

using prefill::decode_work;
using prefill::kTile;
using prefill::Params;
using prefill::Work;

constexpr int kDv = 128;
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kGroupBar0 = 1;                 // named barriers 1, 2: one per consumer warpgroup
constexpr int kBoxBytes = kTile * 128;        // [128 rows x 64 bf16]: 16 KB
constexpr int kQKBytes = 3 * kBoxBytes;       // a Q or K tile, 192 dims: 48 KB
constexpr int kVBytes = 2 * kBoxBytes;        // a V tile, 128 dims: 32 KB
constexpr int kStages = 2;

struct Smem {
  static constexpr int kOffK = 0;                          // kStages x 48 KB
  static constexpr int kOffV = kOffK + kStages * kQKBytes;  // kStages x 32 KB
  static constexpr int kOffQ = kOffV + kStages * kVBytes;   // 48 KB
  static constexpr int kOffBar = kOffQ + kQKBytes;
  static constexpr int kNumBars = 4 * kStages + 2;
  static constexpr int kOffWork = kOffBar + kNumBars * 8;
  static constexpr int kTotal = kOffWork + 4 * (1 + kConsumerWarps);
  static_assert(kTotal <= 232448, "MLA prefill smem exceeds the sm_90 per-block limit");
};

// Barrier protocol as in prefill_bf16.cu: q_full / q_empty per item, k_full / k_empty and
// v_full / v_empty per ring slot. The V slot of the tile holding a request's last key has its rows
// past that key zeroed before the PV: they belong to the next request (or are TMA's zero fill),
// P is 0 there, and 0 * NaN must not reach O.
__global__ void __launch_bounds__(kThreads, 1)
    prefill_mla_kernel(const __grid_constant__ CUtensorMap tmap_q,
                       const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_pe,
                       const __grid_constant__ CUtensorMap tmap_v, const Params p) {
  using L = Smem;
  using MMA = WgmmaBF16<128, 0, 0>;     // S = Q . K^T
  using MMA_PV = WgmmaBF16<128, 0, 1>;  // O += P . V, V MN-major
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* k_smem = smem + L::kOffK;
  uint8_t* v_smem = smem + L::kOffV;
  uint8_t* q_smem = smem + L::kOffQ;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  int* s_work = reinterpret_cast<int*>(smem + L::kOffWork);
  int* s_head = s_work + 1;  // one slot per consumer warp

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
    prefetch_tensormap(&tmap_pe);
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
    const uint64_t pol_kv = make_policy_evict_last();  // K/V re-read by the request's q tiles,
                                                        // k_pe by every head as well
    uint32_t n = 0;     // kv tile counter (rings)
    uint32_t item = 0;  // item counter
    while (true) {
      int w = 0;
      if (lane == 0) w = atomicAdd(p.work_counter, 1);
      w = __shfl_sync(0xffffffffu, w, 0);
      Work k;
      const bool alive = decode_work<true>(p, w, k);
      if (alive && k.rows == 0) continue;  // Q tile beyond this request
      mbar_wait_nocall(q_empty, (item & 1) ^ 1);
      const int u_h = __shfl_sync(0xffffffffu, k.hq, 0);
      const int u_q0 = __shfl_sync(0xffffffffu, k.q0, 0);
      const int u_ntile = __shfl_sync(0xffffffffu, k.num_tile_kv, 0);
      if (elect_one()) {
        s_work[0] = alive ? w : -1;
        if (alive) {
          mbar_arrive_expect_tx(q_full, kQKBytes);
          for (int c = 0; c < 3; c++) {
            tma_load_3d(q_smem + c * kBoxBytes, &tmap_q, q_full, 64 * c, u_h, u_q0);
          }
        } else {
          mbar_arrive(q_full);
        }
      }
      __syncwarp();
      item++;
      if (!alive) {
        // the last CTA out re-arms the work counter for the next launch (host_utils.h
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
      const int u_kv0 = __shfl_sync(0xffffffffu, p.seqlens_kv[k.b], 0);  // request's first key row
      const int kc1 = p.k_head_first ? u_h : 0, kc2 = p.k_head_first ? 0 : u_h;
      const int vc1 = p.v_head_first ? u_h : 0, vc2 = p.v_head_first ? 0 : u_h;
      for (int j = 0; j < u_ntile; j++) {
        const int row = u_kv0 + j * kTile;
        const int kr1 = p.k_head_first ? kc1 : row, kr2 = p.k_head_first ? row : kc2;
        const int vr1 = p.v_head_first ? vc1 : row, vr2 = p.v_head_first ? row : vc2;
        const uint32_t st = n % kStages;
        const uint32_t ph = ((n / kStages) & 1) ^ 1;
        mbar_wait_nocall(&k_empty[st], ph);  // QK(n - kStages) finished
        if (elect_one()) {
          uint8_t* d = k_smem + st * kQKBytes;
          mbar_arrive_expect_tx(&k_full[st], kQKBytes);
          tma_load_3d_hint(d, &tmap_k, &k_full[st], 0, kr1, kr2, pol_kv);
          tma_load_3d_hint(d + kBoxBytes, &tmap_k, &k_full[st], 64, kr1, kr2, pol_kv);
          tma_load_2d_hint(d + 2 * kBoxBytes, &tmap_pe, &k_full[st], 0, row, pol_kv);
        }
        __syncwarp();
        mbar_wait_nocall(&v_empty[st], ph);  // PV(n - kStages) finished
        if (elect_one()) {
          uint8_t* d = v_smem + st * kVBytes;
          mbar_arrive_expect_tx(&v_full[st], kVBytes);
          tma_load_3d_hint(d, &tmap_v, &v_full[st], 0, vr1, vr2, pol_kv);
          tma_load_3d_hint(d + kBoxBytes, &tmap_v, &v_full[st], 64, vr1, vr2, pol_kv);
        }
        __syncwarp();
        n++;
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
    //                   32 B of a row; dims 64c..64c+63 are box c (+16 KB each)
    //  V tile         : MN-major B: the two 64-dim halves are 16 KB apart (LBO), 8-key groups
    //                   1024 B apart (SBO); one k16 step consumes 2048 B
    const uint64_t qdesc = make_smem_desc(smem_u32(q_smem) + wg * 8192, 16, 1024, kLayoutSW128);
    const uint64_t kdesc0 = make_smem_desc(smem_u32(k_smem), 16, 1024, kLayoutSW128);
    const uint64_t vdesc0 = make_smem_desc(smem_u32(v_smem), kBoxBytes, 1024, kLayoutSW128);

    uint32_t n = 0;
    uint32_t item = 0;
    while (true) {
      mbar_wait_nocall(q_full, item & 1);
      const int w = s_work[0];
      if (w < 0) break;
      Work k;
      decode_work<true>(p, w, k);
      const int ntile = k.num_tile_kv;
      // the item's head waits in smem for the epilogue: the tile loop has no register to spare
      __syncwarp();  // every lane has read the previous item's
      if (lane == 0) s_head[warp] = k.hq;
      bool row_ok[2];
      float mrun[2], lrun[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        row_ok[h] = r[h] < k.rows;
        mrun[h] = -INFINITY;  // running maximum of the row, log2 units
        lrun[h] = 0.f;        // this thread's share of the row sum (its 32 columns)
      }
      // key positions visible to tile row r: pos <= tile_lim_min + r and pos < seq_kv
      const int tile_lim_min = k.seq_kv - k.seq_q + k.mq * kTile;
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
        // ---- S = Q . K^T for this warpgroup's 64 rows: 12 k16 steps over 192 dims ----
        mbar_wait_nocall(&k_full[st], ph);
        float sv[64];  // overwritten: the first wgmma does not read D
        wgmma_fence();
#pragma unroll
        for (int b3 = 0; b3 < 3; b3++) {
#pragma unroll
          for (int kk = 0; kk < 4; kk++) {
            MMA::ss(sv, qdesc + b3 * (kBoxBytes >> 4) + kk * 2,
                    kdesc0 + static_cast<uint64_t>(st * (kQKBytes >> 4)) + b3 * (kBoxBytes >> 4) +
                        kk * 2,
                    (b3 | kk) > 0);
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
            sv[i] = (pos > tile_lim_min + r[h] || pos >= k.seq_kv) ? -INFINITY : sv[i];
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
          uint8_t* vs = v_smem + st * kVBytes;
          const int r0 = k.seq_kv - key0;
          for (int e = r0 * 16 + wtid; e < kTile * 16; e += 128) {
            const int row = e >> 4, part = e & 15;
            *reinterpret_cast<uint4*>(vs + (part >> 3) * kBoxBytes + row * 128 + (part & 7) * 16) =
                make_uint4(0, 0, 0, 0);
          }
          fence_proxy_async_smem();
          named_bar_sync(kGroupBar0 + wg, 128);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; kk++) {
          MMA_PV::rs(o, pa + 4 * kk,
                     vdesc0 + static_cast<uint64_t>(st * (kVBytes >> 4)) + kk * (2048 >> 4), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);
        n++;
      }

      // ---- epilogue: O / row sum -> bf16 rows; a row that sees no key has sum 0 and writes 0 ----
      __syncwarp();
      const int head = s_head[warp];
      float inv[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float l = lrun[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[h] = l > 0.f ? 1.f / l : 0.f;
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (!row_ok[h]) continue;
        __nv_bfloat16* dst = p.out + static_cast<long long>(k.q0 + r[h]) * p.ld_out + head * kDv;
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

}  // namespace prefill_mla
}  // namespace b200

using namespace b200;  // NOLINT
using prefill::kTile;

extern "C" int hpc_attention_prefill_mla_bf16_async(
    void* y_ptr, const void* q_ptr, const void* k_nope_ptr, const void* k_pe_ptr,
    const void* v_ptr, const int* cu_seqlens_q_ptr, const int* cu_seqlens_kv_ptr, int num_batch,
    int total_seq_q, int total_seq_kv, int max_seq_q, int num_head, int num_dim_qk, int num_dim_v,
    int ldY, int ldQ, int64_t k_nope_token_stride, int64_t k_nope_head_stride,
    int64_t k_pe_token_stride, int64_t v_token_stride, int64_t v_head_stride, float softmax_scale,
    cudaStream_t stream) {
  const char* who = "attention_prefill_mla_bf16";
  HPC_REQUIRE(num_dim_qk == 192 && num_dim_v == 128,
              "%s: head dims must be 192 for q / k and 128 for v (got %d and %d)", who, num_dim_qk,
              num_dim_v);
  HPC_REQUIRE(num_head >= 1 && num_head <= 128, "%s: num heads must be 1..128 (got %d)", who,
              num_head);
  HPC_REQUIRE(num_batch > 0 && total_seq_q >= 0 && total_seq_kv > 0 && max_seq_q >= 0,
              "%s: bad num_batch / total_seq_q / total_seq_kv / max_seqlen_q (%d, %d, %d, %d)", who,
              num_batch, total_seq_q, total_seq_kv, max_seq_q);
  HPC_REQUIRE(std::isfinite(softmax_scale) && softmax_scale > 0.f,
              "%s: softmax_scale must be finite and positive", who);
  const int64_t max_q_tiles = (static_cast<int64_t>(max_seq_q) + kTile - 1) / kTile;
  HPC_REQUIRE(max_q_tiles * num_batch * num_head < (int64_t{1} << 31),
              "%s: too many work items (%lld q tiles x %d requests x %d heads)", who,
              static_cast<long long>(max_q_tiles), num_batch, num_head);
  const auto al16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  HPC_REQUIRE(al16(q_ptr) && al16(k_nope_ptr) && al16(k_pe_ptr) && al16(v_ptr) && al16(y_ptr),
              "%s: q, k_nope, k_pe, v and output must be 16-byte aligned", who);
  const auto st_ok = [](int64_t s) { return s > 0 && s % 8 == 0 && s < (int64_t{1} << 38); };
  HPC_REQUIRE(st_ok(ldQ) && ldQ >= num_head * 192 && st_ok(ldY) && ldY >= num_head * 128 &&
                  st_ok(k_nope_token_stride) && st_ok(k_nope_head_stride) &&
                  st_ok(k_pe_token_stride) && st_ok(v_token_stride) && st_ok(v_head_stride),
              "%s: token and head strides must be positive multiples of 8 elements", who);
  if (total_seq_q == 0 || max_seq_q == 0) return HPC_OK;

  const CUtensorMapDataType bf16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  // (d, head, token) or, when heads are further apart than tokens, (d, token, head): TMA wants the
  // strides ascending. Either way a box is [128 tokens x 64 dims] of one head, the same smem image.
  const auto heads_tmap = [&](CUtensorMap* t, const void* base, int dim, int64_t tok,
                              int64_t head, int rows, int* head_first) {
    *head_first = head <= tok ? 1 : 0;
    const uint64_t h = static_cast<uint64_t>(num_head), r = static_cast<uint64_t>(rows);
    uint64_t dims[3] = {static_cast<uint64_t>(dim), *head_first ? h : r, *head_first ? r : h};
    uint64_t strides[2] = {static_cast<uint64_t>(*head_first ? head : tok) * 2,
                           static_cast<uint64_t>(*head_first ? tok : head) * 2};
    uint32_t box[3] = {64, *head_first ? 1u : static_cast<uint32_t>(kTile),
                       *head_first ? static_cast<uint32_t>(kTile) : 1u};
    return encode_tmap(t, bf16, 2, base, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  };
  CUtensorMap tq, tk, tpe, tv;
  int qhf = 1, khf = 1, vhf = 1;  // q: always head first (ldQ >= 192 H)
  if (int rc = heads_tmap(&tq, q_ptr, 192, ldQ, 192, total_seq_q, &qhf)) return rc;
  if (int rc = heads_tmap(&tk, k_nope_ptr, 128, k_nope_token_stride, k_nope_head_stride,
                          total_seq_kv, &khf)) {
    return rc;
  }
  if (int rc = heads_tmap(&tv, v_ptr, 128, v_token_stride, v_head_stride, total_seq_kv, &vhf)) {
    return rc;
  }
  {
    uint64_t dims[2] = {64, static_cast<uint64_t>(total_seq_kv)};
    uint64_t strides[1] = {static_cast<uint64_t>(k_pe_token_stride) * 2};
    uint32_t box[2] = {64, static_cast<uint32_t>(kTile)};
    if (int rc = encode_tmap(&tpe, bf16, 2, k_pe_ptr, 2, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)) {
      return rc;
    }
  }

  int* counter = scheduler_counter(stream);  // work-item counter {next item, CTAs done}, self-resetting
  if (counter == nullptr) return HPC_ERR_CUDA;

  prefill::Params p = {};
  p.cu_seqlens_q = cu_seqlens_q_ptr;
  p.seqlens_kv = cu_seqlens_kv_ptr;  // key offsets: decode_work<true>
  p.out = static_cast<__nv_bfloat16*>(y_ptr);
  p.work_counter = counter;
  p.num_batch = num_batch;
  p.num_head_q = num_head;
  p.num_head_kv = num_head;
  p.group = 1;
  p.max_q_tiles = static_cast<int>(max_q_tiles);
  p.ld_out = ldY;
  p.k_head_first = khf;
  p.v_head_first = vhf;
  p.softmax_scale_log2 = static_cast<float>(1.4426950408889634 * static_cast<double>(softmax_scale));

  const int grid = sm_count();  // one resident CTA per SM
  constexpr int smem_bytes = prefill_mla::Smem::kTotal;
  const auto kern = prefill_mla::prefill_mla_kernel;
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(kern), smem_bytes));
  kern<<<grid, prefill_mla::kThreads, smem_bytes, stream>>>(tq, tk, tpe, tv, p);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}
