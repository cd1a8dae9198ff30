// FP8 block-sparse (and dense) causal prefill attention over a paged KV cache (H100 / sm_90a).
//
// Replaces reference src/attention/prefill/kernels.cuh:1978-2554 (q per-token/head, k/v per-tensor)
// and :2558-3150 (q per-token/head, k per-token/head in-cache scales, v per-head), their launcher
// src/attention/prefill/warp_spec_with_kvcache_blocksparse_fp8_dim128.cu:19-253 and the varlen TMA
// patch kernel (kernels.cuh:169-215, not needed here: Q is addressed with a 3-D descriptor).
//
// Work item = (batch, q head, 128-row Q tile); it visits only the 128x128 KV tiles that are set in
// block_mask (absolute KV tile index, Q tile index relative to the request's first new token):
//   active = { j < min(num_tile_kv, Kb) : mask[b, hq, mq, j] } U { Kb if Kb < num_tile_kv }
// Items are handed out heaviest-first (largest mq first) by a global atomic counter.
//
// CTA = 288 threads, one CTA per SM:
//   warp 8     : TMA producer (Q tile, K pages -> 2-slot ring, V pages -> 2-slot ring, per-token k
//                scales), builds the active-tile list of each item with ballot compaction
//   warps 0-7  : two warpgroups, warpgroup w owns query rows [64w, 64w+64) of the tile.
//                S[64 q, 128 keys] = Q . K^T with wgmma (both operands K-major in smem), kept in
//                registers; scale, causal/length mask and base-2 online softmax on the fragment
//                (a row's 128 scores are spread over the 4 threads of a quad) with a lazy
//                reference maximum; P*256 -> e4m3 into 128B-swizzled smem. fp8 wgmma reads only
//                K-major B operands, so both warpgroups first transpose the V tile into a
//                [d][keys] buffer; then O[64 q, 128 d] += P . V with wgmma (B = that buffer), O
//                in registers across the tiles of an item.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "host_utils.h"
#include "prefill_common.cuh"

namespace b200 {
namespace prefill {

constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kConsumerBar = 1;  // named barrier of the two consumer warpgroups
constexpr int kGroupBar0 = 2;    // named barriers 2, 3: one per consumer warpgroup

template <bool kKPerToken>
struct Smem {
  static constexpr int kOffK = 0;                             // kStages x 16 KB
  static constexpr int kOffV = kOffK + kStages * kTileBytes;  // kStages x 16 KB
  static constexpr int kOffVt = kOffV + kStages * kTileBytes; // 2 x 16 KB transposed V
  static constexpr int kOffQ = kOffVt + 2 * kTileBytes;       // 16 KB
  static constexpr int kOffP = kOffQ + kTileBytes;            // 16 KB
  static constexpr int kOffKs = kOffP + kTileBytes;           // kKsBufs x 128 floats
  static constexpr int kOffList = kOffKs + kKsBufs * 128 * 4;
  static constexpr int kListStride = kMaxKvTiles + 8;  // int16 entries
  static constexpr int kOffBar = kOffList + kListStride * 2;
  static constexpr int kNumBars = 4 * kStages + 2;
  static constexpr int kOffWork = kOffBar + kNumBars * 8;
  static constexpr int kTotal = kOffWork + 16;
  static_assert(kTotal <= 227 * 1024, "prefill smem exceeds the sm_90 per-block limit");
};

// Protocol (all mbarriers; "phase" = use-count parity), n = running KV-tile counter of the CTA:
//   q_full      producer: item published (list + work id in smem, Q tile landed)
//   q_empty     the 8 consumer warps finished the item (Q tile, list and work slot reusable)
//   k_full/k_empty[slot]   K ring; a warp releases the slot once its QK(n) wgmma has completed
//   v_full/v_empty[slot]   V ring; released once the tile is transposed into Vt[n % 2]
// Vt[n % 2] is rewritten for tile n + 2 only after both warpgroups passed the consumer barrier of
// tile n + 1, which each reaches after its PV(n) has completed. The k-scale buffer of tile n is
// rewritten for tile n + 4 after the release of K slot n % 2 for tile n + 2, i.e. after both
// warpgroups finished softmax(n).
// kPoly: exponentials per group of 8 scores that take the polynomial path (0, 2 or 4)
template <bool kKPerToken, int kPoly>
__global__ void __launch_bounds__(kThreads, 1)
    prefill_blocksparse_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                   const __grid_constant__ CUtensorMap tmap_k,
                                   const __grid_constant__ CUtensorMap tmap_v, const Params p) {
  using L = Smem<kKPerToken>;
  using MMA = WgmmaE4M3<128>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* k_smem = smem + L::kOffK;
  uint8_t* v_smem = smem + L::kOffV;
  uint8_t* vt_smem = smem + L::kOffVt;
  uint8_t* q_smem = smem + L::kOffQ;
  uint8_t* p_smem = smem + L::kOffP;
  float* ks_smem = reinterpret_cast<float*>(smem + L::kOffKs);
  int16_t* list = reinterpret_cast<int16_t*>(smem + L::kOffList);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  int* s_work = reinterpret_cast<int*>(smem + L::kOffWork);  // work id, number of active tiles

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
    const uint64_t pol_kv = make_policy_evict_last();  // KV of a request is re-read by its q-heads
    uint32_t n = 0;     // kv tile counter (rings)
    uint32_t item = 0;  // item counter
    while (true) {
      int w = 0;
      if (lane == 0) w = atomicAdd(p.work_counter, 1);
      w = __shfl_sync(0xffffffffu, w, 0);
      Work k;
      const bool alive = decode_work(p, w, k);
      if (alive && k.rows == 0) continue;  // Q tile beyond this request
      mbar_wait(q_empty, (item & 1) ^ 1);
      int nact = 0;
      if (alive) {
        // ---- active tile list (ballot compaction, ascending j) ----
        const int kb = p.block_mask ? p.mask_kb : k.num_tile_kv;
        const int lim = k.num_tile_kv < kb ? k.num_tile_kv : kb;
        const uint8_t* mrow =
            p.block_mask
                ? p.block_mask + ((static_cast<long long>(k.b) * p.num_head_q + k.hq) * p.mask_mq +
                                  (k.mq < p.mask_mq ? k.mq : p.mask_mq - 1)) *
                                     p.mask_kb
                : nullptr;
        for (int j0 = 0; j0 < lim; j0 += 32) {
          const int j = j0 + lane;
          const bool on = (j < lim) && (mrow == nullptr || mrow[j] != 0);
          const unsigned m = __ballot_sync(0xffffffffu, on);
          if (on) list[nact + __popc(m & ((1u << lane) - 1))] = static_cast<int16_t>(j);
          nact += __popc(m);
        }
        if (p.block_mask && kb < k.num_tile_kv) {  // one unconditional tile past the mask width
          if (lane == 0) list[nact] = static_cast<int16_t>(kb);
          nact++;
        }
      }
      __syncwarp();
      // warp-uniform copies of what the elected lane's TMA instructions take as operands (the
      // compiler cannot prove values loaded from memory uniform and would wrap every TMA /
      // mbarrier instruction in an elect + broadcast loop)
      const int u_hq = __shfl_sync(0xffffffffu, k.hq, 0);
      const int u_q0 = __shfl_sync(0xffffffffu, k.q0, 0);
      if (elect_one()) {
        s_work[0] = alive ? w : -1;
        s_work[1] = nact;
        if (alive) {
          mbar_arrive_expect_tx(q_full, kTileBytes);
          tma_load_3d(q_smem, &tmap_q, q_full, 0, u_hq, u_q0);
        } else {
          mbar_arrive(q_full);
        }
      }
      __syncwarp();
      item++;
      if (!alive) {
        // the last CTA out re-arms the work counter for the next launch (no memset node between
        // launches; one counter pair per stream or captured launch, see host_utils.h scheduler_counter)
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
      // ---- K/V tiles of the active list ----
      const int hkv = u_hq / p.group;
      const int nblk = (k.seq_kv + kPage - 1) / kPage;
      const int* ids = p.block_ids + static_cast<long long>(k.b) * p.max_blocks;
      const int kc1 = p.k_head_first ? hkv : 0, kc2 = p.k_head_first ? 0 : hkv;
      const int vc1 = p.v_head_first ? hkv : 0, vc2 = p.v_head_first ? 0 : hkv;
      for (int i0 = 0; i0 < nact; i0 += 16) {
        // lanes 2t / 2t+1 fetch the two page ids of tile i0+t
        const int ti = i0 + (lane >> 1);
        int id = 0;
        if (ti < nact) {
          int blk = static_cast<int>(list[ti]) * 2 + (lane & 1);
          blk = blk < nblk ? blk : nblk - 1;  // a missing 2nd page re-reads the 1st (keys masked)
          id = __ldg(ids + blk);
        }
        const int cnt = (nact - i0) < 16 ? (nact - i0) : 16;
        for (int t = 0; t < cnt; t++) {
          const int id0 = __shfl_sync(0xffffffffu, id, 2 * t);
          const int id1 = __shfl_sync(0xffffffffu, id, 2 * t + 1);
          const uint32_t st = n % kStages;
          const uint32_t ph = ((n / kStages) & 1) ^ 1;
          mbar_wait(&k_empty[st], ph);  // QK(n - 2) finished
          if (elect_one()) {
            uint8_t* kd8 = k_smem + st * kTileBytes;
            mbar_arrive_expect_tx(&k_full[st], kTileBytes + (kKPerToken ? 512 : 0));
            tma_load_4d_hint(kd8, &tmap_k, &k_full[st], 0, kc1, kc2, id0, pol_kv);
            tma_load_4d_hint(kd8 + kTileBytes / 2, &tmap_k, &k_full[st], 0, kc1, kc2, id1, pol_kv);
            if constexpr (kKPerToken) {
              // scales of token t of a page: kscale[page, t / 32, hkv, t % 32]
              float* kd = ks_smem + (n % kKsBufs) * 128;
              const float* s0 = p.kscale + id0 * p.ks_stride_blk + hkv * p.ks_stride_head;
              const float* s1 = p.kscale + id1 * p.ks_stride_blk + hkv * p.ks_stride_head;
              bulk_load_1d(kd, s0, 128, &k_full[st]);
              bulk_load_1d(kd + 32, s0 + p.ks_stride_grp, 128, &k_full[st]);
              bulk_load_1d(kd + 64, s1, 128, &k_full[st]);
              bulk_load_1d(kd + 96, s1 + p.ks_stride_grp, 128, &k_full[st]);
            }
          }
          __syncwarp();
          mbar_wait(&v_empty[st], ph);  // V(n - 2) transposed
          if (elect_one()) {
            uint8_t* vd8 = v_smem + st * kTileBytes;
            mbar_arrive_expect_tx(&v_full[st], kTileBytes);
            tma_load_4d_hint(vd8, &tmap_v, &v_full[st], 0, vc1, vc2, id0, pol_kv);
            tma_load_4d_hint(vd8 + kTileBytes / 2, &tmap_v, &v_full[st], 0, vc1, vc2, id1, pol_kv);
          }
          __syncwarp();
          n++;
        }
      }
    }
  } else {
    // =========================== consumer warpgroups =======================================
    const int wg = warp >> 2;
    const int g8 = lane >> 2;
    const int t4 = lane & 3;
    // fragment rows of this thread (query rows of the tile): registers with (i / 2) even -> r[0]
    const int r[2] = {wg * 64 + (warp & 3) * 16 + g8, wg * 64 + (warp & 3) * 16 + g8 + 8};
    const float ks_tensor = kKPerToken ? 1.f : p.kscale[0];
    const uint64_t qdesc = make_smem_desc(smem_u32(q_smem) + wg * 8192, 16, 1024, kLayoutSW128);
    const uint64_t pdesc = make_smem_desc(smem_u32(p_smem) + wg * 8192, 16, 1024, kLayoutSW128);
    const uint64_t kdesc0 = make_smem_desc(smem_u32(k_smem), 16, 1024, kLayoutSW128);
    const uint64_t vtdesc0 = make_smem_desc(smem_u32(vt_smem), 16, 1024, kLayoutSW128);

    uint32_t n = 0;
    uint32_t item = 0;
    while (true) {
      mbar_wait(q_full, item & 1);
      const int w = s_work[0];
      const int nact = s_work[1];
      if (w < 0) break;
      Work k;
      decode_work(p, w, k);
      const int hkv = k.hq / p.group;
      bool row_ok[2];
      float cq[2], mref[2], lrun[2];
      int row_lim[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        row_ok[h] = r[h] < k.rows;
        const float qs =
            row_ok[h] ? __ldg(p.qscale + (static_cast<long long>(k.b) * p.num_head_q + k.hq) *
                                             p.qscale_ld + k.mq * kTile + r[h])
                      : 0.f;
        // > 0 so that a masked score (-inf) stays -inf after scaling (an all-zero q row has
        // qs = 0, and then every raw score is 0 as well)
        cq[h] = fmaxf(qs * ks_tensor * p.softmax_scale_log2, 1e-30f);
        // kv positions visible to this row: pos <= row_lim and pos < seq_kv
        row_lim[h] = k.seq_kv - k.seq_q + k.mq * kTile + r[h];
        // Online softmax with a LAZY reference maximum `mref` (log2 units):
        // P = 256 * 2^(s - mref). mref only moves when the tile maximum exceeds it by more than
        // 0.75 (P would pass ~430 and approach the e4m3 limit 448) or when the row has not seen a
        // key yet; only then is the row of O rescaled.
        mref[h] = -INFINITY;
        lrun[h] = 0.f;  // this thread's share of the row sum (its 32 columns)
      }
      const int tile_lim_min = k.seq_kv - k.seq_q + k.mq * kTile;  // row 0
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; i++) o[i] = 0.f;

      auto softmax_tile = [&](auto mask_tag, float* sv, const int key0, const float* ksr) {
        constexpr bool kMask = decltype(mask_tag)::value;
        // ---- pass 1: dequantised (and masked) scores in place, row maxima ----
        float vmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; i++) {
          const int h = (i >> 1) & 1;
          const int col = 8 * (i >> 2) + 2 * t4 + (i & 1);
          float v = sv[i];
          if constexpr (kKPerToken) v *= ksr[col];
          if constexpr (kMask) {
            const int pos = key0 + col;
            v = (pos > row_lim[h] || pos >= k.seq_kv) ? -INFINITY : v;
          }
          sv[i] = v;
          vmax[h] = fmaxf(vmax[h], v);
        }
        float alpha[2], bias[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          vmax[h] = fmaxf(vmax[h], __shfl_xor_sync(0xffffffffu, vmax[h], 1));
          vmax[h] = fmaxf(vmax[h], __shfl_xor_sync(0xffffffffu, vmax[h], 2));
          float tmax = vmax[h] * cq[h];
          if (!row_ok[h]) tmax = -INFINITY;
          const bool update = (mref[h] == -INFINITY) || (tmax > mref[h] + 0.75f);
          const float mnew = update ? fmaxf(mref[h], tmax) : mref[h];
          const bool dead = (mnew == -INFINITY);
          alpha[h] = (dead || mref[h] == -INFINITY) ? (dead ? 1.f : 0.f) : exp2_approx(mref[h] - mnew);
          mref[h] = mnew;
          bias[h] = dead ? -INFINITY : 8.f - mnew;
        }
        // ---- O rows rescaled (rare after the first tiles of an item) ----
        if (__any_sync(0xffffffffu, alpha[0] != 1.f || alpha[1] != 1.f)) {
#pragma unroll
          for (int i = 0; i < 64; i++) o[i] *= alpha[(i >> 1) & 1];
        }
        // ---- pass 2: P = 256 * 2^(s - mref) -> e4m3 into the swizzled P tile, row sums ----
        float psum[2] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 32; q++) {  // q = pair of adjacent columns: registers 2q, 2q + 1
          const int h = q & 1;
          const int col = 8 * (q >> 1) + 2 * t4;
          const uint64_t x2 = ffma2(pack_f2(sv[2 * q], sv[2 * q + 1]), pack_f2(cq[h], cq[h]),
                                    pack_f2(bias[h], bias[h]));
          float e0, e1;
          if ((q & 3) < kPoly / 2) {
            exp2_poly_pair(x2, e0, e1);
          } else {
            float x0, x1;
            unpack_f2(x2, x0, x1);
            e0 = exp2_approx(x0);
            e1 = exp2_approx(x1);
          }
          psum[h] += e0 + e1;
          *reinterpret_cast<uint16_t*>(p_smem + sw128_offset(r[h], col >> 4) + (col & 15)) =
              cvt_e4m3x2(e0, e1);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) lrun[h] = lrun[h] * alpha[h] + psum[h];
      };

      for (int i = 0; i < nact; i++) {
        const int j = list[i];
        const uint32_t st = n % kStages;
        const uint32_t ph = (n / kStages) & 1;
        // ---- S = Q . K^T for this warpgroup's 64 rows ----
        mbar_wait(&k_full[st], ph);
        float sv[64];  // overwritten: the first wgmma does not read D
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
          MMA::ss(sv, qdesc + kk * 2, kdesc0 + static_cast<uint64_t>(st * (kTileBytes >> 4)) + kk * 2,
                  kk > 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(sv);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[st]);

        const int key0 = j * kTile;
        const bool need_mask = (key0 + kTile - 1 > tile_lim_min) || (key0 + kTile > k.seq_kv);
        const float* ksr = ks_smem + (n % kKsBufs) * 128;
        if (need_mask) {
          softmax_tile(std::true_type{}, sv, key0, ksr);
        } else {
          softmax_tile(std::false_type{}, sv, key0, ksr);
        }

        // ---- V tile -> Vt[n % 2] ([d][keys], 128B swizzle): 4x4-byte blocks, 4 per thread ----
        mbar_wait(&v_full[st], ph);
        {
          const uint8_t* vs = v_smem + st * kTileBytes;
          uint8_t* vt = vt_smem + (n & 1) * kTileBytes;
#pragma unroll
          for (int b = 0; b < 4; b++) {
            const int blk = tid + b * (kConsumerWarps * 32);
            const int kg = blk >> 5;  // keys 4 kg .. 4 kg + 3
            const int dg = blk & 31;  // dims 4 dg .. 4 dg + 3
            uint32_t wv[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
              const int key = 4 * kg + q;
              wv[q] = *reinterpret_cast<const uint32_t*>(vs + sw128_offset(key, dg >> 2) + 4 * (dg & 3));
            }
            const uint32_t lo01 = __byte_perm(wv[0], wv[1], 0x5140), hi01 = __byte_perm(wv[0], wv[1], 0x7362);
            const uint32_t lo23 = __byte_perm(wv[2], wv[3], 0x5140), hi23 = __byte_perm(wv[2], wv[3], 0x7362);
            const uint32_t tr[4] = {__byte_perm(lo01, lo23, 0x5410), __byte_perm(lo01, lo23, 0x7632),
                                    __byte_perm(hi01, hi23, 0x5410), __byte_perm(hi01, hi23, 0x7632)};
#pragma unroll
            for (int c = 0; c < 4; c++) {
              const int d = 4 * dg + c;
              *reinterpret_cast<uint32_t*>(vt + sw128_offset(d, kg >> 2) + 4 * (kg & 3)) = tr[c];
            }
          }
        }
        fence_proxy_async_smem();  // P and Vt writes -> visible to wgmma
        named_bar_sync(kConsumerBar, kConsumerWarps * 32);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);

        // ---- O += P . V ----
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
          MMA::ss(o, pdesc + kk * 2, vtdesc0 + static_cast<uint64_t>((n & 1) * (kTileBytes >> 4)) + kk * 2, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(o);
        // all four warps of this warpgroup are past PV(n) before any of them rewrites P
        named_bar_sync(kGroupBar0 + wg, 128);
        n++;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(q_empty);  // the Q tile, list and work slot may be refilled

      // ---- epilogue: O / sum * vscale -> bf16 rows ----
      const float vs = kKPerToken ? __ldg(p.vscale + hkv) : p.vscale[0];  // (v/256)/(sum/256)
      float inv[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float l = lrun[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        // a row whose every visible tile was skipped has sum 0 -> NaN, as documented for the
        // reference (hpc/attention.py:274-277)
        inv[h] = vs / l;
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (!row_ok[h]) continue;
        __nv_bfloat16* dst = p.out + static_cast<long long>(k.q0 + r[h]) * p.ld_out + k.hq * kD;
#pragma unroll
        for (int jj = 0; jj < 16; jj++) {
          const int col = 8 * jj + 2 * t4;
          *reinterpret_cast<__nv_bfloat162*>(dst + col) =
              __floats2bfloat162_rn(o[4 * jj + 2 * h] * inv[h], o[4 * jj + 2 * h + 1] * inv[h]);
        }
      }
      item++;
    }
  }
}

}  // namespace prefill
}  // namespace b200

using namespace b200;  // NOLINT

constexpr int kDefaultPoly = 2;

static int encode_cache_map(CUtensorMap* tm, const void* base, int heads, int num_blocks,
                            int64_t blk_stride, int64_t tok_stride, int64_t head_stride,
                            int* head_first) {
  *head_first = head_stride <= tok_stride ? 1 : 0;
  uint64_t dims[4];
  uint64_t strides[3];
  uint32_t box[4];
  dims[0] = 128;
  box[0] = 128;
  if (*head_first) {
    dims[1] = static_cast<uint64_t>(heads);
    dims[2] = 64;
    strides[0] = static_cast<uint64_t>(head_stride);
    strides[1] = static_cast<uint64_t>(tok_stride);
    box[1] = 1;
    box[2] = 64;
  } else {
    dims[1] = 64;
    dims[2] = static_cast<uint64_t>(heads);
    strides[0] = static_cast<uint64_t>(tok_stride);
    strides[1] = static_cast<uint64_t>(head_stride);
    box[1] = 64;
    box[2] = 1;
  }
  dims[3] = static_cast<uint64_t>(num_blocks);
  strides[2] = static_cast<uint64_t>(blk_stride);
  box[3] = 1;
  const CUtensorMapL2promotion promo = (tok_stride == 128) ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                                           : CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  return encode_tmap_u8(tm, base, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, promo);
}

// Common launcher of the two quant schemes.
static int prefill_launch(bool k_per_token, void* y_ptr, const void* q_ptr, const void* kcache_ptr,
                          const void* vcache_ptr, const float* qscale_ptr, const float* kscale_ptr,
                          const float* vscale_ptr, const int* cu_seqlens_q_ptr,
                          const int* block_ids_ptr, const int* seqlens_kv_ptr,
                          const uint8_t* block_mask_ptr, int num_batch, int total_seq_q,
                          int max_seq_q, int num_head_q, int num_head_kv, int num_dim,
                          int num_kvcache_blocks, int block_size, int max_blocks, int qscale_ld,
                          int mask_mq, int mask_kb, int ldY, int ldQ, int64_t k_blk, int64_t k_tok,
                          int64_t k_head, int64_t v_blk, int64_t v_tok, int64_t v_head,
                          int64_t ks_blk, int64_t ks_grp, int64_t ks_head, cudaStream_t stream) {
  HPC_REQUIRE(num_dim == 128, "blocksparse prefill: head dim must be 128");
  HPC_REQUIRE(block_size == 64, "blocksparse prefill: paged block size must be 64 in this build");
  HPC_REQUIRE(num_head_kv > 0 && num_head_q % num_head_kv == 0, "bad head counts");
  HPC_REQUIRE(num_batch > 0 && max_seq_q > 0, "bad batch / max_seqlens_q");
  HPC_REQUIRE((ldQ % 16) == 0 && (reinterpret_cast<uintptr_t>(q_ptr) & 15) == 0, "q alignment");
  if (total_seq_q <= 0) return HPC_OK;

  CUtensorMap tq, tk, tv;
  {
    uint64_t dims[3] = {128, static_cast<uint64_t>(num_head_q), static_cast<uint64_t>(total_seq_q)};
    uint64_t strides[2] = {128, static_cast<uint64_t>(ldQ)};
    uint32_t box[3] = {128, 1, 128};
    int rc = encode_tmap_u8(&tq, q_ptr, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc) return rc;
  }
  int khf = 1, vhf = 1;
  int rc = encode_cache_map(&tk, kcache_ptr, num_head_kv, num_kvcache_blocks, k_blk, k_tok, k_head, &khf);
  if (rc) return rc;
  rc = encode_cache_map(&tv, vcache_ptr, num_head_kv, num_kvcache_blocks, v_blk, v_tok, v_head, &vhf);
  if (rc) return rc;

  int* counter = scheduler_counter(stream);  // work-item counter {next item, CTAs done}, self-resetting
  if (counter == nullptr) return HPC_ERR_CUDA;

  prefill::Params p;
  p.cu_seqlens_q = cu_seqlens_q_ptr;
  p.seqlens_kv = seqlens_kv_ptr;
  p.block_ids = block_ids_ptr;
  p.block_mask = block_mask_ptr;
  p.qscale = qscale_ptr;
  p.kscale = kscale_ptr;
  p.vscale = vscale_ptr;
  p.out = static_cast<__nv_bfloat16*>(y_ptr);
  p.work_counter = counter;
  p.ks_stride_blk = ks_blk;
  p.ks_stride_grp = ks_grp;
  p.ks_stride_head = ks_head;
  p.num_batch = num_batch;
  p.num_head_q = num_head_q;
  p.num_head_kv = num_head_kv;
  p.group = num_head_q / num_head_kv;
  p.max_q_tiles = (max_seq_q + prefill::kTile - 1) / prefill::kTile;
  p.mask_mq = mask_mq;
  p.mask_kb = mask_kb;
  p.max_blocks = max_blocks;
  p.qscale_ld = qscale_ld;
  p.ld_out = ldY;
  p.k_head_first = khf;
  p.v_head_first = vhf;
  p.softmax_scale_log2 = 1.4426950408889634f / sqrtf(128.f);

  const int grid = sm_count();  // one resident CTA per SM
  // share of exponentials on the FMA pipe: HPC_B200_PREFILL_POLY = 0 | 2 | 4 (per 8 scores)
  static const int poly = [] {
    const char* e = std::getenv("HPC_B200_PREFILL_POLY");
    const int v = e ? std::atoi(e) : kDefaultPoly;
    return (v == 0 || v == 2 || v == 4) ? v : kDefaultPoly;
  }();
  using KernelFn = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, prefill::Params);
  KernelFn kern;
  int smem_bytes;
  if (k_per_token) {
    smem_bytes = prefill::Smem<true>::kTotal;
    kern = poly == 4   ? prefill::prefill_blocksparse_fp8_kernel<true, 4>
           : poly == 2 ? prefill::prefill_blocksparse_fp8_kernel<true, 2>
                       : prefill::prefill_blocksparse_fp8_kernel<true, 0>;
  } else {
    smem_bytes = prefill::Smem<false>::kTotal;
    kern = poly == 4   ? prefill::prefill_blocksparse_fp8_kernel<false, 4>
           : poly == 2 ? prefill::prefill_blocksparse_fp8_kernel<false, 2>
                       : prefill::prefill_blocksparse_fp8_kernel<false, 0>;
  }
  HPC_CUDA_CHECK(cudaFuncSetAttribute(reinterpret_cast<const void*>(kern),
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  kern<<<grid, prefill::kThreads, smem_bytes, stream>>>(tq, tk, tv, p);
  HPC_CUDA_CHECK(cudaGetLastError());
  return HPC_OK;
}

#define PREFILL_PARAMS                                                                             \
  void *y_ptr, const void *q_ptr, const void *kcache_ptr, const void *vcache_ptr,                 \
      const float *qscale_ptr, const float *kscale_ptr, const float *vscale_ptr,                  \
      const int *cu_seqlens_q_ptr, const int *block_ids_ptr, const int *seqlens_kv_ptr,           \
      const uint8_t *block_mask_ptr, int num_batch, int total_seq_q, int max_seq_q,               \
      int num_head_q, int num_head_kv, int num_dim, int num_kvcache_blocks, int block_size,       \
      int max_blocks, int qscale_ld, int mask_mq, int mask_kb, int ldY, int ldQ, int64_t k_blk,   \
      int64_t k_tok, int64_t k_head, int64_t v_blk, int64_t v_tok, int64_t v_head
#define PREFILL_ARGS                                                                               \
  y_ptr, q_ptr, kcache_ptr, vcache_ptr, qscale_ptr, kscale_ptr, vscale_ptr, cu_seqlens_q_ptr,     \
      block_ids_ptr, seqlens_kv_ptr, block_mask_ptr, num_batch, total_seq_q, max_seq_q,           \
      num_head_q, num_head_kv, num_dim, num_kvcache_blocks, block_size, max_blocks, qscale_ld,    \
      mask_mq, mask_kb, ldY, ldQ, k_blk, k_tok, k_head, v_blk, v_tok, v_head

// replaces reference src/attention/prefill/prefill.h:46-54
// (attention_with_kvcache_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async)
extern "C" int hpc_attention_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async(
    PREFILL_PARAMS, cudaStream_t stream) {
  return prefill_launch(false, PREFILL_ARGS, 0, 0, 0, stream);
}

// replaces reference src/attention/prefill/prefill.h:55-63
// (attention_with_kvcache_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async);
// ks_* = strides in floats of the k-scale tensor [blocks, block/32, Hkv, 32]
extern "C" int hpc_attention_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async(
    PREFILL_PARAMS, int64_t ks_blk, int64_t ks_grp, int64_t ks_head, cudaStream_t stream) {
  HPC_REQUIRE(ks_grp % 4 == 0 && ks_head % 4 == 0 && ks_blk % 4 == 0,
              "k scale strides must be multiples of 4 floats (16-byte bulk copies)");
  return prefill_launch(true, PREFILL_ARGS, ks_blk, ks_grp, ks_head, stream);
}
