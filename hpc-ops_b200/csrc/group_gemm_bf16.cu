// Grouped bf16 GEMM for MoE (H100 / sm_90a).
//
//   Y[rows of group g, :] = X[rows of group g, :] . W[g]^T        X: [M, K] bf16, W: [G, N, K] bf16
//
// epilogues
//   plain     : bf16 Y[M, N]
//   fused act : N = 2*I (gate rows then up rows of W): a = bf16(silu(bf16(gate)) * bf16(up)) into
//               bf16 A[M, I]; the bf16 Gate-Up matrix never goes to HBM.
//
// Kernel: persistent, one CTA per SM, 384 threads, 128 x 256 output tiles:
//   warpgroup 2   producer; its first warp issues TMA: per 64-element K block an A tile of 128 rows
//                 x 128 B and a B tile of 256 rows x 128 B (two 128-row boxes: columns n..n+127 and
//                 n+128..n+255, or for the fused epilogue gate rows n.. and up rows I+n..), 128B
//                 swizzle, 4 stages x 48 KB. Tile ids come from the shared grouped-GEMM scheduler
//                 (group_gemm_sched.cuh), claimed one tile ahead and passed on through a queue.
//   warpgroups 0-1  consumers: warpgroup c multiplies rows 64c..64c+63 of the tile with
//                 m64n256k16 bf16 wgmma straight from the staged tiles (no conversion pass) into
//                 one 128-register fp32 accumulator, keeping one K block's wgmma group in flight.
//                 bf16 needs no per-block promotion, so two consumer warpgroups fit: setmaxnreg
//                 moves registers from the producer warpgroup (40) to the consumers (232).
//   The epilogue works on the accumulator fragment: gate column j is register i of the first
//   128 columns and its up column is register 64 + i, in the same thread.
#include "common.cuh"
#include "group_gemm.h"
#include "group_gemm_sched.cuh"
#include "host_utils.h"

namespace b200 {
namespace ggemm_bf16 {

using ggemm::Sched;
using ggemm::TileInfo;

constexpr int kBM = 128;
constexpr int kBN = 256;
constexpr int kBK = 64;  // bf16 elements per K block: 128-byte rows
constexpr int kStages = 4;
constexpr int kABytes = kBM * kBK * 2;
constexpr int kBBytes = kBN * kBK * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kConsumerWGs = 2;
constexpr int kConsumerWarps = 4 * kConsumerWGs;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 4) * 32;
constexpr int kMaxGroups = 512;
constexpr int kTileQ = 4;
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(kProducerRegs * 128 + kConsumerRegs * 128 * kConsumerWGs <= 65536,
              "setmaxnreg split exceeds the register file");

struct Params {
  const int* seqlens;     // [G] rows per group
  const int* cu_seqlens;  // [G+1] first row of each group in X / Y
  __nv_bfloat16* y;       // plain: [M, N]; fused: [M, N/2]
  int num_group;
  int n;  // rows of W per group
  int k;
  int scale_tile;     // granule of the scheduler's (unused) scale-column scan: kBM
  int* tile_counter;  // dynamic tile scheduler: [0] next tile, [1] CTAs done (self-resetting)
};

// dynamic shared memory: operand stages, schedule arrays, barriers, tile queue
constexpr int kSmemBytes = kStages * kStageBytes + (kMaxGroups + 4 + 3 * kMaxGroups) * 4 +
                           (2 * kStages + 2 * kTileQ) * 8 + kTileQ * 4;
static_assert(kSmemBytes <= 227 * 1024, "bf16 grouped GEMM smem exceeds the sm_90 per-block limit");

template <bool kFused>
__global__ void __launch_bounds__(kThreads, 1)
    group_gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a,
                           const __grid_constant__ CUtensorMap tmap_b, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stages = smem;
  int* s_cu_tiles = reinterpret_cast<int*>(smem + kStages * kStageBytes);
  int* s_pad_base = s_cu_tiles + (kMaxGroups + 4);
  int* s_rows = s_pad_base + kMaxGroups;
  int* s_row_start = s_rows + kMaxGroups;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_row_start + kMaxGroups);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  uint64_t* tq_full = bars + 2 * kStages;  // tile-id queue (kTileQ slots): producer -> consumers
  uint64_t* tq_empty = tq_full + kTileQ;
  int* s_tileq = reinterpret_cast<int*>(tq_empty + kTileQ);

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int KB = p.k / kBK;
  const int nt_count = kFused ? p.n / 2 / 128 : (p.n + kBN - 1) / kBN;

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
  pdl_wait();  // routing (seqlens, gathered rows) / the previous GEMM's output are complete

  // ---- schedule prologue: every CTA derives the same tile list from seqlens ----
  if (warp == 2) {
    GGEMM_SCHEDULE_SCAN(p, kBM, nt_count, s_cu_tiles, s_pad_base, s_rows, s_row_start, lane);
  }
  __syncthreads();

  Sched sched{s_cu_tiles, s_pad_base, s_rows, s_row_start, p.num_group, nt_count};

  if (warp >= kProducerWarp) {
    // =========================== TMA producer ==========================================
    setmaxnreg_dec<kProducerRegs>();
    if (warp != kProducerWarp) return;
    // Whole-warp loop with warp-uniform values, one elected lane issues (see group_gemm_fp8.cu).
    // A rows of a group are re-read by every n-tile -> keep them in L2.
    const uint64_t pol_a = make_policy_evict_last();
    uint32_t it = 0;
    uint32_t tq = 0;
    TileInfo t;
    int next_tile = ggemm::claim_tile(p.tile_counter, lane);
    while (true) {
      const int tile = next_tile;
      bool valid = ggemm::decode_tile<kBM>(sched, tile, t);
      valid = __shfl_sync(0xffffffffu, static_cast<int>(valid), 0) != 0;
      t.g = __shfl_sync(0xffffffffu, t.g, 0);
      t.nt = __shfl_sync(0xffffffffu, t.nt, 0);
      t.row0 = __shfl_sync(0xffffffffu, t.row0, 0);
      const uint32_t qs = tq % kTileQ;
      mbar_wait_nocall(&tq_empty[qs], ((tq / kTileQ) & 1) ^ 1);
      if (elect_one()) {
        s_tileq[qs] = valid ? tile : -1;
        mbar_arrive(&tq_full[qs]);
      }
      __syncwarp();
      tq++;
      if (!valid) break;
      next_tile = ggemm::claim_tile(p.tile_counter, lane);
      const int nrow0 = kFused ? t.nt * 128 : t.nt * kBN;
      const int nrow1 = kFused ? p.n / 2 + t.nt * 128 : t.nt * kBN + 128;
      for (int kb = 0; kb < KB; kb++, it++) {
        const uint32_t s = it % kStages;
        uint8_t* a_dst = stages + s * kStageBytes;
        uint8_t* b_dst = a_dst + kABytes;
        mbar_wait_nocall(&empty[s], ((it / kStages) & 1) ^ 1);
        if (elect_one()) {
          // rows past M or N are zero-filled by TMA and still count towards the stage's bytes
          mbar_arrive_expect_tx(&full[s], kStageBytes);
          tma_load_2d_hint(a_dst, &tmap_a, &full[s], kb * kBK, t.row0, pol_a);
          tma_load_3d(b_dst, &tmap_b, &full[s], kb * kBK, nrow0, t.g);
          tma_load_3d(b_dst + kBBytes / 2, &tmap_b, &full[s], kb * kBK, nrow1, t.g);
        }
        __syncwarp();
      }
    }
    if (lane == 0) ggemm::release_scheduler(p.tile_counter);
  } else {
    // =========================== consumer warpgroups: wgmma + epilogue ====================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;
    const int g8 = lane >> 2;
    const int t4 = lane & 3;
    // fragment rows of this thread within the tile: r_lo (registers with (i / 2) even), r_lo + 8
    const int r_lo = wg * 64 + (warp & 3) * 16 + g8;
    const int r_hi = r_lo + 8;

    uint32_t it = 0;
    uint32_t tq = 0;
    TileInfo t;
    while (true) {
      const uint32_t qs = tq % kTileQ;
      mbar_wait_nocall(&tq_full[qs], (tq / kTileQ) & 1);
      const int tile = s_tileq[qs];
      tq++;
      __syncwarp();
      if (lane == 0) mbar_arrive(&tq_empty[qs]);
      if (tile < 0) break;
      ggemm::decode_tile<kBM>(sched, tile, t);

      // acc[h * 64 + i]: 128-column half h, register i of the m64n128 fragment (the m64n256
      // fragment has the same order: its columns 128..255 are registers 64..127)
      float acc[128];
      for (int kb = 0; kb < KB; kb++, it++) {
        const uint32_t s = it % kStages;
        mbar_wait_nocall(&full[s], (it / kStages) & 1);
        const uint32_t a_base = smem_u32(stages + s * kStageBytes) + wg * (64 * 128);
        const uint64_t a_desc = make_smem_desc(a_base, 16, 1024, kLayoutSW128);
        const uint64_t b_desc = make_smem_desc(smem_u32(stages + s * kStageBytes + kABytes), 16,
                                               1024, kLayoutSW128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; k++) {  // 16 elements = 32 bytes of the 128-byte row per wgmma
          WgmmaBF16<256, 0, 0>::ss(acc, a_desc + k * 2, b_desc + k * 2, (kb | k) > 0);
        }
        wgmma_commit();
        // the previous K block's wgmma group has read its stage: hand that stage back
        if (kb > 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[(it - 1) % kStages]);
        }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[(it - 1) % kStages]);
      wgmma_anchor<128>(acc);

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
            if (ok_lo) *reinterpret_cast<uint32_t*>(p.y + grow_lo * p.n + col) = pack_bf16x2(v[0], v[1]);
            if (ok_hi) *reinterpret_cast<uint32_t*>(p.y + grow_hi * p.n + col) = pack_bf16x2(v[2], v[3]);
          }
        }
      } else {
        // g and u rounded to bf16 (the Gate-Up GEMM's bf16 output), the product in fp32, rounded
        // once more to bf16: the Down GEMM's input
        const int ncols = p.n / 2;
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const int col = t.nt * 128 + 8 * j + 2 * t4;
          float a[4];
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const float g = ggemm::bf16_round(acc[4 * j + q]);
            const float u = ggemm::bf16_round(acc[64 + 4 * j + q]);
            a[q] = ggemm::silu_f(g) * u;
          }
          if (ok_lo) *reinterpret_cast<uint32_t*>(p.y + grow_lo * ncols + col) = pack_bf16x2(a[0], a[1]);
          if (ok_hi) *reinterpret_cast<uint32_t*>(p.y + grow_hi * ncols + col) = pack_bf16x2(a[2], a[3]);
        }
      }
    }
  }
}

template <bool kFused>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Params& p, cudaStream_t stream) {
  auto kern = group_gemm_bf16_kernel<kFused>;
  HPC_CUDA_CHECK(set_max_dynamic_smem(reinterpret_cast<const void*>(kern), kSmemBytes));
  Params pp = p;
  pp.tile_counter = scheduler_counter(stream);  // self-resetting pair: per stream, or per captured launch
  if (pp.tile_counter == nullptr) return HPC_ERR_CUDA;
  HPC_CUDA_CHECK(launch_pdl(kern, dim3(sm_count()), dim3(kThreads), kSmemBytes, stream, 1, ta, tb, pp));
  return HPC_OK;
}

}  // namespace ggemm_bf16

namespace ggemm {

int run_bf16(bool fused, const void* x, const void* w, const int* seqlens, const int* cu_seqlens,
             void* y, int num_group, int m, int n, int k, cudaStream_t stream) {
  using namespace ggemm_bf16;
  HPC_REQUIRE(num_group > 0 && num_group <= kMaxGroups,
              "group_gemm_bf16: num_group %d not in (0, %d]", num_group, kMaxGroups);
  HPC_REQUIRE(k > 0 && k % 128 == 0, "group_gemm_bf16: k (%d) must be a positive multiple of 128", k);
  if (fused) {
    HPC_REQUIRE(n > 0 && n % 256 == 0,
                "fuse_moe_bf16: gate_up rows (%d) must be 2 * I with I a multiple of 128", n);
  } else {
    HPC_REQUIRE(n > 0 && n % 128 == 0, "group_gemm_bf16: n (%d) must be a positive multiple of 128", n);
  }
  HPC_REQUIRE(m >= 0, "group_gemm_bf16: negative row count %d", m);
  HPC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(y) & 15) == 0,
              "group_gemm_bf16: x, weight and output must be 16-byte aligned");
  if (m == 0) return HPC_OK;
  HPC_REQUIRE(seqlens != nullptr && cu_seqlens != nullptr && x != nullptr && w != nullptr && y != nullptr,
              "group_gemm_bf16: null pointer");

  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(m)};
    uint64_t strides[1] = {static_cast<uint64_t>(k) * 2};
    uint32_t box[2] = {static_cast<uint32_t>(kBK), static_cast<uint32_t>(kBM)};
    int rc = encode_tmap(&ta, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, 2, dims, strides, box,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {static_cast<uint64_t>(k), static_cast<uint64_t>(n),
                        static_cast<uint64_t>(num_group)};
    uint64_t strides[2] = {static_cast<uint64_t>(k) * 2, static_cast<uint64_t>(k) * n * 2};
    uint32_t box[3] = {static_cast<uint32_t>(kBK), 128, 1};
    int rc = encode_tmap(&tb, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w, 3, dims, strides, box,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  Params p;
  p.seqlens = seqlens;
  p.cu_seqlens = cu_seqlens;
  p.y = static_cast<__nv_bfloat16*>(y);
  p.num_group = num_group;
  p.n = n;
  p.k = k;
  p.scale_tile = kBM;
  p.tile_counter = nullptr;
  return fused ? launch<true>(ta, tb, p, stream) : launch<false>(ta, tb, p, stream);
}

}  // namespace ggemm
}  // namespace b200

using namespace b200;  // NOLINT

extern "C" int hpc_group_gemm_bf16_async(void* y_ptr, const void* x_ptr, const void* w_ptr,
                                         const void* seqlens_ptr, const void* cu_seqlens_ptr,
                                         int num_group, int m, int n, int k, cudaStream_t stream) {
  return ggemm::run_bf16(false, x_ptr, w_ptr, static_cast<const int*>(seqlens_ptr),
                         static_cast<const int*>(cu_seqlens_ptr), y_ptr, num_group, m, n, k, stream);
}
