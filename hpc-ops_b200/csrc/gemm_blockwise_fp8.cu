// Dense block-scaled FP8 GEMM (H100 / sm_90a): the linear layers of a blockwise-FP8 checkpoint.
//
//   y[m, n] = bf16_rn( sum_kb fl32(xs[m, kb] * ws[n / 128, kb]) * P_kb[m, n] )
//   P_kb = x[m, 128 kb .. 128 kb + 127] . w[n, same columns]      (e4m3 x e4m3, fp32 accumulate)
//   x e4m3 [M, K], xs f32 [M, K / 128], w e4m3 [N, K] (nn.Linear layout), ws f32 [ceil(N / 128),
//   K / 128] (the checkpoint's weight_scale_inv, unpadded), y bf16 [M, N]. No reference counterpart.
//
// Kernel: persistent, warp-specialised, 384 threads, 128 x 128 output tiles, 1 CTA per SM.
//   warpgroup 2   producer; its first warp issues TMA: per 128-column K block an x tile of 128 rows
//                 x 128 B and a w tile of 128 rows x 128 B, 128B swizzle, 6 stages x 32 KB. Rows
//                 past M or N are zero-filled by TMA.
//   warpgroups 0-1  consumers: warpgroup c owns rows 64c..64c+63 of the tile. Per K block it runs
//                 four e4m3 m64n128k32 wgmma straight from the staged tiles into a zeroed block
//                 accumulator P, then promotes: acc = fmaf(P, fl32(xs * ws), acc). A 128-column N
//                 tile is exactly one weight-scale block, so each promotion is one scale per row.
//                 setmaxnreg moves registers from the producer warpgroup (40) to the consumers (232).
// Split-K (decode-sized problems whose tiles cannot fill the SMs): the `split` CTAs of one output
// tile form a thread-block cluster along x; CTA `rank` takes K blocks [KB rank / split,
// KB (rank + 1) / split). Each parks its fp32 tile in its own shared memory (the stages are idle by
// then), the cluster synchronises, and each CTA sums a 1/split share of the tile over all peers
// through distributed shared memory in split order and writes y, as gemm_bf16xfp32.cu does. There
// every cluster owns one tile (the launch has tiles * split CTAs); no global workspace, no counters.
#include "common.cuh"
#include "host_utils.h"

namespace b200 {
namespace bgemm {

constexpr int kBM = 128;
constexpr int kBN = 128;  // one weight-scale block
constexpr int kBK = 128;  // e4m3 elements per K block: one 128-byte swizzle row, one scale block
constexpr int kABytes = kBM * kBK;
constexpr int kBBytes = kBN * kBK;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kStages = 6;
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(kProducerRegs * 128 + kConsumerRegs * kConsumerThreads <= 65536,
              "setmaxnreg split exceeds the register file");
constexpr int kPartLd = kBN + 4;  // floats per row of the parked split-K tile
static_assert(kBM * kPartLd * 4 <= kStages * kStageBytes, "split-K tile must fit the stage region");
constexpr int kEpiBar = 1;
constexpr int kSmemBytes = kStages * kStageBytes + 2 * kStages * 8;
static_assert(kSmemBytes <= 227 * 1024, "blockwise FP8 GEMM smem exceeds the sm_90 per-block limit");

struct Params {
  const float* xs;
  const float* ws;
  __nv_bfloat16* y;
  int m, n, k;
  int split;    // CTAs per cluster = K splits of one output tile
  int tiles_m;  // tile t is (m-tile t % tiles_m, n-tile t / tiles_m)
  int tiles;
};

__global__ void __launch_bounds__(kThreads, 1)
    gemm_blockwise_fp8_kernel(const __grid_constant__ CUtensorMap tmap_x,
                              const __grid_constant__ CUtensorMap tmap_w, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stages = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int KB = p.k / kBK;
  const int rank = static_cast<int>(blockIdx.x) % p.split;  // == rank in the (split x 1 x 1) cluster
  const int kb0 = KB * rank / p.split;
  const int kb1 = KB * (rank + 1) / p.split;
  const int first = static_cast<int>(blockIdx.x) / p.split;
  const int stride = static_cast<int>(gridDim.x) / p.split;

  // ---- set-up that touches no global memory (overlaps the previous kernel under PDL) ----
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tensormap(&tmap_x);
    prefetch_tensormap(&tmap_w);
    for (int i = 0; i < kStages; i++) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp >= kProducerWarp) {
    // =========================== TMA producer ==========================================
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kProducerWarp) {
      uint32_t it = 0;
      for (int tile = first; tile < p.tiles; tile += stride) {
        const int mt = tile % p.tiles_m;
        const int nt = tile / p.tiles_m;
        for (int kb = kb0; kb < kb1; kb++, it++) {
          const uint32_t s = it % kStages;
          uint8_t* a_dst = stages + s * kStageBytes;
          mbar_wait_nocall(&empty[s], ((it / kStages) & 1) ^ 1);
          if (elect_one()) {
            // zero-filled rows past M or N still count towards the stage's bytes
            mbar_arrive_expect_tx(&full[s], kStageBytes);
            tma_load_2d(a_dst, &tmap_x, &full[s], kb * kBK, mt * kBM);
            tma_load_2d(a_dst + kABytes, &tmap_w, &full[s], kb * kBK, nt * kBN);
          }
          __syncwarp();
        }
      }
    }
  } else {
    // =========================== consumer warpgroups: wgmma + promotion ==================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;
    // fragment rows of this thread within the tile: r_lo (registers with (i / 2) even), r_lo + 8
    const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c2 = 2 * (lane & 3);
    uint32_t it = 0;
    for (int tile = first; tile < p.tiles; tile += stride) {
      const int mt = tile % p.tiles_m;
      const int nt = tile / p.tiles_m;
      const int grow_lo = mt * kBM + r_lo;
      const int grow_hi = grow_lo + 8;
      // rows past M multiply zero-filled x rows: any finite scale will do, take row M - 1's
      const float* xs_lo = p.xs + static_cast<long long>(min(grow_lo, p.m - 1)) * KB;
      const float* xs_hi = p.xs + static_cast<long long>(min(grow_hi, p.m - 1)) * KB;
      const float* ws = p.ws + static_cast<long long>(nt) * KB;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; i++) acc[i] = 0.f;
      for (int kb = kb0; kb < kb1; kb++, it++) {
        // scales first: their loads overlap the wait for the stage
        const float w_sc = __ldg(ws + kb);
        const float f_lo = __fmul_rn(__ldg(xs_lo + kb), w_sc);
        const float f_hi = __fmul_rn(__ldg(xs_hi + kb), w_sc);
        const uint32_t s = it % kStages;
        mbar_wait_nocall(&full[s], (it / kStages) & 1);
        const uint32_t a_base = smem_u32(stages + s * kStageBytes) + wg * (64 * 128);
        const uint64_t a_desc = make_smem_desc(a_base, 16, 1024, kLayoutSW128);
        const uint64_t b_desc =
            make_smem_desc(smem_u32(stages + s * kStageBytes + kABytes), 16, 1024, kLayoutSW128);
        float pk[64];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 32; k++) {  // 32 e4m3 = 32 bytes of the 128-byte row per wgmma
          WgmmaE4M3<128>::ss(pk, a_desc + k * 2, b_desc + k * 2, k > 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_anchor<64>(pk);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] = __fmaf_rn(pk[i], (i & 2) ? f_hi : f_lo, acc[i]);
      }

      if (p.split == 1) {
        const bool ok_lo = grow_lo < p.m, ok_hi = grow_hi < p.m;
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const int col = nt * kBN + 8 * j + c2;
          if (col >= p.n) continue;  // n % 8 == 0: a column pair is wholly in or out
          const float* v = acc + 4 * j;
          if (ok_lo) {
            *reinterpret_cast<uint32_t*>(p.y + static_cast<long long>(grow_lo) * p.n + col) =
                pack_bf16x2(v[0], v[1]);
          }
          if (ok_hi) {
            *reinterpret_cast<uint32_t*>(p.y + static_cast<long long>(grow_hi) * p.n + col) =
                pack_bf16x2(v[2], v[3]);
          }
        }
      } else {
        // park the tile once both warpgroups are done reading the stages
        named_bar_sync(kEpiBar, kConsumerThreads);
        wgmma_store_rows<kBN>(reinterpret_cast<float*>(smem), kPartLd, wg * 64, acc);
      }
    }
  }

  if (p.split > 1) {
    // ---------------- cluster reduction over distributed shared memory ----------------
    cluster_sync_all();  // every split's tile is parked
    if (warp < kConsumerWarps) {
      const int mt = first % p.tiles_m;
      const int nt = first / p.tiles_m;
      const int rows = min(p.m - mt * kBM, kBM);
      const int c4_per_row = min(p.n - nt * kBN, kBN) >> 2;
      const int total = rows * c4_per_row;
      const int share = (total + p.split - 1) / p.split;
      const int begin = rank * share;
      const int end = min(begin + share, total);
      const uint32_t part0 = smem_u32(smem);
      for (int f = begin + tid; f < end; f += kConsumerThreads) {
        const int r = f / c4_per_row;
        const int c4 = f - r * c4_per_row;
        const uint32_t off = static_cast<uint32_t>((r * kPartLd + c4 * 4) * 4);
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < p.split; s++) {  // split order: deterministic
          const float4 t = ld_dsmem_f4(map_to_cta(part0 + off, static_cast<uint32_t>(s)));
          a.x += t.x;
          a.y += t.y;
          a.z += t.z;
          a.w += t.w;
        }
        uint2 w;
        w.x = pack_bf16x2(a.x, a.y);
        w.y = pack_bf16x2(a.z, a.w);
        *reinterpret_cast<uint2*>(p.y + static_cast<long long>(mt * kBM + r) * p.n + nt * kBN +
                                  c4 * 4) = w;
      }
    }
    cluster_sync_all();  // no CTA leaves (and frees its smem) while a peer may still read it
  }
}

static int configure_kernel() {
  HPC_CUDA_CHECK(
      set_max_dynamic_smem(reinterpret_cast<const void*>(gemm_blockwise_fp8_kernel), kSmemBytes));
  return HPC_OK;
}

// Clusters of `split` CTAs (one CTA per SM) that can be resident at once. A cluster must sit inside
// one GPC, so this is less than SMs / split for the larger sizes.
static int max_resident_clusters(int split) {
  static int cache[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (cache[split] > 0) return cache[split];
  int n = 0;
  if (configure_kernel() == HPC_OK) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(split, 1, 1);
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = kSmemBytes;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = split;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (cudaOccupancyMaxActiveClusters(&n, gemm_blockwise_fp8_kernel, &cfg) != cudaSuccess) {
      (void)cudaGetLastError();
      n = 0;
    }
  }
  if (n <= 0) {  // no device / query failed: assume 132 SMs, 7/8 usable by clusters
    int sms = sm_count();
    if (sms <= 0) sms = 132;
    n = split == 1 ? sms : (sms * 7 / 8) / split;
  }
  cache[split] = n;
  return n;
}

static int num_tiles(int m, int n) { return ((m + kBM - 1) / kBM) * ((n + kBN - 1) / kBN); }

}  // namespace bgemm
}  // namespace b200

using namespace b200;  // NOLINT

// The K split (cluster size) of an (m, n, k) problem, 1, 2, 4 or 8; the tile is always 128 x 128.
// The largest split whose clusters are all co-resident (a second wave would double the time of a
// latency-bound problem) and that leaves every split at least two K blocks; 1 when the tiles
// alone fill the resident clusters of every split.
extern "C" int hpc_gemm_blockwise_fp8_config(int m, int n, int k) {
  if (m <= 0 || n <= 0 || k < 128) return 1;
  const int tiles = bgemm::num_tiles(m, n);
  const int kblocks = k / bgemm::kBK;
  int split = 1;
  for (int s = 2; s <= 8; s *= 2) {
    if (tiles <= bgemm::max_resident_clusters(s) && kblocks / s >= 2) split = s;
  }
  return split;
}

extern "C" int hpc_gemm_blockwise_fp8_async(void* y_ptr, const void* x_ptr, const float* x_scale_ptr,
                                            const void* w_ptr, const float* w_scale_ptr, int m,
                                            int n, int k, cudaStream_t stream) {
  using namespace bgemm;
  HPC_REQUIRE(k >= 128 && k <= 65536 && k % 128 == 0,
              "gemm_blockwise_fp8: k (%d) must be a multiple of 128 in [128, 65536]", k);
  HPC_REQUIRE(n > 0 && n % 8 == 0, "gemm_blockwise_fp8: n (%d) must be a positive multiple of 8", n);
  HPC_REQUIRE(m >= 0, "gemm_blockwise_fp8: negative row count %d", m);
  HPC_REQUIRE(((reinterpret_cast<uintptr_t>(y_ptr) | reinterpret_cast<uintptr_t>(x_ptr) |
                reinterpret_cast<uintptr_t>(x_scale_ptr) | reinterpret_cast<uintptr_t>(w_ptr) |
                reinterpret_cast<uintptr_t>(w_scale_ptr)) & 15) == 0,
              "gemm_blockwise_fp8: every tensor must be 16-byte aligned");
  if (m == 0) return HPC_OK;
  HPC_REQUIRE(y_ptr != nullptr && x_ptr != nullptr && x_scale_ptr != nullptr && w_ptr != nullptr &&
                  w_scale_ptr != nullptr,
              "gemm_blockwise_fp8: null pointer");
  CUtensorMap tx, tw;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(m)};
    uint64_t strides[1] = {static_cast<uint64_t>(k)};
    uint32_t box[2] = {static_cast<uint32_t>(kBK), static_cast<uint32_t>(kBM)};
    int rc = encode_tmap_u8(&tx, x_ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(n)};
    uint64_t strides[1] = {static_cast<uint64_t>(k)};
    uint32_t box[2] = {static_cast<uint32_t>(kBK), static_cast<uint32_t>(kBN)};
    int rc = encode_tmap_u8(&tw, w_ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  Params p;
  p.xs = x_scale_ptr;
  p.ws = w_scale_ptr;
  p.y = static_cast<__nv_bfloat16*>(y_ptr);
  p.m = m;
  p.n = n;
  p.k = k;
  p.split = hpc_gemm_blockwise_fp8_config(m, n, k);
  p.tiles_m = (m + kBM - 1) / kBM;
  p.tiles = num_tiles(m, n);
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  // split 1: persistent, one CTA per SM at most; split > 1: one cluster per tile
  const int grid = p.split == 1 ? min(p.tiles, sms) : p.tiles * p.split;
  if (int rc = configure_kernel()) return rc;
  HPC_CUDA_CHECK(launch_pdl(gemm_blockwise_fp8_kernel, dim3(grid), dim3(kThreads), kSmemBytes,
                            stream, p.split, tx, tw, p));
  return HPC_OK;
}
