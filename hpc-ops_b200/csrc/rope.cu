// RoPE (NeoX halves) + optional per-head RMSNorm + paged KV-cache store, bf16 and FP8 — the step
// before attention: it writes the paged cache layout the decode / prefill kernels read.
// Written from scratch; semantics of reference src/rope/rope.cu:99-418 (bf16) and
// :420-850 (fp8), launcher contract of src/rope/rope.h:15-38.
//
// HBM-bound streaming kernel: a warp handles (token row, group of 4 q or k heads | the row's whole V
// segment). A lane owns dims {2l, 2l+1} of the lower half and the matching dims of the upper half
// (the NeoX rotation pairs): 4-byte coalesced accesses (128 B per warp per half), 8 of them in
// flight per lane; V is a contiguous 16-byte-vector copy / quantisation. fp32 math, warp-shuffle
// reductions for the RMS and the dynamic Q amax. The warps of a request's LAST token also zero the
// unused tail of that request's last cache page (the "unused slots are zero" contract of attention).
#include "common.cuh"
#include "host_utils.h"

namespace b200 {
namespace rope {

constexpr int kWarpsPerBlock = 8;

struct Params {
  void* out_q;
  void* kcache;
  void* vcache;
  void* out_k;            // optional bypass: [rows, Hkv, Dqk] instead of the cache
  void* out_v;
  int* split_k_flag;      // fp8: [num_req, Hkv], zeroed here
  float* q_scale;         // fp8 dynamic: prefill [num_req, Hq, max_seqlen_aligned], decode [rows, Hq]
  const __nv_bfloat16* qkv;
  const float* cos_sin;   // [max_pos, Dqk]: cos | sin halves
  const int* seqlen;      // [num_req] total length incl. the new tokens
  const int* q_index;     // [num_req + 1]
  const int* kv_indices;  // [num_req, max_blocks]
  const float* q_norm_w;
  const float* k_norm_w;
  const float* k_scale;
  const float* v_scale;
  const float* q_scale_inv;
  float upper_max;
  int max_seqlen_aligned;
  long long kcache_block_stride, vcache_block_stride;  // elements
  int num_req, max_blocks, block_size, num_rows, hq, hkv, dqk, dv;
  int is_prefill, norm_policy, quant_policy;
};

template <typename T>
__device__ __forceinline__ void store2(T* dst, float a, float b);
template <>
__device__ __forceinline__ void store2<__nv_bfloat16>(__nv_bfloat16* dst, float a, float b) {
  *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(a, b);
}
template <>
__device__ __forceinline__ void store2<uint8_t>(uint8_t* dst, float a, float b) {
  *reinterpret_cast<uint16_t*>(dst) = cvt_e4m3x2(a, b);
}

// Work unit of a warp: (token row, unit), units of a row = [groups of kU q heads | groups of kU k heads
// | the whole V segment]. kCH = 64-dim chunks per rotation half (head dim <= 128 * kCH), kU = 4 / kCH
// heads per unit, so that a lane has 8 independent 4-byte loads in flight per unit (a warp per single
// head keeps only 2 in flight).
template <bool kFp8, int kCH>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
    rope_norm_store_kv_kernel(const Params p) {
  using OutT = typename std::conditional<kFp8, uint8_t, __nv_bfloat16>::type;
  constexpr int kU = 4 / kCH;
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  const int qg = (p.hq + kU - 1) / kU, kg = (p.hkv + kU - 1) / kU;
  const int units = qg + kg + 1;
  const long long items = static_cast<long long>(p.num_rows) * units;

  pdl_wait();
  pdl_launch_dependents();
  if (kFp8 && p.split_k_flag != nullptr) {
    const long long n = static_cast<long long>(p.num_req) * p.hkv;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      p.split_k_flag[i] = 0;
    }
  }
  if (warp_global >= items) return;
  const int row = static_cast<int>(warp_global / units);
  const int unit = static_cast<int>(warp_global % units);

  // request of this row: the last r with q_index[r] <= row (padding requests have empty ranges)
  int lo = 0, hi = p.num_req;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(p.q_index + mid) <= row) {
      lo = mid;
    } else {
      hi = mid - 1;
    }
  }
  const int req = lo;
  if (req >= p.num_req) return;
  const int q0 = __ldg(p.q_index + req), q1 = __ldg(p.q_index + req + 1);
  if (row < q0 || row >= q1) return;  // padding row
  const int sl = __ldg(p.seqlen + req);
  const int pos = sl - (q1 - q0) + (row - q0);  // absolute position of this token
  if (pos < 0) return;

  const long long row_elems = static_cast<long long>(p.hq) * p.dqk + static_cast<long long>(p.hkv) * (p.dqk + p.dv);
  const __nv_bfloat16* src = p.qkv + static_cast<long long>(row) * row_elems;
  const bool is_q = unit < qg;
  const bool is_k = !is_q && unit < qg + kg;

  // cache slot of this token
  const int bi = pos / p.block_size, pb = pos - bi * p.block_size;
  long long cb = 0;
  if (!is_q) cb = __ldg(p.kv_indices + static_cast<long long>(req) * p.max_blocks + bi);
  const bool last_tok = pos == sl - 1;

  if (!is_q && !is_k) {
    // ---------------- V: all kv heads of the token are contiguous in the row and in the page ------
    const int n = p.hkv * p.dv;  // elements
    const __nv_bfloat16* v = src + static_cast<long long>(p.hq + p.hkv) * p.dqk;
    OutT* dst = p.out_v != nullptr
                    ? static_cast<OutT*>(p.out_v) + static_cast<long long>(row) * n
                    : static_cast<OutT*>(p.vcache) + cb * p.vcache_block_stride + static_cast<long long>(pb) * n;
    const float mult = kFp8 ? __frcp_rn(__ldg(p.v_scale)) : 1.f;
    if ((n & 7) == 0 && (reinterpret_cast<uintptr_t>(v) & 15) == 0 &&
        (reinterpret_cast<uintptr_t>(dst) & (kFp8 ? 7 : 15)) == 0) {
      for (int e = lane * 8; e < n; e += 256) {
        const uint4 raw = ld_nc_v4(v + e);
        if constexpr (kFp8) {
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
          const float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]);
          const float2 f2 = __bfloat1622float2(h[2]), f3 = __bfloat1622float2(h[3]);
          uint2 o;
          o.x = cvt_e4m3x4(f0.x * mult, f0.y * mult, f1.x * mult, f1.y * mult);
          o.y = cvt_e4m3x4(f2.x * mult, f2.y * mult, f3.x * mult, f3.y * mult);
          *reinterpret_cast<uint2*>(dst + e) = o;
        } else {
          *reinterpret_cast<uint4*>(dst + e) = raw;
        }
      }
    } else {
      for (int e = 2 * lane; e < n; e += 64) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(v + e));
        store2<OutT>(dst + e, f.x * mult, f.y * mult);
      }
    }
    if (p.out_v == nullptr && last_tok) {
      // zero the unused tail of the request's last page: contiguous (block_size - pb - 1) * n elements
      OutT* z = static_cast<OutT*>(p.vcache) + cb * p.vcache_block_stride + static_cast<long long>(pb + 1) * n;
      const long long cnt = static_cast<long long>(p.block_size - pb - 1) * n;
      for (long long e = 2 * lane; e < cnt; e += 64) store2<OutT>(z + e, 0.f, 0.f);
    }
    return;
  }

  // ---------------- Q / K: RoPE (+ RMSNorm) on up to kU heads, loads first ----------------
  const int D = p.dqk, half = D / 2;
  const int nheads = is_q ? p.hq : p.hkv;
  const int h0 = (is_q ? unit : unit - qg) * kU;
  const __nv_bfloat16* xbase = src + (is_q ? 0ll : static_cast<long long>(p.hq) * D);
  const float* cs = p.cos_sin + static_cast<long long>(pos) * D;
  const float* nw = is_q ? p.q_norm_w : p.k_norm_w;

  float a[kU][kCH][2], b[kU][kCH][2];
#pragma unroll
  for (int u = 0; u < kU; u++) {
#pragma unroll
    for (int c = 0; c < kCH; c++) {
      const int d = c * 64 + 2 * lane;
      if (h0 + u < nheads && d < half) {
        const __nv_bfloat16* x = xbase + static_cast<long long>(h0 + u) * D;
        const float2 lo2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + d));
        const float2 hi2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + half + d));
        a[u][c][0] = lo2.x; a[u][c][1] = lo2.y; b[u][c][0] = hi2.x; b[u][c][1] = hi2.y;
      } else {
        a[u][c][0] = a[u][c][1] = b[u][c][0] = b[u][c][1] = 0.f;
      }
    }
  }
  float2 co[kCH], si[kCH];
  float wl[kCH][2], wh[kCH][2];
#pragma unroll
  for (int c = 0; c < kCH; c++) {
    const int d = c * 64 + 2 * lane;
    if (d < half) {
      co[c] = *reinterpret_cast<const float2*>(cs + d);
      si[c] = *reinterpret_cast<const float2*>(cs + half + d);
      if (p.norm_policy != 0) {
        wl[c][0] = __ldg(nw + d); wl[c][1] = __ldg(nw + d + 1);
        wh[c][0] = __ldg(nw + half + d); wh[c][1] = __ldg(nw + half + d + 1);
      }
    } else {
      co[c] = si[c] = make_float2(0.f, 0.f);
    }
  }
  const float k_mult = (kFp8 && !is_q) ? __frcp_rn(__ldg(p.k_scale)) : 1.f;

#pragma unroll
  for (int u = 0; u < kU; u++) {
    if (h0 + u >= nheads) break;  // warp-uniform
    const int head = h0 + u;
    auto rms = [&]() {
      float ssq = 0.f;
#pragma unroll
      for (int c = 0; c < kCH; c++) {
        ssq += a[u][c][0] * a[u][c][0] + a[u][c][1] * a[u][c][1] + b[u][c][0] * b[u][c][0] + b[u][c][1] * b[u][c][1];
      }
      const float r = rsqrtf(warp_sum_f32(ssq) / static_cast<float>(D) + 1e-6f);
#pragma unroll
      for (int c = 0; c < kCH; c++) {
        if (c * 64 + 2 * lane < half) {
          a[u][c][0] *= r * wl[c][0]; a[u][c][1] *= r * wl[c][1];
          b[u][c][0] *= r * wh[c][0]; b[u][c][1] *= r * wh[c][1];
        }
      }
    };
    if (p.norm_policy == 2) rms();
#pragma unroll
    for (int c = 0; c < kCH; c++) {
      const float l0 = a[u][c][0] * co[c].x - b[u][c][0] * si[c].x, l1 = a[u][c][1] * co[c].y - b[u][c][1] * si[c].y;
      const float g0 = b[u][c][0] * co[c].x + a[u][c][0] * si[c].x, g1 = b[u][c][1] * co[c].y + a[u][c][1] * si[c].y;
      a[u][c][0] = l0; a[u][c][1] = l1; b[u][c][0] = g0; b[u][c][1] = g1;
    }
    if (p.norm_policy == 1) rms();

    float mult = k_mult;
    if (kFp8 && is_q) {
      if (p.quant_policy == 1) {
        float m = 0.f;
#pragma unroll
        for (int c = 0; c < kCH; c++) {
          m = fmaxf(m, fmaxf(fmaxf(fabsf(a[u][c][0]), fabsf(a[u][c][1])), fmaxf(fabsf(b[u][c][0]), fabsf(b[u][c][1]))));
        }
        m = warp_max_f32(m);
        const float qs = m / p.upper_max;
        if (lane == 0) {
          if (p.is_prefill) {
            p.q_scale[(static_cast<long long>(req) * p.hq + head) * p.max_seqlen_aligned + (row - q0)] = qs;
          } else {
            p.q_scale[static_cast<long long>(row) * p.hq + head] = qs;
          }
        }
        mult = qs > 0.f ? __frcp_rn(qs) : 0.f;
      } else {
        mult = __ldg(p.q_scale_inv);
      }
    }
    OutT* dst;
    if (is_q) {
      dst = static_cast<OutT*>(p.out_q) + (static_cast<long long>(row) * p.hq + head) * D;
    } else if (p.out_k != nullptr) {
      dst = static_cast<OutT*>(p.out_k) + (static_cast<long long>(row) * p.hkv + head) * D;
    } else {
      dst = static_cast<OutT*>(p.kcache) + cb * p.kcache_block_stride + (static_cast<long long>(pb) * p.hkv + head) * D;
    }
#pragma unroll
    for (int c = 0; c < kCH; c++) {
      const int d = c * 64 + 2 * lane;
      if (d < half) {
        store2<OutT>(dst + d, a[u][c][0] * mult, a[u][c][1] * mult);
        store2<OutT>(dst + half + d, b[u][c][0] * mult, b[u][c][1] * mult);
      }
    }
  }
  if (is_k && unit == qg && p.out_k == nullptr && last_tok) {
    // K tail of the request's last page, all kv heads: contiguous
    const int n = p.hkv * D;
    OutT* z = static_cast<OutT*>(p.kcache) + cb * p.kcache_block_stride + static_cast<long long>(pb + 1) * n;
    const long long cnt = static_cast<long long>(p.block_size - pb - 1) * n;
    for (long long e = 2 * lane; e < cnt; e += 64) store2<OutT>(z + e, 0.f, 0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// head dim 128 (the hot path's only head size): a lane owns 4 consecutive dims -- lanes 0-15 the
// lower rotation half, lanes 16-31 the upper one, partner = lane ^ 16 -- so a head row is ONE
// 256-byte coalesced load (8 B per lane) and one 8-byte (bf16) / 4-byte (fp8) store per lane; a warp
// handles 8 heads with all loads issued first. The generic kernel above keeps 4-byte accesses.
// ------------------------------------------------------------------------------------------------
template <bool kFp8>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
    rope_norm_store_kv_d128_kernel(const Params p) {
  using OutT = typename std::conditional<kFp8, uint8_t, __nv_bfloat16>::type;
  constexpr int kU = 8, D = 128;
  const int lane = threadIdx.x & 31;
  const long long warp_global = static_cast<long long>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  const int qg = (p.hq + kU - 1) / kU, kg = (p.hkv + kU - 1) / kU;
  const int units = qg + kg + 1;
  const long long items = static_cast<long long>(p.num_rows) * units;

  pdl_wait();
  pdl_launch_dependents();
  if (kFp8 && p.split_k_flag != nullptr) {
    const long long n = static_cast<long long>(p.num_req) * p.hkv;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      p.split_k_flag[i] = 0;
    }
  }
  if (warp_global >= items) return;
  const int row = static_cast<int>(warp_global / units);
  const int unit = static_cast<int>(warp_global % units);
  int lo = 0, hi = p.num_req;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(p.q_index + mid) <= row) {
      lo = mid;
    } else {
      hi = mid - 1;
    }
  }
  const int req = lo;
  if (req >= p.num_req) return;
  const int q0 = __ldg(p.q_index + req), q1 = __ldg(p.q_index + req + 1);
  if (row < q0 || row >= q1) return;
  const int sl = __ldg(p.seqlen + req);
  const int pos = sl - (q1 - q0) + (row - q0);
  if (pos < 0) return;

  const long long row_elems = static_cast<long long>(p.hq) * D + static_cast<long long>(p.hkv) * (D + p.dv);
  const __nv_bfloat16* src = p.qkv + static_cast<long long>(row) * row_elems;
  const bool is_q = unit < qg;
  const bool is_k = !is_q && unit < qg + kg;
  const int bi = pos / p.block_size, pb = pos - bi * p.block_size;
  long long cb = 0;
  if (!is_q) cb = __ldg(p.kv_indices + static_cast<long long>(req) * p.max_blocks + bi);
  const bool last_tok = pos == sl - 1;

  if (!is_q && !is_k) {
    const int n = p.hkv * p.dv;
    const __nv_bfloat16* v = src + static_cast<long long>(p.hq + p.hkv) * D;
    OutT* dst = p.out_v != nullptr
                    ? static_cast<OutT*>(p.out_v) + static_cast<long long>(row) * n
                    : static_cast<OutT*>(p.vcache) + cb * p.vcache_block_stride + static_cast<long long>(pb) * n;
    const float mult = kFp8 ? __frcp_rn(__ldg(p.v_scale)) : 1.f;
    for (int e = lane * 8; e < n; e += 256) {
      const uint4 raw = ld_nc_v4(v + e);
      if constexpr (kFp8) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
        const float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]);
        const float2 f2 = __bfloat1622float2(h[2]), f3 = __bfloat1622float2(h[3]);
        uint2 o;
        o.x = cvt_e4m3x4(f0.x * mult, f0.y * mult, f1.x * mult, f1.y * mult);
        o.y = cvt_e4m3x4(f2.x * mult, f2.y * mult, f3.x * mult, f3.y * mult);
        *reinterpret_cast<uint2*>(dst + e) = o;
      } else {
        *reinterpret_cast<uint4*>(dst + e) = raw;
      }
    }
    if (p.out_v == nullptr && last_tok) {
      OutT* z = static_cast<OutT*>(p.vcache) + cb * p.vcache_block_stride + static_cast<long long>(pb + 1) * n;
      const long long cnt = static_cast<long long>(p.block_size - pb - 1) * n;  // multiple of 8 elements
      constexpr int kVec = kFp8 ? 16 : 8;  // elements per 16-byte store
      for (long long e = static_cast<long long>(lane) * kVec; e < cnt; e += 32 * kVec) {
        if (e + kVec <= cnt) {
          *reinterpret_cast<uint4*>(z + e) = make_uint4(0, 0, 0, 0);
        } else {
          for (long long t2 = e; t2 < cnt; t2 += 2) store2<OutT>(z + t2, 0.f, 0.f);
        }
      }
    }
    return;
  }

  const int nheads = is_q ? p.hq : p.hkv;
  const int h0 = (is_q ? unit : unit - qg) * kU;
  const __nv_bfloat16* xbase = src + (is_q ? 0ll : static_cast<long long>(p.hq) * D);
  const int hi_half = lane >> 4;
  const int idx = 4 * (lane & 15);          // dim inside the rotation half
  const int dim0 = hi_half * 64 + idx;      // dim inside the head
  uint2 raw[kU];
#pragma unroll
  for (int u = 0; u < kU; u++) {
    raw[u] = make_uint2(0, 0);
    if (h0 + u < nheads) raw[u] = *reinterpret_cast<const uint2*>(xbase + static_cast<long long>(h0 + u) * D + dim0);
  }
  const float4 co = *reinterpret_cast<const float4*>(p.cos_sin + static_cast<long long>(pos) * D + idx);
  const float4 si = *reinterpret_cast<const float4*>(p.cos_sin + static_cast<long long>(pos) * D + 64 + idx);
  const float sgn = hi_half ? 1.f : -1.f;   // lower half: x1 c - x2 s ; upper half: x2 c + x1 s
  float4 w = make_float4(1.f, 1.f, 1.f, 1.f);
  if (p.norm_policy != 0) w = *reinterpret_cast<const float4*>((is_q ? p.q_norm_w : p.k_norm_w) + dim0);
  const float k_mult = (kFp8 && !is_q) ? __frcp_rn(__ldg(p.k_scale)) : 1.f;

#pragma unroll
  for (int u = 0; u < kU; u++) {
    if (h0 + u >= nheads) break;  // warp-uniform
    const int head = h0 + u;
    const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&raw[u]);
    const float2 f01 = __bfloat1622float2(hb[0]), f23 = __bfloat1622float2(hb[1]);
    float v[4] = {f01.x, f01.y, f23.x, f23.y};
    auto rms = [&]() {
      const float ssq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
      const float r = rsqrtf(warp_sum_f32(ssq) / 128.f + 1e-6f);
      v[0] *= r * w.x; v[1] *= r * w.y; v[2] *= r * w.z; v[3] *= r * w.w;
    };
    if (p.norm_policy == 2) rms();
    {
      const float o0 = __shfl_xor_sync(0xffffffffu, v[0], 16), o1 = __shfl_xor_sync(0xffffffffu, v[1], 16);
      const float o2 = __shfl_xor_sync(0xffffffffu, v[2], 16), o3 = __shfl_xor_sync(0xffffffffu, v[3], 16);
      v[0] = v[0] * co.x + sgn * o0 * si.x;
      v[1] = v[1] * co.y + sgn * o1 * si.y;
      v[2] = v[2] * co.z + sgn * o2 * si.z;
      v[3] = v[3] * co.w + sgn * o3 * si.w;
    }
    if (p.norm_policy == 1) rms();
    float mult = k_mult;
    if (kFp8 && is_q) {
      if (p.quant_policy == 1) {
        const float m = warp_max_f32(fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3]))));
        const float qs = m / p.upper_max;
        if (lane == 0) {
          if (p.is_prefill) {
            p.q_scale[(static_cast<long long>(req) * p.hq + head) * p.max_seqlen_aligned + (row - q0)] = qs;
          } else {
            p.q_scale[static_cast<long long>(row) * p.hq + head] = qs;
          }
        }
        mult = qs > 0.f ? __frcp_rn(qs) : 0.f;
      } else {
        mult = __ldg(p.q_scale_inv);
      }
    }
    OutT* dst;
    if (is_q) {
      dst = static_cast<OutT*>(p.out_q) + (static_cast<long long>(row) * p.hq + head) * D;
    } else if (p.out_k != nullptr) {
      dst = static_cast<OutT*>(p.out_k) + (static_cast<long long>(row) * p.hkv + head) * D;
    } else {
      dst = static_cast<OutT*>(p.kcache) + cb * p.kcache_block_stride + (static_cast<long long>(pb) * p.hkv + head) * D;
    }
    if constexpr (kFp8) {
      *reinterpret_cast<uint32_t*>(dst + dim0) = cvt_e4m3x4(v[0] * mult, v[1] * mult, v[2] * mult, v[3] * mult);
    } else {
      __nv_bfloat162 b0 = __floats2bfloat162_rn(v[0], v[1]), b1 = __floats2bfloat162_rn(v[2], v[3]);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&b0);
      o.y = *reinterpret_cast<uint32_t*>(&b1);
      *reinterpret_cast<uint2*>(dst + dim0) = o;
    }
  }
  if (is_k && unit == qg && p.out_k == nullptr && last_tok) {
    const int n = p.hkv * D;
    OutT* z = static_cast<OutT*>(p.kcache) + cb * p.kcache_block_stride + static_cast<long long>(pb + 1) * n;
    const long long cnt = static_cast<long long>(p.block_size - pb - 1) * n;  // multiple of 128 elements
    constexpr int kVec = kFp8 ? 16 : 8;
    for (long long e = static_cast<long long>(lane) * kVec; e < cnt; e += 32 * kVec) {
      *reinterpret_cast<uint4*>(z + e) = make_uint4(0, 0, 0, 0);
    }
  }
}

template <bool kFp8>
static int launch_d128(const Params& p, cudaStream_t stream) {
  constexpr int kU = 8;
  const long long units = (p.hq + kU - 1) / kU + (p.hkv + kU - 1) / kU + 1;
  const long long items = static_cast<long long>(p.num_rows) * units;
  const long long blocks = (items + kWarpsPerBlock - 1) / kWarpsPerBlock;
  HPC_REQUIRE(blocks < (1ll << 31), "rope: too many rows");
  HPC_CUDA_CHECK(launch_pdl(rope_norm_store_kv_d128_kernel<kFp8>, dim3(static_cast<unsigned>(blocks)),
                            dim3(kWarpsPerBlock * 32), 0, stream, 1, p));
  return HPC_OK;
}

template <bool kFp8, int kCH>
static int launch_impl(const Params& p, cudaStream_t stream) {
  constexpr int kU = 4 / kCH;
  const long long units = (p.hq + kU - 1) / kU + (p.hkv + kU - 1) / kU + 1;
  const long long items = static_cast<long long>(p.num_rows) * units;
  const long long blocks = (items + kWarpsPerBlock - 1) / kWarpsPerBlock;
  HPC_REQUIRE(blocks < (1ll << 31), "rope: too many rows");
  HPC_CUDA_CHECK(launch_pdl(rope_norm_store_kv_kernel<kFp8, kCH>, dim3(static_cast<unsigned>(blocks)),
                            dim3(kWarpsPerBlock * 32), 0, stream, 1, p));
  return HPC_OK;
}

static int launch(bool fp8, const Params& p, cudaStream_t stream) {
  HPC_REQUIRE(p.dqk % 4 == 0 && p.dqk >= 4 && p.dqk <= 512 && p.dv % 2 == 0 && p.dv > 0,
              "rope: head dims qk=%d v=%d unsupported (qk multiple of 4 up to 512, v even)", p.dqk, p.dv);
  HPC_REQUIRE(p.block_size > 0 && p.hq > 0 && p.hkv > 0 && p.num_req > 0, "rope: bad geometry");
  HPC_REQUIRE(p.norm_policy >= 0 && p.norm_policy <= 2, "rope: qk_norm_policy must be 0, 1 or 2");
  if (p.norm_policy != 0) {
    HPC_REQUIRE(p.q_norm_w != nullptr && p.k_norm_w != nullptr, "rope: norm weights required");
  }
  if (p.num_rows <= 0) {
    // no kernel runs, but the split-k flags are still returned zeroed
    if (fp8 && p.split_k_flag != nullptr) {
      HPC_CUDA_CHECK(cudaMemsetAsync(p.split_k_flag, 0, sizeof(int) * p.num_req * p.hkv, stream));
    }
    return HPC_OK;
  }
  const bool aligned16 = ((reinterpret_cast<uintptr_t>(p.qkv) | reinterpret_cast<uintptr_t>(p.cos_sin) |
                           reinterpret_cast<uintptr_t>(p.out_q) | reinterpret_cast<uintptr_t>(p.kcache) |
                           reinterpret_cast<uintptr_t>(p.vcache) | reinterpret_cast<uintptr_t>(p.out_k) |
                           reinterpret_cast<uintptr_t>(p.out_v) | reinterpret_cast<uintptr_t>(p.q_norm_w) |
                           reinterpret_cast<uintptr_t>(p.k_norm_w)) & 15) == 0;
  const int out_bytes = fp8 ? 1 : 2;
  if (p.dqk == 128 && p.dv % 16 == 0 && aligned16 && (p.kcache_block_stride * out_bytes) % 16 == 0 &&
      (p.vcache_block_stride * out_bytes) % 16 == 0) {
    return fp8 ? launch_d128<true>(p, stream) : launch_d128<false>(p, stream);
  }
  const int ch = (p.dqk / 2 + 63) / 64;  // 64-dim chunks per rotation half
  if (fp8) {
    if (ch <= 1) return launch_impl<true, 1>(p, stream);
    if (ch <= 2) return launch_impl<true, 2>(p, stream);
    return launch_impl<true, 4>(p, stream);
  }
  if (ch <= 1) return launch_impl<false, 1>(p, stream);
  if (ch <= 2) return launch_impl<false, 2>(p, stream);
  return launch_impl<false, 4>(p, stream);
}

}  // namespace rope
}  // namespace b200

using namespace b200;  // NOLINT

// replaces reference src/rope/rope.h:15-25 (rope_norm_store_kv_async), same arguments
extern "C" int hpc_rope_norm_store_kv_async(
    void* out_q_ptr, void* kcache_ptr, void* vcache_ptr, void* out_k_ptr, void* out_v_ptr,
    const void* in_qkv_ptr, const float* cos_sin_ptr, const int* num_seqlen_per_req_ptr,
    const int* q_index_ptr, const int* kvcache_indices_ptr, const float* q_norm_weight_ptr,
    const float* k_norm_weight_ptr, int kcache_block_offset, int vcache_block_offset, int num_batch,
    int max_num_kv_block_per_batch, int kv_block_size, int num_rows, int num_q_heads,
    int num_kv_heads, int qk_head_dim, int v_head_dim, int is_prefill, int qk_norm_policy,
    cudaStream_t stream) {
  rope::Params p{};
  p.out_q = out_q_ptr; p.kcache = kcache_ptr; p.vcache = vcache_ptr; p.out_k = out_k_ptr; p.out_v = out_v_ptr;
  p.qkv = static_cast<const __nv_bfloat16*>(in_qkv_ptr);
  p.cos_sin = cos_sin_ptr; p.seqlen = num_seqlen_per_req_ptr; p.q_index = q_index_ptr;
  p.kv_indices = kvcache_indices_ptr; p.q_norm_w = q_norm_weight_ptr; p.k_norm_w = k_norm_weight_ptr;
  p.kcache_block_stride = kcache_block_offset; p.vcache_block_stride = vcache_block_offset;
  p.num_req = num_batch; p.max_blocks = max_num_kv_block_per_batch; p.block_size = kv_block_size;
  p.num_rows = num_rows; p.hq = num_q_heads; p.hkv = num_kv_heads; p.dqk = qk_head_dim; p.dv = v_head_dim;
  p.is_prefill = is_prefill; p.norm_policy = qk_norm_policy; p.quant_policy = 0; p.upper_max = 448.f;
  return rope::launch(false, p, stream);
}

// replaces reference src/rope/rope.h:27-38 (rope_norm_store_kv_fp8_async), same arguments
extern "C" int hpc_rope_norm_store_kv_fp8_async(
    void* out_q_ptr, void* kcache_ptr, void* vcache_ptr, void* out_k_ptr, void* out_v_ptr,
    int32_t* split_k_flag_ptr, float* q_scale_ptr, const void* in_qkv_ptr, const float* cos_sin_ptr,
    const int* num_seqlen_per_req_ptr, const int* q_index_ptr, const int* kvcache_indices_ptr,
    const float* q_norm_weight_ptr, const float* k_norm_weight_ptr, const float* k_scale_ptr,
    const float* v_scale_ptr, const float* q_scale_inv_ptr, float upper_max, int max_seqlens,
    int kcache_block_offset, int vcache_block_offset, int num_batch, int max_num_kv_block_per_batch,
    int kv_block_size, int num_rows, int num_q_heads, int num_kv_heads, int qk_head_dim,
    int v_head_dim, int is_prefill, int qk_norm_policy, int quant_policy, cudaStream_t stream) {
  HPC_REQUIRE(quant_policy == 1 || quant_policy == 2, "rope fp8: quant_policy must be 1 or 2");
  HPC_REQUIRE(k_scale_ptr != nullptr && v_scale_ptr != nullptr, "rope fp8: k/v scales required");
  HPC_REQUIRE(quant_policy == 1 ? q_scale_ptr != nullptr : q_scale_inv_ptr != nullptr,
              "rope fp8: q_scale (policy 1) / q_scale_inv (policy 2) required");
  HPC_REQUIRE(upper_max > 0.f && upper_max <= 448.f, "rope fp8: upper_max must be in (0, 448]");
  rope::Params p{};
  p.out_q = out_q_ptr; p.kcache = kcache_ptr; p.vcache = vcache_ptr; p.out_k = out_k_ptr; p.out_v = out_v_ptr;
  p.split_k_flag = split_k_flag_ptr; p.q_scale = q_scale_ptr;
  p.qkv = static_cast<const __nv_bfloat16*>(in_qkv_ptr);
  p.cos_sin = cos_sin_ptr; p.seqlen = num_seqlen_per_req_ptr; p.q_index = q_index_ptr;
  p.kv_indices = kvcache_indices_ptr; p.q_norm_w = q_norm_weight_ptr; p.k_norm_w = k_norm_weight_ptr;
  p.k_scale = k_scale_ptr; p.v_scale = v_scale_ptr; p.q_scale_inv = q_scale_inv_ptr;
  p.upper_max = upper_max; p.max_seqlen_aligned = (max_seqlens + 127) / 128 * 128;
  p.kcache_block_stride = kcache_block_offset; p.vcache_block_stride = vcache_block_offset;
  p.num_req = num_batch; p.max_blocks = max_num_kv_block_per_batch; p.block_size = kv_block_size;
  p.num_rows = num_rows; p.hq = num_q_heads; p.hkv = num_kv_heads; p.dqk = qk_head_dim; p.dv = v_head_dim;
  p.is_prefill = is_prefill; p.norm_policy = qk_norm_policy; p.quant_policy = quant_policy;
  return rope::launch(true, p, stream);
}
