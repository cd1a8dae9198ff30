#include "host_utils.h"

#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <unordered_map>
#include <utility>
#include <vector>

namespace b200 {

static thread_local char g_last_error[1024] = {0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

int sm_count() {
  // cached per device (H100 SXM: 132)
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cached[dev] = n;
  }
  return cached[dev];
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("HPC_B200_PDL");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

// Current CUDA device clamped to [0, 63] (0 when the runtime is unavailable). One-time state
// (function attributes, scheduler counters) is kept per device: one process may drive several GPUs.
static int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) return 0;
  return dev < 64 ? dev : 63;
}

namespace {

// Zeroed counter pairs of one device, handed out from chunks that are never moved or freed: a pair
// may be baked into a CUDA graph that outlives every stream the process has.
struct CounterPool {
  std::vector<int*> chunks;
  int used = 0;  // pairs handed out from the last chunk
};
constexpr int kChunkPairs = 1024;

// `pairs` consecutive pairs; kChunkPairs is a multiple of every `pairs` a pool is used with.
int* new_counter_pair(CounterPool& pool, int pairs = 1) {
  if (pool.chunks.empty() || pool.used + pairs > kChunkPairs) {
    // May run while this thread captures a stream. cudaMalloc is not allowed under a global-mode
    // capture, so this thread switches to relaxed mode for the allocation; the chunk is zeroed on a
    // private non-blocking stream, so nothing is enqueued on or synchronised with a captured stream.
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    const size_t bytes = kChunkPairs * 2 * sizeof(int);
    int* p = nullptr;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, bytes, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (s != nullptr) cudaStreamDestroy(s);
    if (e != cudaSuccess && p != nullptr) cudaFree(p);
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (e != cudaSuccess) {
      set_last_error("scheduler_counter: allocation failed: %s", cudaGetErrorString(e));
      return nullptr;
    }
    pool.chunks.push_back(p);
    pool.used = 0;
  }
  int* p = pool.chunks.back() + 2 * pool.used;
  pool.used += pairs;
  return p;
}

// Per-stream device storage of `kPairs` zeroed pairs, handed out as scheduler_counter describes.
// Every block handed out gets the next serial number (1, 2, ...) of its table.
template <int kPairs>
struct StreamTable {
  struct Entry {
    int* p = nullptr;
    uint64_t serial = 0;
  };
  CounterPool pools[64];
  std::unordered_map<cudaStream_t, Entry> by_stream[64];
  std::mutex mu;
  uint64_t handed_out = 0;

  int* get(cudaStream_t stream, uint64_t* serial) {
    const int dev = device_slot();
    cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(stream, &status);
    if (e != cudaSuccess) {
      set_last_error("scheduler_counter: cudaStreamIsCapturing failed: %s", cudaGetErrorString(e));
      return nullptr;
    }
    std::lock_guard<std::mutex> lock(mu);
    Entry fresh;
    Entry* slot = &fresh;
    // A captured launch gets a block of its own: graphs captured on one stream may be replayed
    // concurrently on different streams, so the capture stream says nothing about what runs together.
    if (status != cudaStreamCaptureStatusActive) {
      // cudaStreamPerThread is one handle value for a different stream on every host thread
      static thread_local Entry per_thread[64];
      slot = stream == cudaStreamPerThread ? &per_thread[dev] : &by_stream[dev][stream];
    }
    if (slot->p == nullptr) {
      slot->p = new_counter_pair(pools[dev], kPairs);
      if (slot->p == nullptr) return nullptr;
      slot->serial = ++handed_out;
    }
    if (serial != nullptr) *serial = slot->serial;
    return slot->p;
  }
};

}  // namespace

int* scheduler_counter(cudaStream_t stream) {
  static StreamTable<1> table;
  return table.get(stream, nullptr);
}

int* stream_state(cudaStream_t stream, uint64_t* serial) {
  static StreamTable<2> table;
  return table.get(stream, serial);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes, const void* base,
                int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                CUtensorMapSwizzle swizzle, CUtensorMapL2promotion promo) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return HPC_ERR_DRIVER;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; i++) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  (void)elem_bytes;
  CUresult r = fn(out, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr,
                  bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, promo,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error(
        "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] strides [%llu %llu "
        "%llu] box [%u %u %u %u] base %p",
        static_cast<int>(r), rank, (unsigned long long)dims[0],
        (unsigned long long)(rank > 1 ? dims[1] : 0), (unsigned long long)(rank > 2 ? dims[2] : 0),
        (unsigned long long)(rank > 3 ? dims[3] : 0),
        (unsigned long long)(rank > 1 ? strides_bytes[0] : 0),
        (unsigned long long)(rank > 2 ? strides_bytes[1] : 0),
        (unsigned long long)(rank > 3 ? strides_bytes[2] : 0), box[0], rank > 1 ? box[1] : 0,
        rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, base);
    return HPC_ERR_DRIVER;
  }
  return HPC_OK;
}

int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle,
                   CUtensorMapL2promotion promo) {
  return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, base, rank, dims, strides_bytes, box,
                     swizzle, promo);
}

int encode_paged_kv_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes,
                         const void* base, int heads, int page, int num_blocks, int64_t blk_stride,
                         int64_t tok_stride, int64_t head_stride, int* head_first) {
  *head_first = head_stride <= tok_stride ? 1 : 0;
  const uint64_t eb = static_cast<uint64_t>(elem_bytes);
  uint64_t dims[4];
  uint64_t strides[3];
  uint32_t box[4];
  dims[0] = 128;
  box[0] = 128 / elem_bytes;
  if (*head_first) {
    dims[1] = static_cast<uint64_t>(heads);
    dims[2] = static_cast<uint64_t>(page);
    strides[0] = static_cast<uint64_t>(head_stride) * eb;
    strides[1] = static_cast<uint64_t>(tok_stride) * eb;
    box[1] = 1;
    box[2] = static_cast<uint32_t>(page);
  } else {
    dims[1] = static_cast<uint64_t>(page);
    dims[2] = static_cast<uint64_t>(heads);
    strides[0] = static_cast<uint64_t>(tok_stride) * eb;
    strides[1] = static_cast<uint64_t>(head_stride) * eb;
    box[1] = static_cast<uint32_t>(page);
    box[2] = 1;
  }
  dims[3] = static_cast<uint64_t>(num_blocks);
  strides[2] = static_cast<uint64_t>(blk_stride) * eb;
  box[3] = 1;
  // L2 promotion must not exceed the contiguous run of one head's rows: 256 B when they follow each
  // other (token stride = one 128-element row), else 128 B. With the token rows of a head strided by
  // Hkv rows (NHD) a 256 B promotion drags in the neighbouring head's row, which is consumed by
  // another CTA much later.
  // Under the fp8 decode kernel's rotated walk the neighbouring head's row is wanted by another CTA
  // at about the same time, but a 256 B promotion is still slower there on H100: at C2 (NHD,
  // rotated) the kernel takes 0.403 ms with 256 B and 0.367 ms with 128 B (H100 80GB HBM3 SXM,
  // 700 W).
  const CUtensorMapL2promotion promo = tok_stride == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                                         : CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  return encode_tmap(out, dtype, elem_bytes, base, 4, dims, strides, box,
                     CU_TENSOR_MAP_SWIZZLE_128B, promo);
}

cudaError_t set_max_dynamic_smem(const void* kern, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> limit;  // largest size set so far
  const std::pair<const void*, int> key(kern, device_slot());
  std::lock_guard<std::mutex> lock(mu);
  auto it = limit.find(key);
  if (it != limit.end() && it->second >= bytes) return cudaSuccess;
  const cudaError_t e =
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) limit[key] = bytes;
  return e;
}

}  // namespace b200

extern "C" const char* hpc_last_error() { return b200::g_last_error; }

extern "C" int hpc_sm_count() { return b200::sm_count(); }
