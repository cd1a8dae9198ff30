#include "host_utils.h"

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>
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

int device_slot() {
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

int* new_counter_pair(CounterPool& pool) {
  if (pool.chunks.empty() || pool.used == kChunkPairs) {
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
  return pool.chunks.back() + 2 * pool.used++;
}

}  // namespace

int* scheduler_counter(cudaStream_t stream) {
  static CounterPool pools[64];
  static std::unordered_map<cudaStream_t, int*> by_stream[64];
  static std::mutex mu;
  const int dev = device_slot();
  cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
  const cudaError_t e = cudaStreamIsCapturing(stream, &status);
  if (e != cudaSuccess) {
    set_last_error("scheduler_counter: cudaStreamIsCapturing failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  std::lock_guard<std::mutex> lock(mu);
  // A captured launch gets a pair of its own: graphs captured on one stream may be replayed
  // concurrently on different streams, so the capture stream says nothing about what runs together.
  if (status == cudaStreamCaptureStatusActive) return new_counter_pair(pools[dev]);
  // cudaStreamPerThread is one handle value for a different stream on every host thread
  if (stream == cudaStreamPerThread) {
    static thread_local int* per_thread[64] = {nullptr};
    if (per_thread[dev] == nullptr) per_thread[dev] = new_counter_pair(pools[dev]);
    return per_thread[dev];
  }
  auto it = by_stream[dev].find(stream);
  if (it != by_stream[dev].end()) return it->second;
  int* p = new_counter_pair(pools[dev]);
  if (p != nullptr) by_stream[dev].emplace(stream, p);
  return p;
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

}  // namespace b200

extern "C" const char* hpc_last_error() { return b200::g_last_error; }

extern "C" int hpc_sm_count() { return b200::sm_count(); }
