// runtime.cu — process-wide runtime of libtinysql_b200.so: device selection, streams, error text,
// pinned/device memory helpers, device timers (the exclusive scan is in scan.cu).
#include <map>

#include "common.cuh"

namespace tq {

static thread_local char g_err[512] = {0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int32_t cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
  const char *base = strrchr(file, '/');
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), base ? base + 1 : file, line, what);
  if (e == cudaErrorMemoryAllocation) return TQ_ERR_OOM;
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice) return TQ_ERR_NO_DEVICE;
  return TQ_ERR_CUDA;
}

Runtime &rt() {
  static Runtime *r = new Runtime();  // leaked: must outlive every static DevBuf
  return *r;
}

static int32_t init_device(int ordinal) {
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  if (r.inited) {
    if (ordinal >= 0 && ordinal != r.device) {
      set_error("tq_init: already initialised on device %d", r.device);
      return TQ_ERR_STATE;
    }
    return TQ_OK;
  }
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device visible (%s); libtinysql_b200 has no CPU fallback", e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
    return TQ_ERR_NO_DEVICE;
  }
  if (ordinal < 0) ordinal = 0;
  if (ordinal >= n) {
    set_error("device ordinal %d out of range (%d devices)", ordinal, n);
    return TQ_ERR_NO_DEVICE;
  }
  cudaDeviceProp p;
  TQ_CUDA(cudaGetDeviceProperties(&p, ordinal));
  if (p.major != 9 || p.minor != 0) {
    set_error("device %d is sm_%d%d; this library carries sm_90a code only", ordinal, p.major, p.minor);
    return TQ_ERR_NO_DEVICE;
  }
  TQ_CUDA(cudaSetDevice(ordinal));
  r.device = ordinal;
  r.sm_count = p.multiProcessorCount;
  TQ_CUDA(cudaStreamCreateWithFlags(&r.compute, cudaStreamNonBlocking));
  TQ_CUDA(cudaStreamCreateWithFlags(&r.h2d, cudaStreamNonBlocking));
  TQ_CUDA(cudaStreamCreateWithFlags(&r.d2h, cudaStreamNonBlocking));
  TQ_CUDA(cudaEventCreate(&r.t0));
  TQ_CUDA(cudaEventCreate(&r.t1));
  r.inited = true;
  return TQ_OK;
}

int32_t ensure_init() {
  Runtime &r = rt();
  if (!r.inited) TQ_TRY(init_device(-1));
  // cgo calls arrive on arbitrary OS threads: bind the device for this thread every time.
  TQ_CUDA(cudaSetDevice(r.device));
  return TQ_OK;
}

int32_t check_launch(const char *kernel) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("kernel launch failed: %s: %s", kernel, cudaGetErrorString(e));
    return TQ_ERR_CUDA;
  }
  return TQ_OK;
}

// ---------------------------------------------------------------- caching allocators
// cudaMalloc / cudaHostAlloc of GB-sized buffers cost milliseconds; operators are created per query, so
// released blocks are kept and handed back to the next request of a similar size (best fit within 2x).
struct BlockCache {
  std::mutex mu;
  std::multimap<size_t, void *> free_blocks;
  size_t cached_bytes = 0;
  size_t max_cached;
  explicit BlockCache(size_t cap) : max_cached(cap) {}
  void *take(size_t bytes, size_t *got) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = free_blocks.lower_bound(bytes);
    if (it == free_blocks.end() || it->first > bytes * 2 + (1u << 20)) return nullptr;
    void *p = it->second;
    *got = it->first;
    cached_bytes -= it->first;
    free_blocks.erase(it);
    return p;
  }
  bool give(void *p, size_t bytes) {
    std::lock_guard<std::mutex> lk(mu);
    if (cached_bytes + bytes > max_cached) return false;
    free_blocks.emplace(bytes, p);
    cached_bytes += bytes;
    return true;
  }
  template <typename FreeFn> void drain(FreeFn f) {
    std::lock_guard<std::mutex> lk(mu);
    for (auto &kv : free_blocks) f(kv.second);
    free_blocks.clear();
    cached_bytes = 0;
  }
};
// leaked on purpose: DevBuf/PinBuf objects with static storage release into these during exit
static BlockCache &dev_cache() { static BlockCache *c = new BlockCache((size_t)40 << 30); return *c; }  // half of an H100's 80 GB
static BlockCache &pin_cache() { static BlockCache *c = new BlockCache((size_t)24 << 30); return *c; }

int32_t DevBuf::reserve(size_t bytes) {
  if (bytes <= cap) return TQ_OK;
  release();
  size_t want = bytes + (bytes >> 4) + 256;  // a little headroom so slowly growing batches do not realloc
  want = (want + 511) & ~(size_t)511;
  size_t got = 0;
  if (void *q = dev_cache().take(want, &got)) { p = q; cap = got; return TQ_OK; }
  cudaError_t e = cudaMalloc(&p, want);
  if (e == cudaErrorMemoryAllocation) {  // give cached blocks back to the driver and retry once
    cudaGetLastError();
    dev_cache().drain([](void *q) { cudaFree(q); });
    e = cudaMalloc(&p, want);
  }
  if (e != cudaSuccess) {
    p = nullptr;
    cap = 0;
    return cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
  }
  cap = want;
  return TQ_OK;
}
void DevBuf::release() {
  if (p && !dev_cache().give(p, cap)) cudaFree(p);
  p = nullptr;
  cap = 0;
}
int32_t PinBuf::reserve(size_t bytes) {
  if (bytes <= cap) return TQ_OK;
  release();
  size_t want = bytes + (bytes >> 4) + 256;
  want = (want + 4095) & ~(size_t)4095;
  size_t got = 0;
  if (void *q = pin_cache().take(want, &got)) { p = q; cap = got; return TQ_OK; }
  cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    cudaGetLastError();
    pin_cache().drain([](void *q) { cudaFreeHost(q); });
    e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
  }
  if (e != cudaSuccess) {
    p = nullptr;
    cap = 0;
    return cuda_fail(e, "cudaHostAlloc", __FILE__, __LINE__);
  }
  cap = want;
  return TQ_OK;
}
void PinBuf::release() {
  if (p && !pin_cache().give(p, cap)) cudaFreeHost(p);
  p = nullptr;
  cap = 0;
}

bool is_pinned_host(const void *p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

void host_bitmap_append(uint8_t *dst, int64_t dst_off, const uint8_t *src, int64_t n) {
  if (n <= 0) return;
  if ((dst_off & 7) == 0) {
    uint8_t *d = dst + (dst_off >> 3);
    size_t nb = bitmap_bytes(n);
    if (src) memcpy(d, src, nb); else memset(d, 0xFF, nb);
    if (n & 7) d[nb - 1] &= (uint8_t)((1u << (n & 7)) - 1);
    return;
  }
  // unaligned: clear the destination tail then OR bits in
  int sh = (int)(dst_off & 7);
  uint8_t *d = dst + (dst_off >> 3);
  d[0] &= (uint8_t)((1u << sh) - 1);
  size_t nb = bitmap_bytes(n);
  size_t out_bytes = bitmap_bytes(sh + n);
  for (size_t i = 1; i < out_bytes; i++) d[i] = 0;
  for (size_t i = 0; i < nb; i++) {
    uint8_t v = src ? src[i] : 0xFF;
    if (i == nb - 1 && (n & 7)) v &= (uint8_t)((1u << (n & 7)) - 1);
    d[i] |= (uint8_t)(v << sh);
    if (i + 1 < out_bytes) d[i + 1] |= (uint8_t)(v >> (8 - sh));
  }
}

void host_bitmap_extract(uint8_t *dst, const uint8_t *src, int64_t src_off, int64_t n) {
  if (n <= 0) return;
  size_t nb = bitmap_bytes(n);
  const uint8_t *s = src + (src_off >> 3);
  int sh = (int)(src_off & 7);
  if (sh == 0) {
    memcpy(dst, s, nb);
  } else {
    size_t src_bytes = bitmap_bytes(sh + n);
    for (size_t i = 0; i < nb; i++) {
      uint8_t lo = (uint8_t)(s[i] >> sh);
      uint8_t hi = (i + 1 < src_bytes) ? (uint8_t)(s[i + 1] << (8 - sh)) : 0;
      dst[i] = lo | hi;
    }
  }
  if (n & 7) dst[nb - 1] &= (uint8_t)((1u << (n & 7)) - 1);
}

__global__ void k_flush_l2(uint64_t *p, size_t n_words, uint64_t v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n_words; i += stride) p[i] = v + i;
}

}  // namespace tq

// =================================================================== C ABI
using namespace tq;

extern "C" {

int32_t tq_init(int32_t device_ordinal) {
  TQ_TRY(init_device(device_ordinal));
  return ensure_init();
}

int32_t tq_shutdown(void) {
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  if (!r.inited) return TQ_OK;
  cudaSetDevice(r.device);
  cudaDeviceSynchronize();
  dev_cache().drain([](void *q) { cudaFree(q); });
  pin_cache().drain([](void *q) { cudaFreeHost(q); });
  if (r.l2_scratch) cudaFree(r.l2_scratch);
  r.l2_scratch = nullptr;
  cudaEventDestroy(r.t0);
  cudaEventDestroy(r.t1);
  cudaStreamDestroy(r.compute);
  cudaStreamDestroy(r.h2d);
  cudaStreamDestroy(r.d2h);
  r.inited = false;
  return TQ_OK;
}

int32_t tq_last_error(char *buf, int32_t buf_len) {
  if (!buf || buf_len <= 0) return TQ_ERR_INVALID_ARG;
  snprintf(buf, (size_t)buf_len, "%s", g_err);
  return TQ_OK;
}

const char *tq_version(void) { return "tinysql_b200 0.1 (sm_90a)"; }

int32_t tq_pinned_alloc(size_t bytes, void **out) {
  if (!out) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return TQ_OK;
}
int32_t tq_pinned_free(void *p) {
  if (!p) return TQ_OK;
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaFreeHost(p));
  return TQ_OK;
}
int32_t tq_device_alloc(size_t bytes, void **out) {
  if (!out) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  return TQ_OK;
}
int32_t tq_device_free(void *p) {
  if (!p) return TQ_OK;
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaFree(p));
  return TQ_OK;
}
int32_t tq_memcpy_h2d(void *dst_dev, const void *src_host, size_t bytes) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, rt().compute));
  TQ_CUDA(cudaStreamSynchronize(rt().compute));
  return TQ_OK;
}
int32_t tq_memcpy_d2h(void *dst_host, const void *src_dev, size_t bytes) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, rt().compute));
  TQ_CUDA(cudaStreamSynchronize(rt().compute));
  return TQ_OK;
}
int32_t tq_memcpy_d2d(void *dst_dev, const void *src_dev, size_t bytes) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaMemcpyAsync(dst_dev, src_dev, bytes, cudaMemcpyDeviceToDevice, rt().compute));
  TQ_CUDA(cudaStreamSynchronize(rt().compute));
  return TQ_OK;
}
int32_t tq_memset_device(void *dst_dev, int32_t byte_value, size_t bytes) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaMemsetAsync(dst_dev, byte_value, bytes, rt().compute));
  return TQ_OK;
}
int32_t tq_device_synchronize(void) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaDeviceSynchronize());
  return TQ_OK;
}
int32_t tq_compute_synchronize(void) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaStreamSynchronize(rt().compute));
  return TQ_OK;
}
int32_t tq_timer_start(void) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaEventRecord(rt().t0, rt().compute));
  return TQ_OK;
}
int32_t tq_timer_stop(float *elapsed_ms) {
  TQ_TRY(ensure_init());
  TQ_CUDA(cudaEventRecord(rt().t1, rt().compute));
  TQ_CUDA(cudaEventSynchronize(rt().t1));
  float ms = 0;
  TQ_CUDA(cudaEventElapsedTime(&ms, rt().t0, rt().t1));
  if (elapsed_ms) *elapsed_ms = ms;
  return TQ_OK;
}
int64_t tq_kernel_launch_count(void) { return rt().launches.load(); }

int32_t tq_enable_peer_access(int32_t peer_device) {
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  if (peer_device == r.device) return TQ_OK;
  int can = 0;
  TQ_CUDA(cudaDeviceCanAccessPeer(&can, r.device, peer_device));
  if (!can) { set_error("device %d cannot access device %d as a peer", r.device, peer_device); return TQ_ERR_NO_DEVICE; }
  const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return TQ_OK; }
  if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceEnablePeerAccess", __FILE__, __LINE__);
  return TQ_OK;
}

// CUDA IPC for the peer-memory exchange: buffers allocated by tq_device_alloc are exported as 64-byte handles and
// opened by the other ranks' processes while THEIR device is current (lazy peer access), so their kernels can store
// into this buffer over NVLink.
int32_t tq_ipc_get_handle(void *dev_ptr, void *handle64) {
  TQ_TRY(ensure_init());
  if (!dev_ptr || !handle64) return TQ_ERR_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaIpcMemHandle_t h;
  TQ_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
  memcpy(handle64, &h, 64);
  return TQ_OK;
}
int32_t tq_ipc_open_handle(const void *handle64, void **dev_ptr) {
  TQ_TRY(ensure_init());
  if (!handle64 || !dev_ptr) return TQ_ERR_INVALID_ARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  TQ_CUDA(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return TQ_OK;
}
int32_t tq_ipc_close_handle(void *dev_ptr) {
  TQ_TRY(ensure_init());
  if (!dev_ptr) return TQ_OK;
  TQ_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return TQ_OK;
}

int32_t tq_flush_l2(void) {
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  const size_t bytes = 256u << 20;  // 5x the 50 MB L2
  if (!r.l2_scratch) {
    TQ_CUDA(cudaMalloc(&r.l2_scratch, bytes));
    r.l2_scratch_bytes = bytes;
  }
  k_flush_l2<<<r.sm_count * 4, 512, 0, r.compute>>>((uint64_t *)r.l2_scratch, bytes / 8, 0x5bd1e995ULL);
  return check_launch("k_flush_l2");
}

}  // extern "C"
