// common.cuh — shared host runtime + device helpers for libtinysql_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/tinysql_b200.h"

// Kernel launch.  sort.cu and codec.cu launch through this macro so that tests/emu can compile the SAME sources with g++
// against a thread-per-CUDA-thread emulation of the few primitives they use and check them against the oracle without a GPU
// (the emulation's cuda_runtime.h defines TQ_LAUNCH first).
#ifndef TQ_LAUNCH
#define TQ_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif
// A kernel parameter whose address is taken (sort.cu: k_mj_prog) is declared __grid_constant__ so that it stays in the
// parameter space; the emulation build has no such qualifier and takes the parameter by value.
#ifndef __grid_constant__
#define __grid_constant__
#endif

namespace tq {

// ---------------------------------------------------------------- errors (thread-local text)
void set_error(const char *fmt, ...);
int32_t cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define TQ_CUDA(x)                                                        \
  do {                                                                    \
    cudaError_t e__ = (x);                                                \
    if (e__ != cudaSuccess) return ::tq::cuda_fail(e__, #x, __FILE__, __LINE__); \
  } while (0)
#define TQ_TRY(x)                     \
  do {                                \
    int32_t s__ = (x);                \
    if (s__ != TQ_OK) return s__;     \
  } while (0)

// ---------------------------------------------------------------- runtime singleton
// One process drives one GPU.  Every kernel of the library is launched on `compute`;
// `h2d` / `d2h` carry the PCIe copies of the host (cgo) path so they overlap kernels.
struct Runtime {
  bool inited = false;
  int device = -1;
  int sm_count = 0;
  cudaStream_t compute = nullptr, h2d = nullptr, d2h = nullptr;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  std::recursive_mutex mu;  // serialises enqueue sections (handles may be driven by different threads)
  std::atomic<int64_t> launches{0};
  void *l2_scratch = nullptr;
  size_t l2_scratch_bytes = 0;
};
Runtime &rt();
int32_t ensure_init();  // TQ_ERR_NO_DEVICE when there is no usable GPU — never falls back to the CPU
inline void count_launch(int n = 1) { rt().launches.fetch_add(n, std::memory_order_relaxed); }
int32_t check_launch(const char *kernel);  // cudaGetLastError() -> status

// Grow-only device buffer (no frees / mallocs in steady state).
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept { if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; } return *this; }
  ~DevBuf() { release(); }
  int32_t reserve(size_t bytes);
  void release();
  template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};
// Grow-only pinned host buffer.
struct PinBuf {
  void *p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf &) = delete;
  PinBuf &operator=(const PinBuf &) = delete;
  PinBuf(PinBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  PinBuf &operator=(PinBuf &&o) noexcept { if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; } return *this; }
  ~PinBuf() { release(); }
  int32_t reserve(size_t bytes);
  void release();
  template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

inline size_t bitmap_bytes(int64_t n) { return (size_t)((n + 7) >> 3); }
// Bitmaps on the device are handled as 32-bit words; allocations are padded to 8 bytes.
inline size_t bitmap_alloc_bytes(int64_t n) { return (size_t)(((n + 63) >> 6) << 3) + 8; }
bool is_pinned_host(const void *p);

// Append `n` bits of src (bit i of src = row i) at bit offset dst_off of dst; src==nullptr appends 1s.
void host_bitmap_append(uint8_t *dst, int64_t dst_off, const uint8_t *src, int64_t n);
// Extract n bits starting at bit src_off into dst (dst starts at bit 0; tail bits of last byte zeroed).
void host_bitmap_extract(uint8_t *dst, const uint8_t *src, int64_t src_off, int64_t n);

// A device-resident column (8-byte slots).  bm == nullptr means "no NULLs".
struct DCol {
  const uint64_t *data = nullptr;
  const uint32_t *bm = nullptr;
};
struct DColMut {
  uint64_t *data = nullptr;
  uint32_t *bm = nullptr;
};

// device-wide exclusive scan of u32 counts (in place ok); total written to *d_total (u64) if non-null.
int32_t exclusive_scan_u32(const uint32_t *d_in, int in_stride_words, uint32_t *d_out, int out_stride_words,
                           int64_t n, uint64_t *d_total, DevBuf &scratch, cudaStream_t s);

}  // namespace tq

// ================================================================= device helpers
#ifdef __CUDACC__
namespace tqd {

// murmur3 fmix64: the device-side bucket/partition hash.  The reference hashes flag||8 bytes with
// FNV-1 (executor/hash_table.go:64); the hash only chooses buckets — equality is decided by
// (flag, raw bytes) (util/codec/codec.go:363-382) — so a different mixer cannot change results.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return k;
}

// Bucket / partition hash of the join tables: ONE 64-bit multiply.  Top bits = the high bits of a multiplicative
// (Fibonacci) hash, which choose the partition; the low 32 bits are lo32 ^ hi32 of the product, which choose the slot inside
// the partition.  The probe pipeline is instruction-issue-bound, and mix64's two 64-bit multiplies were a
// quarter of its instructions.  Like mix64 it only places rows — equality is always decided on the key itself.
__host__ __device__ __forceinline__ uint64_t hash_key(uint64_t k) {
  k ^= k >> 32;
  k *= 0x9E3779B97F4A7C15ULL;
  return k ^ (k >> 32);
}

__device__ __forceinline__ bool bm_not_null(const uint32_t *bm, int64_t i) {
  return bm == nullptr || ((bm[i >> 5] >> (i & 31)) & 1u);
}

// streaming 128-bit loads / stores (single-use data: keep it out of L1)
__device__ __forceinline__ ulonglong2 ld_stream_u64x2(const void *p) {
  ulonglong2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(r.x), "=l"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_u64x2(void *p, ulonglong2 v) {
  asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
}
__device__ __forceinline__ uint64_t ld_stream_u64(const void *p) {
  uint64_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_u64(void *p, uint64_t v) {
  asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

}  // namespace tqd
#endif
