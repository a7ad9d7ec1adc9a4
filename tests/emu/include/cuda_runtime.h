// cuda_runtime.h of the CPU EMULATION build (tests/emu) — TEST INFRASTRUCTURE, never part of the product library.
//
// tests/emu compiles product sources (tinysql_b200/csrc/sort.cu, codec.cu, dict.cu, strdict.cu, partition.cu ...) unchanged with g++: this header stands in for the CUDA
// runtime and maps the handful of device primitives those kernels use onto host threads — ONE OS thread per CUDA thread of a
// block, blocks run one after another, __syncthreads() and the warp collectives are pthread barriers.  Slow, but it executes
// the real kernel code (indexing, ranking, masks, binary searches) so `-m "not gpu"` can check it against the oracle.
#pragma once
#include <ucontext.h>

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

// ------------------------------------------------------------------ host runtime stand-ins
typedef int cudaError_t;
static const cudaError_t cudaSuccess = 0;
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
static inline cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t n, cudaMemcpyKind, cudaStream_t) { if (n) memcpy(dst, src, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *dst, int v, size_t n, cudaStream_t) { if (n) memset(dst, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = nullptr; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t) { return "emulation"; }

// ------------------------------------------------------------------ device language stand-ins
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

struct ulonglong2 { unsigned long long x, y; };

namespace tq_emu {
// One OS thread runs everything: each CUDA thread of the current block is a FIBER (ucontext); a barrier switches to the next
// fiber until every participant has arrived.  Blocks run one after another.
extern dim3 t_threadIdx, t_blockIdx, t_blockDim, t_gridDim;
extern int cur;                       // fiber (= threadIdx.x) that is running
extern uint64_t warp_slot[32][32];    // exchange slots of the warp collectives: [warp][lane]
void launch(dim3 grid, dim3 block, const std::function<void()> &body);
void block_sync();
void warp_sync();
}  // namespace tq_emu

#define threadIdx tq_emu::t_threadIdx
#define blockIdx tq_emu::t_blockIdx
#define blockDim tq_emu::t_blockDim
#define gridDim tq_emu::t_gridDim
#define TQ_LAUNCH(kernel, grid, block, smem, stream, ...) tq_emu::launch(dim3(grid), dim3(block), [&] { kernel(__VA_ARGS__); })

static inline void __syncthreads() { tq_emu::block_sync(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { tq_emu::warp_sync(); }   // every lane of the warp arrives (see below)

// warp collectives: every lane of the warp takes part (the kernels keep whole warps converged around them)
template <typename T>
static inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  const int w = tq_emu::cur >> 5, lane = tq_emu::cur & 31;
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  tq_emu::warp_slot[w][lane] = bits;
  tq_emu::warp_sync();
  const uint64_t got = tq_emu::warp_slot[w][lane ^ lane_mask];
  tq_emu::warp_sync();
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}
template <typename T>
static inline T __shfl_sync(unsigned, T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  const int w = tq_emu::cur >> 5, lane = tq_emu::cur & 31;
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  tq_emu::warp_slot[w][lane] = bits;
  tq_emu::warp_sync();
  const uint64_t got = tq_emu::warp_slot[w][src_lane & 31];
  tq_emu::warp_sync();
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}
template <typename T>
static inline T __shfl_up_sync(unsigned, T v, unsigned delta) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  const int w = tq_emu::cur >> 5, lane = tq_emu::cur & 31;
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  tq_emu::warp_slot[w][lane] = bits;
  tq_emu::warp_sync();
  const uint64_t got = tq_emu::warp_slot[w][lane >= (int)delta ? lane - (int)delta : lane];   // lanes below delta keep their own value
  tq_emu::warp_sync();
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}
static inline unsigned __ballot_sync(unsigned, bool pred) {
  const int w = tq_emu::cur >> 5, lane = tq_emu::cur & 31;
  tq_emu::warp_slot[w][lane] = pred ? 1 : 0;
  tq_emu::warp_sync();
  unsigned m = 0;
  for (int l = 0; l < 32; l++) if (tq_emu::warp_slot[w][l]) m |= 1u << l;
  tq_emu::warp_sync();
  return m;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred != 0) != 0; }
static inline unsigned __match_any_sync(unsigned, unsigned v) {
  const int w = tq_emu::cur >> 5, lane = tq_emu::cur & 31;
  tq_emu::warp_slot[w][lane] = v;
  tq_emu::warp_sync();
  unsigned m = 0;
  for (int l = 0; l < 32; l++) if (tq_emu::warp_slot[w][l] == (uint64_t)v) m |= 1u << l;
  tq_emu::warp_sync();
  return m;
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }

static inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicCAS(unsigned *p, unsigned expected, unsigned v) {
  __atomic_compare_exchange_n(p, &expected, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;   // the old value, whether or not it was swapped
}
static inline unsigned long long atomicCAS(unsigned long long *p, unsigned long long expected, unsigned long long v) {
  __atomic_compare_exchange_n(p, &expected, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}
static inline unsigned long long atomicMax(unsigned long long *p, unsigned long long v) {
  unsigned long long cur = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (cur < v && !__atomic_compare_exchange_n(p, &cur, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return cur;
}
static inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicOr(unsigned long long *p, unsigned long long v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAnd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_and(p, v, __ATOMIC_SEQ_CST); }

static inline long long __double_as_longlong(double d) { long long r; memcpy(&r, &d, 8); return r; }
static inline double __longlong_as_double(long long v) { double r; memcpy(&r, &v, 8); return r; }
static inline float __uint_as_float(unsigned v) { float r; memcpy(&r, &v, 4); return r; }
static inline unsigned __float_as_uint(float v) { unsigned r; memcpy(&r, &v, 4); return r; }
