// scan.cu — the device-wide exclusive scan of u32 counts that every operator sizes its outputs with (hash-table slot counts,
// partition counts, radix digit counts, merge-join group sizes, var-len cell lengths, string-dictionary arenas).
//
// Three small kernels: 64-bit sums of 4096-element tiles -> exclusive scan of the tile sums by one block -> rescan of each
// tile with its offset.  Kernels launch through TQ_LAUNCH, so tests/emu compiles this file unchanged and the emulated sort,
// merge join and dictionaries run the same scan as the product.
#include "common.cuh"

namespace tq {

static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_ITEMS = 16;  // per thread
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t *s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = (lane < (SCAN_THREADS / 32)) ? s_warp[lane] : 0;
    uint32_t winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += t;
    }
    if (lane < (SCAN_THREADS / 32)) s_warp[lane] = winc - w;
  }
  __syncthreads();
  uint32_t r = inc - v + s_warp[warp];
  __syncthreads();
  return r;
}

// block_sums[b] = sum of tile b, in 64 bits: one tile of 4096 counts can add up to more than 2^32 (4096 outer rows that each
// match 2^20 + 1 inner rows), and the callers' guards against a total >= 2^32 read the sum of these
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block_sums(const uint32_t *in, int stride, int64_t n, uint64_t *block_sums) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
  uint64_t sum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    const int64_t i = base + k;
    if (i < n) sum += in[i * stride];
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t total = 0;
#pragma unroll
    for (int w = 0; w < SCAN_THREADS / 32; w++) total += s_warp[w];
    block_sums[blockIdx.x] = total;
  }
}

// exclusive scan of the per-block sums by ONE CTA: thread t owns a contiguous run of ceil(n / 1024) sums
__global__ void __launch_bounds__(1024) k_scan_sums_serial(uint64_t *block_sums, int64_t n_blocks, uint64_t *total_out) {
  __shared__ uint64_t s_part[1024];
  const int t = threadIdx.x;
  const int64_t per = (n_blocks + 1023) / 1024;
  const int64_t lo = t * per, hi = (lo + per) < n_blocks ? (lo + per) : n_blocks;
  uint64_t sum = 0;
  for (int64_t i = lo; i < hi; i++) sum += block_sums[i];
  s_part[t] = sum;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {  // Hillis-Steele over 1024 partials
    const uint64_t v = t >= d ? s_part[t - d] : 0;
    __syncthreads();
    s_part[t] += v;
    __syncthreads();
  }
  uint64_t run = s_part[t] - sum;  // exclusive prefix of this thread's run
  for (int64_t i = lo; i < hi; i++) {
    const uint64_t v = block_sums[i];
    block_sums[i] = run;
    run += v;
  }
  if (t == 1023 && total_out) *total_out = s_part[1023];
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_final(const uint32_t *in, int in_stride, uint32_t *out, int out_stride, int64_t n,
                                                              const uint64_t *block_offsets) {
  __shared__ uint32_t s_warp[SCAN_THREADS / 32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS];
  uint32_t sum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    const int64_t i = base + k;
    v[k] = (i < n) ? in[i * in_stride] : 0;
    sum += v[k];
  }
  uint32_t run = block_exclusive_scan_256(sum, s_warp) + (uint32_t)block_offsets[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    const int64_t i = base + k;
    if (i < n) out[i * out_stride] = run;
    run += v[k];
  }
}

// The total is exact in 64 bits for any input.  The n exclusive offsets are 32-bit: exact whenever the total is below 2^32,
// which every caller either checks on *d_total before it uses them or bounds by construction; past that they wrap.
int32_t exclusive_scan_u32(const uint32_t *d_in, int in_stride_words, uint32_t *d_out, int out_stride_words, int64_t n,
                           uint64_t *d_total, DevBuf &scratch, cudaStream_t s) {
  if (n <= 0) {
    if (d_total) TQ_CUDA(cudaMemsetAsync(d_total, 0, 8, s));
    return TQ_OK;
  }
  const int64_t n_blocks = (n + SCAN_TILE - 1) / SCAN_TILE;
  TQ_TRY(scratch.reserve((size_t)n_blocks * 8));
  uint64_t *sums = scratch.as<uint64_t>();
  TQ_LAUNCH(k_scan_block_sums, (unsigned)n_blocks, SCAN_THREADS, 0, s, d_in, in_stride_words, n, sums);
  TQ_LAUNCH(k_scan_sums_serial, 1, 1024, 0, s, sums, n_blocks, d_total);
  TQ_LAUNCH(k_scan_final, (unsigned)n_blocks, SCAN_THREADS, 0, s, d_in, in_stride_words, d_out, out_stride_words, n, sums);
  count_launch(3);
  return check_launch("exclusive_scan_u32");
}

}  // namespace tq
