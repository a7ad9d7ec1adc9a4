// partition.cu — radix exchange prep for the multi-GPU path (the device-side shuffleIntermData,
// executor/aggregate.go:352-356): rows are split into n_parts partitions by the high bits of the key
// hash, stable within a partition.  Three launches: per-chunk histogram, exclusive scan over
// (partition-major, chunk-minor) counts, ordered scatter of every column.
#include "common.cuh"

namespace tq {

static constexpr int PART_MAXC = 16;
static constexpr int PART_MAX = 256;
static constexpr int PART_CHUNK = 2048;  // rows owned by one warp, walked in order (=> stable)

struct PartParams {
  int n_cols;
  DCol in[PART_MAXC];
  DColMut out[PART_MAXC];
  int key_col;
  int n_parts;
  int64_t n;
  int64_t n_chunks;
  uint32_t *counts;  // [part * n_chunks + chunk]
};

__device__ __forceinline__ int part_of(const PartParams &p, int64_t r) {
  if (!tqd::bm_not_null(p.in[p.key_col].bm, r)) return (int)(r % p.n_parts);  // NULL keys never match; spread them
  return (int)((tqd::mix64(p.in[p.key_col].data[r]) >> 40) % (uint64_t)p.n_parts);
}

__global__ void __launch_bounds__(256) k_part_hist(const PartParams p) {
  __shared__ uint32_t s_cnt[8][PART_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)blockIdx.x * 8 + warp;
  for (int i = lane; i < p.n_parts; i += 32) s_cnt[warp][i] = 0;
  __syncwarp();
  if (chunk < p.n_chunks) {
    const int64_t lo = chunk * PART_CHUNK;
    const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
    for (int64_t r = lo + lane; r < hi; r += 32) atomicAdd(&s_cnt[warp][part_of(p, r)], 1u);
    __syncwarp();
    for (int i = lane; i < p.n_parts; i += 32) p.counts[(int64_t)i * p.n_chunks + chunk] = s_cnt[warp][i];
  }
}

__global__ void __launch_bounds__(256) k_part_scatter(const PartParams p) {
  __shared__ uint32_t s_base[8][PART_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)blockIdx.x * 8 + warp;
  if (chunk >= p.n_chunks) return;
  for (int i = lane; i < p.n_parts; i += 32) s_base[warp][i] = p.counts[(int64_t)i * p.n_chunks + chunk];  // scanned: global offsets
  __syncwarp();
  const int64_t lo = chunk * PART_CHUNK;
  const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
  for (int64_t r0 = lo; r0 < hi; r0 += 32) {
    const int64_t r = r0 + lane;
    const bool active = r < hi;
    const int part = active ? part_of(p, r) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, part);
    const unsigned rank = __popc(peers & ((1u << lane) - 1));
    uint32_t pos = 0;
    if (active) pos = s_base[warp][part] + rank;
    __syncwarp();
    if (active && rank == (unsigned)__popc(peers) - 1) s_base[warp][part] = pos + 1;  // last peer advances the cursor
    __syncwarp();
    if (active) {
      for (int c = 0; c < p.n_cols; c++) {
        p.out[c].data[pos] = p.in[c].data[r];
        if (p.out[c].bm && tqd::bm_not_null(p.in[c].bm, r)) atomicOr(&p.out[c].bm[pos >> 5], 1u << (pos & 31));
      }
    }
  }
}

__global__ void k_part_offsets(const uint32_t *scanned, int64_t n_chunks, int n_parts, int64_t n, int64_t *offsets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_parts) offsets[i] = scanned[(int64_t)i * n_chunks];
  if (i == n_parts) offsets[i] = n;
}

}  // namespace tq

using namespace tq;

extern "C" int32_t tq_partition_device(int32_t n_cols, const tq_column *cols, const int32_t *types, int32_t key_col, int64_t n, int32_t n_parts,
                                       tq_column *out_cols, int64_t *part_offsets) {
  TQ_TRY(ensure_init());
  if (n_cols < 1 || n_cols > PART_MAXC || !cols || !types || !out_cols || !part_offsets || key_col < 0 || key_col >= n_cols || n_parts < 1 ||
      n_parts > PART_MAX || n < 0 || n > 0xFFFFFFF0ll) {
    set_error("tq_partition_device: bad arguments");
    return TQ_ERR_INVALID_ARG;
  }
  // the kernels move every column as 8-byte words: FLOAT32 slots are 4 bytes and BYTES cells live behind offsets
  for (int c = 0; c < n_cols; c++) {
    const int t = types[c] & 0xFF;
    if ((t != TQ_TYPE_INT64 && t != TQ_TYPE_UINT64 && t != TQ_TYPE_FLOAT64) || cols[c].offsets) {
      set_error("tq_partition_device: column %d is not an 8-byte fixed-width column (type %d)", c, types[c]);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
    if (cols[c].null_bitmap && !out_cols[c].null_bitmap) { set_error("output column %d needs a null bitmap", c); return TQ_ERR_INVALID_ARG; }
  }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.compute;
  if (n == 0) {
    for (int i = 0; i <= n_parts; i++) part_offsets[i] = 0;
    return TQ_OK;
  }
  static DevBuf counts, scan_scratch, d_off;
  static PinBuf h_off;
  PartParams p{};
  p.n_cols = n_cols;
  p.key_col = key_col;
  p.n_parts = n_parts;
  p.n = n;
  p.n_chunks = (n + PART_CHUNK - 1) / PART_CHUNK;
  for (int c = 0; c < n_cols; c++) {
    p.in[c].data = (const uint64_t *)cols[c].data;
    p.in[c].bm = (const uint32_t *)cols[c].null_bitmap;
    p.out[c].data = (uint64_t *)out_cols[c].data;
    p.out[c].bm = cols[c].null_bitmap ? (uint32_t *)out_cols[c].null_bitmap : nullptr;
    if (p.out[c].bm) TQ_CUDA(cudaMemsetAsync(p.out[c].bm, 0, bitmap_alloc_bytes(n) - 8, s));
    out_cols[c].length = n;
  }
  const int64_t n_counts = p.n_chunks * n_parts;
  TQ_TRY(counts.reserve((size_t)n_counts * 4));
  TQ_TRY(d_off.reserve((size_t)(n_parts + 1) * 8));
  TQ_TRY(h_off.reserve((size_t)(n_parts + 1) * 8));
  p.counts = counts.as<uint32_t>();
  const unsigned blocks = (unsigned)((p.n_chunks + 7) / 8);
  TQ_LAUNCH(k_part_hist, blocks, 256, 0, s, p);
  count_launch();
  TQ_TRY(check_launch("k_part_hist"));
  TQ_TRY(exclusive_scan_u32(p.counts, 1, p.counts, 1, n_counts, nullptr, scan_scratch, s));
  TQ_LAUNCH(k_part_offsets, (n_parts + 1 + 255) / 256, 256, 0, s, p.counts, p.n_chunks, n_parts, n, d_off.as<int64_t>());
  TQ_LAUNCH(k_part_scatter, blocks, 256, 0, s, p);
  count_launch(2);
  TQ_TRY(check_launch("k_part_scatter"));
  TQ_CUDA(cudaMemcpyAsync(h_off.p, d_off.p, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  memcpy(part_offsets, h_off.p, (size_t)(n_parts + 1) * 8);
  return TQ_OK;
}
