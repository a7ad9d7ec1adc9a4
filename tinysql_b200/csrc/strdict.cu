// strdict.cu — see strdict.cuh.  One warp per cell: coalesced byte reads for hashing and for the exact comparison with the
// slot's representative string.  Byte movement + L2-resident slot probes: HBM/L2-bound, no tensor cores.
#include "strdict.cuh"

namespace tq {

static constexpr uint32_t SD_EMPTY = 0xFFFFFFFFu, SD_BATCH = 0x80000000u;
static constexpr uint64_t SD_MIN_SLOTS = 1ull << 10;

static int sd_warp_grid(int64_t n_warps) {  // CTAs of 8 warps
  const int64_t blocks = (n_warps + 7) / 8;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}
static int sd_thread_grid(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// 64-bit hash of a byte range, computed by the whole warp: lane l folds the 8-byte groups l, l+32, ... and the lanes'
// states are mixed and summed.  Only a bucket chooser / compare filter: equality is decided on the bytes.
__device__ __forceinline__ uint64_t sd_warp_hash(const uint8_t *p, int64_t len) {
  const int lane = threadIdx.x & 31;
  uint64_t h = 0x9E3779B97F4A7C15ull + (uint64_t)lane * 0xD6E8FEB86659FD93ull;
  for (int64_t o = (int64_t)lane * 8; o < len; o += 256) {
    const int m = (len - o) < 8 ? (int)(len - o) : 8;
    uint64_t w = 0;
    for (int b = 0; b < m; b++) w |= (uint64_t)p[o + b] << (8 * b);
    h = (h ^ w) * 0xff51afd7ed558ccdULL;
    h ^= h >> 32;
  }
  h = tqd::mix64(h);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) h += __shfl_xor_sync(0xffffffffu, h, d);
  return tqd::mix64(h ^ ((uint64_t)len * 0x9E3779B97F4A7C15ull));
}

// exact equality of two byte ranges of the same length (all 32 lanes call)
__device__ __forceinline__ bool sd_warp_equal(const uint8_t *a, const uint8_t *b, int64_t len) {
  const int lane = threadIdx.x & 31;
  for (int64_t o0 = 0; o0 < len; o0 += 256) {
    const int64_t o = o0 + (int64_t)lane * 8;
    bool diff = false;
    if (o < len) {
      const int m = (len - o) < 8 ? (int)(len - o) : 8;
      for (int k = 0; k < m; k++) diff |= a[o + k] != b[o + k];
    }
    if (__any_sync(0xffffffffu, diff)) return false;
  }
  return true;
}

__global__ void __launch_bounds__(256) k_sd_hash(const StrView v, const uint32_t *bm, int64_t n, uint64_t *row_hash) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += n_warps) {
    if (!tqd::bm_not_null(bm, r)) continue;
    const int64_t s0 = v.off[r], s1 = v.off[r + 1];
    const uint64_t h = sd_warp_hash(v.bytes + (s0 - v.base), s1 - s0);
    if (lane == 0) row_hash[r] = h;
  }
}

// Claim a slot per distinct string of the batch.  A slot is claimed with its representative's BATCH ROW (the batch store
// is immutable while this kernel runs, so every other warp can compare against it at once — no waiting on a publisher).
__global__ void __launch_bounds__(256) k_sd_insert(const StrView v, const uint32_t *bm, int64_t n, const uint64_t *row_hash, uint32_t *slots, uint64_t mask,
                                                    const int64_t *a_off, const uint64_t *a_hash, const uint8_t *a_bytes) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += n_warps) {
    if (!tqd::bm_not_null(bm, r)) continue;
    const uint64_t h = row_hash[r];
    const int64_t s0 = v.off[r], len = v.off[r + 1] - s0;
    const uint8_t *p = v.bytes + (s0 - v.base);
    uint64_t s = h & mask;
    for (;;) {
      uint32_t rep = 0;
      int won = 0;
      if (lane == 0) {
        rep = *reinterpret_cast<volatile uint32_t *>(&slots[s]);
        if (rep == SD_EMPTY) {
          const uint32_t prev = atomicCAS(&slots[s], SD_EMPTY, SD_BATCH | (uint32_t)r);
          if (prev == SD_EMPTY) won = 1;
          rep = prev;
        }
      }
      won = __shfl_sync(0xffffffffu, won, 0);
      if (won) break;
      rep = __shfl_sync(0xffffffffu, rep, 0);
      const uint8_t *q;
      int64_t qlen;
      uint64_t qh;
      if (rep & SD_BATCH) {
        const int64_t r2 = (int64_t)(rep & ~SD_BATCH);
        qh = row_hash[r2];
        const int64_t q0 = v.off[r2];
        qlen = v.off[r2 + 1] - q0;
        q = v.bytes + (q0 - v.base);
      } else {
        qh = a_hash[rep];
        const int64_t q0 = a_off[rep];
        qlen = a_off[rep + 1] - q0;
        q = a_bytes + q0;
      }
      if (qh == h && qlen == len && sd_warp_equal(p, q, len)) break;
      s = (s + 1) & mask;
    }
  }
}

// Every slot still holding a batch row becomes a new arena string: draw its id, remember where its bytes come from.
__global__ void __launch_bounds__(256) k_sd_assign(uint32_t *slots, uint64_t n_slots, const StrView v, const uint64_t *row_hash, uint32_t count0, unsigned *n_new,
                                                    uint32_t *new_src, uint32_t *new_len, uint64_t *a_hash) {
  uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; s < n_slots; s += stride) {
    const uint32_t rep = slots[s];
    if (rep == SD_EMPTY || !(rep & SD_BATCH)) continue;
    const uint32_t r = rep & ~SD_BATCH;
    const uint32_t j = atomicAdd(n_new, 1u);
    new_src[j] = r;
    new_len[j] = (uint32_t)(v.off[r + 1] - v.off[r]);
    a_hash[count0 + j] = row_hash[r];
    slots[s] = count0 + j;
  }
}

__global__ void __launch_bounds__(256) k_sd_copy(const StrView v, const uint32_t *new_src, const uint32_t *new_off, uint32_t n_new, uint64_t used0, uint32_t count0,
                                                  const uint64_t *d_total, int64_t *a_off, uint8_t *a_bytes) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  if (warp == 0 && lane == 0) a_off[count0 + n_new] = (int64_t)(used0 + *d_total);
  for (int64_t j = warp; j < (int64_t)n_new; j += n_warps) {
    const uint32_t r = new_src[j];
    const int64_t s0 = v.off[r], len = v.off[r + 1] - s0;
    const uint8_t *src = v.bytes + (s0 - v.base);
    uint8_t *dst = a_bytes + used0 + new_off[j];
    if (lane == 0) a_off[count0 + j] = (int64_t)(used0 + new_off[j]);
    for (int64_t b = lane; b < len; b += 32) dst[b] = src[b];
  }
}

// Rows are handled 32 at a time by one warp so that the validity word of the group is assembled in a register.
__global__ void __launch_bounds__(256) k_sd_lookup(const StrView v, const uint32_t *bm, int64_t n, const uint64_t *row_hash, const uint32_t *slots, uint64_t mask,
                                                    const int64_t *a_off, const uint64_t *a_hash, const uint8_t *a_bytes, uint64_t *ids_out, uint32_t *valid_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n_groups = (n + 31) >> 5;
  for (int64_t g = warp; g < n_groups; g += n_warps) {
    uint32_t word = 0;
    for (int i = 0; i < 32; i++) {
      const int64_t r = g * 32 + i;
      if (r >= n) break;
      uint64_t id = SD_ID_MISS;
      if (tqd::bm_not_null(bm, r)) {
        const uint64_t h = row_hash[r];
        const int64_t s0 = v.off[r], len = v.off[r + 1] - s0;
        const uint8_t *p = v.bytes + (s0 - v.base);
        uint64_t s = h & mask;
        for (;;) {
          const uint32_t rep = slots[s];  // same address in every lane: one transaction
          if (rep == SD_EMPTY) break;
          const int64_t q0 = a_off[rep];
          if (a_hash[rep] == h && a_off[rep + 1] - q0 == len && sd_warp_equal(p, a_bytes + q0, len)) { id = rep; break; }
          s = (s + 1) & mask;
        }
      }
      if (lane == 0) ids_out[r] = id;
      if (id != SD_ID_MISS) word |= 1u << i;
    }
    if (lane == 0 && valid_out) valid_out[g] = word;
  }
}

__global__ void __launch_bounds__(256) k_sd_rehash(uint32_t *slots, uint64_t mask, const uint64_t *a_hash, uint64_t count) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < count; i += stride) {
    uint64_t s = a_hash[i] & mask;
    for (;;) {
      if (atomicCAS(&slots[s], SD_EMPTY, (uint32_t)i) == SD_EMPTY) break;
      s = (s + 1) & mask;
    }
  }
}

// grow a device array, keeping its first `keep` bytes
static int32_t grow_keep(DevBuf &b, size_t keep, size_t want, cudaStream_t s) {
  if (want <= b.cap) return TQ_OK;
  DevBuf nb;
  TQ_TRY(nb.reserve(want + (want >> 1)));
  if (keep) TQ_CUDA(cudaMemcpyAsync(nb.p, b.p, keep, cudaMemcpyDeviceToDevice, s));
  TQ_CUDA(cudaStreamSynchronize(s));  // the old block goes back to the allocator
  b = std::move(nb);
  return TQ_OK;
}

int32_t StringDict::ensure(uint64_t extra_strings, uint64_t extra_bytes, cudaStream_t s) {
  if (count + extra_strings > 0x7FFFFFF0ull) { set_error("string dictionary: more than 2^31 distinct strings"); return TQ_ERR_INVALID_ARG; }
  if (!meta.p) {
    TQ_TRY(meta.reserve(64));
    TQ_TRY(arena.offsets.reserve(8 * 1024));
    TQ_CUDA(cudaMemsetAsync(arena.offsets.p, 0, 8, s));  // offsets[0] = 0
    arena.elem = 0;
    arena.base = 0;
  }
  TQ_TRY(grow_keep(arena.offsets, (size_t)(count + 1) * 8, (size_t)(count + extra_strings + 1) * 8, s));
  TQ_TRY(grow_keep(a_hash, (size_t)count * 8, (size_t)(count + extra_strings + 1) * 8, s));
  TQ_TRY(grow_keep(arena.bytes, (size_t)used_bytes, (size_t)(used_bytes + extra_bytes) + 16, s));
  uint64_t want = n_slots ? n_slots : SD_MIN_SLOTS;
  while (want < (count + extra_strings) * 2) want <<= 1;
  if (want != n_slots) {
    DevBuf ns;
    TQ_TRY(ns.reserve((size_t)want * 4));
    TQ_CUDA(cudaMemsetAsync(ns.p, 0xFF, (size_t)want * 4, s));
    if (count) {
      TQ_LAUNCH(k_sd_rehash, sd_thread_grid((int64_t)count), 256, 0, s, ns.as<uint32_t>(), want - 1, a_hash.as<uint64_t>(), count);
      count_launch();
      TQ_TRY(check_launch("k_sd_rehash"));
    }
    TQ_CUDA(cudaStreamSynchronize(s));
    slots = std::move(ns);
    n_slots = want;
  }
  return TQ_OK;
}

int32_t StringDict::encode(const StrView &v, const uint32_t *bm, int64_t n, int64_t batch_bytes, bool insert, uint64_t *ids_out, uint32_t *valid_out,
                           cudaStream_t s) {
  if (n > 0x7FFFFFF0ll) { set_error("string key batch of %lld rows is too large", (long long)n); return TQ_ERR_INVALID_ARG; }
  TQ_TRY(ensure(insert ? (uint64_t)n : 0, insert ? (uint64_t)(batch_bytes > 0 ? batch_bytes : 0) : 0, s));
  if (n <= 0) return TQ_OK;
  TQ_TRY(row_hash.reserve((size_t)n * 8));
  TQ_LAUNCH(k_sd_hash, sd_warp_grid(n), 256, 0, s, v, bm, n, row_hash.as<uint64_t>());
  count_launch();
  TQ_TRY(check_launch("k_sd_hash"));
  if (insert) {
    TQ_TRY(new_src.reserve((size_t)n * 4));
    TQ_TRY(new_len.reserve((size_t)n * 4 + 8));
    TQ_TRY(new_off.reserve((size_t)n * 4 + 8));
    unsigned *d_n_new = meta.as<unsigned>();
    uint64_t *d_total = reinterpret_cast<uint64_t *>(meta.as<uint8_t>() + 8);
    TQ_CUDA(cudaMemsetAsync(meta.p, 0, 16, s));
    TQ_LAUNCH(k_sd_insert, sd_warp_grid(n), 256, 0, s, v, bm, n, row_hash.as<uint64_t>(), slots.as<uint32_t>(), n_slots - 1, arena.offsets.as<int64_t>(), a_hash.as<uint64_t>(),
              arena.bytes.as<uint8_t>());
    TQ_LAUNCH(k_sd_assign, sd_thread_grid((int64_t)n_slots), 256, 0, s, slots.as<uint32_t>(), n_slots, v, row_hash.as<uint64_t>(), (uint32_t)count, d_n_new, new_src.as<uint32_t>(),
              new_len.as<uint32_t>(), a_hash.as<uint64_t>());
    count_launch(2);
    TQ_TRY(check_launch("k_sd_assign"));
    unsigned n_new = 0;
    TQ_CUDA(cudaMemcpyAsync(&n_new, d_n_new, 4, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    if (n_new) {
      TQ_TRY(exclusive_scan_u32(new_len.as<uint32_t>(), 1, new_off.as<uint32_t>(), 1, (int64_t)n_new, d_total, scan_scratch, s));
      TQ_LAUNCH(k_sd_copy, sd_warp_grid((int64_t)n_new), 256, 0, s, v, new_src.as<uint32_t>(), new_off.as<uint32_t>(), n_new, used_bytes, (uint32_t)count, d_total,
                arena.offsets.as<int64_t>(), arena.bytes.as<uint8_t>());
      count_launch();
      TQ_TRY(check_launch("k_sd_copy"));
      uint64_t total = 0;
      TQ_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, s));
      TQ_CUDA(cudaStreamSynchronize(s));
      if (total > 0xFFFFFFF0ull) { set_error("string dictionary: more than 4 GiB of new distinct strings in one batch"); return TQ_ERR_INVALID_ARG; }
      count += n_new;
      used_bytes += total;
      arena.n = (int64_t)count;
    }
  }
  TQ_LAUNCH(k_sd_lookup, sd_warp_grid((n + 31) >> 5), 256, 0, s, v, bm, n, row_hash.as<uint64_t>(), slots.as<uint32_t>(), n_slots - 1, arena.offsets.as<int64_t>(),
            a_hash.as<uint64_t>(), arena.bytes.as<uint8_t>(), ids_out, valid_out);
  count_launch();
  return check_launch("k_sd_lookup");
}

void StringDict::release() {
  arena.offsets.release();
  arena.bytes.release();
  a_hash.release();
  slots.release();
  row_hash.release();
  new_src.release();
  new_len.release();
  new_off.release();
  n_slots = count = used_bytes = 0;
}

}  // namespace tq
