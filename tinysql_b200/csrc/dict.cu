// dict.cu — value -> dense id dictionaries and the exact N-column key fold (see dict.cuh).
//
// Reference semantics restated here: the key of a row is the tuple of its key-column values; two rows meet iff every
// column is equal by (flag, raw 8 bytes) (util/codec/codec.go:363-382 EqualChunkRow; :212-240 encodeHashChunkRowIdx).
// All kernels are 8-byte gather/scatter work on an L2-resident table: HBM/L2-bound, no tensor cores.
#include "dict.cuh"

namespace tq {

static constexpr uint64_t DICT_EMPTY = 0xA5C3F00DDEADBEEFull;
static constexpr int64_t DICT_SUB_BATCH = 1ll << 24;  // rows per insert launch: bounds how far capacity must run ahead
static constexpr uint64_t DICT_MIN_SLOTS = 1ull << 12;

static int dict_grid(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

__global__ void k_dict_fill(uint64_t *keys, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) keys[i] = DICT_EMPTY;
}

// Claim a slot per distinct value; the claiming thread draws the next dense id.
__global__ void __launch_bounds__(256) k_dict_insert(uint64_t *keys, uint32_t *ids, uint64_t mask, unsigned *next_id, const uint64_t *vals,
                                                      const uint32_t *bm, int64_t r0, int64_t n, int skip_miss) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t r = r0 + i;
    if (!tqd::bm_not_null(bm, r)) continue;
    const uint64_t v = vals[r];
    if (v == DICT_EMPTY) continue;                 // reserved id MK_ID_EMPTYVAL
    if (skip_miss && v == MK_PAIR_MISS) continue;
    uint64_t idx = tqd::mix64(v) & mask;
    for (;;) {
      const unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(keys + idx);
      if (cur == v) break;
      if (cur == DICT_EMPTY) {
        const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(keys + idx), (unsigned long long)DICT_EMPTY, (unsigned long long)v);
        if (prev == DICT_EMPTY) { ids[idx] = atomicAdd(next_id, 1u) + 2u; break; }
        if (prev == v) break;
      }
      idx = (idx + 1) & mask;
    }
  }
}

__global__ void __launch_bounds__(256) k_dict_lookup(const uint64_t *keys, const uint32_t *ids, uint64_t mask, const uint64_t *vals, const uint32_t *bm,
                                                      int64_t n, uint32_t null_id, int no_signbit, int skip_miss, uint32_t *out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint32_t id = MK_ID_MISS;
    if (!tqd::bm_not_null(bm, r)) id = null_id;
    else {
      const uint64_t v = vals[r];
      if (skip_miss && v == MK_PAIR_MISS) id = MK_ID_MISS;
      else if (no_signbit && (v >> 63)) id = MK_ID_MISS;  // signed vs unsigned: equal only when both are < 2^63 (codec.go:219-231)
      else if (v == DICT_EMPTY) id = MK_ID_EMPTYVAL;
      else {
        uint64_t idx = tqd::mix64(v) & mask;
        for (;;) {
          const uint64_t cur = keys[idx];
          if (cur == v) { id = ids[idx]; break; }
          if (cur == DICT_EMPTY) break;
          idx = (idx + 1) & mask;
        }
      }
    }
    out[r] = id;
  }
}

__global__ void __launch_bounds__(256) k_dict_rehash(const uint64_t *old_keys, const uint32_t *old_ids, uint64_t old_slots, uint64_t *new_keys,
                                                      uint32_t *new_ids, uint64_t new_mask) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < old_slots; i += stride) {
    const uint64_t v = old_keys[i];
    if (v == DICT_EMPTY) continue;
    uint64_t idx = tqd::mix64(v) & new_mask;
    for (;;) {
      const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(new_keys + idx), (unsigned long long)DICT_EMPTY, (unsigned long long)v);
      if (prev == DICT_EMPTY) break;
      idx = (idx + 1) & new_mask;
    }
    new_ids[idx] = old_ids[i];
  }
}

// pair = a << 32 | b, or MK_PAIR_MISS when either id is a miss
__global__ void __launch_bounds__(256) k_dict_pair(const uint32_t *a, const uint32_t *b, int64_t n, uint64_t *out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    const uint32_t x = a[r], y = b[r];
    out[r] = (x == MK_ID_MISS || y == MK_ID_MISS) ? MK_PAIR_MISS : (((uint64_t)x << 32) | (uint64_t)y);
  }
}

// NOT-NULL bitmap of the encoded column: one 32-bit word per warp iteration
__global__ void __launch_bounds__(256) k_dict_valid_bitmap(const uint64_t *comb, int64_t n, uint32_t *bm) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_round = (n + 31) & ~31ll;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_round; r += stride) {
    const bool valid = r < n && comb[r] != MK_PAIR_MISS;
    const unsigned w = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0) bm[r >> 5] = w;
  }
}

int32_t KeyDict::ensure(uint64_t extra, cudaStream_t s) {
  uint64_t want = n_slots ? n_slots : DICT_MIN_SLOTS;
  while (want < (count + extra) * 2) want <<= 1;
  if (want == n_slots) return TQ_OK;
  if (want > (1ull << 33)) { set_error("key dictionary too large (%llu distinct values)", (unsigned long long)(count + extra)); return TQ_ERR_OOM; }
  DevBuf nk, ni;
  TQ_TRY(nk.reserve(want * 8));
  TQ_TRY(ni.reserve(want * 4));
  TQ_LAUNCH(k_dict_fill, dict_grid((int64_t)want), 256, 0, s, nk.as<uint64_t>(), want);
  count_launch();
  if (n_slots == 0) {
    TQ_TRY(meta.reserve(64));
    TQ_CUDA(cudaMemsetAsync(meta.p, 0, 64, s));
  } else {
    TQ_LAUNCH(k_dict_rehash, dict_grid((int64_t)n_slots), 256, 0, s, keys.as<uint64_t>(), ids.as<uint32_t>(), n_slots, nk.as<uint64_t>(), ni.as<uint32_t>(), want - 1);
    count_launch();
  }
  TQ_TRY(check_launch("k_dict_rehash"));
  TQ_CUDA(cudaStreamSynchronize(s));  // the old table is released below
  keys = std::move(nk);
  ids = std::move(ni);
  n_slots = want;
  return TQ_OK;
}

int32_t KeyDict::insert(const uint64_t *vals, const uint32_t *bm, int64_t n, bool skip_miss, cudaStream_t s) {
  for (int64_t off = 0; off < n; off += DICT_SUB_BATCH) {
    const int64_t m = n - off < DICT_SUB_BATCH ? n - off : DICT_SUB_BATCH;
    TQ_TRY(ensure((uint64_t)m, s));
    TQ_LAUNCH(k_dict_insert, dict_grid(m), 256, 0, s, keys.as<uint64_t>(), ids.as<uint32_t>(), n_slots - 1, meta.as<unsigned>(), vals, bm, off, m, skip_miss ? 1 : 0);
    count_launch();
    TQ_TRY(check_launch("k_dict_insert"));
    uint32_t c = 0;
    TQ_CUDA(cudaMemcpyAsync(&c, meta.p, 4, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    count = c;
    if (c > 0xFFFFFFF0u) { set_error("key dictionary: more than 2^32 distinct values in one key column"); return TQ_ERR_INVALID_ARG; }
  }
  return TQ_OK;
}

int32_t KeyDict::lookup(const uint64_t *vals, const uint32_t *bm, int64_t n, uint32_t null_id, bool no_signbit, bool skip_miss, uint32_t *out,
                        cudaStream_t s) const {
  if (n <= 0) return TQ_OK;
  if (n_slots == 0) { set_error("internal: lookup in an unallocated key dictionary"); return TQ_ERR_STATE; }
  TQ_LAUNCH(k_dict_lookup, dict_grid(n), 256, 0, s, keys.as<uint64_t>(), ids.as<uint32_t>(), n_slots - 1, vals, bm, n, null_id, no_signbit ? 1 : 0,
            skip_miss ? 1 : 0, out);
  count_launch();
  return check_launch("k_dict_lookup");
}

int32_t MultiKeyEncoder::encode(const DCol *keycols, const bool *no_signbit, int64_t n, bool insert, bool null_is_value, uint64_t *out_comb,
                                uint32_t *out_bm, cudaStream_t s) {
  if (k < 2 || k > MK_MAX_KEYS) { set_error("internal: multi-key encoder over %d columns", k); return TQ_ERR_INVALID_ARG; }
  // dictionaries exist (possibly empty) even when a side never inserts
  for (int i = 0; i < k; i++) {
    TQ_TRY(col[i].ensure(0, s));
    if (i >= 1 && i < k - 1) TQ_TRY(fold[i].ensure(0, s));
  }
  if (n <= 0) return TQ_OK;
  TQ_TRY(acc.reserve((size_t)n * 4));
  TQ_TRY(tmp.reserve((size_t)n * 4));
  if (k > 2) TQ_TRY(pair.reserve((size_t)n * 8));
  const uint32_t null_id = null_is_value ? MK_ID_NULL : MK_ID_MISS;
  if (insert)
    for (int i = 0; i < k; i++) TQ_TRY(col[i].insert(keycols[i].data, keycols[i].bm, n, false, s));
  TQ_TRY(col[0].lookup(keycols[0].data, keycols[0].bm, n, null_id, no_signbit && no_signbit[0], false, acc.as<uint32_t>(), s));
  for (int i = 1; i < k; i++) {
    TQ_TRY(col[i].lookup(keycols[i].data, keycols[i].bm, n, null_id, no_signbit && no_signbit[i], false, tmp.as<uint32_t>(), s));
    uint64_t *dst = (i == k - 1) ? out_comb : pair.as<uint64_t>();
    TQ_LAUNCH(k_dict_pair, dict_grid(n), 256, 0, s, acc.as<uint32_t>(), tmp.as<uint32_t>(), n, dst);
    count_launch();
    TQ_TRY(check_launch("k_dict_pair"));
    if (i < k - 1) {
      if (insert) TQ_TRY(fold[i].insert(dst, nullptr, n, true, s));
      TQ_TRY(fold[i].lookup(dst, nullptr, n, MK_ID_MISS, false, true, acc.as<uint32_t>(), s));
    }
  }
  if (out_bm) {
    TQ_LAUNCH(k_dict_valid_bitmap, dict_grid(n), 256, 0, s, out_comb, n, out_bm);
    count_launch();
    TQ_TRY(check_launch("k_dict_valid_bitmap"));
  }
  return TQ_OK;
}

void MultiKeyEncoder::release() {
  for (int i = 0; i < MK_MAX_KEYS; i++) {
    col[i].keys.release(); col[i].ids.release(); col[i].meta.release();
    fold[i].keys.release(); fold[i].ids.release(); fold[i].meta.release();
    col[i].n_slots = fold[i].n_slots = 0;
    col[i].count = fold[i].count = 0;
  }
  acc.release();
  tmp.release();
  pair.release();
}

}  // namespace tq
