// agg.cu — HashAggExec on the device (replaces executor/aggregate.go and executor/aggfuncs).
//
// One open-addressed table lives in L2: a dense KEY array probed in 4-key buckets (one 32-byte sector holds four
// candidate slots, so a lookup is ~one L2 round trip even at load factor 0.5; slots are claimed lock-free with
// atomicCAS) and an array-of-structs STATE array (the words of one group are contiguous: 16 bytes for SUM(f64) +
// COUNT, i.e. two groups per sector).  An input row costs the key bucket load plus one L2 reduction per updated
// state word (RED.ADD.F64 / RED.ADD.U64 / ATOM.MAX.U64).  Rows whose whole warp lands in one slot
// (scalar aggregates, heavy skew) are combined with warp shuffles first.
// Partial -> final (aggregate.go:96-133) is the same kernel in "merge" mode: COUNT adds partial counts,
// AVG adds (count, sum) pairs — the semantics of MergePartialResult.
#include <deque>
#include <memory>
#include <new>

#include "common.cuh"
#include "dict.cuh"
#include "scatter.cuh"
#include "strdict.cuh"
#include "varlen.cuh"

namespace tq {

static constexpr int AGG_MAXC = 16;
static constexpr int AGG_MAXF = 16;
static constexpr uint64_t AGG_EMPTY = 0xA5C3F00DDEADBEEFull;
static constexpr uint32_t SLOT_NONE = 0xFFFFFFFFu;

enum : unsigned { AERR_BIGINT = 1u };

// state words per function (8 bytes each, zero-initialised; w* are word offsets inside the slot, -1 = absent):
//   COUNT      w0 = count
//   SUM  f64   w0 = sum (double bits)                                 w1 = "a non-NULL input was seen" flag
//   SUM  int   w0 = sum low 64, w2 = sum high 64 (128-bit exact)      w1 = flag
//   AVG        like SUM, but w1 is the COUNT of non-NULL inputs (atomic)
//   MAX / MIN  w0 = order-mapped value (atomicMax)                    w1 = flag
//   FIRSTROW   w0 = value, w1 = 1 claimed | 3 claimed-and-NULL (claim by atomicCAS)
struct AggFuncDev {
  int func;
  int arg_col;     // -1: constant non-NULL 1
  int arg_col2;    // merge mode AVG: the partial-sum column (arg_col is the partial count)
  int arg_type;    // TQ_TYPE_* of the value being aggregated
  int key_passthrough;  // FIRSTROW over the GROUP BY column: answered from the slot key, no state
  int w0, w1, w2;       // word offsets of the state inside the slot
  int use_flag;         // SUM/MAX/MIN: maintain the "seen a non-NULL input" flag in w1
  int arg_not_null;     // the argument column is declared NOT NULL (mysql.NotNullFlag): no flag word, bitmaps ignored
  // string arguments (arg_type == TQ_TYPE_BYTES): the column holds dictionary ids; MAX / MIN compare the arena strings
  const int64_t *str_off;
  const uint8_t *str_bytes;
};

struct AggParams {
  int n_cols;
  DCol cols[AGG_MAXC];
  int key_col;  // -1: no GROUP BY (one group)
  int merge;    // 0: Partial1/Complete (raw rows)  1: Final (partial rows)
  int n_funcs;
  AggFuncDev f[AGG_MAXF];
  uint64_t *keys;             // keys[i] of slot i (AGG_EMPTY = free); probed as aligned buckets of 4
  uint64_t *tbl;              // state record of slot i = tbl[i * stride ...]
  int stride;                 // words per state record (power of two)
  uint64_t mask, n_slots;     // side slots: n_slots = NULL group, n_slots+1 = the AGG_EMPTY key
  uint32_t *side_used;        // [0] NULL group seen, [1] sentinel-key group seen
  unsigned long long *n_used; // occupied regular slots
  uint64_t limit;             // insertion of NEW keys stops here; such rows are deferred
  uint32_t *deferred;
  unsigned *n_deferred;
  const uint32_t *row_list;   // when set: process rows row_list[0..n)
  int64_t n;
};

__device__ __forceinline__ uint64_t order_map(uint64_t bits, int type) {
  // monotone map into unsigned order: signed -> flip sign bit; double -> IEEE total-order trick
  if (type == TQ_TYPE_UINT64) return bits;
  if (type == TQ_TYPE_INT64) return bits ^ 0x8000000000000000ull;
  return (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ uint64_t order_unmap(uint64_t m, int type) {
  if (type == TQ_TYPE_UINT64) return m;
  if (type == TQ_TYPE_INT64) return m ^ 0x8000000000000000ull;
  return (m >> 63) ? (m & 0x7fffffffffffffffull) : ~m;
}

__device__ __forceinline__ void add128(uint64_t *lo, uint64_t *hi, int64_t v) {
  const unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long *>(lo), (unsigned long long)v);
  const unsigned long long carry = (old + (unsigned long long)v) < old ? 1ull : 0ull;
  const unsigned long long hi_add = (unsigned long long)(v >> 63) + carry;  // sign extension + carry
  if (hi_add) atomicAdd(reinterpret_cast<unsigned long long *>(hi), hi_add);
}

// w1 bookkeeping: AVG needs the exact count of non-NULL inputs (atomic); SUM / MAX / MIN only need to know that one
// was seen — a flag that is read (same sector as the state just updated) and stored once, instead of an atomic per row.
// While no batch has carried a NULL bitmap for the argument the flag is not maintained at all (use_flag == 0): a group
// that exists then has a value by construction; the first nullable batch back-fills the flags (k_agg_set_flags).
__device__ __forceinline__ void note_seen(uint64_t *w1, bool exact_count, bool use_flag, long long cnt) {
  if (exact_count) atomicAdd(reinterpret_cast<unsigned long long *>(w1), (unsigned long long)cnt);
  else if (use_flag && *reinterpret_cast<volatile unsigned long long *>(w1) == 0ull) *reinterpret_cast<volatile unsigned long long *>(w1) = 1ull;  // use_flag is 0 when there is no flag word
}

// Apply one input row to its group's state (UpdatePartialResult / MergePartialResult).  Warp-collective: all 32 lanes call.
__device__ __forceinline__ void agg_apply(const AggParams &p, uint32_t slot, int64_t r) {
  const int lane = threadIdx.x & 31;
  const bool live = slot != SLOT_NONE;
  // warp-uniform group? then reduce with shuffles and let lane `leader` do the atomics
  const unsigned live_mask = __ballot_sync(0xffffffffu, live);
  if (live_mask == 0) return;
  const int leader = __ffs(live_mask) - 1;
  const uint32_t lead_slot = __shfl_sync(0xffffffffu, slot, leader);
  const bool uniform = __all_sync(0xffffffffu, !live || slot == lead_slot);
  uint64_t *const sl = p.tbl + (uint64_t)(live ? slot : 0) * p.stride;       // this row's slot record
  uint64_t *const lsl = p.tbl + (uint64_t)lead_slot * p.stride;              // the warp leader's
  for (int fi = 0; fi < p.n_funcs; fi++) {
    const AggFuncDev &f = p.f[fi];
    if (f.key_passthrough) continue;
    bool nn = false;
    uint64_t v = 1;
    if (live) {
      if (f.arg_col < 0) nn = true;
      else { nn = f.arg_not_null ? true : tqd::bm_not_null(p.cols[f.arg_col].bm, r); v = p.cols[f.arg_col].data[r]; }
    }
    switch (f.func) {
      case TQ_AGG_COUNT: {  // func_count.go:33-49 (raw: count non-NULL) / :99-113 (merge: add partial counts)
        const long long add = nn ? (p.merge ? (long long)v : 1ll) : 0ll;
        if (uniform) {  // 64-bit warp sum (counts in merge mode can exceed 32 bits)
          long long s = add;
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
          if (lane == leader && s) atomicAdd(reinterpret_cast<unsigned long long *>(lsl + f.w0), (unsigned long long)s);
        } else if (live && add) {
          atomicAdd(reinterpret_cast<unsigned long long *>(sl + f.w0), (unsigned long long)add);
        }
        break;
      }
      case TQ_AGG_SUM:
      case TQ_AGG_AVG: {
        // raw: func_sum.go:62-82,115-140; func_avg.go:63-83,172-190.   merge: func_sum.go:84-92,142-154; func_avg.go:93-131,200-238
        long long cnt_add = nn ? 1ll : 0ll;
        uint64_t val = v;
        bool val_nn = nn;
        if (p.merge && f.func == TQ_AGG_AVG) {
          // partial row = (count, sum): skipped if either is NULL (func_avg.go:96-110)
          bool nn2 = false; uint64_t v2 = 0;
          if (live) { nn2 = tqd::bm_not_null(p.cols[f.arg_col2].bm, r); v2 = p.cols[f.arg_col2].data[r]; }
          val_nn = nn && nn2;
          cnt_add = val_nn ? (long long)v : 0ll;
          val = v2;
        }
        const bool exact = f.func == TQ_AGG_AVG;
        if (f.arg_type == TQ_TYPE_FLOAT64) {
          double x = val_nn ? __longlong_as_double((long long)val) : 0.0;
          if (uniform) {
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) { x += __shfl_xor_sync(0xffffffffu, x, d); cnt_add += __shfl_xor_sync(0xffffffffu, cnt_add, d); }
            if (lane == leader && cnt_add) {
              atomicAdd(reinterpret_cast<double *>(lsl + f.w0), x);
              note_seen(lsl + f.w1, exact, f.use_flag, cnt_add);
            }
          } else if (live && val_nn) {
            atomicAdd(reinterpret_cast<double *>(sl + f.w0), x);
            note_seen(sl + f.w1, exact, f.use_flag, cnt_add);
          }
        } else {
          if (live && val_nn) {  // exact 128-bit accumulation; range is checked when the group is finalised
            add128(sl + f.w0, sl + f.w2, (int64_t)val);
            note_seen(sl + f.w1, exact, f.use_flag, cnt_add);
          }
        }
        break;
      }
      case TQ_AGG_MAX:
      case TQ_AGG_MIN: {  // func_max_min.go:83-118 (+ Uint / Float64 twins); merge is the same comparison
        if (f.arg_type == TQ_TYPE_BYTES) {
          // maxMin4String (func_max_min.go:337-361): the state word holds id + 1 of the best string so far (0 = none);
          // a candidate replaces it when types.CompareString says so — CAS loop, the compare reads the dictionary arena
          if (live && nn) {
            unsigned long long *w = reinterpret_cast<unsigned long long *>(sl + f.w0);
            unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(w);
            for (;;) {
              if (cur != 0ull) {
                if (cur == v + 1) break;
                const int c = sd_compare_ids(f.str_off, f.str_bytes, (uint32_t)v, (uint32_t)(cur - 1));
                if (!((f.func == TQ_AGG_MAX && c > 0) || (f.func == TQ_AGG_MIN && c < 0))) break;
              }
              const unsigned long long prev = atomicCAS(w, cur, (unsigned long long)v + 1);
              if (prev == cur) break;
              cur = prev;
            }
          }
          break;
        }
        if (live && nn) {
          uint64_t m = order_map(v, f.arg_type);
          if (f.func == TQ_AGG_MIN) m = ~m;
          atomicMax(reinterpret_cast<unsigned long long *>(sl + f.w0), (unsigned long long)m);
          note_seen(sl + f.w1, false, f.use_flag, 1);
        }
        break;
      }
      default: {  // FIRSTROW func_first_row.go:67-89: the first row to claim the group wins
        if (live) {
          const unsigned long long want = nn ? 1ull : 3ull;
          if (*reinterpret_cast<volatile unsigned long long *>(sl + f.w1) == 0ull) {
            const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(sl + f.w1), 0ull, want);
            if (prev == 0ull) sl[f.w0] = v;
          }
        }
        break;
      }
    }
  }
}

// four adjacent keys = one sector; volatile so concurrent inserts are observed (L1 is bypassed)
__device__ __forceinline__ void ld_bucket(const uint64_t *keys, uint64_t b, unsigned long long (&k)[4]) {
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(k[0]), "=l"(k[1]) : "l"(keys + b));
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(k[2]), "=l"(k[3]) : "l"(keys + b + 2));
}

__global__ void __launch_bounds__(256) k_agg_update(const AggParams p) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_round = (p.n + 31) & ~31ll;  // whole warps iterate together
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < n_round; it += stride) {
    uint32_t slot = SLOT_NONE;
    int64_t r = 0;
    bool claimed = false;
    if (it < p.n) {
      r = p.row_list ? (int64_t)p.row_list[it] : it;
      // ---- getGroupKey (aggregate.go:359-394): NULL is its own group (NilFlag, codec.go:718-720)
      if (p.key_col < 0 || !tqd::bm_not_null(p.cols[p.key_col].bm, r)) {
        slot = (uint32_t)p.n_slots;
        if (p.side_used[0] == 0) p.side_used[0] = 1;
      } else {
        const uint64_t key = tqd::ld_stream_u64(p.cols[p.key_col].data + r);
        if (key == AGG_EMPTY) {
          slot = (uint32_t)p.n_slots + 1;
          if (p.side_used[1] == 0) p.side_used[1] = 1;
        } else {
          // ---- getPartialResult (aggregate.go:396-410): find or claim the group's slot, bucket by bucket
          uint64_t b = (tqd::mix64(key) & p.mask) & ~3ull;
          bool defer = false, found = false;
          for (uint64_t buckets = 0; !found && !defer; buckets++) {
            if (buckets * 4 > p.mask) { defer = true; break; }  // table full (cannot happen below `limit`)
            unsigned long long k[4];
            ld_bucket(p.keys, b, k);
#pragma unroll
            for (int j = 0; j < 4; j++) {
              if (found || defer) break;
              if (k[j] == key) { slot = (uint32_t)(b + j); found = true; break; }
              if (k[j] == AGG_EMPTY) {
                if (*reinterpret_cast<volatile unsigned long long *>(p.n_used) >= p.limit) { defer = true; break; }
                const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(&p.keys[b + j]), (unsigned long long)AGG_EMPTY, (unsigned long long)key);
                if (prev == AGG_EMPTY) { claimed = true; slot = (uint32_t)(b + j); found = true; break; }
                if (prev == key) { slot = (uint32_t)(b + j); found = true; break; }
                // another key won this slot: keep scanning
              }
            }
            b = (b + 4) & p.mask;
          }
          if (defer) { slot = SLOT_NONE; p.deferred[atomicAdd(p.n_deferred, 1u)] = (uint32_t)r; }
        }
      }
    }
    // one counter update per warp: 1e6 new groups through a single-address atomic cost 0.4 ms (ncu: the merge of 1e6 partial
    // rows took 413 us the first time, 29 us once the groups existed); `limit` is therefore checked against a slightly stale
    // count — the table can overshoot load 0.5 by the rows in flight, the probe loop still terminates (full table -> defer)
    const unsigned claims = __ballot_sync(0xffffffffu, claimed);
    if (claims && (threadIdx.x & 31) == (unsigned)(__ffs(claims) - 1)) atomicAdd(p.n_used, (unsigned long long)__popc(claims));
    agg_apply(p, slot, r);
  }
}

__global__ void k_agg_set_flags(const uint64_t *keys, uint64_t *tbl, int stride, uint64_t n_slots, const uint32_t *side_used, int w1) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t gstride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n_slots + 2; i += gstride) {
    const bool used = i < n_slots ? keys[i] != AGG_EMPTY : side_used[i - n_slots] != 0;
    if (used) tbl[i * stride + w1] = 1;
  }
}

// value of the SUM/MAX/MIN "seen" word when the flag is not maintained: the group exists, so it has a value
__device__ __forceinline__ uint64_t seen_of(const AggFuncDev &f, const uint64_t *sl) { return (f.func == TQ_AGG_AVG || (f.use_flag && f.w1 >= 0)) ? sl[f.w1] : 1ull; }

struct CollectParams {
  int n_funcs;
  AggFuncDev f[AGG_MAXF];
  DColMut out[AGG_MAXF];
  const uint64_t *keys;
  const uint64_t *tbl;
  int stride;
  uint64_t n_slots;
  const uint32_t *side_used;
  unsigned long long *out_n;
  unsigned *err;
  int has_group_by;
  // partial export (tq_agg_export_partial): key column + raw states instead of final values
  int export_partial;
  DColMut out_key;
  DColMut out_state[2 * AGG_MAXF];
};

__device__ __forceinline__ void put_out(const DColMut &o, unsigned long long pos, uint64_t v, bool nn) {
  o.data[pos] = v;
  if (nn) atomicOr(&o.bm[pos >> 5], 1u << (pos & 31));
}

// getFinalResult (aggregate.go:429-457): one output row per occupied slot, AppendFinalResult2Chunk per function.
__global__ void __launch_bounds__(256) k_agg_collect(const CollectParams p) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t total = p.n_slots + 2;
  for (; i < total; i += stride) {
    bool used;
    uint64_t key = 0;
    bool key_nn = true;
    const uint64_t *sl = p.tbl + i * p.stride;
    if (i < p.n_slots) { key = p.keys[i]; used = key != AGG_EMPTY; }
    else if (i == p.n_slots) { used = p.side_used[0] != 0; key_nn = false; }
    else { used = p.side_used[1] != 0; key = AGG_EMPTY; }
    if (!used) continue;
    const unsigned long long pos = atomicAdd(p.out_n, 1ull);
    if (p.export_partial) {
      if (p.has_group_by) put_out(p.out_key, pos, key_nn ? key : 0, key_nn);
      int w = 0;
      for (int fi = 0; fi < p.n_funcs; fi++) {
        const AggFuncDev &f = p.f[fi];
        if (f.key_passthrough) { put_out(p.out_state[w++], pos, key_nn ? key : 0, key_nn); continue; }
        switch (f.func) {
          case TQ_AGG_COUNT: put_out(p.out_state[w++], pos, sl[f.w0], true); break;
          case TQ_AGG_SUM:
          case TQ_AGG_AVG: {
            const uint64_t cnt = seen_of(f, sl);
            uint64_t sum = sl[f.w0];
            if (f.arg_type != TQ_TYPE_FLOAT64) {
              const int64_t hi = (int64_t)sl[f.w2];
              if (cnt && hi != ((int64_t)sum >> 63)) atomicOr(p.err, AERR_BIGINT);
            }
            if (f.func == TQ_AGG_AVG) put_out(p.out_state[w++], pos, cnt, true);   // AVG partial = (count, sum) descriptor.go:57-92
            put_out(p.out_state[w++], pos, cnt ? sum : 0, cnt != 0);
            break;
          }
          case TQ_AGG_MAX:
          case TQ_AGG_MIN: {
            if (f.arg_type == TQ_TYPE_BYTES) { put_out(p.out_state[w++], pos, sl[f.w0] ? sl[f.w0] - 1 : 0, sl[f.w0] != 0); break; }
            const uint64_t cnt = seen_of(f, sl);
            uint64_t m = sl[f.w0];
            if (f.func == TQ_AGG_MIN) m = ~m;
            put_out(p.out_state[w++], pos, cnt ? order_unmap(m, f.arg_type) : 0, cnt != 0);
            break;
          }
          default: {
            const uint64_t st = sl[f.w1];
            put_out(p.out_state[w++], pos, (st == 1) ? sl[f.w0] : 0, st == 1);
            break;
          }
        }
      }
      continue;
    }
    for (int fi = 0; fi < p.n_funcs; fi++) {
      const AggFuncDev &f = p.f[fi];
      if (f.key_passthrough) { put_out(p.out[fi], pos, key_nn ? key : 0, key_nn); continue; }
      switch (f.func) {
        case TQ_AGG_COUNT: put_out(p.out[fi], pos, sl[f.w0], true); break;            // func_count.go:23-27
        case TQ_AGG_SUM: {                                                          // func_sum.go:53-60,104-113
          const uint64_t cnt = seen_of(f, sl);
          if (cnt == 0) { put_out(p.out[fi], pos, 0, false); break; }
          if (f.arg_type != TQ_TYPE_FLOAT64) {
            const int64_t hi = (int64_t)sl[f.w2];
            if (hi != ((int64_t)sl[f.w0] >> 63)) atomicOr(p.err, AERR_BIGINT);    // types.AddInt64 overflow (types/overflow.go:33-40)
          }
          put_out(p.out[fi], pos, sl[f.w0], true);
          break;
        }
        case TQ_AGG_AVG: {                                                          // func_avg.go:47-55,159-167
          const int64_t cnt = (int64_t)sl[f.w1];
          if (cnt == 0) { put_out(p.out[fi], pos, 0, false); break; }
          if (f.arg_type == TQ_TYPE_FLOAT64) {
            const double r = __longlong_as_double((long long)sl[f.w0]) / (double)cnt;
            put_out(p.out[fi], pos, (uint64_t)__double_as_longlong(r), true);
          } else {
            const int64_t hi = (int64_t)sl[f.w2];
            const int64_t sum = (int64_t)sl[f.w0];
            if (hi != (sum >> 63)) atomicOr(p.err, AERR_BIGINT);
            put_out(p.out[fi], pos, (uint64_t)(sum / cnt), true);                   // Go truncating division
          }
          break;
        }
        case TQ_AGG_MAX:
        case TQ_AGG_MIN: {                                                          // func_max_min.go:73-81
          if (f.arg_type == TQ_TYPE_BYTES) { put_out(p.out[fi], pos, sl[f.w0] ? sl[f.w0] - 1 : 0, sl[f.w0] != 0); break; }   // :327-335
          const uint64_t cnt = seen_of(f, sl);
          uint64_t m = sl[f.w0];
          if (f.func == TQ_AGG_MIN) m = ~m;
          put_out(p.out[fi], pos, cnt ? order_unmap(m, f.arg_type) : 0, cnt != 0);
          break;
        }
        default: {                                                                  // func_first_row.go:91-99
          const uint64_t st = sl[f.w1];
          put_out(p.out[fi], pos, (st == 1) ? sl[f.w0] : 0, st == 1);
          break;
        }
      }
    }
  }
}

__global__ void k_fill_u64(uint64_t *p, uint64_t n, uint64_t v) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// Move every occupied slot (key + state record) of the old table into the new, larger one.
__global__ void __launch_bounds__(256) k_agg_rehash(const uint64_t *old_keys, const uint64_t *old_tbl, uint64_t old_slots, uint64_t *new_keys,
                                                     uint64_t *new_tbl, uint64_t new_mask, int stride) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t gstride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t old_total = old_slots + 2;
  for (; i < old_total; i += gstride) {
    uint64_t dst;
    if (i >= old_slots) dst = (new_mask + 1) + (i - old_slots);  // side slots keep their role
    else {
      const uint64_t key = old_keys[i];
      if (key == AGG_EMPTY) continue;
      uint64_t idx = (tqd::mix64(key) & new_mask) & ~3ull;  // same bucket-aligned probe order as the update kernels
      for (;;) {
        const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(&new_keys[idx]), (unsigned long long)AGG_EMPTY, (unsigned long long)key);
        if (prev == AGG_EMPTY) break;
        idx = (idx + 1) & new_mask;
      }
      dst = idx;
    }
    for (int w = 0; w < stride; w++) new_tbl[dst * stride + w] = old_tbl[i * stride + w];
  }
}

// ------------------------------------------------------------------ shared-memory pre-aggregation
// Large batches over a moderate number of groups do not have to pay one L2 atomic per row and state word.  The batch is
// radix-scattered by the top hash bits of the key (scatter.cuh) so that one partition's groups fit a shared-memory hash
// table; each CTA aggregates its slice of a partition with shared-memory atomics and emits ONE partial row per group
// it saw — (key, COUNT | SUM | (COUNT, SUM) ...), the layout of tq_agg_export_partial — and the partial rows (~groups,
// not ~rows) then go through the ordinary merge path (MergePartialResult semantics, aggregate.go:424-457).  This is the
// reference's own partial -> final split (aggregate.go:96-133) with the partial workers living in shared memory.
enum { PRE_COUNT = 0, PRE_SUM_F64 = 1, PRE_AVG_F64 = 2, PRE_KEY = 3 };
struct PreFunc { int kind, col, w; };
static constexpr uint32_t PRE_SLOTS = 4096;      // shared-memory table entries per CTA
static constexpr int PRE_THREADS = 512;
static constexpr int PRE_MAX_GROUPS_PER_PART = 2400;
static constexpr int PRE_MAX_OUT_COLS = 1 + 2 * AGG_MAXF;
struct PreParams {
  const uint64_t *col[4];        // col[0] = key, then the distinct argument columns (the batch itself when pbits == 0, column slabs on the old scatter)
  const uint64_t *aos;           // non-null: array-of-structs slabs of aos_nc words per row (word 0 = key, word c = argument column c)
  int aos_nc;
  const uint32_t *lo, *hi, *lim; // partition bounds inside the slabs (pbits > 0)
  int64_t n;
  int pbits, split;
  int n_funcs, W;                // W = state words per group
  PreFunc f[AGG_MAXF];
  uint64_t *out[PRE_MAX_OUT_COLS];  // partial-row columns: key, then per function its partial state column(s)
  unsigned long long *out_n;
  unsigned long long out_cap;
  unsigned *fallback;            // non-zero: a table filled up / the marker key appeared / output full -> redo on the general path
};

__global__ void __launch_bounds__(PRE_THREADS) k_agg_preagg(const PreParams p) {
  extern __shared__ __align__(16) uint64_t s_pre[];
  uint64_t *s_keys = s_pre;
  uint64_t *s_st = s_pre + PRE_SLOTS;
  for (uint32_t i = threadIdx.x; i < PRE_SLOTS; i += PRE_THREADS) s_keys[i] = AGG_EMPTY;
  for (uint32_t i = threadIdx.x; i < PRE_SLOTS * (uint32_t)p.W; i += PRE_THREADS) s_st[i] = 0;
  __syncthreads();
  const uint32_t part = blockIdx.x / p.split, sub = blockIdx.x % p.split;
  int64_t lo = 0, hi = p.n;
  if (p.pbits) {
    lo = p.lo[part];
    hi = p.hi[part];
    if (hi > (int64_t)p.lim[part]) hi = p.lim[part];  // overflowed slab: the batch is redone anyway
  }
  const int64_t len = hi - lo;
  const int64_t r_lo = lo + len * sub / p.split, r_hi = lo + len * (sub + 1) / p.split;
  for (int64_t r = r_lo + threadIdx.x; r < r_hi; r += PRE_THREADS) {
    uint64_t key, w1 = 0;
    if (p.aos) {
      if (p.aos_nc == 2) { const ulonglong2 x = tqd::ld_stream_u64x2(p.aos + r * 2); key = x.x; w1 = x.y; }
      else key = tqd::ld_stream_u64(p.aos + r * p.aos_nc);
    } else key = tqd::ld_stream_u64(p.col[0] + r);
    if (key == AGG_EMPTY) { atomicOr(p.fallback, 1u); continue; }
    uint32_t idx = (uint32_t)(tqd::mix64(key) >> 20) & (PRE_SLOTS - 1);  // bits disjoint from the partition bits and the global table's
    bool ok = false;
    for (uint32_t probes = 0; probes < PRE_SLOTS; probes++) {
      const unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(&s_keys[idx]);
      if (cur == key) { ok = true; break; }
      if (cur == AGG_EMPTY) {
        const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(&s_keys[idx]), (unsigned long long)AGG_EMPTY, (unsigned long long)key);
        if (prev == AGG_EMPTY || prev == key) { ok = true; break; }
      }
      idx = (idx + 1) & (PRE_SLOTS - 1);
    }
    if (!ok) { atomicOr(p.fallback, 2u); continue; }
    uint64_t *st = s_st + (size_t)idx * p.W;
    for (int fi = 0; fi < p.n_funcs; fi++) {
      const PreFunc &f = p.f[fi];
      if (f.kind == PRE_COUNT) atomicAdd(reinterpret_cast<unsigned *>(st + f.w), 1u);   // low half of the word: a CTA sees < 2^32 rows, and 32-bit shared atomics are native (64-bit ones are CAS loops)
      else {
        const uint64_t bits = !p.aos ? tqd::ld_stream_u64(p.col[f.col] + r) : (p.aos_nc == 2 ? w1 : tqd::ld_stream_u64(p.aos + r * p.aos_nc + f.col));
        if (f.kind == PRE_SUM_F64) atomicAdd(reinterpret_cast<double *>(st + f.w), __longlong_as_double((long long)bits));
        else if (f.kind == PRE_AVG_F64) {
          atomicAdd(reinterpret_cast<unsigned *>(st + f.w), 1u);
          atomicAdd(reinterpret_cast<double *>(st + f.w + 1), __longlong_as_double((long long)bits));
        }
      }
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < PRE_SLOTS; i += PRE_THREADS) {
    const uint64_t key = s_keys[i];
    if (key == AGG_EMPTY) continue;
    const unsigned long long pos = atomicAdd(p.out_n, 1ull);
    if (pos >= p.out_cap) { atomicOr(p.fallback, 4u); continue; }
    const uint64_t *st = s_st + (size_t)i * p.W;
    p.out[0][pos] = key;
    int oc = 1;
    for (int fi = 0; fi < p.n_funcs; fi++) {
      const PreFunc &f = p.f[fi];
      if (f.kind == PRE_KEY) p.out[oc++][pos] = key;
      else if (f.kind == PRE_AVG_F64) { p.out[oc++][pos] = st[f.w]; p.out[oc++][pos] = st[f.w + 1]; }
      else p.out[oc++][pos] = st[f.w];
    }
  }
}

// ------------------------------------------------------------------ host side
struct AggHostAccum {
  PinBuf data, bm;
  int64_t n = 0, cap = 0;
  bool has_bm = false;
};

}  // namespace tq

using namespace tq;

struct AggResult {
  std::vector<DevBuf> data, bm;
  std::vector<PinBuf> h_data, h_bm;
  std::vector<VarOut> var;   // FLOAT (4-byte slots) and var-len result columns, converted / gathered from `data` (indexed like data)
  int64_t n = 0;
  bool on_host = false;
};

struct tq_agg {
  int n_cols = 0, n_group_by = 0, n_funcs = 0;
  int n_funcs_all = 0;      // n_funcs + one hidden FIRSTROW per GROUP BY column when there are several (their values leave with export_partial)
  int types[AGG_MAXC];      // the 8-byte type the kernels see: FLOAT columns are widened to FLOAT64, var-len columns become dictionary ids (TQ_TYPE_BYTES)
  int in_kind[AGG_MAXC] = {};  // 0 = 8-byte slots as declared, 1 = FLOAT (4-byte slots, widened on the device), 2 = var-len (dictionary-encoded on the device)
  bool any_kind = false;
  StringDict sd[AGG_MAXC];  // one dictionary per var-len input column: GROUP BY items and string arguments work on ids (strdict.cuh)
  int out_kind[AGG_MAXF] = {};  // result column i: 0 = 8-byte, 1 = FLOAT (narrowed back), 2 = var-len (gathered from sd[out_src[i]])
  int out_src[AGG_MAXF] = {};
  DevBuf lens_scratch, scan_scratch;
  int key_col = -1;         // the key column of the update kernel: the GROUP BY column, or the hidden encoded column (index n_cols)
  int gb_cols[MK_MAX_KEYS];
  MultiKeyEncoder mk;       // several GROUP BY columns: exact fold of the key tuple into one 64-bit word (dict.cuh)
  DevBuf mk_comb;
  // shared-memory pre-aggregation of large batches (k_agg_preagg)
  bool pre_disabled = false;
  bool pre_partitioned = true;   // TQ_AGG_PREAGG_PART=0: do not pre-aggregate when the groups need radix partitioning
  int64_t known_groups = 0;  // groups in the table after the last batch
  std::vector<DevBuf> pre_slabs, pre_out;
  DevBuf pre_aos;
  DevBuf pre_lo, pre_hi, pre_lim, pre_meta;
  cudaEvent_t ev_pa = nullptr, ev_pb = nullptr;
  tq_agg_func funcs[AGG_MAXF];
  int arg_type[AGG_MAXF];
  int out_type[AGG_MAXF];
  int key_passthrough[AGG_MAXF];
  int w0[AGG_MAXF], w1[AGG_MAXF], w2[AGG_MAXF];  // state word offsets inside the slot record
  int stride = 1;           // words per slot (power of two)
  bool not_null[AGG_MAXC] = {};    // input column declared NOT NULL (TQ_TYPE_NOT_NULL)
  bool flag_on[AGG_MAXF] = {};  // SUM/MAX/MIN: a batch with a NULL bitmap (or partial rows) has been seen for this argument
  int64_t est_groups = 0;
  int64_t batch_rows = 1 << 22;
  // FinalMode handle (tq_agg_create_final): the child's chunks are PARTIAL rows; internal column j (keys first, then one
  // state column per function, two for AVG) is the caller's input column final_src[j]
  bool final_mode = false;
  int final_src[AGG_MAXC] = {};
  int final_n_in = 0;

  // table
  DevBuf keys, table, meta;   // meta: [0..1] side_used u32, [2] n_deferred u32, [3] err u32, u64@16 n_used, u64@24 out_n
  uint64_t n_slots = 0;
  DevBuf deferred;
  PinBuf meta_host;
  // host staging (double-buffered)
  struct Stage {
    std::vector<PinBuf> data, bm; std::vector<bool> has_bm; int64_t n = 0; std::vector<DevBuf> d_data, d_bm; cudaEvent_t ev_done = nullptr; bool in_flight = false;
    std::vector<HostVarAccum> var;     // cells of the var-len columns of this stage
    std::vector<SideStore> store;      // ... and their device copy
    std::vector<DevBuf> d_raw;         // FLOAT columns: the 4-byte slots before widening
  } stage[2];
  int cur_stage = 0;
  int64_t rows_total = 0, launches = 0, last_update_ns = 0;
  bool eof = false, finalized = false, closed = false;
  bool merge_mode_seen = false, raw_mode_seen = false;
  AggResult result;
  int64_t result_pos = 0;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  ~tq_agg() {
    for (auto &s : stage) if (s.ev_done) cudaEventDestroy(s.ev_done);
    if (ev_a) cudaEventDestroy(ev_a);
    if (ev_b) cudaEventDestroy(ev_b);
    if (ev_pa) cudaEventDestroy(ev_pa);
    if (ev_pb) cudaEventDestroy(ev_pb);
  }
};

namespace tq {

static int agg_grid(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

static int32_t agg_alloc_table(tq_agg *a, uint64_t n_slots) {
  cudaStream_t s = rt().compute;
  a->n_slots = n_slots;
  const uint64_t total = n_slots + 2;
  TQ_TRY(a->keys.reserve((n_slots + 4) * 8));
  TQ_TRY(a->table.reserve(total * a->stride * 8));
  k_fill_u64<<<agg_grid((int64_t)n_slots), 256, 0, s>>>(a->keys.as<uint64_t>(), n_slots, AGG_EMPTY);
  count_launch();
  TQ_CUDA(cudaMemsetAsync(a->table.p, 0, total * a->stride * 8, s));
  return check_launch("k_fill_u64");
}

static void fill_funcs(tq_agg *a, AggFuncDev *f, bool merge) {
  int pcol = a->n_group_by;  // merge-mode input layout: key cols, then partial-state columns in function order
  for (int i = 0; i < a->n_funcs_all; i++) {
    AggFuncDev &d = f[i];
    d.func = a->funcs[i].func;
    d.arg_type = a->arg_type[i];
    d.key_passthrough = a->key_passthrough[i];
    d.arg_col = a->funcs[i].arg_col;
    d.arg_col2 = -1;
    if (merge && i >= a->n_funcs) d.arg_col = i - a->n_funcs;  // hidden FIRSTROW of GROUP BY column j reads key column j of the partial rows
    else if (merge) {
      d.arg_col = pcol++;
      if (d.func == TQ_AGG_AVG && !d.key_passthrough) d.arg_col2 = pcol++;
    }
    d.w0 = a->w0[i];
    d.w1 = a->w1[i];
    d.w2 = a->w2[i];
    d.use_flag = (a->flag_on[i] && a->w1[i] >= 0) ? 1 : 0;
    d.str_off = nullptr;
    d.str_bytes = nullptr;
    if (a->arg_type[i] == TQ_TYPE_BYTES && a->funcs[i].arg_col >= 0) {
      const StringDict &sd = a->sd[a->funcs[i].arg_col];
      d.str_off = sd.arena.offsets.as<int64_t>();
      d.str_bytes = sd.arena.bytes.as<uint8_t>();
    }
    d.arg_not_null = (!merge && a->funcs[i].arg_col >= 0 && a->not_null[a->funcs[i].arg_col]) ? 1 : 0;
  }
}

static int32_t agg_grow(tq_agg *a, uint64_t new_slots) {
  cudaStream_t s = rt().compute;
  DevBuf old_keys = std::move(a->keys), old_tbl = std::move(a->table);
  const uint64_t old_slots = a->n_slots;
  TQ_TRY(agg_alloc_table(a, new_slots));
  k_agg_rehash<<<agg_grid((int64_t)old_slots + 2), 256, 0, s>>>(old_keys.as<uint64_t>(), old_tbl.as<uint64_t>(), old_slots, a->keys.as<uint64_t>(),
                                                                a->table.as<uint64_t>(), new_slots - 1, a->stride);
  count_launch();
  TQ_TRY(check_launch("k_agg_rehash"));
  TQ_CUDA(cudaStreamSynchronize(s));  // the old buffers are released when this scope ends
  return TQ_OK;
}

static int32_t agg_update_device(tq_agg *a, const DCol *cols, int n_in_cols, int64_t n, bool merge);

// Try the shared-memory pre-aggregation path for one raw batch; *done tells whether the batch was consumed.
static int32_t agg_try_preagg(tq_agg *a, const DCol *cols, int64_t n, bool *done) {
  *done = false;
  static const bool disabled_by_env = [] { const char *e = getenv("TQ_AGG_NO_PREAGG"); return e && e[0] == '1'; }();
  if (disabled_by_env || a->pre_disabled || a->any_kind || a->n_group_by != 1 || n < (1 << 20) || n > 0xFFFFFFF0ll) return TQ_OK;
  const int kc = a->key_col;
  if (a->types[kc] == TQ_TYPE_FLOAT64 || cols[kc].bm != nullptr) return TQ_OK;  // integer key without NULLs
  const int64_t g_est = a->known_groups > a->est_groups ? a->known_groups : a->est_groups;
  if (g_est <= 0 || n / g_est < 4) return TQ_OK;  // unknown NDV, or too little reduction to pay for the extra pass
  PreParams p{};
  int col_of[AGG_MAXC];
  for (int c = 0; c < AGG_MAXC; c++) col_of[c] = -1;
  DCol used[4];
  int n_used = 1, W = 0, n_out = 1;
  used[0] = cols[kc];
  col_of[kc] = 0;
  for (int i = 0; i < a->n_funcs; i++) {
    const int fn = a->funcs[i].func, ac = a->funcs[i].arg_col;
    PreFunc &f = p.f[i];
    f.col = 0;
    f.w = W;
    if (a->key_passthrough[i]) { f.kind = PRE_KEY; n_out += 1; continue; }
    const bool arg_ok = ac >= 0 && a->types[ac] == TQ_TYPE_FLOAT64 && cols[ac].bm == nullptr;
    if (fn == TQ_AGG_COUNT && (ac < 0 || cols[ac].bm == nullptr)) { f.kind = PRE_COUNT; W += 1; n_out += 1; continue; }
    if ((fn == TQ_AGG_SUM || fn == TQ_AGG_AVG) && arg_ok) {
      if (col_of[ac] < 0) {
        if (n_used == 4) return TQ_OK;
        used[n_used] = cols[ac];
        col_of[ac] = n_used++;
      }
      f.col = col_of[ac];
      if (fn == TQ_AGG_SUM) { f.kind = PRE_SUM_F64; W += 1; n_out += 1; }
      else { f.kind = PRE_AVG_F64; W += 2; n_out += 2; }
      continue;
    }
    return TQ_OK;  // a function / argument type this path does not cover
  }
  if (W == 0 || W > 5) return TQ_OK;
  int pbits = 0;
  while (((int64_t)PRE_MAX_GROUPS_PER_PART << pbits) < g_est) pbits++;
  if (pbits > 12) return TQ_OK;
  // One table per CTA (<= 2400 groups) beats the general path; with radix partitioning the 64-bit shared-memory atomics can
  // cost more than the L2 atomics they replace, so the partitioned variant is taken only where it wins (below).
  if (pbits > 0 && !a->pre_partitioned) return TQ_OK;
  // Partitioned vs general path (scripts/agg_pre_probe.py, H100): in the middle range (4 to 128 partitions, up to 307,200
  // groups) the general table is still cache-friendly and the scatter is pure overhead, so it stays on the general path.
  static const bool force_part = [] { const char *e = getenv("TQ_AGG_PREAGG_PART"); return e && e[0] == '1'; }();
  if (pbits >= 2 && pbits <= 7 && !force_part) return TQ_OK;
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  const int P = 1 << pbits;
  const int split = P >= 2 * r.sm_count ? 1 : (2 * r.sm_count + P - 1) / P;
  const unsigned long long out_cap = (unsigned long long)P * split * PRE_SLOTS;
  if (!a->ev_pa) { TQ_CUDA(cudaEventCreate(&a->ev_pa)); TQ_CUDA(cudaEventCreate(&a->ev_pb)); }
  TQ_TRY(a->pre_meta.reserve(64));
  TQ_CUDA(cudaMemsetAsync(a->pre_meta.p, 0, 64, s));
  unsigned long long *d_out_n = a->pre_meta.as<unsigned long long>();      // [0] partial rows
  unsigned long long *d_overflow = d_out_n + 1;                            // [1] scatter slab overflow
  unsigned *d_fallback = reinterpret_cast<unsigned *>(d_out_n + 2);        // [2] pre-aggregation gave up
  TQ_CUDA(cudaEventRecord(a->ev_pa, s));
  if (pbits && pbits <= SCATTER_AOS_MAX_PBITS) {
    TQ_TRY(scatter_rows_by_hash_aos(used, n_used, 0, n, pbits, a->pre_aos, a->pre_lo, a->pre_hi, a->pre_lim, d_overflow, s));
    p.aos = a->pre_aos.as<uint64_t>();
    p.aos_nc = n_used;
    p.lo = a->pre_lo.as<uint32_t>();
    p.hi = a->pre_hi.as<uint32_t>();
    p.lim = a->pre_lim.as<uint32_t>();
  } else if (pbits) {
    TQ_TRY(scatter_rows_by_hash(used, n_used, 0, n, pbits, a->pre_slabs, a->pre_lo, a->pre_hi, a->pre_lim, d_overflow, s));
    for (int c = 0; c < n_used; c++) p.col[c] = a->pre_slabs[c].as<uint64_t>();
    p.lo = a->pre_lo.as<uint32_t>();
    p.hi = a->pre_hi.as<uint32_t>();
    p.lim = a->pre_lim.as<uint32_t>();
  } else {
    for (int c = 0; c < n_used; c++) p.col[c] = used[c].data;
  }
  p.n = n;
  p.pbits = pbits;
  p.split = split;
  p.n_funcs = a->n_funcs;
  p.W = W;
  a->pre_out.resize(n_out);
  for (int c = 0; c < n_out; c++) {
    TQ_TRY(a->pre_out[c].reserve((size_t)out_cap * 8));
    p.out[c] = a->pre_out[c].as<uint64_t>();
  }
  p.out_n = d_out_n;
  p.out_cap = out_cap;
  p.fallback = d_fallback;
  const int smem = (int)(PRE_SLOTS * 8 * (1 + W));
  static int smem_set = 0;
  if (smem > smem_set) {
    TQ_CUDA(cudaFuncSetAttribute(k_agg_preagg, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    smem_set = smem;
  }
  k_agg_preagg<<<P * split, PRE_THREADS, smem, s>>>(p);
  count_launch();
  a->launches++;
  TQ_TRY(check_launch("k_agg_preagg"));
  unsigned long long h_meta[3] = {0, 0, 0};
  TQ_CUDA(cudaMemcpyAsync(h_meta, a->pre_meta.p, 24, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  if (h_meta[1] || (unsigned)h_meta[2]) {
    // skewed keys / more groups per partition than estimated / the marker key: nothing was applied to the table yet —
    // this batch and the following ones take the general path
    a->pre_disabled = true;
    return TQ_OK;
  }
  std::vector<DCol> view(n_out);
  for (int c = 0; c < n_out; c++) { view[c].data = a->pre_out[c].as<uint64_t>(); view[c].bm = nullptr; }
  TQ_TRY(agg_update_device(a, view.data(), n_out, (int64_t)h_meta[0], /*merge=*/true));
  TQ_CUDA(cudaEventRecord(a->ev_pb, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  float ms = 0;
  if (cudaEventElapsedTime(&ms, a->ev_pa, a->ev_pb) == cudaSuccess) a->last_update_ns = (int64_t)(ms * 1e6);  // scatter + pre-aggregation + merge
  *done = true;
  return TQ_OK;
}

// Run the update kernel over device columns; handles deferred rows by growing the table.
static int32_t agg_update_device(tq_agg *a, const DCol *cols, int n_in_cols, int64_t n, bool merge) {
  if (n == 0) return TQ_OK;
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  if (!merge) {
    bool done = false;
    TQ_TRY(agg_try_preagg(a, cols, n, &done));
    if (done) return TQ_OK;
  }
  if (a->n_slots == 0) {
    uint64_t want = 1 << 16;
    const uint64_t hint = a->est_groups > 0 ? (uint64_t)a->est_groups : 0;
    while (want < hint * 2) want <<= 1;  // load factor <= 0.5 at the planner's NDV estimate
    TQ_TRY(agg_alloc_table(a, want));
    TQ_CUDA(cudaMemsetAsync(a->meta.p, 0, 64, s));
  }
  if (n > 0xFFFFFFF0ll) { set_error("aggregate batch too large"); return TQ_ERR_INVALID_ARG; }
  std::vector<DCol> wide;
  if (a->n_group_by > 1) {
    // getGroupKey (aggregate.go:359-394) over several GROUP BY items: the key tuple is folded, exactly, into one word
    DCol kc[MK_MAX_KEYS];
    for (int g = 0; g < a->n_group_by; g++) kc[g] = cols[merge ? g : a->gb_cols[g]];
    TQ_TRY(a->mk_comb.reserve((size_t)n * 8));
    TQ_TRY(a->mk.encode(kc, nullptr, n, /*insert=*/true, /*null_is_value=*/true, a->mk_comb.as<uint64_t>(), nullptr, s));
    wide.assign(cols, cols + n_in_cols);
    DCol hidden;
    hidden.data = a->mk_comb.as<uint64_t>();
    hidden.bm = nullptr;
    wide.push_back(hidden);
    cols = wide.data();
    n_in_cols++;
  }
  if (n_in_cols > AGG_MAXC) { set_error("aggregate input of %d columns exceeds the limit of %d", n_in_cols, AGG_MAXC); return TQ_ERR_INVALID_ARG; }
  for (int i = 0; i < a->n_funcs; i++) {
    const int fn = a->funcs[i].func;
    if (a->flag_on[i] || a->w1[i] < 0 || a->key_passthrough[i] || !(fn == TQ_AGG_SUM || fn == TQ_AGG_MAX || fn == TQ_AGG_MIN)) continue;
    const int ac = a->funcs[i].arg_col;
    const bool nullable_now = merge || (ac >= 0 && cols[ac].bm != nullptr);
    if (!nullable_now) continue;
    k_agg_set_flags<<<agg_grid((int64_t)a->n_slots + 2), 256, 0, s>>>(a->keys.as<uint64_t>(), a->table.as<uint64_t>(), a->stride, a->n_slots, a->meta.as<uint32_t>(), a->w1[i]);
    count_launch();
    TQ_TRY(check_launch("k_agg_set_flags"));
    a->flag_on[i] = true;
  }
  TQ_TRY(a->deferred.reserve((size_t)n * 4));
  uint32_t *meta32 = a->meta.as<uint32_t>();
  unsigned long long *meta64 = reinterpret_cast<unsigned long long *>(a->meta.as<uint8_t>() + 16);
  const uint32_t *row_list = nullptr;
  DevBuf row_list_buf;
  int64_t todo = n;
  TQ_CUDA(cudaEventRecord(a->ev_a, s));
  for (int round = 0; round < 64; round++) {
    AggParams p{};
    p.n_cols = n_in_cols;
    for (int c = 0; c < n_in_cols; c++) p.cols[c] = cols[c];
    p.key_col = a->n_group_by ? (a->n_group_by > 1 ? n_in_cols - 1 : (merge ? 0 : a->key_col)) : -1;
    p.merge = merge ? 1 : 0;
    p.n_funcs = a->n_funcs_all;
    fill_funcs(a, p.f, merge);
    p.keys = a->keys.as<uint64_t>();
    p.tbl = a->table.as<uint64_t>();
    p.stride = a->stride;
    p.mask = a->n_slots - 1;
    p.n_slots = a->n_slots;
    p.side_used = meta32;
    p.n_used = meta64;
    p.limit = a->n_slots / 2;
    p.deferred = a->deferred.as<uint32_t>();
    p.n_deferred = meta32 + 2;
    p.row_list = row_list;
    p.n = todo;
    TQ_CUDA(cudaMemsetAsync(meta32 + 2, 0, 4, s));
    k_agg_update<<<agg_grid(todo), 256, 0, s>>>(p);
    count_launch();
    a->launches++;
    TQ_TRY(check_launch("k_agg_update"));
    if (round == 0) TQ_CUDA(cudaEventRecord(a->ev_b, s));
    TQ_CUDA(cudaMemcpyAsync(a->meta_host.p, a->meta.p, 64, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    const uint32_t n_def = a->meta_host.as<uint32_t>()[2];
    if (round == 0) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, a->ev_a, a->ev_b) == cudaSuccess) a->last_update_ns = (int64_t)(ms * 1e6);
    }
    if (n_def == 0) {
      a->known_groups = (int64_t)*reinterpret_cast<unsigned long long *>(a->meta_host.as<uint8_t>() + 16);
      return TQ_OK;
    }
    // the table reached its load limit: grow 4x (at least enough for every deferred row) and redo only those rows
    const uint64_t used = *reinterpret_cast<unsigned long long *>(a->meta_host.as<uint8_t>() + 16);
    uint64_t want = a->n_slots * 4;
    while (want / 2 < used + n_def) want <<= 1;
    TQ_TRY(agg_grow(a, want));
    TQ_TRY(row_list_buf.reserve((size_t)n_def * 4));
    TQ_CUDA(cudaMemcpyAsync(row_list_buf.p, a->deferred.p, (size_t)n_def * 4, cudaMemcpyDeviceToDevice, s));
    row_list = row_list_buf.as<uint32_t>();
    todo = n_def;
  }
  set_error("aggregate table failed to converge");
  return TQ_ERR_CUDA;
}

// layout of input column c: partial rows lent by another handle (tq_agg_merge_partial) are 8-byte words throughout; the partial
// rows of a FinalMode handle come from a child executor and carry their real chunk layout (FLOAT slots, var-len cells)
static inline int col_kind(const tq_agg *a, bool merge, int c) { return (merge && !a->final_mode) ? 0 : a->in_kind[c]; }

static int32_t agg_flush_stage(tq_agg *a, bool merge, int n_in_cols) {
  tq_agg::Stage &st = a->stage[a->cur_stage];
  if (st.n == 0) return TQ_OK;
  Runtime &r = rt();
  st.d_data.resize(n_in_cols);
  st.d_bm.resize(n_in_cols);
  std::vector<DCol> view(n_in_cols);
  if (a->any_kind && (!merge || a->final_mode)) { st.store.resize(n_in_cols); st.d_raw.resize(n_in_cols); }
  for (int c = 0; c < n_in_cols; c++) {
    const int kind = col_kind(a, merge, c);
    TQ_TRY(st.d_data[c].reserve((size_t)st.n * 8));
    view[c].data = st.d_data[c].as<uint64_t>();
    view[c].bm = nullptr;
    if (st.has_bm[c]) {
      TQ_TRY(st.d_bm[c].reserve(bitmap_alloc_bytes(st.n)));
      TQ_CUDA(cudaMemcpyAsync(st.d_bm[c].p, st.bm[c].p, bitmap_bytes(st.n), cudaMemcpyHostToDevice, r.compute));
      view[c].bm = st.d_bm[c].as<uint32_t>();
    }
    if (kind == 0) {
      TQ_CUDA(cudaMemcpyAsync(st.d_data[c].p, st.data[c].p, (size_t)st.n * 8, cudaMemcpyHostToDevice, r.compute));
    } else if (kind == 1) {
      // FLOAT: the 4-byte slots were staged packed; EvalReal / getGroupKey see float64(f) (expression/column.go:95-110)
      TQ_TRY(st.d_raw[c].reserve((size_t)st.n * 4));
      TQ_CUDA(cudaMemcpyAsync(st.d_raw[c].p, st.data[c].p, (size_t)st.n * 4, cudaMemcpyHostToDevice, r.compute));
      TQ_TRY(widen_f32(st.d_raw[c].as<uint32_t>(), st.n, st.d_data[c].as<uint64_t>(), r.compute));
    } else {
      // var-len: cells -> device store -> dictionary ids (the string itself lives once in the dictionary's arena)
      // (insert mode: an id is valid iff the cell is NOT NULL, so the column's own bitmap stays the ids' bitmap)
      TQ_TRY(upload_store(st.var[c], st.store[c], r.compute));
      TQ_TRY(a->sd[c].encode(view_of(st.store[c]), view[c].bm, st.n, st.store[c].nbytes, /*insert=*/true, st.d_data[c].as<uint64_t>(), nullptr, r.compute));
      st.var[c].reset();
    }
  }
  const int64_t n = st.n;
  st.n = 0;
  for (int c = 0; c < n_in_cols; c++) st.has_bm[c] = false;
  a->cur_stage ^= 1;  // (agg_update_device synchronises; the flip keeps the door open for async overlap)
  return agg_update_device(a, view.data(), n_in_cols, n, merge);
}

static int32_t agg_put_common(tq_agg *a, const tq_column *cols, int32_t mem, bool merge, int n_in_cols) {
  if (!a || !cols) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (a->eof) { set_error("put after eof"); return TQ_ERR_STATE; }
  if ((merge && a->raw_mode_seen) || (!merge && a->merge_mode_seen)) { set_error("one handle cannot mix raw rows and partial rows"); return TQ_ERR_STATE; }
  (merge ? a->merge_mode_seen : a->raw_mode_seen) = true;
  const int64_t rows = cols[0].length;
  if (rows < 0) return TQ_ERR_INVALID_ARG;
  for (int c = 0; c < n_in_cols; c++) {
    if (cols[c].length != rows) { set_error("ragged aggregate input chunk"); return TQ_ERR_INVALID_ARG; }
    const int kind = col_kind(a, merge, c);
    if (kind != 2 && cols[c].offsets) { set_error("unsupport column type for encode (var-len data in fixed-width column %d)", c); return TQ_ERR_UNSUPPORTED_TYPE; }
    if (kind == 2 && !cols[c].offsets) { set_error("var-len column %d needs offsets", c); return TQ_ERR_INVALID_ARG; }
    if (rows && !cols[c].data && !(kind == 2 && cols[c].offsets[rows] == cols[c].offsets[0])) return TQ_ERR_INVALID_ARG;
    if (kind != 0 && mem != TQ_MEM_HOST) { set_error("FLOAT / var-len columns are accepted from host memory only"); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  if (rows == 0) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  a->rows_total += rows;
  if (mem == TQ_MEM_DEVICE) {
    TQ_TRY(agg_flush_stage(a, merge, n_in_cols));
    std::vector<DCol> view(n_in_cols);
    for (int c = 0; c < n_in_cols; c++) { view[c].data = (const uint64_t *)cols[c].data; view[c].bm = (const uint32_t *)cols[c].null_bitmap; }
    return agg_update_device(a, view.data(), n_in_cols, rows, merge);
  }
  // host chunks accumulate in pinned staging until a device batch is full
  int64_t done = 0;
  while (done < rows) {
    tq_agg::Stage &st = a->stage[a->cur_stage];
    if ((int)st.data.size() != n_in_cols) { st.data.resize(n_in_cols); st.bm.resize(n_in_cols); st.has_bm.assign(n_in_cols, false); st.var.resize(n_in_cols); }
    int64_t room = a->batch_rows - st.n;
    if (room <= 0) { TQ_TRY(agg_flush_stage(a, merge, n_in_cols)); continue; }
    int64_t take = rows - done < room ? rows - done : room;
    if (take < rows - done) take &= ~7ll;  // keep source bitmap offsets byte aligned when a chunk is split
    if (take == 0) { TQ_TRY(agg_flush_stage(a, merge, n_in_cols)); continue; }
    for (int c = 0; c < n_in_cols; c++) {
      if (st.data[c].cap < (size_t)a->batch_rows * 8) TQ_TRY(st.data[c].reserve((size_t)a->batch_rows * 8));
      if (st.bm[c].cap < bitmap_alloc_bytes(a->batch_rows)) { TQ_TRY(st.bm[c].reserve(bitmap_alloc_bytes(a->batch_rows))); }
      const int kind = col_kind(a, merge, c);
      if (kind == 0) memcpy(st.data[c].as<uint8_t>() + st.n * 8, cols[c].data + done * 8, (size_t)take * 8);
      else if (kind == 1) memcpy(st.data[c].as<uint8_t>() + st.n * 4, cols[c].data + done * 4, (size_t)take * 4);  // packed 4-byte slots
      else {
        tq_column piece = cols[c];
        piece.offsets = cols[c].offsets + done;   // HostVarAccum rebases on offsets[0]
        st.var[c].append(piece, take);
      }
      if (cols[c].null_bitmap && !st.has_bm[c]) { host_bitmap_append(st.bm[c].as<uint8_t>(), 0, nullptr, st.n); st.has_bm[c] = true; }
      if (st.has_bm[c]) {
        if (cols[c].null_bitmap) {
          // source offset `done` is a multiple of 8 by construction
          host_bitmap_append(st.bm[c].as<uint8_t>(), st.n, cols[c].null_bitmap + (done >> 3), take);
        } else host_bitmap_append(st.bm[c].as<uint8_t>(), st.n, nullptr, take);
      }
    }
    st.n += take;
    done += take;
  }
  return TQ_OK;
}

static int32_t agg_finalize(tq_agg *a, bool export_partial, AggResult &res, int n_out_cols) {
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  res.data.resize(n_out_cols);
  res.bm.resize(n_out_cols);
  res.n = 0;
  res.on_host = false;
  if (a->n_slots == 0) return TQ_OK;  // no input at all
  TQ_CUDA(cudaMemcpyAsync(a->meta_host.p, a->meta.p, 64, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  const uint32_t *m32 = a->meta_host.as<uint32_t>();
  const uint64_t used = *reinterpret_cast<unsigned long long *>(a->meta_host.as<uint8_t>() + 16);
  const int64_t groups = (int64_t)used + (m32[0] ? 1 : 0) + (m32[1] ? 1 : 0);
  CollectParams p{};
  p.n_funcs = a->n_funcs;
  fill_funcs(a, p.f, false);
  for (int c = 0; c < n_out_cols; c++) {
    TQ_TRY(res.data[c].reserve((size_t)(groups ? groups : 1) * 8));
    TQ_TRY(res.bm[c].reserve(bitmap_alloc_bytes(groups)));
    TQ_CUDA(cudaMemsetAsync(res.bm[c].p, 0, bitmap_alloc_bytes(groups), s));
  }
  if (export_partial && a->n_group_by > 1) {
    // key columns come from the hidden FIRSTROW states (last in function order), partial states follow them in the row
    p.export_partial = 1;
    p.n_funcs = a->n_funcs_all;
    const int k = a->n_group_by, w_user = n_out_cols - k;
    for (int w = 0; w < w_user; w++) { p.out_state[w].data = res.data[k + w].as<uint64_t>(); p.out_state[w].bm = res.bm[k + w].as<uint32_t>(); }
    for (int g = 0; g < k; g++) { p.out_state[w_user + g].data = res.data[g].as<uint64_t>(); p.out_state[w_user + g].bm = res.bm[g].as<uint32_t>(); }
  } else if (export_partial) {
    p.export_partial = 1;
    int c = 0;
    if (a->n_group_by) { p.out_key.data = res.data[c].as<uint64_t>(); p.out_key.bm = res.bm[c].as<uint32_t>(); c++; }
    for (int w = 0; c < n_out_cols; c++, w++) { p.out_state[w].data = res.data[c].as<uint64_t>(); p.out_state[w].bm = res.bm[c].as<uint32_t>(); }
  } else {
    for (int c = 0; c < n_out_cols; c++) { p.out[c].data = res.data[c].as<uint64_t>(); p.out[c].bm = res.bm[c].as<uint32_t>(); }
  }
  p.keys = a->keys.as<uint64_t>();
  p.tbl = a->table.as<uint64_t>();
  p.stride = a->stride;
  p.n_slots = a->n_slots;
  p.side_used = a->meta.as<uint32_t>();
  p.out_n = reinterpret_cast<unsigned long long *>(a->meta.as<uint8_t>() + 24);
  p.err = a->meta.as<uint32_t>() + 3;
  p.has_group_by = a->n_group_by == 1 ? 1 : 0;
  TQ_CUDA(cudaMemsetAsync(a->meta.as<uint8_t>() + 24, 0, 8, s));
  TQ_CUDA(cudaMemsetAsync(a->meta.as<uint32_t>() + 3, 0, 4, s));
  k_agg_collect<<<agg_grid((int64_t)a->n_slots + 2), 256, 0, s>>>(p);
  count_launch();
  a->launches++;
  TQ_TRY(check_launch("k_agg_collect"));
  TQ_CUDA(cudaMemcpyAsync(a->meta_host.p, a->meta.p, 64, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  const uint64_t out_n = *reinterpret_cast<unsigned long long *>(a->meta_host.as<uint8_t>() + 24);
  if ((int64_t)out_n != groups) { set_error("internal: collected %llu groups, expected %lld", (unsigned long long)out_n, (long long)groups); return TQ_ERR_CUDA; }
  if (a->meta_host.as<uint32_t>()[3] & AERR_BIGINT) { set_error("BIGINT value is out of range in 'sum'"); return TQ_ERR_OVERFLOW_BIGINT; }
  res.n = groups;
  return TQ_OK;
}

static int partial_width(const tq_agg *a) {
  int w = a->n_group_by;
  for (int i = 0; i < a->n_funcs; i++) w += (a->funcs[i].func == TQ_AGG_AVG && !a->key_passthrough[i]) ? 2 : 1;
  return w;
}

}  // namespace tq

extern "C" {

int32_t tq_agg_create(const tq_agg_desc *d, tq_agg **out) {
  if (!d || !out) return TQ_ERR_INVALID_ARG;
  *out = nullptr;
  TQ_TRY(ensure_init());
  if (d->n_input_cols < 0 || d->n_input_cols > AGG_MAXC || d->n_funcs < 0 || d->n_funcs > AGG_MAXF) { set_error("too many columns / functions"); return TQ_ERR_INVALID_ARG; }
  if (d->n_group_by < 0) return TQ_ERR_INVALID_ARG;
  if (d->n_group_by > MK_MAX_KEYS) { set_error("GROUP BY over %d items: at most %d are supported", d->n_group_by, MK_MAX_KEYS); return TQ_ERR_INVALID_ARG; }
  if (d->n_group_by > 1 && (d->n_input_cols + 1 > AGG_MAXC || d->n_funcs + d->n_group_by > AGG_MAXF)) {
    set_error("multi-column GROUP BY needs one spare input column and %d spare function slots", d->n_group_by);
    return TQ_ERR_INVALID_ARG;
  }
  for (int c = 0; c < d->n_input_cols; c++) {
    const int t = d->input_types[c] & 0xFF;
    if (t < TQ_TYPE_INT64 || t > TQ_TYPE_BYTES) { set_error("unsupport column type for encode %d", t); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  for (int i = 0; i < d->n_funcs; i++) {
    const int fn = d->funcs[i].func, ac = d->funcs[i].arg_col;
    if ((fn == TQ_AGG_SUM || fn == TQ_AGG_AVG) && ac >= 0 && ac < d->n_input_cols && (d->input_types[ac] & 0xFF) == TQ_TYPE_BYTES) {
      // the planner wraps a string argument of SUM / AVG in a cast to DOUBLE; HashAgg never sees the raw string
      set_error("SUM / AVG over a var-len column: project cast(col as double) first");
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
  }
  tq_agg *a = new (std::nothrow) tq_agg();
  if (!a) return TQ_ERR_OOM;
  a->n_cols = d->n_input_cols;
  a->n_group_by = d->n_group_by;
  a->n_funcs = d->n_funcs;
  a->est_groups = d->est_groups;
  { const char *e = getenv("TQ_AGG_PREAGG_PART"); a->pre_partitioned = !(e && e[0] == '0'); }  // on by default since the AoS scatter + native 32-bit counts (2.88 vs 3.18 ms at 1e6 groups); =0 turns it off
  for (int c = 0; c < a->n_cols; c++) {
    const int t = d->input_types[c] & 0xFF;
    a->in_kind[c] = t == TQ_TYPE_FLOAT32 ? 1 : (t == TQ_TYPE_BYTES ? 2 : 0);
    a->any_kind |= a->in_kind[c] != 0;
    a->types[c] = t == TQ_TYPE_FLOAT32 ? TQ_TYPE_FLOAT64 : t;   // FLOAT is evaluated as float64(f): EvalReal / VecEvalReal (expression/column.go:95-110)
    a->not_null[c] = (d->input_types[c] & TQ_TYPE_NOT_NULL) != 0;
  }
  for (int g = 0; g < a->n_group_by; g++) {
    a->gb_cols[g] = d->group_by_cols[g];
    if (a->gb_cols[g] < 0 || a->gb_cols[g] >= a->n_cols) { delete a; return TQ_ERR_INVALID_ARG; }
  }
  if (a->n_group_by == 1) a->key_col = a->gb_cols[0];
  else if (a->n_group_by > 1) { a->key_col = a->n_cols; a->mk.k = a->n_group_by; }
  a->n_funcs_all = a->n_funcs + (a->n_group_by > 1 ? a->n_group_by : 0);
  int words = 0;
  for (int i = 0; i < a->n_funcs_all; i++) {
    if (i < a->n_funcs) a->funcs[i] = d->funcs[i];
    else { a->funcs[i].func = TQ_AGG_FIRSTROW; a->funcs[i].arg_col = a->gb_cols[i - a->n_funcs]; }
    const int fn = a->funcs[i].func, ac = a->funcs[i].arg_col;
    if (fn < TQ_AGG_COUNT || fn > TQ_AGG_FIRSTROW || ac >= a->n_cols || ((fn == TQ_AGG_MAX || fn == TQ_AGG_MIN) && ac < 0)) {
      set_error("bad aggregate descriptor %d", i);
      delete a;
      return TQ_ERR_INVALID_ARG;
    }
    a->arg_type[i] = ac >= 0 ? a->types[ac] : TQ_TYPE_INT64;
    if ((fn == TQ_AGG_SUM || fn == TQ_AGG_AVG) && a->arg_type[i] == TQ_TYPE_UINT64) a->arg_type[i] = TQ_TYPE_INT64;  // sum4Int64 reads EvalInt (func_sum.go:118)
    a->out_type[i] = fn == TQ_AGG_COUNT ? TQ_TYPE_INT64 : (ac >= 0 ? a->types[ac] : TQ_TYPE_INT64);
    if ((fn == TQ_AGG_SUM || fn == TQ_AGG_AVG) && a->out_type[i] == TQ_TYPE_UINT64) a->out_type[i] = TQ_TYPE_INT64;
    // MAX / MIN / FIRSTROW keep the argument's own column type: maxMin4Float32 / firstRow4Float32 append a FLOAT,
    // maxMin4String / firstRow4String a string (aggfuncs/builder.go:119-172)
    const bool sel = fn == TQ_AGG_MAX || fn == TQ_AGG_MIN || fn == TQ_AGG_FIRSTROW;
    if (sel && ac >= 0 && a->in_kind[ac] == 1) { a->out_type[i] = TQ_TYPE_FLOAT32; a->out_kind[i] = 1; }
    if (sel && ac >= 0 && a->in_kind[ac] == 2) { a->out_kind[i] = 2; a->out_src[i] = ac; }
    a->key_passthrough[i] = (fn == TQ_AGG_FIRSTROW && a->n_group_by == 1 && ac == a->key_col) ? 1 : 0;
    a->w0[i] = a->w1[i] = a->w2[i] = 0;
    if (!a->key_passthrough[i]) {
      const bool int_sum = (fn == TQ_AGG_SUM || fn == TQ_AGG_AVG) && a->arg_type[i] != TQ_TYPE_FLOAT64;
      const bool arg_nn = ac >= 0 && a->not_null[ac];
      const bool flag_only = (fn == TQ_AGG_SUM || fn == TQ_AGG_MAX || fn == TQ_AGG_MIN);
      a->w0[i] = words++;
      a->w1[i] = -1;
      const bool str_maxmin = (fn == TQ_AGG_MAX || fn == TQ_AGG_MIN) && a->arg_type[i] == TQ_TYPE_BYTES;  // state = id + 1, 0 = no value yet
      if (fn != TQ_AGG_COUNT && !(flag_only && arg_nn) && !str_maxmin) a->w1[i] = words++;
      if (int_sum) a->w2[i] = words++;
    }
  }
  a->stride = 1;
  while (a->stride < words) a->stride <<= 1;
  int32_t st = a->meta.reserve(64);
  if (st == TQ_OK) st = a->meta_host.reserve(64);
  cudaError_t e = cudaEventCreate(&a->ev_a);
  if (e == cudaSuccess) e = cudaEventCreate(&a->ev_b);
  if (st == TQ_OK && e != cudaSuccess) st = cuda_fail(e, "cudaEventCreate", __FILE__, __LINE__);
  if (st != TQ_OK) { delete a; return st; }
  *out = a;
  return TQ_OK;
}

int32_t tq_agg_create_final(const tq_agg_final_desc *d, tq_agg **out) {
  if (!d || !out) return TQ_ERR_INVALID_ARG;
  *out = nullptr;
  if (d->n_input_cols < 0 || d->n_group_by < 0 || d->n_group_by > MK_MAX_KEYS || d->n_funcs < 0 || d->n_funcs > AGG_MAXF) {
    set_error("too many columns / functions");
    return TQ_ERR_INVALID_ARG;
  }
  // internal layout = the one tq_agg_merge_partial reads: GROUP BY columns, then the state columns in function order
  int32_t types[AGG_MAXC], gb[MK_MAX_KEYS], src[AGG_MAXC];
  tq_agg_func fn[AGG_MAXF];
  int n = 0;
  auto in_type = [&](int c) { return d->input_types[c] & 0xFF; };   // TQ_TYPE_NOT_NULL is dropped: a partial SUM / MAX / MIN may be NULL
  auto bad_col = [&](int c) { return c < 0 || c >= d->n_input_cols; };
  for (int g = 0; g < d->n_group_by; g++) {
    if (bad_col(d->group_by_cols[g])) { set_error("GROUP BY item %d is not an input column", g); return TQ_ERR_INVALID_ARG; }
    gb[g] = n; src[n] = d->group_by_cols[g]; types[n] = in_type(src[n]); n++;
  }
  for (int i = 0; i < d->n_funcs; i++) {
    const tq_agg_final_func &f = d->funcs[i];
    const bool avg = f.func == TQ_AGG_AVG;
    if (f.func < TQ_AGG_COUNT || f.func > TQ_AGG_FIRSTROW || bad_col(f.arg_col) || (avg && bad_col(f.arg_col2)) || n + (avg ? 2 : 1) > AGG_MAXC) {
      set_error("bad FinalMode aggregate descriptor %d", i);
      return TQ_ERR_INVALID_ARG;
    }
    // countPartial / avgPartial4* read the partial COUNT with EvalInt (func_count.go:99-113, func_avg.go:86-113,200-227)
    if ((f.func == TQ_AGG_COUNT || avg) && in_type(f.arg_col) != TQ_TYPE_INT64 && in_type(f.arg_col) != TQ_TYPE_UINT64) {
      set_error("partial COUNT column of function %d must be BIGINT", i);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
    src[n] = f.arg_col; types[n] = in_type(f.arg_col); n++;
    fn[i].func = f.func;
    fn[i].arg_col = n - 1;
    if (avg) {
      const int t2 = in_type(f.arg_col2);
      if (t2 != TQ_TYPE_INT64 && t2 != TQ_TYPE_UINT64 && t2 != TQ_TYPE_FLOAT64) { set_error("partial SUM column of AVG %d must be BIGINT or DOUBLE", i); return TQ_ERR_UNSUPPORTED_TYPE; }
      src[n] = f.arg_col2; types[n] = t2; n++;
      fn[i].arg_col = n - 1;   // the value type of AVG is the type of its partial sum (aggfuncs/builder.go:103-109)
    }
    if (f.func == TQ_AGG_SUM && types[fn[i].arg_col] != TQ_TYPE_INT64 && types[fn[i].arg_col] != TQ_TYPE_UINT64 && types[fn[i].arg_col] != TQ_TYPE_FLOAT64) {
      set_error("partial SUM column of function %d must be BIGINT or DOUBLE", i);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
  }
  tq_agg_desc syn{};
  syn.n_input_cols = n;
  syn.input_types = types;
  syn.n_group_by = d->n_group_by;
  syn.group_by_cols = gb;
  syn.n_funcs = d->n_funcs;
  syn.funcs = fn;
  syn.est_groups = d->est_groups;
  tq_agg *a = nullptr;
  TQ_TRY(tq_agg_create(&syn, &a));
  a->final_mode = true;
  a->final_n_in = d->n_input_cols;
  for (int j = 0; j < n; j++) a->final_src[j] = src[j];
  *out = a;
  return TQ_OK;
}

int32_t tq_agg_output_type(tq_agg *a, int32_t i, int32_t *t) {
  if (!a || !t || i < 0 || i >= a->n_funcs) return TQ_ERR_INVALID_ARG;
  *t = a->out_type[i];
  return TQ_OK;
}

int32_t tq_agg_put(tq_agg *a, const tq_column *cols, int32_t mem) {
  if (!a) return TQ_ERR_INVALID_ARG;
  if (a->final_mode) {
    // FinalMode: the chunk holds partial rows in the child's column order; hand them to the merge path in its own order
    if (!cols) return TQ_ERR_INVALID_ARG;
    tq_column view[AGG_MAXC];
    for (int j = 0; j < a->n_cols; j++) view[j] = cols[a->final_src[j]];
    if (a->n_cols == 0) {  // no GROUP BY and no functions: nothing to aggregate, but the row count must still be seen
      if (a->final_n_in == 0) return TQ_ERR_INVALID_ARG;
      return TQ_OK;
    }
    return agg_put_common(a, view, mem, true, a->n_cols);
  }
  return agg_put_common(a, cols, mem, false, a->n_cols);
}

static bool agg_has_varlen(const tq_agg *a) {
  for (int c = 0; c < a->n_cols; c++) if (a->in_kind[c] == 2) return true;
  return false;
}

int32_t tq_agg_merge_partial(tq_agg *a, const tq_column *cols, int32_t mem) {
  if (!a) return TQ_ERR_INVALID_ARG;
  if (a->final_mode) { set_error("a FinalMode handle takes its partial rows through tq_agg_put"); return TQ_ERR_STATE; }
  // partial rows of a var-len column would carry ids of the exporting handle's dictionary
  if (agg_has_varlen(a)) { set_error("partial export / merge with var-len columns is not supported"); return TQ_ERR_UNSUPPORTED_TYPE; }
  return agg_put_common(a, cols, mem, true, partial_width(a));
}

int32_t tq_agg_partial_width(tq_agg *a, int32_t *n) {
  if (!a || !n) return TQ_ERR_INVALID_ARG;
  *n = partial_width(a);
  return TQ_OK;
}

int32_t tq_agg_eof(tq_agg *a) {
  if (!a) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  if (a->eof) return TQ_OK;
  const bool merge = a->merge_mode_seen;
  TQ_TRY(agg_flush_stage(a, merge, merge ? partial_width(a) : a->n_cols));
  a->eof = true;
  return TQ_OK;
}

static int32_t agg_ensure_final(tq_agg *a) {
  if (a->finalized) return TQ_OK;
  if (!a->eof) { set_error("next before eof: HashAgg is a pipeline breaker"); return TQ_ERR_STATE; }
  TQ_TRY(agg_finalize(a, false, a->result, a->n_funcs));
  AggResult &res = a->result;
  res.var.clear();
  if (a->any_kind && res.n > 0) {
    // FLOAT results are narrowed back to 4-byte slots (AppendFloat32), string results gathered from the dictionary arena
    // into offsets + bytes (AppendString): chunk.Column layout of the result type (util/chunk/column.go:28-34)
    cudaStream_t s = rt().compute;
    res.var.resize(a->n_funcs);
    for (int i = 0; i < a->n_funcs; i++) {
      VarOut &v = res.var[i];
      if (a->out_kind[i] == 2) {
        TQ_TRY(gather_cells(a->sd[a->out_src[i]].arena, res.data[i].as<uint64_t>(), res.bm[i].as<uint32_t>(), res.n, v, a->lens_scratch, a->scan_scratch, s));
      } else if (a->out_kind[i] == 1) {
        TQ_TRY(v.bytes.reserve((size_t)res.n * 4));
        TQ_TRY(narrow_f64(res.data[i].as<uint64_t>(), res.n, v.bytes.as<uint32_t>(), s));
        v.elem = 4;
        v.total = res.n * 4;
        v.used = true;
        v.on_host = false;
      }
    }
    TQ_CUDA(cudaStreamSynchronize(s));
  }
  a->finalized = true;
  a->result_pos = 0;
  return TQ_OK;
}

static bool agg_out_indirect(const tq_agg *a, int i) { return a->out_kind[i] != 0 && i < (int)a->result.var.size() && a->result.var[i].used; }

// copy the whole result to pinned host memory once (data, bitmaps, FLOAT / var-len forms)
static int32_t agg_result_to_host(tq_agg *a) {
  AggResult &res = a->result;
  if (res.on_host) return TQ_OK;
  Runtime &r = rt();
  res.h_data.resize(a->n_funcs);
  res.h_bm.resize(a->n_funcs);
  for (int c = 0; c < a->n_funcs; c++) {
    TQ_TRY(res.h_bm[c].reserve(bitmap_alloc_bytes(res.n)));
    TQ_CUDA(cudaMemcpyAsync(res.h_bm[c].p, res.bm[c].p, bitmap_bytes(res.n), cudaMemcpyDeviceToHost, r.compute));
    if (agg_out_indirect(a, c)) {
      VarOut &v = res.var[c];
      TQ_TRY(v.h_bytes.reserve((size_t)v.total + 16));
      if (v.total) TQ_CUDA(cudaMemcpyAsync(v.h_bytes.p, v.bytes.p, (size_t)v.total, cudaMemcpyDeviceToHost, r.compute));
      if (v.elem == 0) {
        TQ_TRY(v.h_off.reserve((size_t)(res.n + 1) * 8));
        TQ_CUDA(cudaMemcpyAsync(v.h_off.p, v.off.p, (size_t)(res.n + 1) * 8, cudaMemcpyDeviceToHost, r.compute));
      }
      v.on_host = true;
    } else {
      TQ_TRY(res.h_data[c].reserve((size_t)res.n * 8));
      TQ_CUDA(cudaMemcpyAsync(res.h_data[c].p, res.data[c].p, (size_t)res.n * 8, cudaMemcpyDeviceToHost, r.compute));
    }
  }
  TQ_CUDA(cudaStreamSynchronize(r.compute));
  res.on_host = true;
  return TQ_OK;
}

int32_t tq_agg_next_bytes(tq_agg *a, int64_t max_rows, int64_t *bytes_per_col) {
  if (!a || !bytes_per_col || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(agg_ensure_final(a));
  AggResult &res = a->result;
  for (int c = 0; c < a->n_funcs; c++) bytes_per_col[c] = 0;
  if (a->rows_total == 0 && a->n_group_by == 0 && a->result_pos == 0) {   // the default row: 8-byte / 4-byte slot, empty string
    for (int c = 0; c < a->n_funcs; c++) bytes_per_col[c] = a->out_kind[c] == 2 ? 0 : (a->out_kind[c] == 1 ? 4 : 8);
    return TQ_OK;
  }
  if (a->rows_total == 0 || a->result_pos >= res.n) return TQ_OK;
  TQ_TRY(agg_result_to_host(a));
  const int64_t take = res.n - a->result_pos < max_rows ? res.n - a->result_pos : max_rows;
  for (int c = 0; c < a->n_funcs; c++) {
    if (!agg_out_indirect(a, c)) bytes_per_col[c] = take * 8;
    else if (res.var[c].elem == 4) bytes_per_col[c] = take * 4;
    else {
      const int64_t *off = res.var[c].h_off.as<int64_t>() + a->result_pos;
      bytes_per_col[c] = off[take] - off[0];
    }
  }
  return TQ_OK;
}

int32_t tq_agg_next(tq_agg *a, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!a || !n_rows || !eof || max_rows <= 0 || (a->n_funcs && !out_cols)) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  *n_rows = 0;
  *eof = 0;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(agg_ensure_final(a));
  AggResult &res = a->result;
  // empty input without GROUP BY: one default row — COUNT 0, everything else NULL (aggregate.go:572-574,
  // builder.go:517-540); all-FIRSTROW aggregates produce no row
  if (a->rows_total == 0 && a->n_group_by == 0 && a->result_pos == 0) {
    bool all_first = true;
    for (int i = 0; i < a->n_funcs; i++) if (a->funcs[i].func != TQ_AGG_FIRSTROW) all_first = false;
    a->result_pos = 1;
    if (!all_first && a->n_funcs) {
      for (int i = 0; i < a->n_funcs; i++) {
        if (!out_cols[i].null_bitmap || (a->out_kind[i] != 2 && !out_cols[i].data) || (a->out_kind[i] == 2 && !out_cols[i].offsets)) return TQ_ERR_INVALID_ARG;
        if (a->out_kind[i] == 2) { out_cols[i].offsets[0] = 0; out_cols[i].offsets[1] = 0; }
        else memset(out_cols[i].data, 0, a->out_kind[i] == 1 ? 4 : 8);
        out_cols[i].null_bitmap[0] = (a->funcs[i].func == TQ_AGG_COUNT) ? 1 : 0;
        out_cols[i].length = 1;
      }
      *n_rows = 1;
      return TQ_OK;
    }
  }
  if (a->rows_total == 0 || a->result_pos >= res.n) { *eof = 1; for (int i = 0; i < a->n_funcs; i++) out_cols[i].length = 0; return TQ_OK; }
  TQ_TRY(agg_result_to_host(a));
  const int64_t take = res.n - a->result_pos < max_rows ? res.n - a->result_pos : max_rows;
  for (int c = 0; c < a->n_funcs; c++) {
    const bool ind = agg_out_indirect(a, c), var = ind && res.var[c].elem == 0;
    if (!out_cols[c].null_bitmap || (!out_cols[c].data && !var) || (var && !out_cols[c].offsets)) {
      set_error("output column %d needs data and null_bitmap buffers (and offsets for a var-len column)", c);
      return TQ_ERR_INVALID_ARG;
    }
    if (var) {   // offsets rebased to 0 + the cells' bytes (chunk.Column layout)
      const int64_t *off = res.var[c].h_off.as<int64_t>() + a->result_pos;
      const int64_t b0 = off[0];
      for (int64_t i = 0; i <= take; i++) out_cols[c].offsets[i] = off[i] - b0;
      if (off[take] > b0) {
        if (!out_cols[c].data) { set_error("output column %d needs a data buffer (tq_agg_next_bytes tells its size)", c); return TQ_ERR_INVALID_ARG; }
        memcpy(out_cols[c].data, res.var[c].h_bytes.as<uint8_t>() + b0, (size_t)(off[take] - b0));
      }
    } else if (ind) memcpy(out_cols[c].data, res.var[c].h_bytes.as<uint8_t>() + a->result_pos * 4, (size_t)take * 4);
    else memcpy(out_cols[c].data, res.h_data[c].as<uint8_t>() + a->result_pos * 8, (size_t)take * 8);
    host_bitmap_extract(out_cols[c].null_bitmap, res.h_bm[c].as<uint8_t>(), a->result_pos, take);
    out_cols[c].length = take;
  }
  a->result_pos += take;
  *n_rows = take;
  return TQ_OK;
}

int32_t tq_agg_next_device(tq_agg *a, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!a || !out_cols || !n_rows || !eof) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  *n_rows = 0;
  *eof = 0;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(agg_ensure_final(a));
  if (a->result_pos > 0 || a->result.n == 0) { *eof = 1; return TQ_OK; }
  for (int c = 0; c < a->n_funcs; c++) {
    out_cols[c].length = a->result.n;
    out_cols[c].data = a->result.data[c].as<uint8_t>();
    out_cols[c].null_bitmap = a->result.bm[c].as<uint8_t>();
    out_cols[c].offsets = nullptr;
    if (agg_out_indirect(a, c)) {   // FLOAT slots / gathered strings, device resident
      out_cols[c].data = a->result.var[c].bytes.as<uint8_t>();
      if (a->result.var[c].elem == 0) out_cols[c].offsets = a->result.var[c].off.as<int64_t>();
    }
  }
  *n_rows = a->result.n;
  a->result_pos = a->result.n;
  return TQ_OK;
}

int32_t tq_agg_export_partial(tq_agg *a, tq_column *out_cols, int64_t *n_rows) {
  if (!a || !out_cols || !n_rows) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  if (agg_has_varlen(a)) { set_error("partial export / merge with var-len columns is not supported"); return TQ_ERR_UNSUPPORTED_TYPE; }
  if (!a->eof) TQ_TRY(tq_agg_eof(a));
  const int w = partial_width(a);
  TQ_TRY(agg_finalize(a, true, a->result, w));
  for (int c = 0; c < w; c++) {
    out_cols[c].length = a->result.n;
    out_cols[c].data = a->result.data[c].as<uint8_t>();
    out_cols[c].null_bitmap = a->result.bm[c].as<uint8_t>();
    out_cols[c].offsets = nullptr;
  }
  *n_rows = a->result.n;
  return TQ_OK;
}

int32_t tq_agg_stats(tq_agg *a, int64_t *s) {
  if (!a || !s) return TQ_ERR_INVALID_ARG;
  s[0] = a->rows_total;
  s[1] = a->result.n;
  s[2] = a->last_update_ns;
  s[3] = a->launches;
  return TQ_OK;
}

int32_t tq_agg_destroy(tq_agg *a) {
  if (!a) return TQ_OK;
  if (rt().inited) {
    cudaSetDevice(rt().device);
    cudaDeviceSynchronize();  // Close may run after Open without Next (aggregate.go:187-197)
  }
  delete a;
  return TQ_OK;
}

}  // extern "C"
