// join.cu — HashJoinExec on the device (replaces executor/join.go, hash_table.go, joiner.go).
//
// Table.  Open-addressed entries of 2 or 4 eight-byte words, word 0 = the join key.  Large build sides
// are split by the TOP bits of the key hash into 2^pbits partition tables stored back to back (linear
// probing wraps inside a partition), so the probe side can be radix-scattered the same way and only a
// few partition tables are live — in L2, or in shared memory when a partition image is <= 128 KB.
//   ROW mode (unique build keys, <= 4 words per row — the PK-FK join): the entry IS the build row:
//       word0 = key, then the other build columns, then an optional NOT-NULL mask word.
//       One 16/32-byte sector per probe; the build is: init, insert (atomicCAS), write rows.
//   CSR mode (duplicate keys or wide rows): word1 = (offset | count << 32) into build rows packed
//       row-major in key order; duplicates keep build insertion order (rowHashMap.Get, hash_table.go:259-272).
//       Build: insert+count, exclusive scan, fill, sort duplicate segments, gather rows.
//   Large NOT NULL build sides that fit an entry first try the streaming build (try_stream_build, gated by stream_build_ok):
//       k_scatter_aos into AoS slabs, then k_build_cta builds each sub-table in one CTA's shared memory (k_build_cluster, in
//       cluster shared memory, where no sub-table size that one CTA holds stays within PART_MAX_BITS).
// Probe.  Small build (one table): k_probe, ordered output (probe row asc, build insertion asc) via
//   ticketed tiles + decoupled look-back.
//   Large build, PK-FK shape (stream_probe_ok, no probe NULL bitmap): the streaming positional path of join_stream.cuh
//   (launch_probe_stream): k_pos_reset -> k_scatter_cols (the probe columns straight into result pages claimed on the fly)
//   -> k_pos_pages -> k_probe_pos (key column in, build columns out) -> hole filling; the result is a multiset.
//   Any other large build: k_probe_part_hist (only after a slab overflow) -> scan -> k_probe_scatter(_fast) (shared-memory
//   counting sort of 4096-row tiles, coalesced full-sector stores) -> k_probe_part_fast / k_probe_part(_uniq).
#include <chrono>
#include <cstdlib>
#include <deque>
#include <memory>
#include <new>

#include "common.cuh"
#include "dict.cuh"
#include "varlen.cuh"
#include "strdict.cuh"
#include "push.cuh"
#include "scatter.cuh"
#include "othercond.cuh"
#include "nlj.cuh"

namespace tq {

static constexpr int MAXC = 16;  // columns per join side

// Bits [off, off + rows) of a concatenated device bitmap from one chunk's bitmap (bit i = row i of the chunk), for a chunk that
// does not start on a byte boundary: each thread owns one 32-bit destination word and rewrites only the chunk's bits in it.
__global__ void k_bitmap_append(uint32_t *dst, int64_t off, const uint8_t *src, int64_t rows) {
  const int64_t w1 = (off + rows + 31) >> 5;
  for (int64_t w = (off >> 5) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < w1; w += (int64_t)gridDim.x * blockDim.x) {
    uint32_t v = dst[w];
    for (int b = 0; b < 32; b++) {
      const int64_t i = (w << 5) + b - off;
      if (i < 0 || i >= rows) continue;
      v = (v & ~(1u << b)) | ((uint32_t)((src[i >> 3] >> (i & 7)) & 1) << b);
    }
    dst[w] = v;
  }
}
static constexpr uint64_t EMPTY_KEY = 0xA5C3F00DDEADBEEFull;  // empty-entry marker; a real key with this value lives in a side entry/segment
static constexpr uint32_t ROW_INVALID = 0xFFFFFFFFu, ROW_SENTINEL = 0xFFFFFFFEu;
static constexpr uint32_t OFF_MISS = 0xFFFFFFFFu;
static constexpr int64_t PART_MIN_BUILD_ROWS = 1 << 18;  // below this the whole table (<= 8 MB) is L2-resident anyway
static constexpr int PART_MAX_BITS = 12;
static constexpr uint64_t PART_MAX_SMEM_BYTES = 128 << 10;  // a partition table image that still fits in shared memory
static const int64_t g_tiles_per_cta = 8;
static constexpr int64_t PART_TARGET_ROWS = 150000;      // build rows per partition: a partition table ~ 4-8 MB, a few live ones fit in L2
static const int64_t g_max_load_pct = 50;                // partition-table load-factor bound (pair probing keeps chains short)
static bool g_no_fast_kernel = false;                    // TQ_JOIN_NO_FAST=1: use the generic kernels (tests)

// key_mode: how (flag, raw bytes) equality (util/codec/codec.go:212-240,363-382) maps onto raw 8-byte equality
//   0: flags always agree (both signed, both unsigned, or both DOUBLE)  -> raw equality
//   1: one side UNSIGNED, the other signed: values with the sign bit set carry different flags
//      (uvarintFlag vs varintFlag) and can never match -> such rows are treated like NULL keys
//   2: int-class vs DOUBLE: flags never agree -> nothing matches
enum { KEYMODE_RAW = 0, KEYMODE_NO_SIGNBIT = 1, KEYMODE_NEVER = 2 };

struct JoinTable {
  uint64_t *words;  // entry e = words[e << shift ...]
  uint32_t cap;     // entries per partition table (even; partition table t starts at entry t * cap)
  int pbits;        // log2(#partition tables); 0 = one table
  int shift;        // log2(words per entry): 1 or 2
  int row_mode;
  uint32_t sent_off, sent_cnt;  // CSR: CSR segment of the EMPTY_KEY-valued key.  ROW: sent_off = entry index of that row, sent_cnt = 0/1
};
__device__ __forceinline__ uint64_t part_of_hash(uint64_t h, int pbits) { return pbits ? (h >> (64 - pbits)) : 0; }

__device__ __forceinline__ bool key_valid(uint64_t key, bool not_null, int key_mode) {
  if (!not_null) return false;
  if (key_mode == KEYMODE_RAW) return true;
  if (key_mode == KEYMODE_NO_SIGNBIT) return (key >> 63) == 0;
  return false;
}

// The slot arithmetic of every partition table (builders and probers alike).  A table of `cap` entries need not be a power
// of two: the home slot scales the low 32 hash bits onto [0, cap) (the partition comes from the top bits), and probing wraps
// inside the table.  16-byte entries (shift == 1) start on an even slot, so a 32-byte sector holds a whole entry PAIR.
__device__ __forceinline__ uint32_t home_slot(uint64_t h, uint32_t cap, int shift) {
  const uint32_t s = __umulhi((uint32_t)h, cap);
  return shift == 1 ? (s & ~1u) : s;
}
__device__ __forceinline__ uint32_t next_slot(uint32_t loc, uint32_t step, uint32_t cap) {
  loc += step;
  return loc >= cap ? loc - cap : loc;
}

// (word0, word1) of an entry with one 128-bit load
__device__ __forceinline__ ulonglong2 ld_entry(const uint64_t *words, uint64_t e, int shift) {
  return *reinterpret_cast<const ulonglong2 *>(words + (e << shift));
}

__global__ void k_init_table(uint64_t *words, uint64_t n_entries, int shift) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t n_words = n_entries << shift, wmask = (1ull << shift) - 1;
  for (; i < n_words; i += stride) words[i] = (i & wmask) ? 0ull : EMPTY_KEY;
}

// counters: [0] EMPTY_KEY-valued rows, [1] their fill cursor, [2] distinct regular keys, [3] large-segment worklist length,
//           [4] max rows of a build partition, [5] valid regular rows, u64 @ [8] scan total
// The thread whose atomicCAS claims an entry also writes its row into it when the row fits the entry (ROW-mode
// candidate): if the keys then turn out to be unique the table is complete after this one kernel.
struct InsertParams {
  int n_cols, key_col, key_mode;
  DCol cols[MAXC];
  int word_of_col[MAXC];  // word inside the entry (key column -> 0); only used when write_rows
  int mask_word;          // -1: no NOT-NULL mask word
  int write_rows;
  int64_t n;
  uint64_t *words;
  uint32_t cap;           // entries per partition table
  int pbits, shift;
  uint32_t sent_entry;
  uint32_t *row_slot;
  uint32_t *counters;
};
__device__ __forceinline__ void write_row_words(const InsertParams &b, uint64_t *ent, int64_t i, bool with_key) {
  uint64_t m = 0;
  for (int c = 0; c < b.n_cols; c++) {
    if (c != b.key_col || with_key) ent[b.word_of_col[c]] = b.cols[c].data[i];
    m |= (uint64_t)tqd::bm_not_null(b.cols[c].bm, i) << c;
  }
  if (b.mask_word >= 0) ent[b.mask_word] = m;
}
__global__ void __launch_bounds__(256) k_build_insert(const InsertParams b) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const uint64_t *keys = b.cols[b.key_col].data;
  const uint32_t *bm = b.cols[b.key_col].bm;
  unsigned my_valid = 0, my_new = 0;
  for (; i < b.n; i += stride) {
    const uint64_t key = keys[i];
    if (!key_valid(key, tqd::bm_not_null(bm, i), b.key_mode)) { b.row_slot[i] = ROW_INVALID; continue; }  // hash_table.go:161-163
    if (key == EMPTY_KEY) {
      const uint32_t prior = atomicAdd(&b.counters[0], 1u);
      b.row_slot[i] = ROW_SENTINEL;
      if (b.write_rows && prior == 0) write_row_words(b, b.words + ((uint64_t)b.sent_entry << b.shift), i, true);
      continue;
    }
    const uint64_t h = tqd::hash_key(key);
    const uint64_t base = part_of_hash(h, b.pbits) * b.cap;
    uint32_t loc = home_slot(h, b.cap, b.shift);
    my_valid++;
    for (;;) {
      const uint64_t e = base + loc;
      const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(&b.words[e << b.shift]), (unsigned long long)EMPTY_KEY,
                                                (unsigned long long)key);
      if (prev == EMPTY_KEY) {
        my_new++;
        if (b.write_rows) write_row_words(b, b.words + (e << b.shift), i, false);
      }
      if (prev == EMPTY_KEY || prev == key) { b.row_slot[i] = (uint32_t)e; break; }
      loc = next_slot(loc, 1, b.cap);
    }
  }
  my_valid = __reduce_add_sync(0xffffffffu, my_valid);
  my_new = __reduce_add_sync(0xffffffffu, my_new);
  if ((threadIdx.x & 31) == 0) {
    if (my_valid) atomicAdd(&b.counters[5], my_valid);
    if (my_new) atomicAdd(&b.counters[2], my_new);
  }
}

// CSR mode only (duplicate keys): clear word 1 of every entry (it may hold an inlined column), then count rows per key.
__global__ void k_clear_word1(uint64_t *words, uint64_t n_entries, int shift) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n_entries; i += stride) words[(i << shift) + 1] = 0;
}
__global__ void __launch_bounds__(256) k_build_count(const uint32_t *row_slot, int64_t n, uint64_t *words, int shift) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const uint32_t e = row_slot[i];
    if (e == ROW_INVALID || e == ROW_SENTINEL) continue;
    atomicAdd(reinterpret_cast<uint32_t *>(&words[((uint64_t)e << shift) + 1]) + 1, 1u);  // count = high half of word 1
  }
}

// rows per build partition (valid keys only) — decides the partition table capacity.  Per-CTA shared-memory
// histogram, then one global atomic per non-empty bin per CTA.
__global__ void __launch_bounds__(256) k_build_part_hist(const uint64_t *keys, const uint32_t *bm, int64_t n, int key_mode, int pbits,
                                                          uint32_t *part_cnt) {
  __shared__ uint32_t s_hist[1 << PART_MAX_BITS];
  const int n_bins = 1 << pbits;
  for (int b = threadIdx.x; b < n_bins; b += blockDim.x) s_hist[b] = 0;
  __syncthreads();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const uint64_t key = keys[i];
    if (!key_valid(key, tqd::bm_not_null(bm, i), key_mode) || key == EMPTY_KEY) continue;
    atomicAdd(&s_hist[part_of_hash(tqd::hash_key(key), pbits)], 1u);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < n_bins; b += blockDim.x)
    if (s_hist[b]) atomicAdd(&part_cnt[b], s_hist[b]);
}

__global__ void k_max_u32(const uint32_t *v, int n, uint32_t *out) {
  uint32_t m = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = max(m, v[i]);
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// ---- CSR mode build kernels
__global__ void __launch_bounds__(256) k_build_fill(const uint32_t *row_slot, int64_t n, uint64_t *words, int shift, uint32_t sent_off,
                                                     uint32_t *counters, uint32_t *row_ids) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const uint32_t s = row_slot[i];
    if (s == ROW_INVALID) continue;
    uint32_t pos;
    if (s == ROW_SENTINEL) pos = sent_off + atomicAdd(&counters[1], 1u);
    else pos = atomicAdd(reinterpret_cast<uint32_t *>(&words[((uint64_t)s << shift) + 1]), 1u);  // offset = low half of word 1
    row_ids[pos] = (uint32_t)i;
  }
}

// Restores the offsets (k_build_fill advanced them by count) and sorts duplicate-key segments ascending by row id.
__global__ void __launch_bounds__(256) k_build_fixsort(uint64_t *words, uint64_t n_entries, int shift, uint32_t *row_ids, uint32_t *counters,
                                                        uint2 *worklist, uint32_t worklist_cap) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n_entries; i += stride) {
    uint32_t *w1 = reinterpret_cast<uint32_t *>(&words[(i << shift) + 1]);
    const uint32_t cnt = w1[1];
    if (cnt == 0) continue;
    const uint32_t off = w1[0] - cnt;
    w1[0] = off;
    if (cnt == 1) continue;
    if (cnt <= 32) {
      uint32_t *seg = row_ids + off;  // insertion sort: segments are tiny
      for (uint32_t a = 1; a < cnt; a++) {
        const uint32_t v = seg[a];
        uint32_t b = a;
        while (b > 0 && seg[b - 1] > v) { seg[b] = seg[b - 1]; b--; }
        seg[b] = v;
      }
    } else {
      const uint32_t w = atomicAdd(&counters[3], 1u);
      if (w < worklist_cap) worklist[w] = make_uint2(off, cnt);
    }
  }
}

// One CTA per large duplicate segment: bitonic sort in global memory (indices >= cnt act as +inf).
__global__ void __launch_bounds__(256) k_sort_large(const uint2 *worklist, uint32_t *row_ids) {
  const uint2 w = worklist[blockIdx.x];
  uint32_t *seg = row_ids + w.x;
  const uint32_t n = w.y;
  uint32_t p2 = 1;
  while (p2 < n) p2 <<= 1;
  // all comparators ascending (first stage of each merge mirrors: partner = t ^ (k-1)), so the virtual
  // +inf tail never has to move and comparators touching it are skipped
  for (uint32_t k = 2; k <= p2; k <<= 1) {
    for (uint32_t t = threadIdx.x; t < p2; t += blockDim.x) {
      const uint32_t partner = t ^ (k - 1);
      if (partner > t && partner < n) {
        const uint32_t a = seg[t], b = seg[partner];
        if (a > b) { seg[t] = b; seg[partner] = a; }
      }
    }
    __syncthreads();
    for (uint32_t j = k >> 2; j > 0; j >>= 1) {
      for (uint32_t t = threadIdx.x; t < p2; t += blockDim.x) {
        const uint32_t partner = t ^ j;
        if (partner > t && partner < n) {
          const uint32_t a = seg[t], b = seg[partner];
          if (a > b) { seg[t] = b; seg[partner] = a; }
        }
      }
      __syncthreads();
    }
  }
}

// B'[pos] = B[row_ids[pos]] packed row-major (+ NOT-NULL mask per row): build rows in CSR order.
struct GatherParams {
  int n_cols;
  DCol cols[MAXC];
  const uint32_t *row_ids;
  int64_t n;
  uint64_t *out_rows;
  uint32_t *out_mask;  // nullptr: no build column holds NULLs
};
__global__ void __launch_bounds__(256) k_gather_rows(const GatherParams g) {
  int64_t pos = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; pos < g.n; pos += stride) {
    const uint32_t r = g.row_ids[pos];
    uint32_t mask = 0;
    for (int c = 0; c < g.n_cols; c++) {
      g.out_rows[pos * g.n_cols + c] = g.cols[c].data[r];
      mask |= (uint32_t)tqd::bm_not_null(g.cols[c].bm, r) << c;
    }
    if (g.out_mask) g.out_mask[pos] = mask;
  }
}

// ------------------------------------------------------------------ probe
static constexpr int PROBE_THREADS = 256;
static constexpr int PROBE_ROWS_PER_THREAD = 4;
static constexpr int PROBE_TILE = PROBE_THREADS * PROBE_ROWS_PER_THREAD;

struct ProbeParams {
  int n_probe_cols, n_build_cols;
  DCol probe[MAXC];           // probe columns (the partitioned copies on the partitioned path)
  DColMut out_probe[MAXC];    // destination of probe column c (bm == nullptr: column cannot hold NULLs, bitmap pre-filled)
  DColMut out_build[MAXC];
  // build rows: CSR mode = rows packed row-major in key order; ROW mode = the table entries themselves
  const uint64_t *build_rows;
  int build_stride;           // words between consecutive build rows
  int build_word[MAXC];       // word of build column c inside a row
  const uint32_t *build_mask; // CSR mode: NOT-NULL mask per row (nullptr: no NULLs)
  int build_mask_word;        // ROW mode: word holding the NOT-NULL mask (-1: none)
  const uint8_t *selected;    // outerSideFilter result or nullptr (one-table path only; the scatter applies it on the partitioned path)
  int key_col;
  int key_mode;
  int is_outer;               // LeftOuter / RightOuter: misses emit probe row ++ defaultInner (joiner.go:274-277,337-340)
  uint64_t def_val[MAXC];     // defaultInner (PhysicalHashJoin.DefaultValues, joiner.go:139-143): value of build column c in a miss row
  uint32_t def_mask;          // ... and its NOT-NULL bits (0 = the usual all-NULL inner side)
  int64_t n;
  uint64_t capacity;          // rows the output columns can hold
  unsigned long long *cursor; // [0] rows produced (may exceed capacity: then the batch is re-run), [1] matched probe rows
  // ordered output (one-table path): tiles are handed out by ticket and each tile learns the output offset of all
  // earlier tiles by decoupled look-back over tile_state (bits 63..62: 1 = tile total, 2 = inclusive prefix)
  unsigned long long *tile_state;
  unsigned *ticket;
  // partitioned path: rows of partition q are [part_off[q], part_off[q+1]) of the probe columns; partition
  // 2^pbits holds the rows that cannot match (NULL / filtered keys) and exists only for outer joins
  const uint32_t *part_lo, *part_hi;  // exact path: hi == lo + 1 (one offsets array); optimistic slabs: hi = scatter cursors
  const uint32_t *part_lim;           // optimistic slabs: end of each partition's slab (nullptr on the exact path)
  int split;                  // CTAs per partition
  int table_in_smem;          // partition table images fit in shared memory (TMA bulk-loaded)
};

struct TileSmem {
  unsigned long long prefix[PROBE_TILE + 1];
  uint32_t off[PROBE_TILE];
  unsigned long long warp_sums[PROBE_THREADS / 32 + 1];
  unsigned long long base;
  long long tile;
};

// build-side values of one match.  `off` = build row index (CSR position or entry index), OFF_MISS = pad with NULLs.
struct BuildRow {
  const uint64_t *row;
  uint32_t mask;
  uint64_t w0, w1;  // words 0 and 1 of the row when the caller already holds them in registers (ROW mode)
  bool have01;
  __device__ __forceinline__ uint64_t word(int w) const { return (have01 && w < 2) ? (w ? w1 : w0) : row[w]; }
};
__device__ __forceinline__ BuildRow build_row_of(const ProbeParams &p, bool want, uint32_t off, bool have01 = false, uint64_t w0 = 0, uint64_t w1 = 0) {
  BuildRow b;
  b.row = nullptr;
  b.mask = want ? p.def_mask : 0u;   // a miss row carries defaultInner; lanes past the tile's rows contribute no bits
  b.have01 = have01;
  b.w0 = w0;
  b.w1 = w1;
  if (want && off != OFF_MISS) {
    b.row = p.build_rows + (uint64_t)off * (uint64_t)p.build_stride;
    if (p.build_mask) b.mask = p.build_mask[off];
    else if (p.build_mask_word >= 0) b.mask = (uint32_t)b.word(p.build_mask_word);
    else b.mask = 0xFFFFFFFFu;
  }
  return b;
}

// Look one key up.  Returns (off, cnt): CSR mode = CSR segment; ROW mode = (entry index, 1).  cnt == 0: miss.
// `first` is the already-loaded (word0, word1) of the home entry at partition-local index loc.
template <bool SMEM>
__device__ __forceinline__ uint2 resolve(const JoinTable &t, const uint64_t *tbl /*partition base (global or smem)*/, uint64_t ebase, uint64_t key,
                                         uint32_t loc, ulonglong2 &cur /* in: home entry; out: matched entry (word0, word1) */) {
  while (cur.x != key && cur.x != EMPTY_KEY) {  // linear probing; short at load factor <= 0.5
    loc = next_slot(loc, 1, t.cap);
    cur = ld_entry(tbl, loc, t.shift);
  }
  if (cur.x != key) return make_uint2(OFF_MISS, 0);
  if (t.row_mode) return make_uint2((uint32_t)(ebase + loc), 1u);
  return make_uint2((uint32_t)cur.y, (uint32_t)(cur.y >> 32));
}

// Phase B: exclusive scan of the tile's PROBE_TILE match counts (held in sm.prefix as counts on entry).
// Returns the tile total M; sm.prefix[0..TILE] holds the exclusive prefix afterwards.
__device__ __forceinline__ unsigned long long tile_scan(TileSmem &sm, unsigned &matched_acc, bool &any_multi) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned long long c4[PROBE_ROWS_PER_THREAD], tsum = 0;
  unsigned matched = 0;
#pragma unroll
  for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
    c4[k] = sm.prefix[tid * PROBE_ROWS_PER_THREAD + k];
    tsum += c4[k];
    matched += (sm.off[tid * PROBE_ROWS_PER_THREAD + k] != OFF_MISS);
  }
  const bool my_multi = (c4[0] > 1) | (c4[1] > 1) | (c4[2] > 1) | (c4[3] > 1);
  unsigned long long inc = tsum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += v;
  }
  matched = __reduce_add_sync(0xffffffffu, matched);
  if (lane == 31) sm.warp_sums[warp] = inc;
  any_multi = __syncthreads_or(my_multi) != 0;  // (barrier) also orders the c4 reads before the prefix writes below
  if (warp == 0) {
    unsigned long long w = (lane < PROBE_THREADS / 32) ? sm.warp_sums[lane] : 0;
    unsigned long long winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long v = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += v;
    }
    if (lane < PROBE_THREADS / 32) sm.warp_sums[lane] = winc - w;
    if (lane == PROBE_THREADS / 32 - 1) sm.warp_sums[PROBE_THREADS / 32] = winc;
  }
  if (lane == 0) matched_acc += matched;  // per-warp running total; flushed once per CTA (one same-address atomic, not one per tile)
  __syncthreads();
  unsigned long long run = inc - tsum + sm.warp_sums[warp];
#pragma unroll
  for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
    sm.prefix[tid * PROBE_ROWS_PER_THREAD + k] = run;
    run += c4[k];
  }
  const unsigned long long M = sm.warp_sums[PROBE_THREADS / 32];
  if (tid == 0) sm.prefix[PROBE_TILE] = M;
  return M;
}

// Phase D, general: output-centric expansion.  Thread per OUTPUT row q in [base, base+M): binary search of the
// tile prefix gives the probe row r and the index j of the match inside the key's CSR segment; column stores are
// coalesced along q and the null-bitmap words are assembled with ballots (warp iterations are aligned to
// 32-row bitmap words; the partial first/last words of the tile are merged with atomicOr).
__device__ __forceinline__ void tile_expand(const ProbeParams &p, const TileSmem &sm, int64_t tile_base, unsigned long long base,
                                            unsigned long long M) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long base_al = base & ~31ull;
  const unsigned long long end = base + M;
  for (unsigned long long q0 = base_al + (unsigned long long)warp * 32; q0 < end; q0 += PROBE_THREADS) {
    const unsigned long long q = q0 + lane;
    const bool active = q >= base && q < end;
    const bool full_word = q0 >= base && q0 + 32 <= end;
    int r = 0;
    unsigned long long j = 0;
    uint32_t off = OFF_MISS;
    if (active) {
      const unsigned long long o = q - base;
      int lo = 0, hi = PROBE_TILE;  // find r: prefix[r] <= o < prefix[r+1]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (sm.prefix[mid] <= o) lo = mid; else hi = mid;
      }
      r = lo;
      j = o - sm.prefix[r];
      off = sm.off[r];
    }
    const int64_t row = tile_base + r;
    for (int c = 0; c < p.n_probe_cols; c++) {
      bool nn = false;
      if (active) {
        tqd::st_stream_u64(p.out_probe[c].data + q, p.probe[c].data[row]);
        nn = tqd::bm_not_null(p.probe[c].bm, row);
      }
      if (p.out_probe[c].bm) {
        const unsigned word = __ballot_sync(0xffffffffu, nn);
        if (lane == 0 && word) {
          if (full_word) p.out_probe[c].bm[q0 >> 5] = word;
          else atomicOr(&p.out_probe[c].bm[q0 >> 5], word);
        }
      }
    }
    const BuildRow b = build_row_of(p, active, off == OFF_MISS ? OFF_MISS : (uint32_t)(off + j));
    for (int c = 0; c < p.n_build_cols; c++) {
      if (active) tqd::st_stream_u64(p.out_build[c].data + q, b.row ? b.word(p.build_word[c]) : p.def_val[c]);  // miss: defaultInner (builder.go:463-465)
      if (p.out_build[c].bm) {
        const unsigned word = __ballot_sync(0xffffffffu, (b.mask >> c) & 1u);
        if (lane == 0 && word) {
          if (full_word) p.out_build[c].bm[q0 >> 5] = word;
          else atomicOr(&p.out_build[c].bm[q0 >> 5], word);
        }
      }
    }
  }
}

// OR `bit` into bm[q >> 5] for every active lane, one atomic per distinct word in the warp (q is monotone in the
// lane index, so there are 1-2 distinct words).  All 32 lanes must call.
__device__ __forceinline__ void warp_set_bits(uint32_t *bm, bool active, unsigned long long q, bool nn) {
  const int lane = threadIdx.x & 31;
  unsigned pending = __ballot_sync(0xffffffffu, active);
  const unsigned long long widx = q >> 5;
  const unsigned bit = (active && nn) ? (1u << (q & 31)) : 0u;
  while (pending) {
    const int leader = __ffs(pending) - 1;
    const unsigned long long w = __shfl_sync(0xffffffffu, widx, leader);
    const bool in_group = active && widx == w;
    const unsigned word = __reduce_or_sync(0xffffffffu, in_group ? bit : 0u);
    if (lane == leader && word) atomicOr(&bm[w], word);
    pending &= ~__ballot_sync(0xffffffffu, in_group);
  }
}

// Emit one output row (row-centric paths): probe columns of `row` + build row `off` at output position q.
// All 32 lanes of the warp must call (the bitmap helper is warp-collective).
__device__ __forceinline__ void emit_row(const ProbeParams &p, bool emit, int64_t row, uint64_t key, uint32_t off, unsigned long long q,
                                         bool have01 = false, uint64_t w0 = 0, uint64_t w1 = 0) {
  for (int c = 0; c < p.n_probe_cols; c++) {
    bool nn = false;
    if (emit) {
      const uint64_t v = (c == p.key_col) ? key : tqd::ld_stream_u64(p.probe[c].data + row);
      tqd::st_stream_u64(p.out_probe[c].data + q, v);
      nn = tqd::bm_not_null(p.probe[c].bm, row);
    }
    if (p.out_probe[c].bm) warp_set_bits(p.out_probe[c].bm, emit, q, nn);
  }
  const BuildRow b = build_row_of(p, emit, off, have01, w0, w1);
  for (int c = 0; c < p.n_build_cols; c++) {
    if (emit) tqd::st_stream_u64(p.out_build[c].data + q, b.row ? b.word(p.build_word[c]) : p.def_val[c]);
    if (p.out_build[c].bm) warp_set_bits(p.out_build[c].bm, emit, q, (b.mask >> c) & 1u);
  }
}

// Phase D for tiles in which every probe row has at most one output (unique build keys / misses): row-centric.
__device__ __forceinline__ void tile_emit_rowwise(const ProbeParams &p, const TileSmem &sm, int64_t tile_base, unsigned long long base,
                                                  const uint64_t (&key)[PROBE_ROWS_PER_THREAD]) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
    const int rl = k * PROBE_THREADS + tid;
    const unsigned long long pre = sm.prefix[rl];
    const bool emit = sm.prefix[rl + 1] != pre;
    emit_row(p, emit, tile_base + rl, key[k], sm.off[rl], base + pre);
  }
}

// ---- one-table probe (small build sides): ordered output
__global__ void __launch_bounds__(PROBE_THREADS) k_probe(const ProbeParams p, const JoinTable t) {
  __shared__ TileSmem sm;
  const int tid = threadIdx.x;
  const int64_t n_tiles = (p.n + PROBE_TILE - 1) / PROBE_TILE;
  const uint64_t *keys = p.probe[p.key_col].data;
  const uint32_t *kbm = p.probe[p.key_col].bm;
  unsigned matched_acc = 0;

  for (;;) {
    if (tid == 0) sm.tile = (long long)atomicAdd(p.ticket, 1u);
    __syncthreads();
    const int64_t tile = sm.tile;
    if (tile >= n_tiles) break;
    const int64_t tile_base = tile * PROBE_TILE;
    // ---- phase A: look up PROBE_ROWS_PER_THREAD keys per thread (coalesced: row = base + k*256 + tid)
    uint64_t key[PROBE_ROWS_PER_THREAD];
    bool valid[PROBE_ROWS_PER_THREAD];
    ulonglong2 first[PROBE_ROWS_PER_THREAD];
    uint64_t ebase[PROBE_ROWS_PER_THREAD];
    uint32_t loc[PROBE_ROWS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
      const int64_t r = tile_base + k * PROBE_THREADS + tid;
      key[k] = 0;
      valid[k] = false;
      if (r < p.n) {
        key[k] = tqd::ld_stream_u64(keys + r);
        const bool sel = p.selected ? (p.selected[r] != 0) : true;          // join.go:344 `!selected[i] || hasNull[i]` -> miss
        valid[k] = sel && key_valid(key[k], tqd::bm_not_null(kbm, r), p.key_mode);
      }
      const uint64_t h = tqd::hash_key(key[k]);
      ebase[k] = part_of_hash(h, t.pbits) * t.cap;
      loc[k] = home_slot(h, t.cap, t.shift);
    }
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {  // the 4 random entry loads are issued back to back
      first[k] = make_ulonglong2(EMPTY_KEY, 0);
      if (valid[k] && key[k] != EMPTY_KEY) first[k] = ld_entry(t.words, ebase[k] + loc[k], t.shift);
    }
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
      uint2 m = make_uint2(OFF_MISS, 0);
      if (valid[k]) {
        if (key[k] == EMPTY_KEY) { if (t.sent_cnt) m = make_uint2(t.sent_off, t.sent_cnt); }
        else m = resolve<false>(t, t.words + (ebase[k] << t.shift), ebase[k], key[k], loc[k], first[k]);
      }
      const int64_t r = tile_base + k * PROBE_THREADS + tid;
      const uint32_t c = m.y ? m.y : ((p.is_outer && r < p.n) ? 1u : 0u);  // onMissMatch
      sm.off[k * PROBE_THREADS + tid] = m.y ? m.x : OFF_MISS;
      sm.prefix[k * PROBE_THREADS + tid] = c;
    }
    __syncthreads();
    bool any_multi;
    const unsigned long long M = tile_scan(sm, matched_acc, any_multi);
    if (tid == 0) {
      // ---- phase C: output offset = sum of the totals of all earlier tiles (decoupled look-back), which
      // makes the result order (probe row asc, build insertion asc) — the reference's order inside a chunk
      constexpr unsigned long long FLAG_AGG = 1ull << 62, FLAG_INC = 2ull << 62, VAL = (1ull << 62) - 1;
      volatile unsigned long long *st = p.tile_state;
      unsigned long long excl = 0;
      if (tile > 0) {
        st[tile] = FLAG_AGG | M;
        for (int64_t prev = tile - 1;; prev--) {
          unsigned long long v;
          do { v = st[prev]; } while ((v >> 62) == 0);
          excl += v & VAL;
          if ((v >> 62) == 2) break;
        }
      }
      st[tile] = FLAG_INC | (excl + M);
      if (M) atomicAdd(p.cursor, M);
      sm.base = excl;
    }
    __syncthreads();
    const unsigned long long base = sm.base;
    if (M && base + M <= p.capacity) {  // else: the host re-runs the batch with the exact size
      if (any_multi) tile_expand(p, sm, tile_base, base, M);
      else tile_emit_rowwise(p, sm, tile_base, base, key);
    }
    __syncthreads();  // smem is reused by the next tile
  }
  if ((tid & 31) == 0 && matched_acc) atomicAdd(p.cursor + 1, (unsigned long long)matched_acc);
}

__global__ void k_init_slabs(uint32_t *lo, uint32_t *cursor, uint32_t *lim, int n_parts, uint32_t slab, uint32_t tail_rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_parts) return;
  const uint32_t start = (uint32_t)i * slab;  // bin n_parts (rows that cannot match, outer joins) takes the tail
  lo[i] = start;
  cursor[i] = start;
  lim[i] = (i < n_parts) ? start + slab : start + tail_rows;
}
// Rows per partition slab of the optimistic (histogram-free) scatter of n rows into P partitions: hash partitions of a batch
// are near-uniform, so the mean plus 25% and 4096 rows.  AoS slabs are rounded up to 32 rows so that every slab starts
// 16-byte aligned whatever the row width, as the bulk copies of the positional probe require.
static uint64_t slab_rows(int64_t n, int P, bool aos) {
  const uint64_t slab = (uint64_t)n / P + (uint64_t)n / P / 4 + 4096;
  return aos ? (slab + 31) & ~31ull : slab;
}

// ---- probe-side radix scatter -------------------------------------------------------------------------
static constexpr int SCAT_THREADS = 256;
static constexpr int SCAT_ROWS_PER_THREAD = 16;
static constexpr int SCAT_TILE = SCAT_THREADS * SCAT_ROWS_PER_THREAD;
static constexpr uint32_t PID_DROP = 0xFFFFFFFFu;

struct ScatterParams {
  int n_cols;
  DCol in[MAXC];
  DColMut out[MAXC];
  const uint8_t *selected;
  int key_col, key_mode, is_outer, pbits;
  int64_t n;
  uint32_t *part_cnt;     // histogram (2^pbits + 1 bins; the last bin = rows that cannot match)
  uint32_t *part_cursor;  // scatter cursors, initialised to the first row of each partition
  const uint32_t *part_lim;  // optimistic slabs: one past the last row a partition may hold (nullptr: exact offsets, cannot overflow)
  unsigned long long *overflow;  // set when a slab was too small
  // multi-GPU push scatter: partition = (hash >> 40) % n_parts_mod and partition q's rows go to out_bin[q][c] — the
  // receive buffer of rank q, a PEER pointer mapped through CUDA IPC: the stores travel over NVLink.  With is_outer the rows
  // that cannot match go to out_bin[n_parts_mod][c], local columns of this rank.
  int n_parts_mod;
  uint64_t *out_bin[9][4];
};
__host__ __device__ __forceinline__ int scatter_bins(const ScatterParams &p) { return (p.n_parts_mod ? p.n_parts_mod : (1 << p.pbits)) + 1; }
__device__ __forceinline__ uint32_t scatter_pid(const ScatterParams &p, uint64_t key) {
  // multi-GPU destination rank: (mix64 >> 40) % world (dist.py mirrors it in numpy); table partition: top bits of the table hash
  return p.n_parts_mod ? (uint32_t)((tqd::mix64(key) >> 40) % (uint64_t)p.n_parts_mod) : (uint32_t)part_of_hash(tqd::hash_key(key), p.pbits);
}

__device__ __forceinline__ uint32_t probe_pid(const ScatterParams &p, int64_t r, uint64_t key) {
  const bool sel = p.selected ? (p.selected[r] != 0) : true;
  if (sel && key_valid(key, tqd::bm_not_null(p.in[p.key_col].bm, r), p.key_mode)) return scatter_pid(p, key);
  return p.is_outer ? (uint32_t)(scatter_bins(p) - 1) : PID_DROP;  // inner join: a row that cannot match produces nothing (joiner.go:405)
}

__global__ void __launch_bounds__(SCAT_THREADS) k_probe_part_hist(const ScatterParams p) {
  extern __shared__ uint32_t s_hist[];
  const int n_bins = scatter_bins(p);
  for (int i = threadIdx.x; i < n_bins; i += SCAT_THREADS) s_hist[i] = 0;
  __syncthreads();
  const uint64_t *keys = p.in[p.key_col].data;
  int64_t i = (int64_t)blockIdx.x * SCAT_THREADS + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * SCAT_THREADS;
  for (; i < p.n; i += stride) {
    const uint32_t pid = probe_pid(p, i, tqd::ld_stream_u64(keys + i));
    if (pid != PID_DROP) atomicAdd(&s_hist[pid], 1u);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < n_bins; b += SCAT_THREADS)
    if (s_hist[b]) atomicAdd(&p.part_cnt[b], s_hist[b]);
}

// Exclusive scan of one value per thread over a CTA of THREADS threads (s_warp: THREADS / 32 + 1 words): returns the
// thread's prefix, and s_warp[THREADS / 32] holds the CTA's sum.  Two barriers; a caller that writes s_warp again needs one
// more between.
template <int THREADS>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *s_warp) {
  static_assert(THREADS % 32 == 0 && THREADS <= 1024, "whole warps, at most 32 of them");
  constexpr int NW = THREADS / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += x; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = lane < NW ? s_warp[lane] : 0u;
    uint32_t winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, winc, d); if (lane >= d) winc += x; }
    if (lane < NW) s_warp[lane] = winc - w;
    if (lane == NW - 1) s_warp[NW] = winc;
  }
  __syncthreads();
  return inc - v + s_warp[warp];
}

// Shared-memory image of k_probe_scatter and k_probe_scatter_fast (the fast kernel leaves `nn` unused).
struct ScatterSmem {
  uint64_t *stage;  // [SCAT_TILE] one column of the tile, sorted
  uint32_t *bins;   // [n_bins] tile counts, then local exclusive offsets
  uint32_t *gdelta; // [n_bins] (claimed global run start) - (local offset)
  uint32_t *imax;   // [n_bins] first sorted position of the tile that no longer fits the slab
  uint16_t *spid;   // [SCAT_TILE] sorted position -> partition
  uint8_t *nn;      // [SCAT_TILE] sorted position -> NOT NULL flag
};
__host__ __device__ constexpr int scatter_smem_bytes(int n_bins) { return SCAT_TILE * (8 + 2 + 1) + n_bins * 4 * 3; }  // stage, spid, nn; 3 bin tables
__device__ __forceinline__ ScatterSmem scatter_smem(unsigned char *raw, int n_bins) {
  ScatterSmem m;
  m.stage = reinterpret_cast<uint64_t *>(raw);
  m.bins = reinterpret_cast<uint32_t *>(raw + SCAT_TILE * 8);
  m.gdelta = m.bins + n_bins;
  m.imax = m.gdelta + n_bins;
  m.spid = reinterpret_cast<uint16_t *>(m.imax + n_bins);
  m.nn = reinterpret_cast<uint8_t *>(m.spid + SCAT_TILE);
  return m;
}

// From the partition pid[k] and the rank spos[k] of each of a thread's ROWS rows (sm.bins holds the tile's counts): scans the
// bins, lets every non-empty bin claim its run with ONE global atomicAdd on part_cursor (clipped at part_lim, which raises the
// overflow flag), turns each rank into the row's sorted position in the tile and records its partition in sm.spid.  Returns
// the rows of the tile that go somewhere.
template <int THREADS, int ROWS>
__device__ __forceinline__ uint32_t scatter_claim(const ScatterParams &p, const ScatterSmem &sm, int n_bins, const uint32_t (&pid)[ROWS],
                                                  uint32_t (&spos)[ROWS], uint32_t *s_warp) {
  const int tid = threadIdx.x;
  const int bpt = (n_bins + THREADS - 1) / THREADS;  // thread t owns bins [t*bpt, (t+1)*bpt)
  __syncthreads();
  uint32_t tsum = 0;
  for (int q = 0; q < bpt; q++) { const int b = tid * bpt + q; if (b < n_bins) tsum += sm.bins[b]; }
  uint32_t run = block_excl_scan<THREADS>(tsum, s_warp);
  for (int q = 0; q < bpt; q++) {
    const int b = tid * bpt + q;
    if (b < n_bins) {
      const uint32_t c = sm.bins[b];
      sm.bins[b] = run;
      if (c) {
        const uint32_t g = atomicAdd(&p.part_cursor[b], c);
        sm.gdelta[b] = g - run;
        uint32_t imax = 0xFFFFFFFFu;
        if (p.part_lim) {
          const uint32_t lim = p.part_lim[b];
          if (g + c > lim) { imax = (g < lim) ? run + (lim - g) : run; atomicOr(p.overflow, 1ull); }
        }
        sm.imax[b] = imax;
      }
      run += c;
    }
  }
  const uint32_t total = s_warp[THREADS / 32];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < ROWS; k++) {
    if (pid[k] == PID_DROP) continue;
    spos[k] += sm.bins[pid[k]];
    sm.spid[spos[k]] = (uint16_t)pid[k];
  }
  return total;
}

// One tile = SCAT_TILE (4096) rows.  The tile is counting-sorted by partition in shared memory (histogram -> local
// exclusive scan -> sorted position per row), each non-empty partition claims its run with ONE global
// atomicAdd, and every column then goes global -> shared (coalesced, at the row's sorted position) ->
// global (coalesced, consecutive lanes store consecutive destinations: whole 32-byte sectors).
__global__ void __launch_bounds__(SCAT_THREADS, 4) k_probe_scatter(const ScatterParams p) {
  extern __shared__ __align__(16) unsigned char s_scat[];
  const int n_bins = scatter_bins(p);
  const ScatterSmem sm = scatter_smem(s_scat, n_bins);
  __shared__ uint32_t s_warp[SCAT_THREADS / 32 + 1];
  const int tid = threadIdx.x;
  const uint64_t *keys = p.in[p.key_col].data;
  const int64_t n_tiles = (p.n + SCAT_TILE - 1) / SCAT_TILE;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t tile_base = tile * SCAT_TILE;
    for (int b = tid; b < n_bins; b += SCAT_THREADS) sm.bins[b] = 0;
    __syncthreads();
    uint32_t pid[SCAT_ROWS_PER_THREAD], spos[SCAT_ROWS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < SCAT_ROWS_PER_THREAD; k++) {
      const int64_t r = tile_base + k * SCAT_THREADS + tid;
      pid[k] = PID_DROP;
      if (r < p.n) pid[k] = probe_pid(p, r, keys[r]);
      spos[k] = (pid[k] != PID_DROP) ? atomicAdd(&sm.bins[pid[k]], 1u) : 0u;  // rank inside the partition
    }
    const uint32_t total = scatter_claim<SCAT_THREADS>(p, sm, n_bins, pid, spos, s_warp);
    for (int c = 0; c < p.n_cols; c++) {
      const bool has_bm = p.out[c].bm != nullptr;
#pragma unroll
      for (int k = 0; k < SCAT_ROWS_PER_THREAD; k++) {
        if (pid[k] == PID_DROP) continue;
        const int64_t r = tile_base + k * SCAT_THREADS + tid;
        sm.stage[spos[k]] = p.in[c].data[r];
        if (has_bm) sm.nn[spos[k]] = (uint8_t)tqd::bm_not_null(p.in[c].bm, r);
      }
      __syncthreads();
      for (uint32_t i = tid; i < total; i += SCAT_THREADS) {
        const uint32_t bin = sm.spid[i];
        if (i >= sm.imax[bin]) continue;  // slab full (optimistic path only)
        const uint32_t dst = sm.gdelta[bin] + i;
        tqd::st_stream_u64(p.out[c].data + dst, sm.stage[i]);
        if (has_bm && sm.nn[i]) atomicOr(&p.out[c].bm[dst >> 5], 1u << (dst & 31));
      }
      __syncthreads();
    }
  }
}

// Scatter fast path: no input column carries a NULL bitmap and the column count is a template parameter.  All
// columns of the tile are requested up front (8 rows x NP columns in flight per thread), then each column goes
// registers -> shared (sorted position) -> global (coalesced).  512 threads x 8 rows = the same 4096-row tile.
static constexpr int SCATF_THREADS = 512;
static constexpr int SCATF_ROWS = SCAT_TILE / SCATF_THREADS;
template <int NP>
__global__ void __launch_bounds__(SCATF_THREADS, (NP <= 2 ? 2 : 1)) k_probe_scatter_fast(const ScatterParams p) {
  extern __shared__ __align__(16) unsigned char s_scat[];
  const int n_bins = scatter_bins(p);
  const ScatterSmem sm = scatter_smem(s_scat, n_bins);
  __shared__ uint32_t s_warp[SCATF_THREADS / 32 + 1];
  const int tid = threadIdx.x;
  const uint64_t *in[NP];
  uint64_t *out[NP];
#pragma unroll
  for (int c = 0; c < NP; c++) { in[c] = p.in[c].data; out[c] = p.out[c].data; }
  const int kc = p.key_col;
  const int64_t n_tiles = (p.n + SCAT_TILE - 1) / SCAT_TILE;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t tile_base = tile * SCAT_TILE;
    for (int b = tid; b < n_bins; b += SCATF_THREADS) sm.bins[b] = 0;
    uint64_t v[NP][SCATF_ROWS];
#pragma unroll
    for (int k = 0; k < SCATF_ROWS; k++) {
      const int64_t r = tile_base + k * SCATF_THREADS + tid;
#pragma unroll
      for (int c = 0; c < NP; c++) v[c][k] = (r < p.n) ? tqd::ld_stream_u64(in[c] + r) : 0;
    }
    __syncthreads();
    uint32_t pid[SCATF_ROWS], spos[SCATF_ROWS];
#pragma unroll
    for (int k = 0; k < SCATF_ROWS; k++) {
      const int64_t r = tile_base + k * SCATF_THREADS + tid;
      uint64_t key = v[0][k];
#pragma unroll
      for (int c = 1; c < NP; c++) if (c == kc) key = v[c][k];
      pid[k] = PID_DROP;
      if (r < p.n) {
        const bool sel = p.selected ? (p.selected[r] != 0) : true;
        if (sel && key_valid(key, true, p.key_mode)) pid[k] = scatter_pid(p, key);
        else if (p.is_outer) pid[k] = (uint32_t)(n_bins - 1);
      }
      spos[k] = (pid[k] != PID_DROP) ? atomicAdd(&sm.bins[pid[k]], 1u) : 0u;
    }
    const uint32_t total = scatter_claim<SCATF_THREADS>(p, sm, n_bins, pid, spos, s_warp);
#pragma unroll
    for (int c = 0; c < NP; c++) {
#pragma unroll
      for (int k = 0; k < SCATF_ROWS; k++)
        if (pid[k] != PID_DROP) sm.stage[spos[k]] = v[c][k];
      __syncthreads();
      for (uint32_t i = tid; i < total; i += SCATF_THREADS) {
        const uint32_t bin = sm.spid[i];
        if (i >= sm.imax[bin]) continue;
        uint64_t *dst = p.n_parts_mod ? p.out_bin[bin][c] : out[c];
        const uint32_t d32 = sm.gdelta[bin] + i;  // 32-bit wrap-around arithmetic: (run start - local offset) + sorted position
        tqd::st_stream_u64(dst + d32, sm.stage[i]);
      }
      __syncthreads();
    }
  }
}

// Launches k_probe_scatter_fast for sp.n_cols (1..4) NULL-free columns on stream s; `what` names the launch in errors.
static int32_t launch_scatter_fast(const ScatterParams &sp, cudaStream_t s, const char *what) {
  typedef void (*ScatterKernel)(const ScatterParams);
  static const ScatterKernel kernels[5] = {nullptr, k_probe_scatter_fast<1>, k_probe_scatter_fast<2>, k_probe_scatter_fast<3>, k_probe_scatter_fast<4>};
  static bool attr_set[5] = {};
  const int np = sp.n_cols;
  if (np < 1 || np > 4) { set_error("internal: %s of %d columns", what, np); return TQ_ERR_INVALID_ARG; }
  if (!attr_set[np]) {
    TQ_CUDA(cudaFuncSetAttribute(kernels[np], cudaFuncAttributeMaxDynamicSharedMemorySize, scatter_smem_bytes((1 << PART_MAX_BITS) + 1)));
    attr_set[np] = true;
  }
  const int64_t tiles = (sp.n + SCAT_TILE - 1) / SCAT_TILE;
  const int64_t cap = (int64_t)rt().sm_count * (np <= 2 ? 2 : 1);
  kernels[np]<<<(int)(tiles < cap ? tiles : cap), SCATF_THREADS, scatter_smem_bytes(scatter_bins(sp)), s>>>(sp);
  count_launch();
  return check_launch(what);
}

// scatter.cuh: the same scatter for other operators (HashAgg pre-aggregation)
int32_t scatter_rows_by_hash(const DCol *cols, int n_cols, int key_col, int64_t n, int pbits, std::vector<DevBuf> &out, DevBuf &lo, DevBuf &hi, DevBuf &lim,
                             unsigned long long *d_overflow, cudaStream_t s) {
  if (n_cols < 1 || n_cols > 4 || pbits < 1 || pbits > PART_MAX_BITS || n <= 0 || n > 0xFFFFFFF0ll) { set_error("internal: scatter_rows_by_hash arguments"); return TQ_ERR_INVALID_ARG; }
  const int P = 1 << pbits, n_bins = P + 1;
  const uint64_t slab = slab_rows(n, P, false);
  if (slab * P > 0xFFFFFFF0ull) { set_error("batch too large for 32-bit partition offsets"); return TQ_ERR_INVALID_ARG; }
  out.resize(n_cols);
  ScatterParams sp{};
  sp.n_cols = n_cols;
  for (int c = 0; c < n_cols; c++) {
    TQ_TRY(out[c].reserve((size_t)slab * P * 8));
    sp.in[c] = cols[c];
    sp.out[c].data = out[c].as<uint64_t>();
    sp.out[c].bm = nullptr;
  }
  TQ_TRY(lo.reserve((size_t)(n_bins + 1) * 4));
  TQ_TRY(hi.reserve((size_t)(n_bins + 1) * 4));
  TQ_TRY(lim.reserve((size_t)(n_bins + 1) * 4));
  k_init_slabs<<<(n_bins + 255) / 256, 256, 0, s>>>(lo.as<uint32_t>(), hi.as<uint32_t>(), lim.as<uint32_t>(), P, (uint32_t)slab, 0u);
  count_launch();
  sp.selected = nullptr;
  sp.key_col = key_col;
  sp.key_mode = KEYMODE_RAW;
  sp.is_outer = 0;
  sp.pbits = pbits;
  sp.n = n;
  sp.part_cnt = nullptr;
  sp.part_cursor = hi.as<uint32_t>();
  sp.part_lim = lim.as<uint32_t>();
  sp.overflow = d_overflow;
  return launch_scatter_fast(sp, s, "k_probe_scatter_fast");
}

// ---- partitioned probe: the partition's table image lives in shared memory ------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
               "r"(bytes), "r"(smem_u32(mbar))
               : "memory");
}
__device__ __forceinline__ void mbar_init(uint64_t *mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(mbar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *mbar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(mbar)),
      "r"(parity)
      : "memory");
}

// Common prologue of the partitioned probe kernels: which rows does this CTA own, where is its table.
struct PartCtx {
  uint32_t part;
  int64_t p_lo, p_hi, t_lo, t_hi;
  bool has_table, use_smem;
  const uint64_t *tbl;  // partition table (global memory, or the shared-memory image once loaded)
  uint64_t ebase;       // first entry index of the partition
};
__device__ __forceinline__ bool part_prologue(const ProbeParams &p, const JoinTable &t, unsigned char *s_dyn, uint64_t *s_mbar, PartCtx &c) {
  const uint32_t n_parts = 1u << t.pbits;
  c.part = blockIdx.x / p.split;
  const uint32_t sub = blockIdx.x % p.split;
  c.p_lo = p.part_lo[c.part];
  c.p_hi = p.part_hi[c.part];
  if (p.part_lim && c.p_hi > (int64_t)p.part_lim[c.part]) c.p_hi = p.part_lim[c.part];  // overflowed slab: the batch is re-run anyway
  const int64_t p_tiles = (c.p_hi - c.p_lo + PROBE_TILE - 1) / PROBE_TILE;
  c.t_lo = p_tiles * sub / p.split;
  c.t_hi = p_tiles * (sub + 1) / p.split;
  if (c.t_lo >= c.t_hi) return false;
  c.has_table = c.part < n_parts;  // partition n_parts: rows that cannot match (outer joins only)
  const uint64_t cap = t.cap;
  c.ebase = (uint64_t)(c.has_table ? c.part : 0) * cap;
  c.tbl = t.words + (c.ebase << t.shift);
  // Small partition tables are copied into shared memory by TMA; larger ones are probed in place — consecutive
  // CTAs work on the same partition, so only a few partition tables are live at a time and they stay in L2.
  c.use_smem = c.has_table && p.table_in_smem;
  if (c.use_smem) {
    if (threadIdx.x == 0) {
      mbar_init(s_mbar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const uint32_t bytes = (uint32_t)((cap << t.shift) * 8);
      mbar_expect_tx(s_mbar, bytes);
      const unsigned char *src = reinterpret_cast<const unsigned char *>(c.tbl);
      for (uint32_t o = 0; o < bytes; o += 16384) tma_load_1d(s_dyn + o, src + o, min(16384u, bytes - o), s_mbar);
    }
    c.tbl = reinterpret_cast<const uint64_t *>(s_dyn);
  }
  return true;
}

// ---- partitioned probe, UNIQUE build keys (PK-FK joins): every probe row yields 0 or 1 rows ---------------
// Lean variant: warp w of the CTA owns rows [w*128, w*128+128) of the tile; matches are compacted with
// ballots, a shared-memory atomic orders the 8 warps inside the tile and one global atomic claims the tile's
// output range — two barriers per tile, no prefix arrays, no search.
__global__ void __launch_bounds__(PROBE_THREADS) k_probe_part_uniq(const ProbeParams p, const JoinTable t) {
  extern __shared__ __align__(128) unsigned char s_dyn[];
  __shared__ __align__(8) uint64_t s_mbar;
  __shared__ unsigned s_total[2];
  __shared__ unsigned long long s_base[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  PartCtx cx;
  if (!part_prologue(p, t, s_dyn, &s_mbar, cx)) return;
  if (tid == 0) { s_total[0] = 0; s_total[1] = 0; }
  __syncthreads();
  const uint64_t *keys = p.probe[p.key_col].data;
  const unsigned lt_mask = (1u << lane) - 1;
  unsigned matched_acc = 0;
  bool table_ready = !cx.use_smem;
  constexpr int R = PROBE_ROWS_PER_THREAD;
  for (int64_t tile = cx.t_lo; tile < cx.t_hi; tile++) {
    const int par = (int)(tile & 1);
    const int64_t wbase = cx.p_lo + tile * PROBE_TILE + warp * (32 * R);  // this warp's 128 rows
    uint64_t key[R];
    bool inb[R];
#pragma unroll
    for (int k = 0; k < R; k++) {
      const int64_t r = wbase + k * 32 + lane;
      inb[k] = r < cx.p_hi;
      key[k] = inb[k] ? tqd::ld_stream_u64(keys + r) : 0;
    }
    if (!table_ready) { mbar_wait(&s_mbar, 0); table_ready = true; }  // the key loads above overlap the table copy
    uint32_t loc[R];
    ulonglong2 first[R];
#pragma unroll
    for (int k = 0; k < R; k++) {  // independent entry loads issued back to back
      loc[k] = home_slot(tqd::hash_key(key[k]), t.cap, t.shift);
      first[k] = make_ulonglong2(EMPTY_KEY, 0);
      if (inb[k] && cx.has_table && key[k] != EMPTY_KEY) first[k] = ld_entry(cx.tbl, loc[k], t.shift);
    }
    uint32_t off[R];
    unsigned bal[R];
    unsigned wcnt = 0;
#pragma unroll
    for (int k = 0; k < R; k++) {
      off[k] = OFF_MISS;
      if (inb[k] && cx.has_table) {  // every row of a regular partition has a valid key (the scatter filtered the rest)
        if (key[k] == EMPTY_KEY) { if (t.sent_cnt) off[k] = t.sent_off; }
        else off[k] = resolve<true>(t, cx.tbl, cx.ebase, key[k], loc[k], first[k]).x;  // first[k] now holds the matched entry
      }
      const bool emit = inb[k] && (off[k] != OFF_MISS || p.is_outer);
      bal[k] = __ballot_sync(0xffffffffu, emit);
      wcnt += __popc(bal[k]);
      const unsigned mb = __ballot_sync(0xffffffffu, off[k] != OFF_MISS);
      if (lane == 0) matched_acc += __popc(mb);
    }
    unsigned woff = 0;
    if (lane == 0 && wcnt) woff = atomicAdd(&s_total[par], wcnt);
    __syncthreads();
    if (tid == 0) {
      const unsigned tot = s_total[par];
      s_base[par] = tot ? atomicAdd(p.cursor, (unsigned long long)tot) : 0ull;
      s_total[par] = 0;  // next use of this parity is two tiles away, behind two more barriers
    }
    __syncthreads();
    unsigned long long q0 = s_base[par] + __shfl_sync(0xffffffffu, woff, 0);
#pragma unroll
    for (int k = 0; k < R; k++) {
      const unsigned long long q = q0 + __popc(bal[k] & lt_mask);
      q0 += __popc(bal[k]);
      const bool emit = ((bal[k] >> lane) & 1u) && q < p.capacity;  // capacity == probe rows: always fits for unique keys
      // ROW mode: words 0/1 of the build row are already in registers (the matched entry)
      emit_row(p, emit, wbase + k * 32 + lane, key[k], off[k], q, t.row_mode && key[k] != EMPTY_KEY, first[k].x, first[k].y);
    }
  }
  if (lane == 0 && matched_acc) atomicAdd(p.cursor + 1, (unsigned long long)matched_acc);
}

// ---- the PK-FK fast path: inner join, ROW-mode table, no output column can hold NULLs ------------------------
// Same structure as k_probe_part_uniq with the column counts as template parameters: column pointers live in
// registers, the loops unroll, words 0/1 of the build row come straight from the matched entry.  16-byte
// entries are fetched as 32-byte aligned PAIRS (the insert starts probing on an even entry), so one sector
// read checks two candidate slots and dependent collision round-trips are rare.
struct EntryPair {
  ulonglong2 a, b;
};
__device__ __forceinline__ EntryPair ld_pair(const uint64_t *tbl, uint32_t loc_even, bool smem) {
  EntryPair e;
  const uint64_t *p = tbl + ((uint64_t)loc_even << 1);
  if (smem) {
    e.a = *reinterpret_cast<const ulonglong2 *>(p);
    e.b = *reinterpret_cast<const ulonglong2 *>(p + 2);
  } else {  // two 128-bit loads of the same 32-byte sector (sm_90 has no 256-bit global load)
    asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(e.a.x), "=l"(e.a.y) : "l"(p));
    asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(e.b.x), "=l"(e.b.y) : "l"(p + 2));
  }
  return e;
}

template <int NP, int NB>
__global__ void __launch_bounds__(PROBE_THREADS, 4) k_probe_part_fast(const ProbeParams p, const JoinTable t) {
  extern __shared__ __align__(128) unsigned char s_dyn[];
  __shared__ __align__(8) uint64_t s_mbar;
  __shared__ unsigned s_total[2];
  __shared__ unsigned long long s_base[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  PartCtx cx;
  if (!part_prologue(p, t, s_dyn, &s_mbar, cx)) return;
  if (tid == 0) { s_total[0] = 0; s_total[1] = 0; }
  __syncthreads();
  const uint64_t *pin[NP];
  uint64_t *pout[NP];
  uint64_t *bout[NB];
  int bw[NB];
#pragma unroll
  for (int c = 0; c < NP; c++) { pin[c] = p.probe[c].data; pout[c] = p.out_probe[c].data; }
#pragma unroll
  for (int c = 0; c < NB; c++) { bout[c] = p.out_build[c].data; bw[c] = p.build_word[c]; }
  const int kc = p.key_col;
  const uint64_t *keys = pin[0];
#pragma unroll
  for (int c = 1; c < NP; c++) if (c == kc) keys = pin[c];
  const unsigned lt_mask = (1u << lane) - 1;
  const uint32_t cap = t.cap;
  const int shift = t.shift;
  const bool smem = cx.use_smem;
  unsigned matched_acc = 0;
  bool table_ready = !cx.use_smem;
  constexpr int R = PROBE_ROWS_PER_THREAD;
  // software pipeline: the keys of tile i+1 are requested before the barriers / atomics of tile i
  uint64_t nkey[R];
  {
    const int64_t wb = cx.p_lo + cx.t_lo * PROBE_TILE + warp * (32 * R) + lane;
#pragma unroll
    for (int k = 0; k < R; k++) nkey[k] = (wb + k * 32 < cx.p_hi) ? tqd::ld_stream_u64(keys + wb + k * 32) : EMPTY_KEY;
  }
  for (int64_t tile = cx.t_lo; tile < cx.t_hi; tile++) {
    const int par = (int)(tile & 1);
    const int64_t wbase = cx.p_lo + tile * PROBE_TILE + warp * (32 * R) + lane;  // this lane's first row
    uint64_t key[R];
#pragma unroll
    for (int k = 0; k < R; k++) key[k] = nkey[k];
    if (!table_ready) { mbar_wait(&s_mbar, 0); table_ready = true; }
    uint32_t loc[R];
    ulonglong2 ent[R];
    unsigned bal[R];
    unsigned wcnt = 0;
    uint64_t pay[NP][R];
    if (shift == 1) {
      EntryPair pr[R];
#pragma unroll
      for (int k = 0; k < R; k++) {  // R independent sector loads in flight
        loc[k] = home_slot(tqd::hash_key(key[k]), cap, 1);
        pr[k].a = make_ulonglong2(EMPTY_KEY, 0);
        pr[k].b = pr[k].a;
        if (key[k] != EMPTY_KEY) pr[k] = ld_pair(cx.tbl, loc[k], smem);
      }
      if (tile + 1 < cx.t_hi) {
        const int64_t wb = wbase + PROBE_TILE;
#pragma unroll
        for (int k = 0; k < R; k++) nkey[k] = (wb + k * 32 < cx.p_hi) ? tqd::ld_stream_u64(keys + wb + k * 32) : EMPTY_KEY;
      }
#pragma unroll
      for (int k = 0; k < R; k++) {
        bool hit = false;
        ent[k] = pr[k].a;
        if (key[k] != EMPTY_KEY) {
          for (;;) {
            if (pr[k].a.x == key[k]) { ent[k] = pr[k].a; hit = true; break; }
            if (pr[k].a.x == EMPTY_KEY) break;
            if (pr[k].b.x == key[k]) { ent[k] = pr[k].b; loc[k] += 1; hit = true; break; }
            if (pr[k].b.x == EMPTY_KEY) break;
            loc[k] = next_slot(loc[k], 2, cap);
            pr[k] = ld_pair(cx.tbl, loc[k], smem);
          }
        } else if ((wbase + k * 32) < cx.p_hi && t.sent_cnt) {  // a probe key equal to the empty marker: its row is the side entry
          loc[k] = (uint32_t)(t.sent_off - cx.ebase);
          ent[k] = ld_entry(t.words, t.sent_off, 1);
          hit = true;
        }
        bal[k] = __ballot_sync(0xffffffffu, hit);
        wcnt += __popc(bal[k]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < R; k++) {
        loc[k] = home_slot(tqd::hash_key(key[k]), cap, shift);
        ent[k] = make_ulonglong2(EMPTY_KEY, 0);
        if (key[k] != EMPTY_KEY) ent[k] = ld_entry(cx.tbl, loc[k], shift);
      }
      if (tile + 1 < cx.t_hi) {
        const int64_t wb = wbase + PROBE_TILE;
#pragma unroll
        for (int k = 0; k < R; k++) nkey[k] = (wb + k * 32 < cx.p_hi) ? tqd::ld_stream_u64(keys + wb + k * 32) : EMPTY_KEY;
      }
#pragma unroll
      for (int k = 0; k < R; k++) {
        bool hit = false;
        if (key[k] != EMPTY_KEY) {
          while (ent[k].x != key[k] && ent[k].x != EMPTY_KEY) {
            loc[k] = next_slot(loc[k], 1, cap);
            ent[k] = ld_entry(cx.tbl, loc[k], shift);
          }
          hit = ent[k].x == key[k];
        } else if ((wbase + k * 32) < cx.p_hi && t.sent_cnt) {
          loc[k] = (uint32_t)(t.sent_off - cx.ebase);
          ent[k] = ld_entry(t.words, t.sent_off, shift);
          hit = true;
        }
        bal[k] = __ballot_sync(0xffffffffu, hit);
        wcnt += __popc(bal[k]);
      }
    }
    unsigned woff = 0;
    if (lane == 0) {
      matched_acc += wcnt;
      if (wcnt) woff = atomicAdd(&s_total[par], wcnt);
    }
    // the other probe columns of the matched rows are requested NOW: their latency hides behind the two barriers and
    // the global atomic below (only word 1 of the matched entry stays live: word 0 is the key itself)
#pragma unroll
    for (int k = 0; k < R; k++) {
      const bool hit = (bal[k] >> lane) & 1u;
#pragma unroll
      for (int c = 0; c < NP; c++) {
        pay[c][k] = 0;
        if (c != kc && hit) pay[c][k] = tqd::ld_stream_u64(pin[c] + wbase + k * 32);
      }
    }
    __syncthreads();
    if (tid == 0) {
      const unsigned tot = s_total[par];
      s_base[par] = tot ? atomicAdd(p.cursor, (unsigned long long)tot) : 0ull;
      s_total[par] = 0;
    }
    __syncthreads();
    unsigned long long q0 = s_base[par] + __shfl_sync(0xffffffffu, woff, 0);
#pragma unroll
    for (int k = 0; k < R; k++) {
      const unsigned long long q = q0 + __popc(bal[k] & lt_mask);
      q0 += __popc(bal[k]);
      if (((bal[k] >> lane) & 1u) && q < p.capacity) {
#pragma unroll
        for (int c = 0; c < NP; c++) tqd::st_stream_u64(pout[c] + q, (c == kc) ? key[k] : pay[c][k]);
#pragma unroll
        for (int c = 0; c < NB; c++) {
          uint64_t v;
          if (bw[c] == 0) v = ent[k].x;
          else if (bw[c] == 1) v = ent[k].y;
          else v = t.words[((cx.ebase + loc[k]) << shift) + bw[c]];  // words 2..3 of a 32-byte entry: same sector, L1/L2 hit
          tqd::st_stream_u64(bout[c] + q, v);
        }
      }
    }
  }
  if (lane == 0 && matched_acc) atomicAdd(p.cursor + 1, (unsigned long long)matched_acc);
}

typedef void (*ProbeKernel)(const ProbeParams, const JoinTable);
template <int NP>
static ProbeKernel fast_kernel_nb(int nb) {
  switch (nb) {
    case 1: return k_probe_part_fast<NP, 1>;
    case 2: return k_probe_part_fast<NP, 2>;
    case 3: return k_probe_part_fast<NP, 3>;
    case 4: return k_probe_part_fast<NP, 4>;
  }
  return nullptr;
}
static ProbeKernel fast_kernel(int np, int nb) {
  switch (np) {
    case 1: return fast_kernel_nb<1>(nb);
    case 2: return fast_kernel_nb<2>(nb);
    case 3: return fast_kernel_nb<3>(nb);
    case 4: return fast_kernel_nb<4>(nb);
  }
  return nullptr;
}

// ---- partitioned probe, general (duplicate build keys): block scan + output-centric expansion ------------
__global__ void __launch_bounds__(PROBE_THREADS) k_probe_part(const ProbeParams p, const JoinTable t) {
  extern __shared__ __align__(128) unsigned char s_dyn[];
  __shared__ TileSmem sm;
  __shared__ __align__(8) uint64_t s_mbar;

  const int tid = threadIdx.x;
  PartCtx cx;
  if (!part_prologue(p, t, s_dyn, &s_mbar, cx)) return;
  const uint64_t *keys = p.probe[p.key_col].data;
  unsigned matched_acc = 0;
  bool table_ready = !cx.use_smem;
  for (int64_t tile = cx.t_lo; tile < cx.t_hi; tile++) {
    const int64_t tile_base = cx.p_lo + tile * PROBE_TILE;
    uint64_t key[PROBE_ROWS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
      const int64_t r = tile_base + k * PROBE_THREADS + tid;
      key[k] = (r < cx.p_hi) ? tqd::ld_stream_u64(keys + r) : 0;
    }
    if (!table_ready) { mbar_wait(&s_mbar, 0); table_ready = true; }
    uint32_t loc[PROBE_ROWS_PER_THREAD];
    ulonglong2 first[PROBE_ROWS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
      const int64_t r = tile_base + k * PROBE_THREADS + tid;
      loc[k] = home_slot(tqd::hash_key(key[k]), t.cap, t.shift);
      first[k] = make_ulonglong2(EMPTY_KEY, 0);
      if (r < cx.p_hi && cx.has_table && key[k] != EMPTY_KEY) first[k] = ld_entry(cx.tbl, loc[k], t.shift);
    }
#pragma unroll
    for (int k = 0; k < PROBE_ROWS_PER_THREAD; k++) {
      const int64_t r = tile_base + k * PROBE_THREADS + tid;
      uint2 m = make_uint2(OFF_MISS, 0);
      if (r < cx.p_hi && cx.has_table) {
        if (key[k] == EMPTY_KEY) { if (t.sent_cnt) m = make_uint2(t.sent_off, t.sent_cnt); }
        else m = resolve<true>(t, cx.tbl, cx.ebase, key[k], loc[k], first[k]);
      }
      const uint32_t c = m.y ? m.y : ((p.is_outer && r < cx.p_hi) ? 1u : 0u);
      sm.off[k * PROBE_THREADS + tid] = m.y ? m.x : OFF_MISS;
      sm.prefix[k * PROBE_THREADS + tid] = c;
    }
    __syncthreads();
    bool any_multi;
    const unsigned long long M = tile_scan(sm, matched_acc, any_multi);
    if (tid == 0) sm.base = M ? atomicAdd(p.cursor, M) : 0ull;  // partition-major output: order across tiles is free
    __syncthreads();
    const unsigned long long base = sm.base;
    if (M && base + M <= p.capacity) {
      if (any_multi) tile_expand(p, sm, tile_base, base, M);
      else tile_emit_rowwise(p, sm, tile_base, base, key);
    }
    __syncthreads();
  }
  if ((tid & 31) == 0 && matched_acc) atomicAdd(p.cursor + 1, (unsigned long long)matched_acc);
}

}  // namespace tq
#include "join_stream.cuh"
namespace tq {

// The optimistic AoS scatter of one batch.  The caller describes the input in q (columns, key, key_mode, selected, pbits, n,
// overflow flag, segments); this sizes the slabs (slab_rows), reserves them and lo / hi / lim, initialises the slab bounds
// and launches k_scatter_aos — with TMA bulk copies when every input column is 16-byte aligned, plain loads otherwise.
static int32_t scatter_aos(ScatterAosParams &q, DevBuf &aos, DevBuf &lo, DevBuf &hi, DevBuf &lim, cudaStream_t s) {
  const int nc = q.sp.n_cols, pbits = q.sp.pbits;
  const int64_t n = q.sp.n;
  if (nc < 1 || nc > 4 || pbits < 1 || pbits > SA_MAX_PBITS || n <= 0 || n > 0xFFFFFFF0ll) { set_error("internal: AoS scatter arguments"); return TQ_ERR_INVALID_ARG; }
  const int P = 1 << pbits;
  const uint64_t slab = slab_rows(n, P, true);
  if (slab * P > 0xFFFFFFF0ull) { set_error("batch too large for 32-bit partition offsets"); return TQ_ERR_INVALID_ARG; }
  TQ_TRY(aos.reserve((size_t)slab * P * nc * 8 + 256));
  TQ_TRY(lo.reserve((size_t)(P + 3) * 4));
  TQ_TRY(hi.reserve((size_t)(P + 3) * 4));
  TQ_TRY(lim.reserve((size_t)(P + 3) * 4));
  k_init_slabs<<<(P + 1 + 255) / 256, 256, 0, s>>>(lo.as<uint32_t>(), hi.as<uint32_t>(), lim.as<uint32_t>(), P, (uint32_t)slab, 0u);
  count_launch();
  set_use_tma(q);
  q.sp.part_cursor = hi.as<uint32_t>();
  q.sp.part_lim = lim.as<uint32_t>();
  q.out = aos.as<uint64_t>();
  return launch_scatter_aos(q, nc, s);
}

// scatter.cuh: the streaming AoS scatter for other operators (HashAgg pre-aggregation)
int32_t scatter_rows_by_hash_aos(const DCol *cols, int n_cols, int key_col, int64_t n, int pbits, DevBuf &aos, DevBuf &lo, DevBuf &hi, DevBuf &lim,
                                 unsigned long long *d_overflow, cudaStream_t s) {
  ScatterAosParams q{};
  q.sp.n_cols = n_cols;
  for (int c = 0; c < n_cols && c < 4; c++) q.sp.in[c] = cols[c];
  q.sp.key_col = key_col;
  q.sp.key_mode = KEYMODE_RAW;
  q.sp.pbits = pbits;
  q.sp.n = n;
  q.sp.overflow = d_overflow;
  return scatter_aos(q, aos, lo, hi, lim, s);
}

// ------------------------------------------------------------------ host side
// Pinned accumulation of ≤1024-row host chunks into one column.
struct HostAccum {
  PinBuf data, bm;
  int64_t n = 0, cap = 0, bm_cap = 0;
  bool has_bm = false;
  int32_t ensure(int64_t rows) {
    if (rows <= cap) return TQ_OK;
    int64_t ncap = cap ? cap : 4096;
    while (ncap < rows) ncap *= 2;
    PinBuf nd, nb;
    TQ_TRY(nd.reserve((size_t)ncap * 8));
    TQ_TRY(nb.reserve(bitmap_alloc_bytes(ncap)));
    if (n) {
      memcpy(nd.p, data.p, (size_t)n * 8);
      memcpy(nb.p, bm.p, bitmap_bytes(n));
    }
    std::swap(data.p, nd.p); std::swap(data.cap, nd.cap);
    std::swap(bm.p, nb.p); std::swap(bm.cap, nb.cap);
    cap = ncap;
    bm_cap = ncap;
    return TQ_OK;
  }
  int32_t append(const tq_column &c, int64_t rows) {
    TQ_TRY(ensure(n + rows));
    memcpy(data.as<uint8_t>() + n * 8, c.data, (size_t)rows * 8);
    host_bitmap_append(bm.as<uint8_t>(), n, c.null_bitmap, rows);
    if (c.null_bitmap) has_bm = true;
    n += rows;
    return TQ_OK;
  }
  // indirect (FLOAT / var-len) columns: only the NULL bitmap is staged here, the cells go to a HostVarAccum
  int32_t append_nulls(const tq_column &c, int64_t rows) {
    if (n + rows > bm_cap) {  // bitmap-only growth (no 8-byte slots behind it)
      int64_t ncap = bm_cap ? bm_cap : 4096;
      while (ncap < n + rows) ncap *= 2;
      PinBuf nb;
      TQ_TRY(nb.reserve(bitmap_alloc_bytes(ncap)));
      if (n) memcpy(nb.p, bm.p, bitmap_bytes(n));
      std::swap(bm.p, nb.p); std::swap(bm.cap, nb.cap);
      bm_cap = ncap;
    }
    host_bitmap_append(bm.as<uint8_t>(), n, c.null_bitmap, rows);
    if (c.null_bitmap) has_bm = true;
    n += rows;
    return TQ_OK;
  }
  void reset() { n = 0; has_bm = false; }
};

struct DevColBuf {
  DevBuf data, bm;
};

struct ResultBatch {
  std::vector<DevColBuf> cols;
  int64_t n = 0;
  uint64_t capacity = 0;
  // host copies (host-consumer path)
  std::vector<PinBuf> h_data, h_bm;
  std::vector<VarOut> var;   // gathered FLOAT / var-len output columns (indexed like cols)
  std::vector<DevColBuf> alt;  // OtherConditions: the filtered copy of cols (swapped in)
  unsigned oc_err = 0;         // OtherConditions: ops that raised on its rows (bit i: op i); the call that delivers the batch reports the first
  bool on_host = false;
  cudaEvent_t ev_ready = nullptr;
  ~ResultBatch() { if (ev_ready) cudaEventDestroy(ev_ready); }
};

struct ProbeInputSet {  // device copy of one host probe batch
  std::vector<DevColBuf> cols;
  std::vector<SideStore> store;  // cells of the indirect probe columns of this batch
  DevBuf selected;
  cudaEvent_t ev_h2d = nullptr;
  ~ProbeInputSet() { if (ev_h2d) cudaEventDestroy(ev_h2d); }
};

// A segmented probe batch (tq_join_put_probe_segments): n device regions of `cap` rows each; region g holds *cnt[g] rows,
// column c of it starts at col[g][c].  n == 0: an ordinary batch.
struct SegSpec { int n = 0; int64_t cap = 0; const uint64_t *col[SA_MAX_SEGS][4]; const unsigned long long *cnt[SA_MAX_SEGS]; };

struct PendingBatch {  // a launched probe batch whose row count has not been read back yet
  bool active = false;
  std::unique_ptr<ResultBatch> rb;
  // inputs, kept for a possible re-run on output overflow
  std::vector<DCol> probe;
  const uint8_t *d_selected = nullptr;
  int64_t n = 0;
  bool want_host = false;
  int cursor_slot = 0;
  cudaEvent_t ev_k = nullptr;
};

// Key-less join (n_keys == 0, nlj.cuh): one probe batch, owned by the handle, and its position in its pair space.  The batch is
// walked in sub-ranges of whole probe rows; result batches are slices of the current sub-range's output.
struct KlProbe {
  ProbeInputSet in;            // the probe rows (+ FLOAT / var-len cells, selected bytes)
  std::vector<DCol> view;
  const uint8_t *d_sel = nullptr;
  int64_t n = 0;
  int64_t next_row = 0;        // first probe row of the next sub-range
  int64_t r0 = 0, rows = 0;    // the current sub-range
  uint64_t sub_total = 0, sub_pos = 0;
  bool sub_open = false;
};

}  // namespace tq

using namespace tq;

struct tq_join {
  // descriptor
  int join_type = 0, outer_is_right = 0;
  int n_build_cols = 0, n_probe_cols = 0, n_keys = 0;
  int build_types[MAXC], probe_types[MAXC];
  int build_key = 0, probe_key = 0;
  int key_mode = KEYMODE_RAW;
  // Several key columns (n_keys > 1): each side carries one hidden column — the key tuple folded exactly into one
  // 64-bit word (dict.cuh) — which is the key of the single-key kernels.  n_build_cols / n_probe_cols count it;
  // nb_user / np_user are what the caller passes and receives.
  int nb_user = 0, np_user = 0;
  int bkeys[MK_MAX_KEYS], pkeys[MK_MAX_KEYS];
  bool mk_no_signbit[MK_MAX_KEYS] = {};
  MultiKeyEncoder mk;
  DevBuf mk_build_key, mk_build_bm, mk_probe_key[2], mk_probe_bm[2];
  // FLOAT / var-len KEY columns (codec.go:226-233,276-333): a FLOAT key is compared as float64(f) — widened into an 8-byte
  // column; a var-len key is compared byte for byte — replaced by its id in a string dictionary built from the build side
  // (strdict.cuh).  Either makes the key "hidden" (an extra 8-byte column per side), like a multi-column key.
  uint64_t def_val[MAXC] = {};            // defaultInner per build column (+ NOT-NULL bits); all NULL unless the descriptor says otherwise
  uint32_t def_mask = 0;
  bool key_hidden = false;
  int bkey_kind[MK_MAX_KEYS] = {}, pkey_kind[MK_MAX_KEYS] = {};   // 0 = 8-byte column as is, 1 = FLOAT widened, 2 = var-len via dictionary
  StringDict sdict[MK_MAX_KEYS];
  DevBuf kx_b_data[MK_MAX_KEYS], kx_b_bm[MK_MAX_KEYS], kx_p_data[2][MK_MAX_KEYS], kx_p_bm[2][MK_MAX_KEYS];
  std::vector<int> out_map;               // caller's output column -> column of the result batch
  // FLOAT / var-len payload columns travel through the kernels as row ids into a side store (varlen.cuh)
  bool b_ind[MAXC] = {}, p_ind[MAXC] = {}, any_ind = false;
  int b_elem[MAXC] = {}, p_elem[MAXC] = {};
  SideStore b_store[MAXC];
  HostVarAccum b_var[MAXC], p_var[MAXC];
  int out_side[2 * MAXC] = {};            // per result-batch column: 0 = plain, 1 = build-side store, 2 = probe-side store
  int out_col[2 * MAXC] = {};
  DevBuf lens_scratch, scan_scratch3;
  DevBuf var_meta;                        // read-back record of append_cells_device (var-len columns of device chunks)
  // OtherConditions (othercond.cuh): applied to every finished result batch
  bool has_oc = false;
  OcPlan oc;
  int64_t oc_warnings = 0;                // division-by-zero warnings of the condition program so far
  int p_hidden_rowid = -1;                // outer joins: hidden probe column carrying the row id within the batch
  DevBuf oc_rowid[2], oc_scratch, oc_scan;
  int64_t batch_rows = 1 << 22;

  enum State { BUILDING, PROBING, CLOSED } state = BUILDING;

  // ---- build side
  std::vector<HostAccum> b_host;          // host chunks accumulate here
  std::vector<std::vector<tq_column>> b_dev_chunks;  // borrowed device chunks
  int build_mem = -1;
  int64_t n_build = 0;
  int flags = 0;                          // TQ_JOIN_* flags of the descriptor
  // large host build chunks skip the pinned staging copy: data goes straight to these device columns (H2D from the
  // caller's buffer inside the call), only the NULL bitmaps are staged on the host
  bool b_direct = false;
  std::vector<DevBuf> b_ddata;
  int64_t b_dcap = 0;
  std::vector<DevColBuf> b_cols;          // materialised inner side (owned) ...
  std::vector<DCol> b_view;               // ... or borrowed view
  DevBuf csr_rows, csr_mask;              // build rows in CSR order, row-major (+ per-row NOT-NULL mask)
  bool build_has_nulls = false;
  DevBuf slots, row_slot, row_ids, counters, worklist, scan_scratch;
  int shift = 1;                          // log2(words per table entry)
  bool row_mode = false;                  // unique build keys: the entries hold the build rows
  int row_word[MAXC];                     // ROW mode: word of build column c inside the entry
  int row_mask_word = -1;
  JoinTable table{};
  uint64_t n_slots = 0;
  int pbits = 0;                          // log2(#partition tables); 0 = one global table
  DevBuf b_part_cnt;
  int64_t n_valid = 0, n_distinct = 0;
  bool build_unique = true;
  int64_t build_ns = 0;
  int32_t build_path = TQ_JOIN_BUILD_GENERAL;
  int64_t part_rows = PART_TARGET_ROWS;   // build rows per partition table (TQ_JOIN_PART_ROWS at tq_join_create, tests)

  // ---- probe side
  std::vector<HostAccum> p_host;
  std::vector<uint8_t> p_sel_host;        // selected bytes of the staged chunks (lazily all-ones)
  bool p_sel_any = false;
  ProbeInputSet in_set[2];
  int in_flip = 0;
  PinBuf p_sel_pin[2];
  DevBuf cursors;                         // 2 x {rows, matched} device counters
  DevBuf tile_state[2];                   // per cursor slot: look-back words + ticket
  std::vector<DevColBuf> part_cols[2];    // per cursor slot: probe columns in partition order
  DevBuf part_cnt[2], part_off[2], part_cursor[2], part_lim[2];
  bool optimistic_scatter = true;         // general partitioned path: skip the histogram pass, fixed slabs with 25% slack (falls back on overflow)
  // streaming PK-FK pipeline (join_stream.cuh): exact partition counts, positional output, hole filling
  DevBuf pos_meta[2], pos_pt[2], pos_valid[2], hole_runs[2], hole_scan;
  uint32_t pos_epoch[2] = {0, 0};          // page-table epoch of the last positional batch in each cursor slot
  size_t pos_pt_cleared[2] = {0, 0};       // bytes of pos_pt cleared since it was allocated
  DevBuf b_aos;                           // build-side AoS slabs (released after the build)
  // segmented probe batch (tq_join_put_probe_segments): consumed by the next launch_probe_stream
  SegSpec seg;
  DevBuf scan_scratch2;
  PinBuf cursors_host;
  PendingBatch pending;
  std::deque<std::unique_ptr<ResultBatch>> results;
  std::vector<std::unique_ptr<ResultBatch>> free_list;
  std::unique_ptr<ResultBatch> lent;      // batch handed out by next_device
  std::unique_ptr<ResultBatch> host_cur;  // batch being sliced by next()
  int64_t host_cur_pos = 0;
  bool probe_eof = false;
  int64_t probe_rows_total = 0, joined_rows_total = 0, probe_launches = 0, last_probe_ns = 0;
  cudaEvent_t ev_a[2] = {nullptr, nullptr}, ev_b[2] = {nullptr, nullptr};  // per cursor slot
  // ---- key-less join (n_keys == 0): no table; probe batches become pair cursors, result batches are built on demand
  bool keyless = false;
  std::deque<std::unique_ptr<KlProbe>> kl;
  DevBuf kl_mask, kl_wpre, kl_cnt, kl_off, kl_miss, kl_meta, kl_scan;
  PinBuf kl_back;
  bool kl_timed = false;                  // ev_a[0] / ev_b[0] bracket the last result batch's kernels

  ~tq_join() {
    if (pending.ev_k) cudaEventDestroy(pending.ev_k);
    for (int i = 0; i < 2; i++) {
      if (ev_a[i]) cudaEventDestroy(ev_a[i]);
      if (ev_b[i]) cudaEventDestroy(ev_b[i]);
    }
  }
};

namespace tq {

static int probe_grid(int64_t n) {
  const int64_t tiles = (n + PROBE_TILE - 1) / PROBE_TILE;
  const int64_t cap = (int64_t)rt().sm_count * 6;
  return (int)(tiles < cap ? (tiles < 1 ? 1 : tiles) : cap);
}
static int stream_grid(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

static bool type_ok(int t) { return t == TQ_TYPE_INT64 || t == TQ_TYPE_UINT64 || t == TQ_TYPE_FLOAT64; }
static bool type_indirect(int t) { return t == TQ_TYPE_FLOAT32 || t == TQ_TYPE_BYTES; }

// Result row ids -> cells, for every indirect column of a finished result batch.
static int32_t materialize_indirect(tq_join *j, ResultBatch *rb, const std::vector<SideStore> &probe_store) {
  const int ncols = j->n_build_cols + j->n_probe_cols;
  rb->var.resize(ncols);
  for (int ic = 0; ic < ncols; ic++) {
    if (!j->out_side[ic]) continue;
    const SideStore &st = j->out_side[ic] == 1 ? j->b_store[j->out_col[ic]] : probe_store[j->out_col[ic]];
    TQ_TRY(gather_cells(st, rb->cols[ic].data.as<uint64_t>(), rb->cols[ic].bm.as<uint32_t>(), rb->n, rb->var[ic], j->lens_scratch, j->scan_scratch3,
                        rt().compute));
  }
  return TQ_OK;
}
static int32_t materialize_indirect(tq_join *j, ResultBatch *rb, int slot) { return materialize_indirect(j, rb, j->in_set[slot].store); }

static int32_t upload_col(const HostAccum &h, DevColBuf &d, cudaStream_t s) {
  TQ_TRY(d.data.reserve((size_t)(h.n ? h.n : 1) * 8));
  TQ_TRY(d.bm.reserve(bitmap_alloc_bytes(h.n)));
  if (h.n) {
    // (bitmap-only accumulators — row-id columns — have no staged data: the caller fills d.data itself)
    if (h.data.p) TQ_CUDA(cudaMemcpyAsync(d.data.p, h.data.p, (size_t)h.n * 8, cudaMemcpyHostToDevice, s));
    TQ_CUDA(cudaMemcpyAsync(d.bm.p, h.bm.p, bitmap_bytes(h.n), cudaMemcpyHostToDevice, s));
  }
  return TQ_OK;
}

// The 8-byte form of key column i of one side: the column itself, a FLOAT column widened to float64 bits, or the
// dictionary ids of a var-len column (the build side inserts, the probe side only looks up: a string the build side
// never had gets a 0 validity bit = "cannot match", exactly like a NULL key).
static int32_t key_source(tq_join *j, bool build, int i, const std::vector<DCol> &view, const SideStore *store, int64_t n, DevBuf &xd, DevBuf &xb, DCol *out,
                          cudaStream_t s) {
  const int col = build ? j->bkeys[i] : j->pkeys[i];
  const int kind = build ? j->bkey_kind[i] : j->pkey_kind[i];
  if (kind == 0) { *out = view[col]; return TQ_OK; }
  if (!store) { set_error("internal: FLOAT / var-len key column without a side store"); return TQ_ERR_STATE; }
  TQ_TRY(xd.reserve((size_t)(n ? n : 1) * 8));
  out->data = xd.as<uint64_t>();
  if (kind == 1) {
    TQ_TRY(widen_f32(store[col].bytes.as<uint32_t>(), n, xd.as<uint64_t>(), s));
    out->bm = view[col].bm;
    return TQ_OK;
  }
  TQ_TRY(xb.reserve(bitmap_alloc_bytes(n)));
  TQ_TRY(j->sdict[i].encode(view_of(store[col]), view[col].bm, n, store[col].nbytes, /*insert=*/build, xd.as<uint64_t>(), xb.as<uint32_t>(), s));
  out->bm = xb.as<uint32_t>();
  return TQ_OK;
}

// Whether the build side may try the streaming build (try_stream_build): a large NOT NULL build side whose rows fit a table
// entry and whose keys can match at all.  Unlike stream_probe_ok this does not depend on the join type: a stream-built table
// also serves outer joins, through the general partitioned probe.
static bool stream_build_ok(const tq_join *j) {
  return j->n_build >= PART_MIN_BUILD_ROWS && !g_no_fast_kernel && !j->build_has_nulls && j->n_build_cols <= 4 && j->key_mode != KEYMODE_NEVER;
}

// Whether probe batches may take the streaming positional path (launch_probe_stream) as far as the operator and its table
// decide: a partitioned ROW-mode table with unique NOT NULL build rows, an inner join without OtherConditions, and at most 4
// columns per side.  launch_probe adds what depends on the batch: no probe NULL bitmap.  Segmented batches only ever take
// this path (only its scatter reads regions).
static bool stream_probe_ok(const tq_join *j) {
  return j->pbits > 0 && j->pbits <= SA_MAX_PBITS && j->row_mode && j->join_type == TQ_JOIN_INNER && !j->build_has_nulls &&
         j->n_probe_cols <= 4 && j->n_build_cols <= 4 && !j->has_oc && !g_no_fast_kernel;
}

// Partition-local build (join_stream.cuh): scatter the build rows into AoS slabs, then build every sub-table in shared
// memory: one CTA per sub-table where a sub-table fits one CTA (k_build_cta), else one thread-block cluster per slab, in
// distributed shared memory (k_build_cluster).  The table has 2^(pbits + sbits) sub-tables; the probe side keeps the 2^pbits
// coarse partitions.  Covers the PK-FK shape — NOT NULL build columns that fit
// a table entry, unique keys; anything else (*done == false) takes the general build below.
static int32_t try_stream_build(tq_join *j, bool *done) {
  *done = false;
  cudaStream_t s = rt().compute;
  const int64_t n = j->n_build;
  const int NB = j->n_build_cols;
  int pbits = 0;
  while (((uint64_t)j->part_rows << pbits) < (uint64_t)n) pbits++;
  if (pbits > SA_MAX_PBITS) pbits = SA_MAX_PBITS;
  if (pbits < 1) return TQ_OK;
  const int P = 1 << pbits;
  // Table capacity from the row count alone (no host round trip for the partition histogram): hash partitions of m rows hold
  // m +- a few sqrt(m); a sub-table that turns out fuller than the load limit allows is flagged by the build kernel and the
  // general path takes over.  cap is that estimate at the load limit, rounded up to 16 entries so that every CTA's slice of a
  // cluster-built sub-table holds whole 32-byte sectors.  sbits: the fewest sub-tables per partition for which one fits the
  // shared memory of ONE CTA (k_build_cta) — or, where no such sbits stays within PART_MAX_BITS (the general probe path
  // scatters into one bin per sub-table), of a cluster (k_build_cluster).
  const int shift = NB > 2 ? 2 : 1;
  auto cap_of = [&](int sb) {
    const double mean = (double)n / (double)((uint64_t)P << sb);
    const uint64_t est_max = (uint64_t)(mean + 8.0 * sqrt(mean) + 64.0);
    return (est_max * 100 / (uint64_t)g_max_load_pct + 15) & ~15ull;
  };
  int sbits = 0;
  uint64_t cap = 0;
  bool cta = false;
  for (sbits = 0; pbits + sbits <= PART_MAX_BITS; sbits++) {
    cap = cap_of(sbits);
    if (((cap << shift) * 8) <= (uint64_t)BT_MAX_BYTES) { cta = true; break; }
  }
  if (!cta) {
    for (sbits = 0;; sbits++) {
      if (pbits + sbits > PART_MAX_BITS) return TQ_OK;
      cap = cap_of(sbits);
      if (((cap << shift) * 8) / BC_CLUSTER <= (uint64_t)BC_MAX_SLICE_BYTES) break;
    }
  }
  const uint64_t n_slots = ((uint64_t)P << sbits) * cap;
  if (n_slots > (uint64_t)n * 12 + 4096 || n_slots > 0xFFFFFFF0ull) return TQ_OK;
  // The build rows are scattered straight into one slab per sub-table when the scatter has that many bins; beyond
  // SA_MAX_PBITS bits each slab holds 2^(pbits + sbits - bbits) sub-tables: one CTA each reads the slab (k_build_cta), or
  // the slab's cluster builds them one after another (k_build_cluster).
  const int tbits = pbits + sbits;
  const int bbits = tbits < SA_MAX_PBITS ? tbits : SA_MAX_PBITS;
  const int n_bins = 1 << bbits;
  const uint64_t bin_slab = slab_rows(n, n_bins, true);
  if (bin_slab * n_bins > 0xFFFFFFF0ull) return TQ_OK;
  const int table_bytes = (int)((cap << shift) * 8);  // one sub-table
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute cl[1];
  cfg.blockDim = dim3(cta ? BT_THREADS : BC_THREADS);
  cfg.stream = s;
  const BuildKernel kb = cta ? build_cta_kernel(NB) : build_cluster_kernel(NB);
  if (cta) {
    static bool smem_set[5] = {false, false, false, false, false};
    if (!smem_set[NB]) {
      TQ_CUDA(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, BT_MAX_BYTES));
      smem_set[NB] = true;
    }
    cfg.gridDim = dim3(1u << tbits);  // one CTA per sub-table, those of one slab adjacent
    cfg.dynamicSmemBytes = (size_t)table_bytes;
  } else {
    cl[0].id = cudaLaunchAttributeClusterDimension;
    cl[0].val.clusterDim.x = BC_CLUSTER;
    cl[0].val.clusterDim.y = 1;
    cl[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)(n_bins * BC_CLUSTER));
    cfg.attrs = cl;
    cfg.numAttrs = 1;
    // once per kernel: the largest slice must fit, and the device must be able to run such a cluster at all
    static int cluster_ok[5] = {-1, -1, -1, -1, -1};
    if (cluster_ok[NB] < 0) {
      TQ_CUDA(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, BC_MAX_SLICE_BYTES));
      cfg.dynamicSmemBytes = BC_MAX_SLICE_BYTES;
      int n_clusters = 0;
      TQ_CUDA(cudaOccupancyMaxActiveClusters(&n_clusters, kb, &cfg));
      cluster_ok[NB] = n_clusters > 0 ? 1 : 0;
    }
    if (!cluster_ok[NB]) return TQ_OK;
    cfg.dynamicSmemBytes = (size_t)(table_bytes / BC_CLUSTER);
  }
  DevBuf &off = j->part_off[0], &hi = j->part_cursor[0], &lim = j->part_lim[0];
  unsigned long long *cur = j->cursors.as<unsigned long long>();
  TQ_CUDA(cudaMemsetAsync(cur, 0, 64, s));
  ScatterAosParams q{};
  q.sp.n_cols = NB;
  for (int c = 0; c < NB; c++) q.sp.in[c] = j->b_view[c];
  q.sp.key_col = j->build_key;
  q.sp.key_mode = j->key_mode;   // rows whose key can never match are dropped here (hash_table.go:161-163 skips NULL keys; none here)
  q.sp.pbits = bbits;
  q.sp.n = n;
  q.sp.overflow = cur + 2;
  TQ_TRY(scatter_aos(q, j->b_aos, off, hi, lim, s));
  TQ_TRY(j->slots.reserve(((n_slots + 1) << shift) * 8));  // (+ the side entry of the empty-marker key, unused on this path)
  uint64_t *words = j->slots.as<uint64_t>();
  BuildParams bp{};
  bp.slab = j->b_aos.as<uint64_t>();
  bp.lo = off.as<uint32_t>();
  bp.hi = hi.as<uint32_t>();
  bp.lim = lim.as<uint32_t>();
  bp.words = words;
  bp.cap = (uint32_t)cap;
  bp.max_rows = (uint32_t)(cap * (uint64_t)g_max_load_pct / 100);
  bp.tbits = tbits;
  bp.lbits = tbits - bbits;
  bp.key_col = j->build_key;
  {
    int w = 1;
    for (int c = 0; c < NB; c++) {
      j->row_word[c] = (c == j->build_key) ? 0 : w++;
      bp.word_of_col[c] = j->row_word[c];
    }
    j->row_mask_word = -1;
  }
  bp.rows = cur;
  bp.flags = reinterpret_cast<unsigned *>(cur + 3);
  TQ_CUDA(cudaLaunchKernelEx(&cfg, kb, bp));
  count_launch();
  TQ_TRY(check_launch(cta ? "k_build_cta" : "k_build_cluster"));
  // {rows inserted, -, slab overflow, flags}: one copy into pinned memory
  const unsigned long long *h_cur = j->cursors_host.as<unsigned long long>();
  TQ_CUDA(cudaMemcpyAsync(j->cursors_host.p, cur, 32, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  if (h_cur[2]) return TQ_OK;  // a slab overflowed: skewed hash partitions
  if (h_cur[3]) return TQ_OK;  // duplicate keys, the empty-marker key, or a partition over the load limit: the general build handles them
  const uint64_t n_valid = h_cur[0];
  j->shift = shift;
  j->pbits = pbits;
  j->n_slots = n_slots;
  j->n_valid = (int64_t)n_valid;
  j->n_distinct = (int64_t)n_valid;
  j->build_unique = true;
  j->row_mode = true;
  j->table.words = words;
  j->table.cap = (uint32_t)cap;
  j->table.pbits = tbits;
  j->table.shift = shift;
  j->table.row_mode = 1;
  j->table.sent_off = (uint32_t)n_slots;
  j->table.sent_cnt = 0;
  j->build_path = cta ? TQ_JOIN_BUILD_CTA : TQ_JOIN_BUILD_CLUSTER;
  *done = true;
  return TQ_OK;
}

static int32_t join_build(tq_join *j) {
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  const int64_t n = j->n_build;
  TQ_CUDA(cudaEventRecord(j->ev_a[0], s));
  const DCol key = j->b_view[j->build_key];
  TQ_TRY(j->counters.reserve(64));
  uint32_t *counters = j->counters.as<uint32_t>();
  TQ_CUDA(cudaMemsetAsync(counters, 0, 64, s));
  j->build_has_nulls = false;
  j->build_path = TQ_JOIN_BUILD_GENERAL;
  for (int c = 0; c < j->n_build_cols; c++) j->build_has_nulls |= (j->b_view[c].bm != nullptr);
  if (stream_build_ok(j)) {
    bool done = false;
    TQ_TRY(try_stream_build(j, &done));
    j->b_aos.release();
    if (done) {
      TQ_CUDA(cudaEventRecord(j->ev_b[0], s));
      TQ_CUDA(cudaStreamSynchronize(s));
      float ms = 0;
      TQ_CUDA(cudaEventElapsedTime(&ms, j->ev_a[0], j->ev_b[0]));
      j->build_ns = (int64_t)(ms * 1e6);
      j->b_cols.clear();
      j->b_view.clear();
      return TQ_OK;
    }
  }
  // entry layout: ROW mode needs key + other columns (+ mask word) to fit 2 or 4 words
  const int row_words = j->n_build_cols + (j->build_has_nulls ? 1 : 0);
  const bool row_candidate = row_words <= 4;
  const int shift = (row_candidate && row_words > 2) ? 2 : 1;
  j->shift = shift;
  // Partitioning: ~j->part_rows build rows per partition table; small build sides keep ONE table.
  uint64_t n_slots = 64, cap = 0;
  int pbits = 0;
  if (n >= PART_MIN_BUILD_ROWS) {
    uint64_t P = 1;
    while (P * (uint64_t)j->part_rows < (uint64_t)n) P <<= 1;
    while ((1ull << pbits) < P) pbits++;
    if (pbits > PART_MAX_BITS) pbits = PART_MAX_BITS;
    P = 1ull << pbits;
    TQ_TRY(j->b_part_cnt.reserve(P * 4));
    TQ_CUDA(cudaMemsetAsync(j->b_part_cnt.p, 0, P * 4, s));
    k_build_part_hist<<<stream_grid(n), 256, 0, s>>>(key.data, key.bm, n, j->key_mode, pbits, j->b_part_cnt.as<uint32_t>());
    k_max_u32<<<1, 1024, 0, s>>>(j->b_part_cnt.as<uint32_t>(), (int)P, counters + 4);
    count_launch(2);
    TQ_TRY(check_launch("k_build_part_hist"));
    uint32_t max_cnt = 0;
    TQ_CUDA(cudaMemcpyAsync(&max_cnt, counters + 4, 4, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    cap = 64;
    while (cap * (uint64_t)g_max_load_pct < (uint64_t)max_cnt * 100) cap <<= 1;  // load factor <= g_max_load_pct % in the fullest partition
    if (cap * P > (uint64_t)n * 12 + 4096) { pbits = 0; cap = 0; }  // heavily skewed hash partitions: one table instead
    else n_slots = P * cap;
  }
  if (pbits == 0) {
    while (n_slots < (uint64_t)n * 2) n_slots <<= 1;       // one table at load factor <= 0.5
    cap = n_slots;
  }
  j->pbits = pbits;
  if (n_slots > 0xFFFFFFF0ull) { set_error("build side too large: %lld rows", (long long)n); return TQ_ERR_INVALID_ARG; }
  j->n_slots = n_slots;
  const uint64_t n_entries = n_slots + 1;  // +1: side entry for the EMPTY_KEY-valued key in ROW mode
  TQ_TRY(j->slots.reserve((n_entries << shift) * 8));
  TQ_TRY(j->row_slot.reserve((size_t)(n ? n : 1) * 4));
  uint64_t *words = j->slots.as<uint64_t>();
  k_init_table<<<stream_grid((int64_t)(n_entries << shift)), 256, 0, s>>>(words, n_entries, shift);
  count_launch();
  InsertParams ip{};
  ip.n_cols = j->n_build_cols;
  ip.key_col = j->build_key;
  ip.key_mode = j->key_mode;
  {
    int w = 1;
    for (int c = 0; c < j->n_build_cols; c++) {
      ip.cols[c] = j->b_view[c];
      j->row_word[c] = (c == j->build_key) ? 0 : w++;
      ip.word_of_col[c] = j->row_word[c];
    }
    j->row_mask_word = j->build_has_nulls ? w : -1;
  }
  ip.mask_word = j->row_mask_word;
  ip.write_rows = row_candidate ? 1 : 0;
  ip.n = n;
  ip.words = words;
  ip.cap = (uint32_t)cap;
  ip.pbits = pbits;
  ip.shift = shift;
  ip.sent_entry = (uint32_t)n_slots;
  ip.row_slot = j->row_slot.as<uint32_t>();
  ip.counters = counters;
  if (n > 0) {
    k_build_insert<<<stream_grid(n), 256, 0, s>>>(ip);
    count_launch();
  }
  TQ_TRY(check_launch("k_build_insert"));
  uint32_t h_counters[16];
  TQ_CUDA(cudaMemcpyAsync(h_counters, counters, 64, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  const uint32_t sent_cnt = h_counters[0];
  const int64_t valid_regular = h_counters[5], distinct_regular = h_counters[2];
  j->n_valid = valid_regular + sent_cnt;
  j->n_distinct = distinct_regular + (sent_cnt ? 1 : 0);
  j->build_unique = (j->n_distinct == j->n_valid);
  j->table.words = words;
  j->table.cap = (uint32_t)cap;
  j->table.pbits = pbits;
  j->table.shift = shift;
  j->row_mode = j->build_unique && row_candidate;
  j->table.row_mode = j->row_mode ? 1 : 0;
  if (j->row_mode) {
    // ---- ROW mode: every key is unique, so the claiming rows have already written the whole table
    j->table.sent_off = (uint32_t)n_slots;
    j->table.sent_cnt = sent_cnt;
  } else {
    // ---- CSR mode: count rows per key, then exclusive scan of the counts (high half of word 1) into the offsets (low half)
    k_clear_word1<<<stream_grid((int64_t)n_entries), 256, 0, s>>>(words, n_entries, shift);
    if (n > 0) k_build_count<<<stream_grid(n), 256, 0, s>>>(j->row_slot.as<uint32_t>(), n, words, shift);
    count_launch(2);
    TQ_TRY(check_launch("k_build_count"));
    TQ_TRY(j->row_ids.reserve((size_t)(n ? n : 1) * 4));
    const uint32_t worklist_cap = (uint32_t)((n / 33) + 2);
    TQ_TRY(j->worklist.reserve((size_t)worklist_cap * 8));
    uint32_t *w32 = reinterpret_cast<uint32_t *>(words);
    const int stride32 = 2 << shift;
    uint64_t *d_total = reinterpret_cast<uint64_t *>(counters + 8);
    TQ_TRY(exclusive_scan_u32(w32 + 3, stride32, w32 + 2, stride32, (int64_t)n_slots, d_total, j->scan_scratch, s));
    j->table.sent_off = (uint32_t)valid_regular;  // the EMPTY_KEY-valued key's segment follows all regular segments
    j->table.sent_cnt = sent_cnt;
    if (n > 0) {
      k_build_fill<<<stream_grid(n), 256, 0, s>>>(j->row_slot.as<uint32_t>(), n, words, shift, j->table.sent_off, counters, j->row_ids.as<uint32_t>());
      count_launch();
    }
    k_build_fixsort<<<stream_grid((int64_t)n_slots), 256, 0, s>>>(words, n_slots, shift, j->row_ids.as<uint32_t>(), counters, j->worklist.as<uint2>(), worklist_cap);
    count_launch();
    TQ_TRY(check_launch("k_build_fixsort"));
    TQ_CUDA(cudaMemcpyAsync(h_counters, counters, 64, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    uint32_t n_large = h_counters[3];
    if (sent_cnt > 1) {  // the sentinel-key segment is sorted like any other large segment
      uint2 w = make_uint2(j->table.sent_off, sent_cnt);
      TQ_CUDA(cudaMemcpyAsync(j->worklist.as<uint2>() + n_large, &w, sizeof(w), cudaMemcpyHostToDevice, s));
      n_large++;
    }
    if (n_large) {
      k_sort_large<<<n_large, 256, 0, s>>>(j->worklist.as<uint2>(), j->row_ids.as<uint32_t>());
      count_launch();
      TQ_TRY(check_launch("k_sort_large"));
    }
    // build rows into CSR order, packed row-major
    const int64_t nv = j->n_valid;
    TQ_TRY(j->csr_rows.reserve((size_t)(nv ? nv : 1) * 8 * j->n_build_cols));
    if (j->build_has_nulls) TQ_TRY(j->csr_mask.reserve((size_t)(nv ? nv : 1) * 4));
    if (nv) {
      GatherParams g{};
      g.n_cols = j->n_build_cols;
      for (int c = 0; c < j->n_build_cols; c++) g.cols[c] = j->b_view[c];
      g.row_ids = j->row_ids.as<uint32_t>();
      g.n = nv;
      g.out_rows = j->csr_rows.as<uint64_t>();
      g.out_mask = j->build_has_nulls ? j->csr_mask.as<uint32_t>() : nullptr;
      k_gather_rows<<<stream_grid(nv), 256, 0, s>>>(g);
      count_launch();
    }
    TQ_TRY(check_launch("k_gather_rows"));
  }
  TQ_CUDA(cudaEventRecord(j->ev_b[0], s));
  TQ_CUDA(cudaStreamSynchronize(s));
  float ms = 0;
  TQ_CUDA(cudaEventElapsedTime(&ms, j->ev_a[0], j->ev_b[0]));
  j->build_ns = (int64_t)(ms * 1e6);
  // the row-order copies are no longer needed
  j->row_slot.release();
  j->row_ids.release();
  j->b_cols.clear();
  j->b_view.clear();
  return TQ_OK;
}

static std::unique_ptr<ResultBatch> get_result_batch(tq_join *j) {
  std::unique_ptr<ResultBatch> rb;
  if (!j->free_list.empty()) { rb = std::move(j->free_list.back()); j->free_list.pop_back(); }
  else rb.reset(new ResultBatch());
  rb->n = 0;
  rb->on_host = false;
  for (auto &v : rb->var) v.used = false;
  return rb;
}

// Hole filling, fast path: when every probe row of the batch found its match (the foreign-key join) the only holes of the
// positional result are the unfilled tails of the partitions' last pages, and both lists — the hole slots below M and the real
// rows at or above M — are a few runs of slots that follow from the final cursors and the page table alone: one run of holes
// per partition, and one run of real rows per page at or above M (at most P such pages, since the P last pages leave less
// than P pages unfilled).  k_hole_pages writes the runs with their prefix offsets; k_hole_move_pages finds the k-th hole and
// the k-th tail row by binary search over them.  A batch with misses (M != rows scattered) is completed by fill_holes_host
// once the counts are on the host.
static constexpr int HOLE_PAD_THREADS = 512;   // >= partitions of the streaming path (SA_MAX_PBITS)
struct HoleRuns {
  uint32_t *h_start, *h_off;   // [n_parts], [n_parts + 1]: partition q's holes below M start at h_start[q], the h_off[q]-th hole
  uint32_t *t_start, *t_off;   // [n_parts], [n_parts + 1]: the i-th page at or above M: its real rows there, likewise
};
__global__ void __launch_bounds__(HOLE_PAD_THREADS) k_hole_pages(const PosPages m, int n_parts, unsigned long long *cur, const HoleRuns h) {
  __shared__ uint32_t s_warp[HOLE_PAD_THREADS / 32 + 1];
  __shared__ uint32_t s_fill[HOLE_PAD_THREADS];
  const int q = threadIdx.x;
  const uint64_t M = cur[0], PG = m.page_rows;
  uint32_t c = 0, n_h = 0;
  uint64_t last = 0, fill = 0, h_lo = 0;
  if (q < n_parts) c = m.cursor[q];
  if (c) {
    const uint32_t k = (c - 1) / (uint32_t)PG;
    last = (uint32_t)m.pt[(uint64_t)q * m.kmax + k];   // the partition's last page, filled up to `fill`
    fill = c - (uint64_t)k * PG;
    h_lo = last * PG + fill;
    const uint64_t h_hi = (last + 1) * PG < M ? (last + 1) * PG : M;
    n_h = h_hi > h_lo ? (uint32_t)(h_hi - h_lo) : 0u;
  }
  block_excl_scan<HOLE_PAD_THREADS>(c, s_warp);
  const uint32_t rows = s_warp[HOLE_PAD_THREADS / 32];
  __syncthreads();   // s_warp is scanned again
  const uint32_t h_off = block_excl_scan<HOLE_PAD_THREADS>(n_h, s_warp);
  const uint32_t n_holes = s_warp[HOLE_PAD_THREADS / 32];
  if (q == 0) {
    cur[6] = rows;                    // rows the scatter placed: == M iff no probe row missed
    cur[5] = n_holes;                 // holes to fill
  }
  if ((uint64_t)rows != M) return;    // misses among the probe rows: fill_holes_host builds exact lists (CTA-uniform exit)
  if (q < n_parts) {
    h.h_start[q] = (uint32_t)h_lo;
    h.h_off[q] = h_off;
  }
  // pages first .. n_pages - 1 hold the real rows at or above M: every one full but the partitions' last pages
  const uint64_t first = M / PG, n_tail = m.cursor[n_parts] - first;
  s_fill[q] = (uint32_t)PG;
  __syncthreads();
  if (c && last >= first) s_fill[last - first] = (uint32_t)fill;
  __syncthreads();
  uint32_t n_t = 0;
  uint64_t t_lo = 0;
  if ((uint64_t)q < n_tail) {
    const uint64_t pb = (first + q) * PG;
    t_lo = pb > M ? pb : M;
    n_t = pb + s_fill[q] > t_lo ? (uint32_t)(pb + s_fill[q] - t_lo) : 0u;
  }
  const uint32_t t_off = block_excl_scan<HOLE_PAD_THREADS>(n_t, s_warp);
  const uint32_t n_tail_rows = s_warp[HOLE_PAD_THREADS / 32];   // == n_holes
  if (q < n_parts) {
    h.t_start[q] = (uint32_t)t_lo;
    h.t_off[q] = (uint64_t)q < n_tail ? t_off : n_tail_rows;   // (past the tail pages: no row, never found)
  }
  if (q == 0) {
    h.h_off[n_parts] = n_holes;
    h.t_off[n_parts] = n_tail_rows;
  }
}
struct HoleMoveDevParams {
  int n_cols, n_parts;
  uint64_t *col[8];
  HoleRuns runs;
  const unsigned long long *cur;
};
// the last index i < n with off[i] <= k (off ascending, off[0] = 0)
__device__ __forceinline__ int run_of(const uint32_t *off, int n, uint32_t k) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= k) lo = mid;
    else hi = mid;
  }
  return lo;
}
__global__ void __launch_bounds__(256) k_hole_move_pages(const HoleMoveDevParams h) {
  __shared__ uint32_t s_hs[HOLE_PAD_THREADS], s_ho[HOLE_PAD_THREADS], s_ts[HOLE_PAD_THREADS], s_to[HOLE_PAD_THREADS];
  if (h.cur[6] != h.cur[0]) return;  // misses: the host-sized pass does the whole job
  const uint64_t H = h.cur[5];
  if ((uint64_t)blockIdx.x * blockDim.x >= H) return;
  for (int i = threadIdx.x; i < h.n_parts; i += blockDim.x) {
    s_hs[i] = h.runs.h_start[i];
    s_ho[i] = h.runs.h_off[i];
    s_ts[i] = h.runs.t_start[i];
    s_to[i] = h.runs.t_off[i];
  }
  __syncthreads();
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < H; k += stride) {
    const int a = run_of(s_ho, h.n_parts, (uint32_t)k), b = run_of(s_to, h.n_parts, (uint32_t)k);
    const uint32_t d = s_hs[a] + ((uint32_t)k - s_ho[a]), sidx = s_ts[b] + ((uint32_t)k - s_to[b]);
#pragma unroll
    for (int c = 0; c < 8; c++)
      if (c < h.n_cols) h.col[c][d] = h.col[c][sidx];
  }
}

// column-wise scatter into result pages claimed on the fly -> key-only positional probe -> device-driven hole filling.
// Nothing is read back to the host.
static int32_t launch_probe_stream(tq_join *j, const ProbeParams &p, const std::vector<DCol> &probe, const uint8_t *d_selected, int64_t n,
                                   unsigned long long *cur, int slot, uint64_t alloc_rows) {
  cudaStream_t s = rt().compute;
  const int P = 1 << j->pbits, NP = j->n_probe_cols, NB = j->n_build_cols;
  const uint32_t page = pos_page_rows(n, P, NP);
  if (n + (int64_t)P * page > 0xFFFFFFF0ll) { set_error("probe batch too large for 32-bit result slots; feed smaller batches"); return TQ_ERR_INVALID_ARG; }
  TQ_TRY(j->pos_meta[slot].reserve((size_t)2 * (P + 1) * 4));
  PosPages m;
  m.cursor = j->pos_meta[slot].as<uint32_t>();
  m.chunk = m.cursor + (P + 1);
  m.page_rows = page;
  m.kmax = (uint32_t)(n / page + 1);   // virtual pages of one partition holding the whole batch
  // The page table is cleared only when a batch needs more of it than was cleared before (the first batch of a handle) and
  // when the epoch wraps; otherwise a batch writes only the entries it uses, and older entries carry an older epoch.
  const size_t pt_bytes = (size_t)P * m.kmax * 8;
  uint32_t &epoch = j->pos_epoch[slot];
  if (j->pos_pt_cleared[slot] < pt_bytes || epoch == 0xFFFFFFFFu) {
    TQ_TRY(j->pos_pt[slot].reserve(pt_bytes));
    TQ_CUDA(cudaMemsetAsync(j->pos_pt[slot].p, 0, pt_bytes, s));   // (not the whole block: a cached one may be far larger)
    j->pos_pt_cleared[slot] = pt_bytes;
    epoch = 0;
  }
  m.epoch = ++epoch;
  m.pt = j->pos_pt[slot].as<unsigned long long>();
  m.err = cur + 4;
  const int64_t n_words_max = (int64_t)(alloc_rows >> 5) + 1;
  TQ_TRY(j->pos_valid[slot].reserve((size_t)(n_words_max + 2) * 4));
  TQ_TRY(j->hole_runs[slot].reserve((size_t)4 * (P + 1) * 4));
  HoleRuns hr;
  hr.h_start = j->hole_runs[slot].as<uint32_t>();
  hr.h_off = hr.h_start + (P + 1);
  hr.t_start = hr.h_off + (P + 1);
  hr.t_off = hr.t_start + (P + 1);
  const ProbePosVariant pv = probe_pos_kernel(NB);
  if (!pv.k || NP < 1 || NP > 4) { set_error("internal: positional probe of %d x %d columns", NP, NB); return TQ_ERR_INVALID_ARG; }
  ScatterAosParams q{};
  q.sp.n_cols = NP;
  for (int c = 0; c < NP; c++) {
    q.sp.in[c] = probe[c];
    q.sp.out[c].data = p.out_probe[c].data;   // the result's probe columns
  }
  int64_t seg_rows = 0;
  if (j->seg.n) {  // regions filled by the peers' push kernels; row counts live on the device
    seg_rows = (j->seg.cap + POS_SEG_ROWS_ALIGN - 1) / POS_SEG_ROWS_ALIGN * POS_SEG_ROWS_ALIGN;
    q.n_segs = j->seg.n;
    for (int g = 0; g < j->seg.n; g++) {
      q.seg_cnt[g] = j->seg.cnt[g];
      for (int c = 0; c < NP; c++) q.seg_in[g][c] = j->seg.col[g][c];
    }
  }
  q.sp.selected = d_selected;
  q.sp.key_col = j->probe_key;
  q.sp.key_mode = j->key_mode;
  q.sp.pbits = j->pbits;
  q.sp.n = n;
  TQ_TRY(launch_pos_scatter(q, seg_rows, m, cur + 3, s));
  ProbePosParams pp{};
  pp.keys = p.out_probe[j->probe_key].data;
  pp.cnt = m.cursor;
  pp.chunk = m.chunk;
  pp.pt = m.pt;
  pp.page_rows = m.page_rows;
  pp.kmax = m.kmax;
  pp.n_parts = P;
  for (int c = 0; c < NB; c++) { pp.out_build[c] = p.out_build[c].data; pp.build_word[c] = p.build_word[c]; }
  pp.valid = j->pos_valid[slot].as<uint32_t>();
  pp.cursor = cur;
  { const char *e = getenv("TQ_JOIN_PP_DEBUG"); const int f = e ? atoi(e) : 0; pp.dbg_no_tma = f & 1; pp.dbg_late_release = (f >> 1) & 1; }
  // CTAs: at most one per PP_CHUNK_TILES tiles of rows plus one per partition (its last, partial chunk); the unused ones exit
  const int64_t grid = n / ((int64_t)pv.tile * PP_CHUNK_TILES) + P + 1;
  const int smem = PP_STAGES * pv.tile * 8;
  TQ_CUDA(cudaFuncSetAttribute(pv.k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  pv.k<<<(unsigned)grid, pv.threads, smem, s>>>(pp, j->table);
  count_launch();
  TQ_TRY(check_launch("k_probe_pos"));
  // holes: the unfilled tails of the last pages (filled here) + probe rows without a match (finalize_pending)
  k_hole_pages<<<1, HOLE_PAD_THREADS, 0, s>>>(m, P, cur, hr);
  HoleMoveDevParams hm{};
  hm.n_cols = NP + NB;
  hm.n_parts = P;
  for (int c = 0; c < NP; c++) hm.col[c] = p.out_probe[c].data;
  for (int c = 0; c < NB; c++) hm.col[NP + c] = p.out_build[c].data;
  hm.runs = hr;
  hm.cur = cur;
  k_hole_move_pages<<<rt().sm_count * 4, 256, 0, s>>>(hm);
  count_launch(2);
  TQ_TRY(check_launch("k_hole_move_pages"));
  j->probe_launches += 6;
  return TQ_OK;
}

// misses among the probe rows (a join with many misses): exact-size lists, after the counts are on the host
static int32_t fill_holes_host(tq_join *j, ResultBatch *rb, int slot, uint64_t M, uint64_t S) {
  cudaStream_t s = rt().compute;
  const int64_t n_words = (int64_t)(S >> 5);
  if (n_words == 0 || S == M) return TQ_OK;
  const uint64_t max_holes = S - M;
  // prefix popcounts of the validity bitmap (n_words + 1 entries: the last one is the total), then the two lists, then the moves
  DevBuf cnt, pre, hp, hs;
  TQ_TRY(cnt.reserve((size_t)(n_words + 2) * 4));
  TQ_TRY(pre.reserve((size_t)(n_words + 2) * 4));
  TQ_TRY(hp.reserve((size_t)(max_holes + 64) * 4));
  TQ_TRY(hs.reserve((size_t)(max_holes + 64) * 4));
  const uint32_t *valid = j->pos_valid[slot].as<uint32_t>();
  TQ_CUDA(cudaMemsetAsync(cnt.as<uint32_t>() + n_words, 0, 4, s));
  k_hole_popc<<<stream_grid(n_words), 256, 0, s>>>(valid, n_words, cnt.as<uint32_t>());
  count_launch();
  TQ_TRY(exclusive_scan_u32(cnt.as<uint32_t>(), 1, pre.as<uint32_t>(), 1, n_words + 1, nullptr, j->hole_scan, s));
  k_hole_lists<<<stream_grid(n_words), 256, 0, s>>>(valid, pre.as<uint32_t>(), n_words, M, hp.as<uint32_t>(), hs.as<uint32_t>());
  HoleMoveParams hm{};
  hm.n_cols = (int)rb->cols.size();
  if (hm.n_cols > 8) { set_error("internal: positional result with %d columns", hm.n_cols); return TQ_ERR_STATE; }
  for (int c = 0; c < hm.n_cols; c++) hm.col[c] = rb->cols[c].data.as<uint64_t>();
  hm.hole_pos = hp.as<uint32_t>();
  hm.tail_src = hs.as<uint32_t>();
  hm.valid = valid;
  hm.vpre = pre.as<uint32_t>();
  hm.n_words = n_words;
  hm.M = M;
  k_hole_move<<<stream_grid((int64_t)max_holes), 256, 0, s>>>(hm);
  count_launch(2);
  TQ_TRY(check_launch("k_hole_move"));
  TQ_CUDA(cudaStreamSynchronize(s));  // the scratch arrays go back to the allocator
  return TQ_OK;
}

// Enqueue one probe launch for `n` rows of device columns `probe` into rb (capacity rows).
static int32_t launch_probe(tq_join *j, const std::vector<DCol> &probe, const uint8_t *d_selected, int64_t n, ResultBatch *rb, uint64_t capacity,
                            int cursor_slot) {
  if (n > 0xFFFFFFF0ll) { set_error("probe batch of %lld rows exceeds the 32-bit partition offsets; feed smaller batches", (long long)n); return TQ_ERR_INVALID_ARG; }
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  const int ncols = j->n_build_cols + j->n_probe_cols;
  rb->cols.resize(ncols);
  rb->capacity = capacity;
  const int build_base = j->outer_is_right ? 0 : j->n_probe_cols;   // joiner.go:145-150: lhs ++ rhs
  const int probe_base = j->outer_is_right ? j->n_build_cols : 0;
  ProbeParams p{};
  p.n_probe_cols = j->n_probe_cols;
  p.n_build_cols = j->n_build_cols;
  p.selected = d_selected;
  p.key_col = j->probe_key;
  p.key_mode = j->key_mode;
  p.is_outer = (j->join_type != TQ_JOIN_INNER);
  for (int c = 0; c < MAXC; c++) p.def_val[c] = j->def_val[c];
  p.def_mask = j->def_mask;
  p.n = n;
  p.capacity = capacity;
  unsigned long long *cur = j->cursors.as<unsigned long long>() + 8 * cursor_slot;  // [0] rows, [1] matched probe rows, [2] slab overflow (general path), [3] span of the positional result, [4] a result page id never appeared, [5] page-tail holes, [6] rows the scatter placed
  p.cursor = cur;
  TQ_CUDA(cudaMemsetAsync(cur, 0, 64, s));
  {
    const int64_t n_tiles = (n + PROBE_TILE - 1) / PROBE_TILE;
    DevBuf &ts = j->tile_state[cursor_slot];
    TQ_TRY(ts.reserve((size_t)(n_tiles + 1) * 8));
    TQ_CUDA(cudaMemsetAsync(ts.p, 0, (size_t)(n_tiles + 1) * 8, s));
    p.tile_state = ts.as<unsigned long long>();
    p.ticket = reinterpret_cast<unsigned *>(ts.as<unsigned long long>() + n_tiles);
  }
  // The streaming PK-FK pipeline (join_stream.cuh) when the operator allows it and this batch has no probe NULL bitmap.  Its
  // result is paged: room for the unfilled tail of every partition's last page.
  bool any_in_bm = false;
  for (int c = 0; c < j->n_probe_cols; c++) any_in_bm |= (probe[c].bm != nullptr);
  const bool pos_path = stream_probe_ok(j) && !any_in_bm;
  const uint64_t alloc_rows = capacity + (pos_path ? (uint64_t)pos_page_rows(n, 1 << j->pbits, j->n_probe_cols) << j->pbits : 0);
  for (int c = 0; c < ncols; c++) {
    TQ_TRY(rb->cols[c].data.reserve((size_t)(alloc_rows ? alloc_rows : 1) * 8));
    TQ_TRY(rb->cols[c].bm.reserve(bitmap_alloc_bytes((int64_t)alloc_rows)));
  }
  for (int c = 0; c < j->n_probe_cols; c++) {
    p.probe[c] = probe[c];
    DevColBuf &o = rb->cols[probe_base + c];
    p.out_probe[c].data = o.data.as<uint64_t>();
    const bool may_null = probe[c].bm != nullptr;
    TQ_CUDA(cudaMemsetAsync(o.bm.p, may_null ? 0x00 : 0xFF, bitmap_alloc_bytes((int64_t)capacity), s));
    p.out_probe[c].bm = may_null ? o.bm.as<uint32_t>() : nullptr;
  }
  if (j->row_mode) {
    p.build_rows = j->slots.as<uint64_t>();
    p.build_stride = 1 << j->shift;
    for (int c = 0; c < j->n_build_cols; c++) p.build_word[c] = j->row_word[c];
    p.build_mask = nullptr;
    p.build_mask_word = j->row_mask_word;
  } else {
    p.build_rows = j->csr_rows.as<uint64_t>();
    p.build_stride = j->n_build_cols;
    for (int c = 0; c < j->n_build_cols; c++) p.build_word[c] = c;
    p.build_mask = j->build_has_nulls ? j->csr_mask.as<uint32_t>() : nullptr;
    p.build_mask_word = -1;
  }
  for (int c = 0; c < j->n_build_cols; c++) {
    DevColBuf &o = rb->cols[build_base + c];
    p.out_build[c].data = o.data.as<uint64_t>();
    const bool may_null = p.is_outer || j->build_has_nulls;  // outer-join misses pad the inner side with NULLs
    TQ_CUDA(cudaMemsetAsync(o.bm.p, may_null ? 0x00 : 0xFF, bitmap_alloc_bytes((int64_t)capacity), s));
    p.out_build[c].bm = may_null ? o.bm.as<uint32_t>() : nullptr;
  }
  TQ_CUDA(cudaEventRecord(j->ev_a[cursor_slot], s));
  if (pos_path) {
    TQ_TRY(launch_probe_stream(j, p, probe, d_selected, n, cur, cursor_slot, alloc_rows));
  } else if (j->pbits == 0) {
    k_probe<<<probe_grid(n), PROBE_THREADS, 0, s>>>(p, j->table);
    count_launch();
    j->probe_launches++;
    TQ_TRY(check_launch("k_probe"));
  } else {
    // ---- partitioned pipeline: histogram -> scan -> scatter -> per-partition probe with the table in smem.  One bin per
    // partition TABLE: a stream-built table has more tables (sub-tables) than the build had partitions.
    const int P = 1 << j->table.pbits;
    const int n_bins = P + 1;
    static bool attr_done = false;
    if (!attr_done) {
      TQ_CUDA(cudaFuncSetAttribute(k_probe_part, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PART_MAX_SMEM_BYTES));
      TQ_CUDA(cudaFuncSetAttribute(k_probe_part_uniq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PART_MAX_SMEM_BYTES));
      TQ_CUDA(cudaFuncSetAttribute(k_probe_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, scatter_smem_bytes((1 << PART_MAX_BITS) + 1)));
      TQ_CUDA(cudaFuncSetAttribute(k_probe_part_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(((1 << PART_MAX_BITS) + 1) * 4)));
      attr_done = true;
    }
    DevBuf &cnt = j->part_cnt[cursor_slot], &off = j->part_off[cursor_slot], &cur_b = j->part_cursor[cursor_slot];
    TQ_TRY(cnt.reserve((size_t)(n_bins + 1) * 4));
    TQ_TRY(off.reserve((size_t)(n_bins + 1) * 4));
    TQ_TRY(cur_b.reserve((size_t)(n_bins + 1) * 4));
    TQ_CUDA(cudaMemsetAsync(cnt.p, 0, (size_t)(n_bins + 1) * 4, s));
    std::vector<DevColBuf> &pc = j->part_cols[cursor_slot];
    pc.resize(j->n_probe_cols);
    ScatterParams sp{};
    sp.n_cols = j->n_probe_cols;
    sp.selected = d_selected;
    sp.key_col = j->probe_key;
    sp.key_mode = j->key_mode;
    sp.is_outer = p.is_outer;
    sp.pbits = j->table.pbits;
    sp.n = n;
    sp.part_cnt = cnt.as<uint32_t>();
    sp.part_cursor = cur_b.as<uint32_t>();
    // Optimistic slabs: every partition gets a fixed slab (slab_rows) and the histogram pass (a full extra read of the key
    // column) is skipped; the scatter flags a slab that would overflow and finalize_pending re-runs the batch on the exact path.
    const bool optimistic = j->optimistic_scatter;
    const uint64_t slab = slab_rows(n, P, false);
    const uint64_t part_rows = optimistic ? slab * P + (p.is_outer ? (uint64_t)n : 0) : (uint64_t)n;
    if (part_rows > 0xFFFFFFF0ull) { set_error("probe batch too large for 32-bit partition offsets"); return TQ_ERR_INVALID_ARG; }
    for (int c = 0; c < j->n_probe_cols; c++) {
      TQ_TRY(pc[c].data.reserve((size_t)part_rows * 8));
      sp.in[c] = probe[c];
      sp.out[c].data = pc[c].data.as<uint64_t>();
      sp.out[c].bm = nullptr;
      if (probe[c].bm) {
        TQ_TRY(pc[c].bm.reserve(bitmap_alloc_bytes((int64_t)part_rows)));
        TQ_CUDA(cudaMemsetAsync(pc[c].bm.p, 0, bitmap_alloc_bytes((int64_t)part_rows), s));
        sp.out[c].bm = pc[c].bm.as<uint32_t>();
      }
      p.probe[c].data = pc[c].data.as<uint64_t>();
      p.probe[c].bm = sp.out[c].bm;
    }
    const int smem_bins = n_bins * 4;
    if (optimistic) {
      DevBuf &lim = j->part_lim[cursor_slot];
      TQ_TRY(lim.reserve((size_t)(n_bins + 1) * 4));
      k_init_slabs<<<(n_bins + 255) / 256, 256, 0, s>>>(off.as<uint32_t>(), cur_b.as<uint32_t>(), lim.as<uint32_t>(), P, (uint32_t)slab, (uint32_t)n);
      count_launch();
      sp.part_lim = lim.as<uint32_t>();
      sp.overflow = cur + 2;
      p.part_lo = off.as<uint32_t>();
      p.part_hi = cur_b.as<uint32_t>();   // after the scatter: one past the last row written into each slab
      p.part_lim = lim.as<uint32_t>();
    } else {
      const int hist_grid = rt().sm_count * 4;
      k_probe_part_hist<<<hist_grid, SCAT_THREADS, smem_bins, s>>>(sp);
      count_launch();
      TQ_TRY(check_launch("k_probe_part_hist"));
      // off[q] = first row of partition q; the extra zero bin makes off[n_bins] the total
      TQ_TRY(exclusive_scan_u32(cnt.as<uint32_t>(), 1, off.as<uint32_t>(), 1, n_bins + 1, nullptr, j->scan_scratch2, s));
      TQ_CUDA(cudaMemcpyAsync(cur_b.p, off.p, (size_t)(n_bins + 1) * 4, cudaMemcpyDeviceToDevice, s));
      sp.part_lim = nullptr;
      sp.overflow = cur + 2;
      p.part_lo = off.as<uint32_t>();
      p.part_hi = off.as<uint32_t>() + 1;
      p.part_lim = nullptr;
    }
    if (!any_in_bm && !g_no_fast_kernel && j->n_probe_cols <= 4) {
      TQ_TRY(launch_scatter_fast(sp, s, "k_probe_scatter_fast"));
    } else {
      const int64_t scat_tiles = (n + SCAT_TILE - 1) / SCAT_TILE;
      const int64_t scat_cap = (int64_t)rt().sm_count * 4;
      k_probe_scatter<<<(int)(scat_tiles < scat_cap ? scat_tiles : scat_cap), SCAT_THREADS, scatter_smem_bytes(n_bins), s>>>(sp);
      count_launch();
      TQ_TRY(check_launch("k_probe_scatter"));
    }
    p.selected = nullptr;
    const int work_parts = p.is_outer ? n_bins : P;
    // ~g_tiles_per_cta tiles per CTA: enough CTAs per partition that only a handful of partitions are live at once
    const int64_t tiles_per_part = (n / work_parts + PROBE_TILE - 1) / PROBE_TILE;
    int64_t split64 = tiles_per_part / g_tiles_per_cta;
    if (split64 < 1) split64 = 1;
    if (split64 * work_parts > (1ll << 30)) split64 = (1ll << 30) / work_parts;
    int split = (int)split64;
    p.split = split;
    const size_t image_bytes = ((size_t)j->table.cap << j->shift) * 8;
    const bool in_smem = image_bytes <= PART_MAX_SMEM_BYTES;
    p.table_in_smem = in_smem ? 1 : 0;
    const size_t table_bytes = in_smem ? image_bytes : 0;
    bool any_out_bm = false;
    for (int c = 0; c < j->n_probe_cols; c++) any_out_bm |= (p.out_probe[c].bm != nullptr);
    for (int c = 0; c < j->n_build_cols; c++) any_out_bm |= (p.out_build[c].bm != nullptr);
    ProbeKernel fast = (j->row_mode && !p.is_outer && !any_out_bm && !g_no_fast_kernel) ? fast_kernel(j->n_probe_cols, j->n_build_cols) : nullptr;
    if (fast) {
      static bool fast_attr[5][5] = {};
      if (!fast_attr[j->n_probe_cols][j->n_build_cols]) {
        TQ_CUDA(cudaFuncSetAttribute(fast, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PART_MAX_SMEM_BYTES));
        fast_attr[j->n_probe_cols][j->n_build_cols] = true;
      }
      fast<<<work_parts * split, PROBE_THREADS, table_bytes, s>>>(p, j->table);
    } else if (j->build_unique) k_probe_part_uniq<<<work_parts * split, PROBE_THREADS, table_bytes, s>>>(p, j->table);
    else k_probe_part<<<work_parts * split, PROBE_THREADS, table_bytes, s>>>(p, j->table);
    count_launch();
    j->probe_launches += 3;
    TQ_TRY(check_launch("k_probe_part"));
  }
  TQ_CUDA(cudaEventRecord(j->ev_b[cursor_slot], s));
  TQ_CUDA(cudaMemcpyAsync(j->cursors_host.as<unsigned long long>() + 8 * cursor_slot, cur, 64, cudaMemcpyDeviceToHost, s));
  return TQ_OK;
}

static int32_t enqueue_d2h(tq_join *j, ResultBatch *rb) {
  Runtime &r = rt();
  const int ncols = (int)rb->cols.size();
  rb->h_data.resize(ncols);
  rb->h_bm.resize(ncols);
  if (!rb->ev_ready) TQ_CUDA(cudaEventCreateWithFlags(&rb->ev_ready, cudaEventDisableTiming));
  for (int c = 0; c < ncols; c++) {
    TQ_TRY(rb->h_data[c].reserve((size_t)(rb->n ? rb->n : 1) * 8));
    TQ_TRY(rb->h_bm[c].reserve(bitmap_alloc_bytes(rb->n)));
    const bool ind = c < (int)rb->var.size() && rb->var[c].used;
    if (rb->n) {
      if (!ind) TQ_CUDA(cudaMemcpyAsync(rb->h_data[c].p, rb->cols[c].data.p, (size_t)rb->n * 8, cudaMemcpyDeviceToHost, r.d2h));
      TQ_CUDA(cudaMemcpyAsync(rb->h_bm[c].p, rb->cols[c].bm.p, bitmap_bytes(rb->n), cudaMemcpyDeviceToHost, r.d2h));
    }
    if (ind) {
      VarOut &v = rb->var[c];
      TQ_TRY(v.h_bytes.reserve((size_t)v.total + 16));
      if (v.total) TQ_CUDA(cudaMemcpyAsync(v.h_bytes.p, v.bytes.p, (size_t)v.total, cudaMemcpyDeviceToHost, r.d2h));
      if (v.elem == 0) {
        TQ_TRY(v.h_off.reserve((size_t)(rb->n + 1) * 8));
        TQ_CUDA(cudaMemcpyAsync(v.h_off.p, v.off.p, (size_t)(rb->n + 1) * 8, cudaMemcpyDeviceToHost, r.d2h));
      }
      v.on_host = true;
    }
  }
  TQ_CUDA(cudaEventRecord(rb->ev_ready, r.d2h));
  rb->on_host = true;
  return TQ_OK;
}

// OtherConditions: filter the finished result batch in place (joiner.go:155-167; all-failed outer rows become miss rows).
static int32_t apply_other_conditions(tq_join *j, ResultBatch *rb, int64_t n_probe_rows) {
  const int ncols = j->n_build_cols + j->n_probe_cols;
  if (rb->n == 0) return TQ_OK;
  rb->alt.resize(ncols);
  OcCols oc_cols;
  oc_cols.n = ncols;
  for (int c = 0; c < ncols; c++) {
    TQ_TRY(rb->alt[c].data.reserve((size_t)rb->n * 8));
    TQ_TRY(rb->alt[c].bm.reserve(bitmap_alloc_bytes(rb->n)));
    oc_cols.data[c] = rb->cols[c].data.as<uint64_t>();
    oc_cols.bm[c] = rb->cols[c].bm.as<uint32_t>();
    oc_cols.out_data[c] = rb->alt[c].data.as<uint64_t>();
    oc_cols.out_bm[c] = rb->alt[c].bm.as<uint32_t>();
  }
  int64_t kept = 0, warnings = 0;
  TQ_TRY(oc_filter(j->oc, oc_cols, rb->n, n_probe_rows, j->oc_scratch, j->oc_scan, &kept, &rb->oc_err, &warnings, rt().compute));
  std::swap(rb->cols, rb->alt);
  rb->n = kept;
  j->oc_warnings += warnings;
  return TQ_OK;
}

// Wait for the pending batch, re-run it if the output did not fit, queue its result.
static int32_t finalize_pending(tq_join *j) {
  PendingBatch &pb = j->pending;
  if (!pb.active) return TQ_OK;
  Runtime &r = rt();
  TQ_CUDA(cudaEventSynchronize(pb.ev_k));
  unsigned long long *hc = j->cursors_host.as<unsigned long long>() + 8 * pb.cursor_slot;
  uint64_t produced = hc[0];
  float ms = 0;
  if (cudaEventElapsedTime(&ms, j->ev_a[pb.cursor_slot], j->ev_b[pb.cursor_slot]) == cudaSuccess) j->last_probe_ns = (int64_t)(ms * 1e6);
  else cudaGetLastError();
  if (hc[2]) {
    // a partition slab of the general path's optimistic (histogram-free) scatter was too small — skewed keys: exact offsets
    // from now on (the positional path counts exactly and never overflows)
    j->optimistic_scatter = false;
    TQ_TRY(launch_probe(j, pb.probe, pb.d_selected, pb.n, pb.rb.get(), pb.rb->capacity, pb.cursor_slot));
    TQ_CUDA(cudaStreamSynchronize(r.compute));
    produced = hc[0];
  }
  if (hc[4]) { set_error("internal: a page of the positional result was never handed out"); return TQ_ERR_CUDA; }
  if (hc[3] && hc[6] != hc[0]) TQ_TRY(fill_holes_host(j, pb.rb.get(), pb.cursor_slot, hc[0], hc[3]));  // positional result with misses among the probe rows
  if (produced > pb.rb->capacity) {
    // duplicate build keys: the first launch served as the count pass; run again with the exact size
    TQ_TRY(launch_probe(j, pb.probe, pb.d_selected, pb.n, pb.rb.get(), produced, pb.cursor_slot));
    TQ_CUDA(cudaStreamSynchronize(r.compute));
    produced = hc[0];
    if (produced > pb.rb->capacity) { set_error("join output size changed between passes"); return TQ_ERR_CUDA; }
    if (cudaEventElapsedTime(&ms, j->ev_a[pb.cursor_slot], j->ev_b[pb.cursor_slot]) == cudaSuccess) j->last_probe_ns = (int64_t)(ms * 1e6);
  }
  pb.rb->n = (int64_t)produced;
  pb.rb->oc_err = 0;
  if (j->has_oc) TQ_TRY(apply_other_conditions(j, pb.rb.get(), pb.n));
  j->joined_rows_total += pb.rb->n;
  if (j->any_ind) TQ_TRY(materialize_indirect(j, pb.rb.get(), pb.cursor_slot));  // synchronises the compute stream
  if (pb.want_host) {
    TQ_CUDA(cudaStreamWaitEvent(r.d2h, pb.ev_k, 0));
    TQ_TRY(enqueue_d2h(j, pb.rb.get()));
  }
  j->results.push_back(std::move(pb.rb));
  pb.active = false;
  return TQ_OK;
}

// Start a probe batch on device columns in cursor/input slot `slot`; the PREVIOUS batch (other slot) is
// finalised after this one is enqueued, so the host-side wait overlaps GPU work.
static int32_t start_batch(tq_join *j, const std::vector<DCol> &probe, const uint8_t *d_selected, int64_t n, bool want_host, int slot) {
  if (n == 0) return TQ_OK;
  Runtime &r = rt();
  if (j->pending.active && j->pending.cursor_slot == slot) TQ_TRY(finalize_pending(j));
  std::vector<DCol> encoded;
  const std::vector<DCol> *pin = &probe;
  if (j->key_hidden && j->n_keys == 1) {
    DCol kc;
    const std::vector<SideStore> &st = j->in_set[slot].store;
    TQ_TRY(key_source(j, false, 0, probe, st.empty() ? nullptr : st.data(), n, j->kx_p_data[slot][0], j->kx_p_bm[slot][0], &kc, r.compute));
    encoded = probe;
    encoded[j->np_user] = kc;
    pin = &encoded;
  } else if (j->key_hidden) {
    // probe-side key tuples -> the hidden key column (lookup only: a value the build side never had is a miss)
    DCol kc[MK_MAX_KEYS];
    const std::vector<SideStore> &st = j->in_set[slot].store;
    for (int i = 0; i < j->n_keys; i++)
      TQ_TRY(key_source(j, false, i, probe, st.empty() ? nullptr : st.data(), n, j->kx_p_data[slot][i], j->kx_p_bm[slot][i], &kc[i], r.compute));
    TQ_TRY(j->mk_probe_key[slot].reserve((size_t)n * 8));
    TQ_TRY(j->mk_probe_bm[slot].reserve(bitmap_alloc_bytes(n)));
    TQ_TRY(j->mk.encode(kc, j->mk_no_signbit, n, /*insert=*/false, /*null_is_value=*/false, j->mk_probe_key[slot].as<uint64_t>(),
                        j->mk_probe_bm[slot].as<uint32_t>(), r.compute));
    encoded = probe;
    encoded[j->np_user].data = j->mk_probe_key[slot].as<uint64_t>();
    encoded[j->np_user].bm = j->mk_probe_bm[slot].as<uint32_t>();
    pin = &encoded;
  }
  if (j->p_hidden_rowid >= 0) {
    // OtherConditions on an outer join: every joined row has to know which probe row it came from
    if (pin == &probe) { encoded = probe; pin = &encoded; }
    TQ_TRY(j->oc_rowid[slot].reserve((size_t)n * 8));
    TQ_TRY(iota_u64(j->oc_rowid[slot].as<uint64_t>(), n, r.compute));
    encoded[j->p_hidden_rowid].data = j->oc_rowid[slot].as<uint64_t>();
    encoded[j->p_hidden_rowid].bm = nullptr;
  }
  // a join on unique build keys produces at most one row per probe row; with duplicate keys the
  // first launch doubles as the count pass (finalize_pending re-runs with the exact size)
  const uint64_t capacity = (uint64_t)n;
  std::unique_ptr<ResultBatch> rb = get_result_batch(j);
  TQ_TRY(launch_probe(j, *pin, d_selected, n, rb.get(), capacity, slot));
  j->seg.n = 0;  // consumed by this launch: a re-run of the previous batch in finalize_pending must not read these regions
  cudaEvent_t ev = nullptr;
  TQ_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  TQ_CUDA(cudaEventRecord(ev, r.compute));
  TQ_TRY(finalize_pending(j));
  PendingBatch &pb = j->pending;
  if (pb.ev_k) cudaEventDestroy(pb.ev_k);
  pb.ev_k = ev;
  pb.active = true;
  pb.rb = std::move(rb);
  pb.probe = *pin;
  pb.d_selected = d_selected;
  pb.n = n;
  pb.want_host = want_host;
  pb.cursor_slot = slot;
  j->probe_rows_total += n;
  return TQ_OK;
}

// ---- key-less join (n_keys == 0) -------------------------------------------------------------------------------------------
// A probe batch produces no rows when it arrives: it becomes a pair cursor (KlProbe) that owns its rows, and result batches of
// at most batch_rows rows are built from it when a tq_join_next* call needs rows.  Memory does not depend on |probe| x |build|:
// a sub-range's survivor bits are bounded by KL_MASK_WORDS (or one probe row's words), its counts by the batch's rows.
static constexpr int64_t KL_MASK_WORDS = 1 << 23;   // survivor words of one sub-range: 32 MB, 2^28 pairs

// Takes the probe rows of `in` (its buffers move into the cursor; `in` gets empty ones) as a new pair cursor.
static void kl_take(tq_join *j, ProbeInputSet &in, const std::vector<DCol> &view, const uint8_t *d_sel, int64_t n) {
  std::unique_ptr<KlProbe> k(new KlProbe());
  std::swap(k->in.cols, in.cols);
  std::swap(k->in.store, in.store);
  std::swap(k->in.selected, in.selected);
  k->view = view;
  k->d_sel = d_sel;
  k->n = n;
  j->kl.push_back(std::move(k));
  j->probe_rows_total += n;
}

// A device chunk: copied (D2D; var-len cells into the cursor's own store) so the cursor does not depend on the caller's buffers.
static int32_t kl_put_device(tq_join *j, const tq_column *cols, const uint8_t *selected, int64_t rows) {
  cudaStream_t s = rt().compute;
  ProbeInputSet in;
  in.cols.resize(j->n_probe_cols);
  if (j->any_ind) in.store.resize(j->np_user);
  std::vector<DCol> view(j->n_probe_cols);
  for (int c = 0; c < j->np_user; c++) {
    DevColBuf &d = in.cols[c];
    TQ_TRY(d.data.reserve((size_t)rows * 8));
    if (j->p_ind[c]) {   // (FLOAT columns were refused): row ids into the store
      int64_t longest = 0;
      TQ_TRY(append_cells_device(in.store[c], cols[c].offsets, cols[c].data, rows, &longest, j->var_meta, s));
      TQ_TRY(iota_u64(d.data.as<uint64_t>(), rows, s));
    } else {
      TQ_CUDA(cudaMemcpyAsync(d.data.p, cols[c].data, (size_t)rows * 8, cudaMemcpyDeviceToDevice, s));
    }
    view[c].data = d.data.as<uint64_t>();
    if (cols[c].null_bitmap) {
      TQ_TRY(d.bm.reserve(bitmap_alloc_bytes(rows)));
      TQ_CUDA(cudaMemcpyAsync(d.bm.p, cols[c].null_bitmap, bitmap_bytes(rows), cudaMemcpyDeviceToDevice, s));
      view[c].bm = d.bm.as<uint32_t>();
    }
  }
  const uint8_t *d_sel = nullptr;
  if (selected) {   // host memory by contract
    TQ_TRY(in.selected.reserve((size_t)rows));
    TQ_CUDA(cudaMemcpyAsync(in.selected.p, selected, (size_t)rows, cudaMemcpyHostToDevice, s));
    d_sel = in.selected.as<uint8_t>();
  }
  TQ_CUDA(cudaStreamSynchronize(s));   // the caller's columns are not read after the call
  kl_take(j, in, view, d_sel, rows);
  return TQ_OK;
}

// Opens the next sub-range of cursor k: survivor bits (conditions only), per-row counts, their 64-bit scan.  *err = the ops
// that raised on a pair of the sub-range's evaluation set.
static int32_t kl_open_subrange(tq_join *j, KlProbe &k, unsigned *err) {
  cudaStream_t s = rt().compute;
  const uint32_t B = (uint32_t)j->n_build;
  const uint32_t W = (j->has_oc && B) ? (B + 31) / 32 : 0;
  int64_t rows = k.n - k.next_row;
  if (W) {
    const int64_t fit = KL_MASK_WORDS / W;
    if (rows > fit) rows = fit < 1 ? 1 : fit;
  }
  k.r0 = k.next_row;
  k.rows = rows;
  TQ_TRY(j->kl_cnt.reserve((size_t)rows * 8));
  TQ_TRY(j->kl_off.reserve((size_t)(rows + 1) * 8));
  TQ_TRY(j->kl_miss.reserve((size_t)rows));
  TQ_TRY(j->kl_meta.reserve(16));
  TQ_TRY(j->kl_back.reserve(32));
  TQ_CUDA(cudaMemsetAsync(j->kl_meta.p, 0, 16, s));
  if (W) {
    TQ_TRY(j->kl_mask.reserve((size_t)rows * W * 4));
    TQ_TRY(j->kl_wpre.reserve((size_t)rows * W * 4));
    NljEvalParams e;
    e.prog = j->oc.prog;
    const int bbase = j->outer_is_right ? 0 : j->n_probe_cols, pbase = j->outer_is_right ? j->n_build_cols : 0;
    for (int q = 0; q < e.prog.n_in; q++) {
      const int ic = j->oc.prog.in_col[q];
      const bool build = ic >= bbase && ic < bbase + j->n_build_cols;
      e.in_build[q] = build ? 1 : 0;
      e.in[q] = build ? j->b_view[ic - bbase] : k.view[ic - pbase];
    }
    e.selected = k.d_sel;
    e.r0 = k.r0;
    e.rows = rows;
    e.n_build = B;
    e.words = W;
    e.mask = j->kl_mask.as<uint32_t>();
    e.err = reinterpret_cast<unsigned *>(j->kl_meta.as<uint64_t>() + 1);
    e.warn = j->kl_meta.as<unsigned long long>();
    TQ_TRY(nlj_eval(e, s));
  }
  NljCountParams c;
  c.selected = k.d_sel;
  c.r0 = k.r0;
  c.rows = rows;
  c.n_build = B;
  c.words = W;
  c.mask = W ? j->kl_mask.as<uint32_t>() : nullptr;
  c.wpre = W ? j->kl_wpre.as<uint32_t>() : nullptr;
  c.outer = j->join_type != TQ_JOIN_INNER;
  c.cnt = j->kl_cnt.as<uint64_t>();
  c.miss = j->kl_miss.as<uint8_t>();
  TQ_TRY(nlj_count(c, s));
  TQ_TRY(nlj_scan_u64(j->kl_cnt.as<uint64_t>(), j->kl_off.as<uint64_t>(), rows, j->kl_scan, s));
  uint64_t *back = j->kl_back.as<uint64_t>();
  TQ_CUDA(cudaMemcpyAsync(back, j->kl_off.as<uint64_t>() + rows, 8, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaMemcpyAsync(back + 1, j->kl_meta.p, 16, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  k.sub_total = back[0];
  k.sub_pos = 0;
  k.sub_open = true;
  j->oc_warnings += (int64_t)back[1];
  *err = (unsigned)back[2];
  return TQ_OK;
}

// Builds the next result batch of the key-less join and queues it; queues nothing when every cursor is drained.  A sub-range
// whose pairs raised queues a batch that carries only the error: the call that takes it up returns the status, as on the keyed
// path (DESIGN.md §3).
static int32_t kl_produce(tq_join *j) {
  Runtime &r = rt();
  cudaStream_t s = r.compute;
  while (!j->kl.empty()) {
    KlProbe &k = *j->kl.front();
    if (!k.sub_open) {
      if (k.next_row >= k.n) {
        TQ_CUDA(cudaStreamSynchronize(s));   // the last batch's kernels read the cursor's buffers
        j->kl.pop_front();
        continue;
      }
      unsigned err = 0;
      TQ_TRY(kl_open_subrange(j, k, &err));
      if (err) {
        std::unique_ptr<ResultBatch> rb = get_result_batch(j);
        rb->oc_err = err;
        if (!rb->ev_ready) TQ_CUDA(cudaEventCreateWithFlags(&rb->ev_ready, cudaEventDisableTiming));
        TQ_CUDA(cudaEventRecord(rb->ev_ready, s));
        j->results.push_back(std::move(rb));
        j->kl.clear();
        return TQ_OK;
      }
    }
    if (k.sub_pos == k.sub_total) {
      k.sub_open = false;
      k.next_row = k.r0 + k.rows;
      continue;
    }
    const uint64_t left = k.sub_total - k.sub_pos;
    const int64_t len = left < (uint64_t)j->batch_rows ? (int64_t)left : j->batch_rows;
    std::unique_ptr<ResultBatch> rb = get_result_batch(j);
    const int ncols = j->n_build_cols + j->n_probe_cols;
    const int build_base = j->outer_is_right ? 0 : j->n_probe_cols, probe_base = j->outer_is_right ? j->n_build_cols : 0;
    rb->cols.resize(ncols);
    rb->capacity = (uint64_t)len;
    for (int c = 0; c < ncols; c++) {
      TQ_TRY(rb->cols[c].data.reserve((size_t)len * 8));
      TQ_TRY(rb->cols[c].bm.reserve(bitmap_alloc_bytes(len)));
    }
    NljOutParams o;
    o.n_probe_cols = j->n_probe_cols;
    o.n_build_cols = j->n_build_cols;
    for (int c = 0; c < j->n_probe_cols; c++) {
      o.probe[c] = k.view[c];
      o.out_probe[c].data = rb->cols[probe_base + c].data.as<uint64_t>();
      o.out_probe[c].bm = rb->cols[probe_base + c].bm.as<uint32_t>();
    }
    for (int c = 0; c < j->n_build_cols; c++) {
      o.build[c] = j->b_view[c];
      o.out_build[c].data = rb->cols[build_base + c].data.as<uint64_t>();
      o.out_build[c].bm = rb->cols[build_base + c].bm.as<uint32_t>();
      o.def_val[c] = j->def_val[c];
    }
    o.def_mask = j->def_mask;
    o.off = j->kl_off.as<uint64_t>();
    o.miss = j->kl_miss.as<uint8_t>();
    const bool masked = j->has_oc && j->n_build;
    o.mask = masked ? j->kl_mask.as<uint32_t>() : nullptr;
    o.wpre = masked ? j->kl_wpre.as<uint32_t>() : nullptr;
    o.words = masked ? (uint32_t)((j->n_build + 31) / 32) : 0;
    o.r0 = k.r0;
    o.rows = k.rows;
    o.q0 = k.sub_pos;
    o.len = len;
    TQ_CUDA(cudaEventRecord(j->ev_a[0], s));
    TQ_TRY(nlj_materialize(o, s));
    TQ_CUDA(cudaEventRecord(j->ev_b[0], s));
    j->kl_timed = true;
    j->probe_launches++;
    rb->n = len;
    rb->oc_err = 0;
    if (j->any_ind) TQ_TRY(materialize_indirect(j, rb.get(), k.in.store));   // synchronises the compute stream
    if (!rb->ev_ready) TQ_CUDA(cudaEventCreateWithFlags(&rb->ev_ready, cudaEventDisableTiming));
    TQ_CUDA(cudaEventRecord(rb->ev_ready, s));   // the batch is complete: its D2H waits for this, next_device syncs on it
    k.sub_pos += (uint64_t)len;
    j->joined_rows_total += len;
    j->results.push_back(std::move(rb));
    return TQ_OK;
  }
  return TQ_OK;
}

// Ship one piece of host rows to the device (double-buffered input sets) and start its probe.
static int32_t process_host_piece(tq_join *j, const tq_column *cols, int64_t row0, int64_t rows, const uint8_t *selected, bool eager_d2h = true) {
  Runtime &r = rt();
  const int slot = j->in_flip;
  j->in_flip ^= 1;
  // the batch that last read this input set must be complete before the set is overwritten
  if (j->pending.active && j->pending.cursor_slot == slot) TQ_TRY(finalize_pending(j));
  ProbeInputSet &in = j->in_set[slot];
  if (!in.ev_h2d) TQ_CUDA(cudaEventCreateWithFlags(&in.ev_h2d, cudaEventDisableTiming));
  in.cols.resize(j->n_probe_cols);
  std::vector<DCol> view(j->n_probe_cols);
  if ((row0 & 7) != 0) { set_error("internal: unaligned host piece"); return TQ_ERR_INVALID_ARG; }
  if (j->any_ind) in.store.resize(j->np_user);
  for (int c = 0; c < j->np_user; c++) {
    TQ_TRY(in.cols[c].data.reserve((size_t)rows * 8));
    if (j->p_ind[c]) {
      // the cells go to this batch's side store; the join sees row ids 0..rows-1 (+ the column's NULL bitmap)
      SideStore &st = in.store[c];
      st.elem = j->p_elem[c];
      st.n = rows;
      if (st.elem == 4) {
        st.base = 0;
        TQ_TRY(st.bytes.reserve((size_t)rows * 4 + 16));
        TQ_CUDA(cudaMemcpyAsync(st.bytes.p, cols[c].data + row0 * 4, (size_t)rows * 4, cudaMemcpyHostToDevice, r.h2d));
      } else {
        const int64_t b0 = cols[c].offsets[row0], b1 = cols[c].offsets[row0 + rows];
        st.base = b0;
        st.nbytes = b1 - b0;
        TQ_TRY(st.offsets.reserve((size_t)(rows + 1) * 8));
        TQ_TRY(st.bytes.reserve((size_t)(b1 - b0) + 16));
        TQ_CUDA(cudaMemcpyAsync(st.offsets.p, cols[c].offsets + row0, (size_t)(rows + 1) * 8, cudaMemcpyHostToDevice, r.h2d));
        if (b1 > b0) TQ_CUDA(cudaMemcpyAsync(st.bytes.p, cols[c].data + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, r.h2d));
      }
      TQ_TRY(iota_u64(in.cols[c].data.as<uint64_t>(), rows, r.compute));
    } else {
      TQ_CUDA(cudaMemcpyAsync(in.cols[c].data.p, cols[c].data + row0 * 8, (size_t)rows * 8, cudaMemcpyHostToDevice, r.h2d));
    }
    view[c].data = in.cols[c].data.as<uint64_t>();
    view[c].bm = nullptr;
    if (cols[c].null_bitmap) {
      TQ_TRY(in.cols[c].bm.reserve(bitmap_alloc_bytes(rows)));
      TQ_CUDA(cudaMemcpyAsync(in.cols[c].bm.p, cols[c].null_bitmap + (row0 >> 3), bitmap_bytes(rows), cudaMemcpyHostToDevice, r.h2d));
      view[c].bm = in.cols[c].bm.as<uint32_t>();
    }
  }
  const uint8_t *d_sel = nullptr;
  if (selected) {
    TQ_TRY(in.selected.reserve((size_t)rows));
    TQ_TRY(j->p_sel_pin[slot].reserve((size_t)rows));
    memcpy(j->p_sel_pin[slot].p, selected + row0, (size_t)rows);
    TQ_CUDA(cudaMemcpyAsync(in.selected.p, j->p_sel_pin[slot].p, (size_t)rows, cudaMemcpyHostToDevice, r.h2d));
    d_sel = in.selected.as<uint8_t>();
  }
  TQ_CUDA(cudaEventRecord(in.ev_h2d, r.h2d));
  TQ_CUDA(cudaStreamWaitEvent(r.compute, in.ev_h2d, 0));
  if (j->keyless) {
    // the rows become a pair cursor, which takes this input set's buffers: the slot is free again at once.  (p_sel_pin[slot]
    // is refilled by the next piece of this slot, so its upload has to be complete.)
    TQ_CUDA(cudaStreamSynchronize(r.h2d));
    kl_take(j, in, view, d_sel, rows);
    return TQ_OK;
  }
  return start_batch(j, view, d_sel, rows, /*want_host=*/eager_d2h, slot);
}

static int32_t flush_probe_staging(tq_join *j) {
  if (j->p_host.empty() || j->p_host[0].n == 0) return TQ_OK;
  const int64_t rows = j->p_host[0].n;
  std::vector<tq_column> cols(j->np_user);
  for (int c = 0; c < j->np_user; c++) {
    cols[c].length = rows;
    cols[c].data = j->p_host[c].data.as<uint8_t>();
    cols[c].null_bitmap = j->p_host[c].has_bm ? j->p_host[c].bm.as<uint8_t>() : nullptr;
    cols[c].offsets = nullptr;
    if (j->p_ind[c]) {
      cols[c].data = j->p_var[c].bytes.data();
      cols[c].offsets = j->p_elem[c] == 0 ? j->p_var[c].off.data() : nullptr;
    }
  }
  const uint8_t *sel = j->p_sel_any ? j->p_sel_host.data() : nullptr;
  // The staging buffers are reused right after this call, so the H2D copies must have completed.
  int32_t st = process_host_piece(j, cols.data(), 0, rows, sel);
  if (st == TQ_OK) {
    cudaError_t e = cudaStreamSynchronize(rt().h2d);
    if (e != cudaSuccess) st = cuda_fail(e, "sync h2d", __FILE__, __LINE__);
  }
  for (auto &h : j->p_host) h.reset();
  for (int c = 0; c < j->np_user; c++) j->p_var[c].reset();
  j->p_sel_host.clear();
  j->p_sel_any = false;
  return st;
}

static void recycle(tq_join *j, std::unique_ptr<ResultBatch> rb) {
  if (rb) j->free_list.push_back(std::move(rb));
}

}  // namespace tq

extern "C" {

int32_t tq_join_create(const tq_join_desc *d, tq_join **out) {
  if (!d || !out) return TQ_ERR_INVALID_ARG;
  *out = nullptr;
  TQ_TRY(ensure_init());
  if (d->join_type < TQ_JOIN_INNER || d->join_type > TQ_JOIN_RIGHT_OUTER) { set_error("unsupported join type %d", d->join_type); return TQ_ERR_INVALID_ARG; }
  if (d->n_build_cols < 1 || d->n_build_cols > MAXC || d->n_probe_cols < 1 || d->n_probe_cols > MAXC) {
    set_error("join sides must have 1..%d columns", MAXC);
    return TQ_ERR_INVALID_ARG;
  }
  if (d->n_keys < 0 || d->n_keys > MK_MAX_KEYS) { set_error("hash join on %d key columns: 0..%d are supported", d->n_keys, MK_MAX_KEYS); return TQ_ERR_INVALID_ARG; }
  for (int i = 0; i < d->n_keys; i++)
    if (d->build_key_idx[i] < 0 || d->build_key_idx[i] >= d->n_build_cols || d->probe_key_idx[i] < 0 || d->probe_key_idx[i] >= d->n_probe_cols) return TQ_ERR_INVALID_ARG;
  // a hidden key column per side: several key columns, or a FLOAT / var-len key (compared as float64 / byte string)
  int hidden = d->n_keys > 1 ? 1 : 0;
  for (int i = 0; i < d->n_keys; i++)
    if (type_indirect(d->build_types[d->build_key_idx[i]]) || type_indirect(d->probe_types[d->probe_key_idx[i]])) hidden = 1;
  if (d->n_build_cols + hidden > MAXC || d->n_probe_cols + hidden > MAXC) { set_error("multi-column / FLOAT / var-len join keys need one spare column per side"); return TQ_ERR_INVALID_ARG; }
  for (int c = 0; c < d->n_build_cols; c++)
    if (!type_ok(d->build_types[c]) && !type_indirect(d->build_types[c])) { set_error("unsupport column type for encode %d", d->build_types[c]); return TQ_ERR_UNSUPPORTED_TYPE; }
  for (int c = 0; c < d->n_probe_cols; c++)
    if (!type_ok(d->probe_types[c]) && !type_indirect(d->probe_types[c])) { set_error("unsupport column type for encode %d", d->probe_types[c]); return TQ_ERR_UNSUPPORTED_TYPE; }
  // LeftOuter keeps the left child as the outer side, RightOuter the right child (builder.go:451-477)
  if (d->join_type == TQ_JOIN_LEFT_OUTER && d->outer_is_right) { set_error("left outer join needs outer_is_right == 0"); return TQ_ERR_INVALID_ARG; }
  if (d->join_type == TQ_JOIN_RIGHT_OUTER && !d->outer_is_right) { set_error("right outer join needs outer_is_right == 1"); return TQ_ERR_INVALID_ARG; }
  { const char *e = getenv("TQ_JOIN_NO_FAST"); g_no_fast_kernel = e && e[0] == '1'; }
  tq_join *j = new (std::nothrow) tq_join();
  if (!j) return TQ_ERR_OOM;
  // per handle: unset or not a positive number means the default, whatever an earlier handle was created with
  { const char *e = getenv("TQ_JOIN_PART_ROWS"); if (e && atoll(e) > 0) j->part_rows = atoll(e); }
  j->join_type = d->join_type;
  j->outer_is_right = d->outer_is_right ? 1 : 0;
  j->nb_user = d->n_build_cols;
  j->np_user = d->n_probe_cols;
  j->n_build_cols = d->n_build_cols + hidden;
  j->n_probe_cols = d->n_probe_cols + hidden;
  j->n_keys = d->n_keys;
  j->flags = d->flags;
  for (int c = 0; c < d->n_build_cols; c++) j->build_types[c] = d->build_types[c];
  for (int c = 0; c < d->n_probe_cols; c++) j->probe_types[c] = d->probe_types[c];
  // key comparison across types (codec.go:219-231,363-382): a DOUBLE never equals an integer key; signed vs unsigned
  // integers are equal only when both are below 2^63
  // flags: varintFlag / uvarintFlag for the integer types, floatFlag for FLOAT and DOUBLE (a FLOAT is hashed and compared as
  // float64(f): float32(1) == float64(1), codec_test.go:735-769), compactBytesFlag for the var-len types
  auto class_of = [](int t) { return (t == TQ_TYPE_FLOAT64 || t == TQ_TYPE_FLOAT32) ? 1 : (t == TQ_TYPE_BYTES ? 2 : 0); };
  auto mode_of = [&](int bt, int pt) {
    if (class_of(bt) != class_of(pt)) return (int)KEYMODE_NEVER;
    if (class_of(bt) == 0 && bt != pt) return (int)KEYMODE_NO_SIGNBIT;
    return (int)KEYMODE_RAW;
  };
  auto kind_of = [](int t) { return t == TQ_TYPE_FLOAT32 ? 1 : (t == TQ_TYPE_BYTES ? 2 : 0); };
  j->key_hidden = hidden != 0;
  if (d->n_keys == 0) {
    // key-less join (nlj.cuh): every build row is a candidate of every selected probe row; no key columns, no table
    j->keyless = true;
    j->build_key = j->probe_key = 0;
    j->key_mode = KEYMODE_RAW;
  } else if (!hidden) {
    j->build_key = d->build_key_idx[0];
    j->probe_key = d->probe_key_idx[0];
    j->key_mode = mode_of(j->build_types[j->build_key], j->probe_types[j->probe_key]);
  } else {
    j->build_key = j->nb_user;
    j->probe_key = j->np_user;
    j->build_types[j->nb_user] = TQ_TYPE_UINT64;
    j->probe_types[j->np_user] = TQ_TYPE_UINT64;
    j->key_mode = KEYMODE_RAW;
    j->mk.k = d->n_keys;
    for (int i = 0; i < d->n_keys; i++) {
      j->bkeys[i] = d->build_key_idx[i];
      j->pkeys[i] = d->probe_key_idx[i];
      j->bkey_kind[i] = kind_of(j->build_types[j->bkeys[i]]);
      j->pkey_kind[i] = kind_of(j->probe_types[j->pkeys[i]]);
      const int m = mode_of(j->build_types[j->bkeys[i]], j->probe_types[j->pkeys[i]]);
      if (m == KEYMODE_NEVER) j->key_mode = KEYMODE_NEVER;
      j->mk_no_signbit[i] = (m == KEYMODE_NO_SIGNBIT);
    }
    // one key column: the hidden column IS that column's 8-byte form, so the signed/unsigned rule stays with the kernels
    if (d->n_keys == 1 && j->key_mode != KEYMODE_NEVER && j->mk_no_signbit[0]) j->key_mode = KEYMODE_NO_SIGNBIT;
  }
  {
    const int bbase = j->outer_is_right ? 0 : j->n_probe_cols, pbase = j->outer_is_right ? j->n_build_cols : 0;
    for (int c = 0; c < j->nb_user; c++)
      if (type_indirect(j->build_types[c])) {
        j->b_ind[c] = j->any_ind = true;
        j->b_elem[c] = j->b_var[c].elem = (j->build_types[c] == TQ_TYPE_FLOAT32) ? 4 : 0;
        j->out_side[bbase + c] = 1;
        j->out_col[bbase + c] = c;
      }
    for (int c = 0; c < j->np_user; c++)
      if (type_indirect(j->probe_types[c])) {
        j->p_ind[c] = j->any_ind = true;
        j->p_elem[c] = j->p_var[c].elem = (j->probe_types[c] == TQ_TYPE_FLOAT32) ? 4 : 0;
        j->out_side[pbase + c] = 2;
        j->out_col[pbase + c] = c;
      }
  }
  {
    const int first_user = j->outer_is_right ? j->nb_user : j->np_user, first_int = j->outer_is_right ? j->n_build_cols : j->n_probe_cols;
    for (int u = 0; u < j->nb_user + j->np_user; u++) j->out_map.push_back(u < first_user ? u : u - first_user + first_int);
  }
  if (d->default_inner_not_null) {
    // defaultInner of an outer join (joiner.go:139-143; set by the aggregation push-down, rule_aggregation_push_down.go:211-214)
    if (d->join_type == TQ_JOIN_INNER) { set_error("default_inner is only meaningful for outer joins"); delete j; return TQ_ERR_INVALID_ARG; }
    for (int c = 0; c < j->nb_user; c++) {
      if (!d->default_inner_not_null[c]) continue;
      if (!type_ok(j->build_types[c]) || !d->default_inner_bits) { set_error("default_inner: non-NULL defaults are supported for the 8-byte column types"); delete j; return TQ_ERR_UNSUPPORTED_TYPE; }
      j->def_val[c] = d->default_inner_bits[c];
      j->def_mask |= 1u << c;
    }
  }
  if (d->probe_batch_rows > 0) j->batch_rows = (d->probe_batch_rows + 63) & ~63ll;
  j->b_host.resize(j->nb_user);
  j->p_host.resize(j->np_user);
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < 2 && e == cudaSuccess; i++) {
    e = cudaEventCreate(&j->ev_a[i]);
    if (e == cudaSuccess) e = cudaEventCreate(&j->ev_b[i]);
  }
  if (e != cudaSuccess) { delete j; return cuda_fail(e, "cudaEventCreate", __FILE__, __LINE__); }
  int32_t st = j->cursors.reserve(128);
  if (st == TQ_OK) st = j->cursors_host.reserve(128);
  if (st != TQ_OK) { delete j; return st; }
  *out = j;
  return TQ_OK;
}

}  // extern "C"

// user output column (lhs ++ rhs) -> (build side?, column of that side)
static void join_user_col(const tq_join *j, int u, bool *is_build, int *col) {
  const int first_user = j->outer_is_right ? j->nb_user : j->np_user;
  const bool first = u < first_user;
  *is_build = j->outer_is_right ? first : !first;
  *col = first ? u : u - first_user;
}
static int join_user_type(const tq_join *j, int u) {
  bool is_build; int col;
  join_user_col(j, u, &is_build, &col);
  return is_build ? j->build_types[col] : j->probe_types[col];
}

static int32_t join_oc_settable(const tq_join *j) {
  if (j->state != tq_join::BUILDING || j->n_build != 0 || j->has_oc) { set_error("OtherConditions must be set once, right after tq_join_create"); return TQ_ERR_STATE; }
  return TQ_OK;
}

// Installs the OtherConditions program of either setter.  prog's input registers name user output columns.  An outer join
// gets the hidden probe row-id column (last on the probe side), which moves the result-batch layout.
static int32_t join_set_oc(tq_join *j, const JoinProg &prog, bool cmp_list) {
  const bool outer = j->join_type != TQ_JOIN_INNER;
  if (outer && !j->keyless && j->n_probe_cols + 1 > MAXC) { set_error("OtherConditions on an outer join need one spare probe column"); return TQ_ERR_INVALID_ARG; }
  const int n_user = j->nb_user + j->np_user;
  if (outer && !j->keyless) {   // (the key-less path knows each pair's probe row without a column)
    j->p_hidden_rowid = j->n_probe_cols;
    j->probe_types[j->n_probe_cols] = TQ_TYPE_INT64;
    j->n_probe_cols++;
    // the result-batch layout moved: recompute the caller -> batch column map and the indirect-column table
    const int bbase = j->outer_is_right ? 0 : j->n_probe_cols, pbase = j->outer_is_right ? j->n_build_cols : 0;
    for (int c = 0; c < 2 * MAXC; c++) { j->out_side[c] = 0; j->out_col[c] = 0; }
    for (int c = 0; c < j->nb_user; c++) if (j->b_ind[c]) { j->out_side[bbase + c] = 1; j->out_col[bbase + c] = c; }
    for (int c = 0; c < j->np_user; c++) if (j->p_ind[c]) { j->out_side[pbase + c] = 2; j->out_col[pbase + c] = c; }
    const int first_user = j->outer_is_right ? j->nb_user : j->np_user, first_int = j->outer_is_right ? j->n_build_cols : j->n_probe_cols;
    j->out_map.clear();
    for (int u = 0; u < n_user; u++) j->out_map.push_back(u < first_user ? u : u - first_user + first_int);
  }
  const int bbase = j->outer_is_right ? 0 : j->n_probe_cols, pbase = j->outer_is_right ? j->n_build_cols : 0;
  j->oc = OcPlan();
  j->oc.prog = prog;
  j->oc.cmp_list = cmp_list ? 1 : 0;
  for (int k = 0; k < prog.n_in; k++) j->oc.prog.in_col[k] = j->out_map[prog.in_col[k]];
  j->oc.outer = outer ? 1 : 0;
  j->oc.build_key_col = bbase + j->build_key;
  j->oc.rowid_col = outer ? pbase + j->p_hidden_rowid : -1;
  j->oc.build_lo = bbase;
  j->oc.build_hi = bbase + j->n_build_cols;
  for (int c = 0; c < j->n_build_cols; c++) j->oc.def_val[c] = j->def_val[c];
  j->oc.def_mask = j->def_mask;
  j->has_oc = true;
  return TQ_OK;
}

extern "C" {

int32_t tq_join_set_other_conditions(tq_join *j, int32_t n_conds, const tq_join_cond *conds) {
  if (!j || n_conds < 0 || n_conds > JP_MAX_CONDS || (n_conds && !conds)) { set_error("OtherConditions: 0..%d conditions", JP_MAX_CONDS); return TQ_ERR_INVALID_ARG; }
  TQ_TRY(join_oc_settable(j));
  if (n_conds == 0) return TQ_OK;
  const int n_user = j->nb_user + j->np_user;
  for (int k = 0; k < n_conds; k++) {
    const tq_join_cond &q = conds[k];
    if (q.op < TQ_CMP_LT || q.op > TQ_CMP_NE || q.lhs_col < 0 || q.lhs_col >= n_user || q.rhs_col >= n_user) { set_error("OtherConditions: bad condition %d", k); return TQ_ERR_INVALID_ARG; }
    const int ta = join_user_type(j, q.lhs_col), tb = q.rhs_col >= 0 ? join_user_type(j, q.rhs_col) : q.const_type;
    const bool fa = ta == TQ_TYPE_FLOAT64, fb = tb == TQ_TYPE_FLOAT64;
    if (!type_ok(ta) || !type_ok(tb) || fa != fb) { set_error("OtherConditions compare BIGINT with BIGINT or DOUBLE with DOUBLE columns"); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  JoinProg prog;
  join_prog_from_conds(n_conds, conds, [&](int u) { return join_user_type(j, u); }, &prog);
  return join_set_oc(j, prog, true);
}

int32_t tq_join_set_other_program(tq_join *j, int32_t n_inputs, const int32_t *input_cols, int32_t n_ops, const tq_expr_op *ops) {
  if (!j) return TQ_ERR_INVALID_ARG;
  TQ_TRY(join_oc_settable(j));
  JoinProg prog;
  TQ_TRY(join_prog_from_ops(n_inputs, input_cols, n_ops, ops, j->nb_user + j->np_user, [&](int u) { return join_user_type(j, u); }, &prog));
  return join_set_oc(j, prog, false);
}

int32_t tq_join_warnings(tq_join *j, int64_t *div_by_zero) {
  if (!j || !div_by_zero) return TQ_ERR_INVALID_ARG;
  *div_by_zero = j->oc_warnings;
  return TQ_OK;
}

int32_t tq_join_put_build(tq_join *j, const tq_column *cols, int32_t mem) {
  if (!j || !cols) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state != tq_join::BUILDING) { set_error("put_build after finalize_build"); return TQ_ERR_STATE; }
  if (j->build_mem >= 0 && j->build_mem != mem) { set_error("build chunks must all be host or all device"); return TQ_ERR_INVALID_ARG; }
  j->build_mem = mem;
  const int64_t rows = cols[0].length;
  if (rows < 0) return TQ_ERR_INVALID_ARG;
  for (int c = 0; c < j->nb_user; c++) {
    const bool var = j->b_ind[c] && j->b_elem[c] == 0;
    if (cols[c].length != rows) { set_error("ragged build chunk"); return TQ_ERR_INVALID_ARG; }
    if (!var && cols[c].offsets) { set_error("unsupport column type for encode (var-len data in fixed-width column %d)", c); return TQ_ERR_UNSUPPORTED_TYPE; }
    if (var && !cols[c].offsets) { set_error("var-len column %d needs offsets", c); return TQ_ERR_INVALID_ARG; }
    // (the offsets of a device column are not read here: append_cells_device checks them on the device)
    if (mem == TQ_MEM_HOST && rows && !cols[c].data && !(var && cols[c].offsets[rows] == cols[c].offsets[0])) return TQ_ERR_INVALID_ARG;
    if (mem != TQ_MEM_HOST && rows && !cols[c].data && !var) return TQ_ERR_INVALID_ARG;
    if (j->b_ind[c] && !var && mem != TQ_MEM_HOST) { set_error("FLOAT columns are accepted from host memory only"); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  if (rows == 0) return TQ_OK;
  if (mem == TQ_MEM_HOST) {
    if (j->n_build == 0) {
      j->b_direct = rows >= (1 << 18);
      for (int c = 0; c < j->nb_user; c++) if (j->b_ind[c]) j->b_direct = false;
    }
    if (j->b_direct) {
      Runtime &r = rt();
      std::lock_guard<std::recursive_mutex> lk(r.mu);
      const int64_t need = j->n_build + rows;
      if (need > j->b_dcap) {
        const int64_t ncap = need > j->b_dcap * 2 ? need : j->b_dcap * 2;
        j->b_ddata.resize(j->nb_user);
        TQ_CUDA(cudaStreamSynchronize(r.h2d));  // earlier chunks may still be uploading into the blocks that are about to move
        for (int c = 0; c < j->nb_user; c++) {
          DevBuf nb;
          TQ_TRY(nb.reserve((size_t)ncap * 8));
          if (j->n_build) TQ_CUDA(cudaMemcpyAsync(nb.p, j->b_ddata[c].p, (size_t)j->n_build * 8, cudaMemcpyDeviceToDevice, r.compute));
          TQ_CUDA(cudaStreamSynchronize(r.compute));  // the old block goes back to the allocator below
          j->b_ddata[c] = std::move(nb);
        }
        j->b_dcap = ncap;
      }
      for (int c = 0; c < j->nb_user; c++) {
        TQ_CUDA(cudaMemcpyAsync(j->b_ddata[c].as<uint8_t>() + j->n_build * 8, cols[c].data, (size_t)rows * 8, cudaMemcpyHostToDevice, r.h2d));
        TQ_TRY(j->b_host[c].append_nulls(cols[c], rows));
      }
      // cgo pointers are only valid during the call — unless the caller declared its input buffers stable
      if (!(j->flags & TQ_JOIN_STABLE_INPUT)) TQ_CUDA(cudaStreamSynchronize(r.h2d));
    } else {
      for (int c = 0; c < j->nb_user; c++) {
        if (j->b_ind[c]) { j->b_var[c].append(cols[c], rows); TQ_TRY(j->b_host[c].append_nulls(cols[c], rows)); }
        else TQ_TRY(j->b_host[c].append(cols[c], rows));
      }
    }
  } else {
    // var-len cells are copied into the build store now (the caller may reuse those buffers on return); the 8-byte columns
    // and every NULL bitmap are borrowed until tq_join_finalize_build
    Runtime &r = rt();
    std::lock_guard<std::recursive_mutex> lk(r.mu);
    int64_t before[MAXC][2];
    for (int c = 0; c < j->nb_user; c++) {
      if (!j->b_ind[c]) continue;
      before[c][0] = j->b_store[c].n;
      before[c][1] = j->b_store[c].nbytes;
      int64_t longest = 0;
      const int32_t st = append_cells_device(j->b_store[c], cols[c].offsets, cols[c].data, rows, &longest, j->var_meta, r.compute);
      if (st != TQ_OK) {   // a refused chunk leaves the stores as they were
        for (int d = 0; d < c; d++)
          if (j->b_ind[d]) { j->b_store[d].n = before[d][0]; j->b_store[d].nbytes = before[d][1]; }
        return st;
      }
    }
    j->b_dev_chunks.emplace_back(cols, cols + j->nb_user);
  }
  j->n_build += rows;
  return TQ_OK;
}

int32_t tq_join_finalize_build(tq_join *j) {
  if (!j) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state != tq_join::BUILDING) { set_error("finalize_build called twice"); return TQ_ERR_STATE; }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  j->b_view.assign(j->n_build_cols, DCol());
  if (j->build_mem == TQ_MEM_DEVICE) {
    // var-len columns: the cells are in b_store (put_build); the kernels see row ids, exactly as on the host path
    j->b_cols.resize(j->nb_user);
    for (int c = 0; c < j->nb_user; c++) {
      if (!j->b_ind[c]) continue;
      if (j->b_elem[c] == 4) {   // FLOAT is refused from device memory: the side is empty
        j->b_store[c].elem = 4;
        TQ_TRY(j->b_store[c].bytes.reserve(16));
      } else {
        int64_t unused = 0;
        TQ_TRY(append_cells_device(j->b_store[c], nullptr, nullptr, 0, &unused, j->var_meta, r.compute));   // offsets[0] of an empty side
      }
      TQ_TRY(j->b_cols[c].data.reserve((size_t)(j->n_build ? j->n_build : 1) * 8));
      TQ_TRY(iota_u64(j->b_cols[c].data.as<uint64_t>(), j->n_build, r.compute));
    }
  }
  if (j->build_mem == TQ_MEM_DEVICE && j->b_dev_chunks.size() == 1) {
    for (int c = 0; c < j->nb_user; c++) {
      j->b_view[c].data = j->b_ind[c] ? j->b_cols[c].data.as<uint64_t>() : (const uint64_t *)j->b_dev_chunks[0][c].data;
      j->b_view[c].bm = (const uint32_t *)j->b_dev_chunks[0][c].null_bitmap;
    }
  } else if (j->build_mem == TQ_MEM_DEVICE) {
    // several device chunks: concatenate (data D2D; a bitmap copied whole where its chunk starts on a byte, bit-shifted where not)
    for (int c = 0; c < j->nb_user; c++) {
      if (!j->b_ind[c]) TQ_TRY(j->b_cols[c].data.reserve((size_t)j->n_build * 8));
      TQ_TRY(j->b_cols[c].bm.reserve(bitmap_alloc_bytes(j->n_build)));
      int64_t off = 0;
      bool any_bm = false;
      for (auto &ch : j->b_dev_chunks) any_bm |= (ch[c].null_bitmap != nullptr);
      if (any_bm) TQ_CUDA(cudaMemsetAsync(j->b_cols[c].bm.p, 0xFF, bitmap_alloc_bytes(j->n_build), r.compute));
      for (auto &ch : j->b_dev_chunks) {
        const int64_t rows = ch[c].length;
        if (!j->b_ind[c])
          TQ_CUDA(cudaMemcpyAsync(j->b_cols[c].data.as<uint8_t>() + off * 8, ch[c].data, (size_t)rows * 8, cudaMemcpyDeviceToDevice, r.compute));
        if (ch[c].null_bitmap && (off & 7)) {
          const int64_t words = ((off + rows + 31) >> 5) - (off >> 5), cap = (int64_t)r.sm_count * 4;
          TQ_LAUNCH(k_bitmap_append, (unsigned)(words < 256 ? 1 : (words / 256 < cap ? words / 256 : cap)), 256, 0, r.compute, j->b_cols[c].bm.as<uint32_t>(), off,
                    (const uint8_t *)ch[c].null_bitmap, rows);
          count_launch();
          TQ_TRY(check_launch("k_bitmap_append"));
        } else if (ch[c].null_bitmap) {
          TQ_CUDA(cudaMemcpyAsync(j->b_cols[c].bm.as<uint8_t>() + (off >> 3), ch[c].null_bitmap, bitmap_bytes(rows), cudaMemcpyDeviceToDevice, r.compute));
        }
        off += rows;
      }
      j->b_view[c].data = j->b_cols[c].data.as<uint64_t>();
      j->b_view[c].bm = any_bm ? j->b_cols[c].bm.as<uint32_t>() : nullptr;
    }
  } else {
    j->b_cols.resize(j->nb_user);
    for (int c = 0; c < j->nb_user; c++) {
      if (j->b_direct) {
        // data is already in HBM (put_build); only the staged NULL bitmap is uploaded
        TQ_CUDA(cudaStreamSynchronize(r.h2d));
        j->b_cols[c].data = std::move(j->b_ddata[c]);
        TQ_TRY(j->b_cols[c].bm.reserve(bitmap_alloc_bytes(j->n_build)));
        TQ_CUDA(cudaMemcpyAsync(j->b_cols[c].bm.p, j->b_host[c].bm.p, bitmap_bytes(j->n_build), cudaMemcpyHostToDevice, r.compute));
      } else {
        TQ_TRY(upload_col(j->b_host[c], j->b_cols[c], r.compute));
      }
      if (j->b_ind[c]) {  // the column the kernels see: row ids into the side store
        TQ_TRY(iota_u64(j->b_cols[c].data.as<uint64_t>(), j->n_build, r.compute));
        TQ_TRY(upload_store(j->b_var[c], j->b_store[c], r.compute));
        j->b_var[c].reset();
      }
      j->b_view[c].data = j->b_cols[c].data.as<uint64_t>();
      j->b_view[c].bm = j->b_host[c].has_bm ? j->b_cols[c].bm.as<uint32_t>() : nullptr;
    }
  }
  if (j->key_hidden && j->n_keys == 1) {
    DCol kc;
    TQ_TRY(key_source(j, true, 0, j->b_view, j->b_store, j->n_build, j->kx_b_data[0], j->kx_b_bm[0], &kc, r.compute));
    j->b_view[j->nb_user] = kc;
  } else if (j->key_hidden) {
    // build-side key tuples -> the hidden key column; a NULL in any key column leaves the row out of the table (hash_table.go:161-163)
    DCol kc[MK_MAX_KEYS];
    bool any_bm = false;
    for (int i = 0; i < j->n_keys; i++) {
      TQ_TRY(key_source(j, true, i, j->b_view, j->b_store, j->n_build, j->kx_b_data[i], j->kx_b_bm[i], &kc[i], r.compute));
      any_bm |= (kc[i].bm != nullptr);
    }
    TQ_TRY(j->mk_build_key.reserve((size_t)(j->n_build ? j->n_build : 1) * 8));
    if (any_bm) TQ_TRY(j->mk_build_bm.reserve(bitmap_alloc_bytes(j->n_build)));
    TQ_TRY(j->mk.encode(kc, nullptr, j->n_build, /*insert=*/true, /*null_is_value=*/false, j->mk_build_key.as<uint64_t>(),
                        any_bm ? j->mk_build_bm.as<uint32_t>() : nullptr, r.compute));
    j->b_view[j->nb_user].data = j->mk_build_key.as<uint64_t>();
    j->b_view[j->nb_user].bm = any_bm ? j->mk_build_bm.as<uint32_t>() : nullptr;
  }
  if (j->keyless) {
    // no table: the build rows stay as device columns in insertion order.  A single device chunk is still the caller's
    // memory, which is only lent until this call returns, so it is copied.
    const auto t0 = std::chrono::steady_clock::now();
    if (j->n_build > 0xFFFFFFFFll) { set_error("key-less join: the build side holds 2^32 rows or more"); return TQ_ERR_INVALID_ARG; }
    if (j->build_mem == TQ_MEM_DEVICE && j->b_dev_chunks.size() == 1) {
      for (int c = 0; c < j->nb_user; c++) {
        const tq_column &ch = j->b_dev_chunks[0][c];
        if (!j->b_ind[c]) {
          TQ_TRY(j->b_cols[c].data.reserve((size_t)j->n_build * 8));
          TQ_CUDA(cudaMemcpyAsync(j->b_cols[c].data.p, ch.data, (size_t)j->n_build * 8, cudaMemcpyDeviceToDevice, r.compute));
          j->b_view[c].data = j->b_cols[c].data.as<uint64_t>();
        }
        if (ch.null_bitmap) {
          TQ_TRY(j->b_cols[c].bm.reserve(bitmap_alloc_bytes(j->n_build)));
          TQ_CUDA(cudaMemcpyAsync(j->b_cols[c].bm.p, ch.null_bitmap, bitmap_bytes(j->n_build), cudaMemcpyDeviceToDevice, r.compute));
          j->b_view[c].bm = j->b_cols[c].bm.as<uint32_t>();
        }
      }
    }
    TQ_CUDA(cudaStreamSynchronize(r.compute));   // the staging buffers are released below
    j->n_valid = j->n_build;
    j->build_ns = (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
  } else {
    TQ_TRY(join_build(j));
  }
  j->mk_build_key.release();
  j->mk_build_bm.release();
  for (int i = 0; i < j->n_keys; i++) { j->kx_b_data[i].release(); j->kx_b_bm[i].release(); }
  for (auto &h : j->b_host) { h.data.release(); h.bm.release(); }
  j->b_dev_chunks.clear();
  j->state = tq_join::PROBING;
  return TQ_OK;
}

int32_t tq_join_put_probe(tq_join *j, const tq_column *cols, const uint8_t *selected, int32_t mem) {
  if (!j || !cols) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state != tq_join::PROBING) { set_error("put_probe before finalize_build"); return TQ_ERR_STATE; }
  if (j->probe_eof) { set_error("put_probe after probe_eof"); return TQ_ERR_STATE; }
  const int64_t rows = cols[0].length;
  if (rows < 0) return TQ_ERR_INVALID_ARG;
  for (int c = 0; c < j->np_user; c++) {
    const bool var = j->p_ind[c] && j->p_elem[c] == 0;
    if (cols[c].length != rows) { set_error("ragged probe chunk"); return TQ_ERR_INVALID_ARG; }
    if (!var && cols[c].offsets) { set_error("unsupport column type for encode (var-len data in fixed-width column %d)", c); return TQ_ERR_UNSUPPORTED_TYPE; }
    if (var && !cols[c].offsets) { set_error("var-len column %d needs offsets", c); return TQ_ERR_INVALID_ARG; }
    // (the offsets of a device column are not read here: append_cells_device checks them on the device)
    if (mem == TQ_MEM_HOST && rows && !cols[c].data && !(var && cols[c].offsets[rows] == cols[c].offsets[0])) return TQ_ERR_INVALID_ARG;
    if (mem != TQ_MEM_HOST && rows && !cols[c].data && !var) return TQ_ERR_INVALID_ARG;
    if (j->p_ind[c] && !var && mem != TQ_MEM_HOST) { set_error("FLOAT columns are accepted from host memory only"); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  if (rows == 0) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  if (mem == TQ_MEM_DEVICE) {
    TQ_TRY(flush_probe_staging(j));
    if (j->keyless) return kl_put_device(j, cols, selected, rows);
    std::vector<DCol> view(j->n_probe_cols);
    for (int c = 0; c < j->np_user; c++) {
      view[c].data = (const uint64_t *)cols[c].data;
      view[c].bm = (const uint32_t *)cols[c].null_bitmap;
    }
    const int slot = j->pending.active ? 1 - j->pending.cursor_slot : 0;
    if (j->any_ind) {
      // var-len cells are copied into this batch's side store (no batch reads this input set any more: the one in flight
      // uses the other slot); the join sees row ids 0..rows-1 + the column's NULL bitmap, as for a host piece
      ProbeInputSet &in = j->in_set[slot];
      in.store.resize(j->np_user);
      in.cols.resize(j->n_probe_cols);
      for (int c = 0; c < j->np_user; c++) {
        if (!j->p_ind[c]) continue;
        SideStore &st = in.store[c];
        st.n = st.nbytes = 0;
        int64_t longest = 0;
        TQ_TRY(append_cells_device(st, cols[c].offsets, cols[c].data, rows, &longest, j->var_meta, r.compute));
        TQ_TRY(in.cols[c].data.reserve((size_t)rows * 8));
        TQ_TRY(iota_u64(in.cols[c].data.as<uint64_t>(), rows, r.compute));
        view[c].data = in.cols[c].data.as<uint64_t>();
      }
    }
    const uint8_t *d_sel = nullptr;
    if (selected) {  // `selected` is host memory by contract
      ProbeInputSet &in = j->in_set[slot];
      TQ_TRY(in.selected.reserve((size_t)rows));
      TQ_CUDA(cudaMemcpyAsync(in.selected.p, selected, (size_t)rows, cudaMemcpyHostToDevice, r.compute));
      TQ_CUDA(cudaStreamSynchronize(r.compute));
      d_sel = in.selected.as<uint8_t>();
    }
    return start_batch(j, view, d_sel, rows, /*want_host=*/false, slot);
  }
  if (rows >= j->batch_rows) {
    // a large host column (not the ≤1024-row chunk protocol): stream it in batch-sized pieces straight from the caller's buffer
    TQ_TRY(flush_probe_staging(j));
    for (int64_t row0 = 0; row0 < rows; row0 += j->batch_rows) {
      const int64_t piece = rows - row0 < j->batch_rows ? rows - row0 : j->batch_rows;
      TQ_TRY(process_host_piece(j, cols, row0, piece, selected, /*eager_d2h=*/false));
    }
    // the caller may reuse its buffers on return — unless it declared them stable (TQ_JOIN_STABLE_INPUT): then the
    // upload keeps running while the caller drains the previous batch (H2D and D2H overlap on the full-duplex link)
    if (!(j->flags & TQ_JOIN_STABLE_INPUT)) TQ_CUDA(cudaStreamSynchronize(r.h2d));
    return TQ_OK;
  }
  if (j->p_host[0].n + rows > j->batch_rows) TQ_TRY(flush_probe_staging(j));
  const int64_t before = j->p_host[0].n;
  for (int c = 0; c < j->np_user; c++) {
    if (j->p_ind[c]) { j->p_var[c].append(cols[c], rows); TQ_TRY(j->p_host[c].append_nulls(cols[c], rows)); }
    else TQ_TRY(j->p_host[c].append(cols[c], rows));
  }
  if (selected && !j->p_sel_any) { j->p_sel_host.assign((size_t)before, 1); j->p_sel_any = true; }
  if (j->p_sel_any) {
    if (selected) j->p_sel_host.insert(j->p_sel_host.end(), selected, selected + rows);
    else j->p_sel_host.insert(j->p_sel_host.end(), (size_t)rows, 1);
  }
  return TQ_OK;
}

int32_t tq_join_put_probe_segments(tq_join *j, int32_t n_segs, const tq_column *cols, const uint64_t *const *seg_counts, int64_t seg_cap) {
  if (!j || !cols || !seg_counts || n_segs < 1 || n_segs > SA_MAX_SEGS || seg_cap < 1) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state != tq_join::PROBING) { set_error("put_probe before finalize_build"); return TQ_ERR_STATE; }
  if (j->probe_eof) { set_error("put_probe after probe_eof"); return TQ_ERR_STATE; }
  // segmented input can only run the streaming path (its scatter alone reads the regions), and it has no pass that would
  // encode a hidden key column or FLOAT / var-len columns
  if (j->keyless || !stream_probe_ok(j) || j->key_hidden || j->any_ind) {
    set_error("segmented probe batches need the streaming PK-FK path (inner join, unique NOT NULL build side >= 2^18 rows, <= 4 columns per side)");
    return TQ_ERR_UNSUPPORTED_TYPE;
  }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(flush_probe_staging(j));
  const int64_t seg_rows = (seg_cap + POS_SEG_ROWS_ALIGN - 1) / POS_SEG_ROWS_ALIGN * POS_SEG_ROWS_ALIGN;
  std::vector<DCol> view(j->n_probe_cols);
  j->seg.n = n_segs;
  j->seg.cap = seg_cap;
  for (int g = 0; g < n_segs; g++) {
    j->seg.cnt[g] = reinterpret_cast<const unsigned long long *>(seg_counts[g]);
    for (int c = 0; c < j->n_probe_cols; c++) {
      const tq_column &col = cols[g * j->n_probe_cols + c];
      if (!col.data || col.null_bitmap || col.offsets) { j->seg.n = 0; set_error("segment columns: NOT NULL 8-byte device columns"); return TQ_ERR_INVALID_ARG; }
      j->seg.col[g][c] = reinterpret_cast<const uint64_t *>(col.data);
    }
  }
  for (int c = 0; c < j->n_probe_cols; c++) { view[c].data = j->seg.col[0][c]; view[c].bm = nullptr; }
  const int slot = j->pending.active ? 1 - j->pending.cursor_slot : 0;
  const int32_t st = start_batch(j, view, nullptr, (int64_t)n_segs * seg_rows, /*want_host=*/false, slot);
  j->seg.n = 0;
  return st;
}

int32_t tq_join_probe_eof(tq_join *j) {
  if (!j) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state != tq_join::PROBING) { set_error("probe_eof before finalize_build"); return TQ_ERR_STATE; }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(flush_probe_staging(j));
  TQ_TRY(finalize_pending(j));
  j->probe_eof = true;
  return TQ_OK;
}

// Make j->host_cur the result batch the next rows come from (waiting / copying as needed).  *have == 0: no rows now
// (*eof tells whether the stream has ended).
static int32_t join_current_batch(tq_join *j, int64_t max_rows, int *have, int32_t *eof) {
  Runtime &r = rt();
  *have = 0;
  for (;;) {
    if (j->host_cur && j->host_cur_pos < j->host_cur->n) break;
    if (j->host_cur) { recycle(j, std::move(j->host_cur)); j->host_cur_pos = 0; }
    // The batch in flight is only waited for at end of input: until then "no rows yet" means "feed more", so the
    // D2H of batch i overlaps the H2D + kernels of batch i+1.
    if (j->results.empty() && j->keyless) TQ_TRY(kl_produce(j));
    if (j->results.empty() && j->probe_eof) TQ_TRY(finalize_pending(j));
    if (j->results.empty()) {
      *eof = j->probe_eof ? 1 : 0;
      return TQ_OK;
    }
    j->host_cur = std::move(j->results.front());
    j->results.pop_front();
    j->host_cur_pos = 0;
    if (j->host_cur->oc_err) return xp_err_to_status(j->host_cur->oc_err, j->oc.prog.ops, "other conditions");
    if (j->keyless && !j->host_cur->on_host) {
      // copies of this batch wait for its kernels only; then the next batch is built while this one is copied and sliced
      TQ_CUDA(cudaStreamWaitEvent(r.d2h, j->host_cur->ev_ready, 0));
      if (j->results.empty()) TQ_TRY(kl_produce(j));
    }
    if (!j->host_cur->on_host) {
      // Large consumer buffers: copy straight from HBM into the caller's columns (no staging, no CPU memcpy).
      // (a queued batch is complete: finalize_pending waited for its kernels — no stream-wide sync here, so the copy
      // below runs while the NEXT batch is still uploading / probing)
      const bool direct = !j->any_ind && max_rows >= (1 << 18) && (max_rows & 7) == 0;
      if (direct) break;
      TQ_TRY(enqueue_d2h(j, j->host_cur.get()));
    }
    TQ_CUDA(cudaEventSynchronize(j->host_cur->ev_ready));
  }
  *have = 1;
  return TQ_OK;
}

int32_t tq_join_next_bytes(tq_join *j, int64_t max_rows, int64_t *bytes_per_col) {
  if (!j || !bytes_per_col || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (j->state == tq_join::BUILDING) { set_error("next before finalize_build"); return TQ_ERR_STATE; }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  const int ncols = j->nb_user + j->np_user;
  for (int c = 0; c < ncols; c++) bytes_per_col[c] = 0;
  int have = 0;
  int32_t eof = 0;
  TQ_TRY(join_current_batch(j, max_rows, &have, &eof));
  if (!have) return TQ_OK;
  ResultBatch *rb = j->host_cur.get();
  const int64_t take = (rb->n - j->host_cur_pos) < max_rows ? (rb->n - j->host_cur_pos) : max_rows;
  for (int c = 0; c < ncols; c++) {
    const int ic = j->out_map[c];
    if (!j->out_side[ic]) bytes_per_col[c] = take * 8;
    else if (rb->var[ic].elem == 4) bytes_per_col[c] = take * 4;
    else {
      const int64_t *off = rb->var[ic].h_off.as<int64_t>() + j->host_cur_pos;
      bytes_per_col[c] = off[take] - off[0];
    }
  }
  return TQ_OK;
}

int32_t tq_join_next(tq_join *j, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!j || !out_cols || !n_rows || !eof || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  *n_rows = 0;
  *eof = 0;
  if (j->state == tq_join::BUILDING) { set_error("next before finalize_build"); return TQ_ERR_STATE; }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  const int ncols = j->nb_user + j->np_user;  // hidden key columns stay behind (out_map)
  int have = 0;
  TQ_TRY(join_current_batch(j, max_rows, &have, eof));
  if (!have) {
    for (int c = 0; c < ncols; c++) out_cols[c].length = 0;
    return TQ_OK;
  }
  ResultBatch *rb = j->host_cur.get();
  const int64_t take = (rb->n - j->host_cur_pos) < max_rows ? (rb->n - j->host_cur_pos) : max_rows;
  for (int c = 0; c < ncols; c++) {
    const bool var = j->out_side[j->out_map[c]] && rb->var[j->out_map[c]].elem == 0;
    if (!out_cols[c].null_bitmap || (!out_cols[c].data && !var) || (var && !out_cols[c].offsets)) {
      set_error("output column %d needs data and null_bitmap buffers (and offsets for a var-len column)", c);
      return TQ_ERR_INVALID_ARG;
    }
  }
  if (!rb->on_host) {
    if ((j->host_cur_pos & 7) != 0) { set_error("internal: unaligned direct result copy"); return TQ_ERR_STATE; }
    for (int c = 0; c < ncols; c++) {
      const int ic = j->out_map[c];
      TQ_CUDA(cudaMemcpyAsync(out_cols[c].data, rb->cols[ic].data.as<uint8_t>() + j->host_cur_pos * 8, (size_t)take * 8, cudaMemcpyDeviceToHost, r.d2h));
      TQ_CUDA(cudaMemcpyAsync(out_cols[c].null_bitmap, rb->cols[ic].bm.as<uint8_t>() + (j->host_cur_pos >> 3), bitmap_bytes(take), cudaMemcpyDeviceToHost, r.d2h));
      out_cols[c].length = take;
    }
    TQ_CUDA(cudaStreamSynchronize(r.d2h));
    if (take & 7) for (int c = 0; c < ncols; c++) out_cols[c].null_bitmap[bitmap_bytes(take) - 1] &= (uint8_t)((1u << (take & 7)) - 1);
    j->host_cur_pos += take;
    // a partially consumed batch continues on the staged path if the next call asks for a small / unaligned slice
    if (j->host_cur_pos < rb->n && (j->host_cur_pos & 7) != 0) { TQ_TRY(enqueue_d2h(j, rb)); TQ_CUDA(cudaEventSynchronize(rb->ev_ready)); }
    *n_rows = take;
    return TQ_OK;
  }
  for (int c = 0; c < ncols; c++) {
    const int ic = j->out_map[c];
    if (j->out_side[ic]) {
      // FLOAT: 4-byte slots; var-len: offsets rebased to 0 + the cells' bytes (chunk.Column layout, column.go:28-34)
      const VarOut &v = rb->var[ic];
      if (v.elem == 4) memcpy(out_cols[c].data, v.h_bytes.as<uint8_t>() + j->host_cur_pos * 4, (size_t)take * 4);
      else {
        const int64_t *off = v.h_off.as<int64_t>() + j->host_cur_pos;
        const int64_t b0 = off[0];
        for (int64_t i = 0; i <= take; i++) out_cols[c].offsets[i] = off[i] - b0;
        if (off[take] > b0) memcpy(out_cols[c].data, v.h_bytes.as<uint8_t>() + b0, (size_t)(off[take] - b0));
      }
    } else {
      memcpy(out_cols[c].data, rb->h_data[ic].as<uint8_t>() + j->host_cur_pos * 8, (size_t)take * 8);
    }
    host_bitmap_extract(out_cols[c].null_bitmap, rb->h_bm[ic].as<uint8_t>(), j->host_cur_pos, take);
    out_cols[c].length = take;
  }
  j->host_cur_pos += take;
  *n_rows = take;
  return TQ_OK;
}

int32_t tq_join_next_device(tq_join *j, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!j || !out_cols || !n_rows || !eof) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  *n_rows = 0;
  *eof = 0;
  if (j->state == tq_join::BUILDING) { set_error("next before finalize_build"); return TQ_ERR_STATE; }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  recycle(j, std::move(j->lent));
  if (j->results.empty() && j->keyless) TQ_TRY(kl_produce(j));
  if (j->results.empty()) TQ_TRY(finalize_pending(j));
  if (j->results.empty()) {
    *eof = j->probe_eof ? 1 : 0;
    return TQ_OK;
  }
  j->lent = std::move(j->results.front());
  j->results.pop_front();
  if (j->lent->oc_err) return xp_err_to_status(j->lent->oc_err, j->oc.prog.ops, "other conditions");
  if (j->keyless) {   // build the next batch while the caller works on this one, which is complete when the call returns
    if (j->results.empty()) TQ_TRY(kl_produce(j));
    TQ_CUDA(cudaEventSynchronize(j->lent->ev_ready));
  }
  const int ncols = j->nb_user + j->np_user;
  for (int c = 0; c < ncols; c++) {
    out_cols[c].length = j->lent->n;
    const int ic = j->out_map[c];
    out_cols[c].data = j->lent->cols[ic].data.as<uint8_t>();
    out_cols[c].null_bitmap = j->lent->cols[ic].bm.as<uint8_t>();
    out_cols[c].offsets = nullptr;
    if (j->out_side[ic]) {  // gathered FLOAT / var-len column, device resident
      out_cols[c].data = j->lent->var[ic].bytes.as<uint8_t>();
      if (j->lent->var[ic].elem == 0) out_cols[c].offsets = j->lent->var[ic].off.as<int64_t>();
    }
  }
  *n_rows = j->lent->n;
  return TQ_OK;
}

int32_t tq_join_stats(tq_join *j, int64_t *s) {
  if (!j || !s) return TQ_ERR_INVALID_ARG;
  if (j->keyless && j->kl_timed) {   // [5]: the last result batch's kernels
    float ms = 0;
    if (cudaEventSynchronize(j->ev_b[0]) == cudaSuccess && cudaEventElapsedTime(&ms, j->ev_a[0], j->ev_b[0]) == cudaSuccess)
      j->last_probe_ns = (int64_t)(ms * 1e6);
    else cudaGetLastError();
  }
  s[0] = j->n_valid;
  s[1] = j->n_distinct;
  s[2] = j->keyless ? 0 : 1ll << j->pbits;
  s[3] = j->probe_rows_total;
  s[4] = j->joined_rows_total;
  s[5] = j->last_probe_ns;
  s[6] = j->build_ns;
  s[7] = j->probe_launches;
  return TQ_OK;
}

int32_t tq_join_build_path(tq_join *j, int32_t *path) {
  if (!j || !path) return TQ_ERR_INVALID_ARG;
  *path = j->build_path;
  return TQ_OK;
}

// ---- multi-GPU shard boundary: push into per-source REGIONS of the peers' receive buffers, no count exchange first --------
// Every destination rank reserves one region of `region_cap` rows per source rank and per column; this rank scatters its rows
// straight into "its" region on every peer (stores over NVLink) and then publishes how many rows it wrote to each peer in
// that peer's count table (one 8-byte peer store per destination).  The receiver joins the regions as ONE segmented batch
// (tq_join_put_probe_segments) whose kernels read the counts from device memory — between the exchange and the join there
// is no host round trip, only the cross-rank barrier that says "all pushes of this chunk have landed".  The slots and the
// device-side wait live in push.cu.

// One region push (include/tinysql_b200.h): every argument is checked before anything is enqueued, so a refused push writes
// no region and publishes no slot.  Then the scatter of n rows into n_parts destinations (+ the miss bin with keep_misses)
// runs on the push stream, followed by k_publish_counts.
int32_t tq_partition_push_regions(int32_t n_cols, const tq_column *cols, int32_t key_col, int64_t n, int32_t n_parts,
                                  const uint8_t *selected, int32_t keep_misses, void *const *dest_data, void *const *dest_counts,
                                  int64_t region_cap, void *const *miss_data, void *miss_count, int64_t miss_cap, int32_t slot,
                                  uint64_t epoch) {
  TQ_TRY(ensure_init());
  const char *fn = "tq_partition_push_regions";
  if (!cols || n_cols < 1 || key_col < 0 || key_col >= n_cols || n < 0 || n > 0xFFFFFFF0ll) {
    set_error("%s: needs columns, 0 <= key_col < n_cols and < 2^32 rows", fn);
    return TQ_ERR_INVALID_ARG;
  }
  if (keep_misses && (!miss_data || !miss_count || miss_cap < 0 || miss_cap > 0xFFFFFFF0ll)) {
    set_error("%s: keep_misses needs miss columns, a miss slot and 0 <= miss_cap < 2^32", fn);
    return TQ_ERR_INVALID_ARG;
  }
  // a NULL bitmap anywhere: the mask word travels as wire column n_cols, and a NULL key routes like an unselected row
  bool pack = false;
  for (int c = 0; c < n_cols; c++) pack = pack || cols[c].null_bitmap;
  const int n_wire = n_cols + (pack ? 1 : 0);
  if (n_wire > 4) { set_error("%s: %d columns%s: the push moves at most 4 words per row", fn, n_cols, pack ? " and the NULL mask word" : ""); return TQ_ERR_UNSUPPORTED_TYPE; }
  TQ_TRY(push_check_dests(fn, n_parts, n_wire, dest_data, dest_counts, region_cap, slot));
  ScatterParams sp{};
  sp.n_cols = n_wire;
  sp.key_col = key_col;
  sp.key_mode = KEYMODE_RAW;
  sp.n = n;
  sp.n_parts_mod = n_parts;
  sp.is_outer = keep_misses ? 1 : 0;
  sp.selected = selected;
  for (int c = 0; c < n_cols; c++) {
    sp.in[c].data = (const uint64_t *)cols[c].data;
    sp.in[c].bm = (const uint32_t *)cols[c].null_bitmap;
  }
  for (int q = 0; q < n_parts; q++)
    for (int c = 0; c < n_wire; c++) sp.out_bin[q][c] = (uint64_t *)dest_data[q * n_wire + c];
  if (keep_misses)
    for (int c = 0; c < n_wire; c++) sp.out_bin[n_parts][c] = (uint64_t *)miss_data[c];

  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.h2d;  // the push stream: rows cross NVLink while the compute stream joins what has already arrived
  PushSlot *slot_state = nullptr;
  // the previous push of this slot no longer reads the pinned tables or the mask below
  TQ_TRY(push_begin(slot, n_parts, dest_counts, keep_misses ? miss_count : nullptr, s, &slot_state));
  PushSlot &ps = *slot_state;
  const int n_pub = n_parts + (keep_misses ? 1 : 0);
  for (int q = 0; q < 16; q++) ps.h_lim.as<uint32_t>()[q] = (uint32_t)region_cap;
  if (keep_misses) ps.h_lim.as<uint32_t>()[n_parts] = (uint32_t)miss_cap;
  TQ_CUDA(cudaMemcpyAsync(ps.lim.p, ps.h_lim.p, 64, cudaMemcpyHostToDevice, s));
  if (n > 0) {
    if (pack) {  // the mask word and the effective selection first
      TQ_TRY(ps.mask.reserve((size_t)n * 8));
      TQ_TRY(ps.sel.reserve((size_t)n));
      TQ_TRY(pack_null_mask(sp.in, n_cols, key_col, selected, n, ps.mask.as<uint64_t>(), ps.sel.as<uint8_t>(), s));
      sp.selected = ps.sel.as<uint8_t>();
      sp.in[n_cols] = DCol{ps.mask.as<uint64_t>(), nullptr};
    }
    sp.part_cursor = ps.cursor.as<uint32_t>();
    sp.part_lim = ps.lim.as<uint32_t>();
    sp.overflow = ps.ovf.as<unsigned long long>();
    TQ_TRY(launch_scatter_fast(sp, s, "k_probe_scatter_fast(push regions)"));
  }
  return push_publish(ps, n_pub, epoch, s);
}

int32_t tq_join_destroy(tq_join *j) {
  if (!j) return TQ_OK;
  if (rt().inited) {
    cudaSetDevice(rt().device);
    cudaDeviceSynchronize();  // Close may arrive with work in flight (join_test.go:175-182 early Close)
  }
  delete j;
  return TQ_OK;
}

}  // extern "C"
