// partition.cu — radix exchange prep for the multi-GPU path (the device-side shuffleIntermData,
// executor/aggregate.go:352-356): rows are split into n_parts partitions by the high bits of the key
// hash, stable within a partition.  Three launches: per-chunk histogram, exclusive scan over
// (partition-major, chunk-minor) counts, ordered scatter of every column.
// Also both ends of the nullable region exchange: the mask word a pushing rank packs (k_pack_null_mask) and the receiver's
// tq_region_gather, which copies the arrived regions into contiguous columns and expands the mask word into NULL bitmaps.
// And the GROUP BY push's kernels (tq_agg_push_partial): the destination of a partial row from its group, the same histogram /
// scan / scatter writing each destination's run column-wise into that destination's region with the mask word packed on the
// way, and the mask word's expansion into NULL bitmaps on the receiving side.
// And the ORDER BY range push's kernels (tq_partition_push_sample / _ranges): the sample gather and the destination of a row
// from the sorted sample's splitters, on the sort's own key words (sortkey.cuh).
#include "scatter.cuh"
#include "sortkey.cuh"

namespace tq {

static constexpr int PART_MAXC = 16;
static constexpr int PART_MAX = 256;
static constexpr int PART_CHUNK = 2048;  // rows owned by one warp, walked in order (=> stable)

// k_part_hist / k_part_scatter take their routing and their stores from the parameter struct (the policy):
//   dest_of(r)         destination of row r
//   run_base(q)        subtracted from destination q's scanned offsets (0: one output array; its first offset: one region per q)
//   store(r, q, pos)   writes row r at position pos of destination q
// PartParams is tq_partition_device (destination from the key's hash, every column into one output array at the global offset);
// RegionParams is the GROUP BY push (destination from an array, column-wise into per-destination regions with the mask word).
struct PartParams {
  int n_cols;
  DCol in[PART_MAXC];
  DColMut out[PART_MAXC];
  int key_col;
  int n_parts;
  int64_t n;
  int64_t n_chunks;
  uint32_t *counts;  // [part * n_chunks + chunk]

  __device__ __forceinline__ int dest_of(int64_t r) const {
    if (!tqd::bm_not_null(in[key_col].bm, r)) return (int)(r % n_parts);  // NULL keys never match; spread them
    return (int)((tqd::mix64(in[key_col].data[r]) >> 40) % (uint64_t)n_parts);
  }
  __device__ __forceinline__ uint32_t run_base(int) const { return 0; }
  __device__ __forceinline__ void store(int64_t r, int, uint32_t pos) const {
    for (int c = 0; c < n_cols; c++) {
      out[c].data[pos] = in[c].data[r];
      if (out[c].bm && tqd::bm_not_null(in[c].bm, r)) atomicOr(&out[c].bm[pos >> 5], 1u << (pos & 31));
    }
  }
};

struct RegionParams {
  int n_cols;  // wire columns before the mask word
  int n_parts;
  int64_t n;
  int64_t n_chunks;
  uint32_t *counts;
  DCol in[REGION_MAXW];
  const uint8_t *dest;
  uint64_t *const *out;  // DEVICE table: out[q * n_areas + a] = destination q's area a: wire columns, the mask word, byte areas
  uint32_t cap;          // rows per region: a row at or past it is not written (the push publishes ~0)
  int n_areas;           // n_cols + 1 + n_var
  // var-len wire columns (scatter_to_regions_var): their words are not copied, k_region_scatter_var writes offsets and cells
  int n_var;
  uint64_t var_mask;     // bit c: wire column c is var-len
  RegionVar var[REGION_MAXV];
  uint32_t *bcounts;     // [(v * n_parts + q) * n_chunks + chunk] cell bytes, scanned in place
  unsigned long long *btotal;  // [v * n_parts + q] cell bytes of the region, exact

  __device__ __forceinline__ int dest_of(int64_t r) const { return dest[r]; }
  __device__ __forceinline__ uint32_t run_base(int q) const { return counts[(int64_t)q * n_chunks]; }
  __device__ __forceinline__ void store(int64_t r, int q, uint32_t pos) const {
    if (pos >= cap) return;
    uint64_t *const *o = out + (int64_t)q * n_areas;
    uint64_t m = 0;
    for (int c = 0; c < n_cols; c++) {
      if (!((var_mask >> c) & 1)) o[c][pos] = in[c].data[r];
      m |= (uint64_t)tqd::bm_not_null(in[c].bm, r) << c;
    }
    o[n_cols][pos] = m;
  }
  // the arena id of row r's cell in var-len column v: its id word, or r itself for a column without ids (a device column
  // whose offsets are the arena, as the range push sends one)
  __device__ __forceinline__ uint64_t cell_id(int v, int64_t r) const {
    const DCol &c = in[var[v].col];
    return c.data ? c.data[r] : (uint64_t)r;
  }
  // bytes of row r's cell in var-len column v (0 for NULL)
  __device__ __forceinline__ uint64_t cell_len(int v, int64_t r) const {
    if (!tqd::bm_not_null(in[var[v].col].bm, r)) return 0;
    const uint64_t id = cell_id(v, r);
    return (uint64_t)(var[v].off[id + 1] - var[v].off[id]);
  }
};

template <class P>
__global__ void __launch_bounds__(256) k_part_hist(const P p) {
  __shared__ uint32_t s_cnt[8][PART_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)blockIdx.x * 8 + warp;
  for (int i = lane; i < p.n_parts; i += 32) s_cnt[warp][i] = 0;
  __syncwarp();
  if (chunk < p.n_chunks) {
    const int64_t lo = chunk * PART_CHUNK;
    const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
    for (int64_t r = lo + lane; r < hi; r += 32) atomicAdd(&s_cnt[warp][p.dest_of(r)], 1u);
    __syncwarp();
    for (int i = lane; i < p.n_parts; i += 32) p.counts[(int64_t)i * p.n_chunks + chunk] = s_cnt[warp][i];
  }
}

template <class P>
__global__ void __launch_bounds__(256) k_part_scatter(const P p) {
  __shared__ uint32_t s_base[8][PART_MAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)blockIdx.x * 8 + warp;
  if (chunk >= p.n_chunks) return;
  for (int i = lane; i < p.n_parts; i += 32) s_base[warp][i] = p.counts[(int64_t)i * p.n_chunks + chunk] - p.run_base(i);  // scanned offsets
  __syncwarp();
  const int64_t lo = chunk * PART_CHUNK;
  const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
  for (int64_t r0 = lo; r0 < hi; r0 += 32) {
    const int64_t r = r0 + lane;
    const bool active = r < hi;
    const int part = active ? p.dest_of(r) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, part);
    const unsigned rank = __popc(peers & ((1u << lane) - 1));
    uint32_t pos = 0;
    if (active) pos = s_base[warp][part] + rank;
    __syncwarp();
    if (active && rank == (unsigned)__popc(peers) - 1) s_base[warp][part] = pos + 1;  // last peer advances the cursor
    __syncwarp();
    if (active) p.store(r, part, pos);
  }
}

__global__ void k_part_offsets(const uint32_t *scanned, int64_t n_chunks, int n_parts, int64_t n, int64_t *offsets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_parts) offsets[i] = scanned[(int64_t)i * n_chunks];
  if (i == n_parts) offsets[i] = n;
}

// ---- the nullable wire format of the region exchange (scatter.cuh): mask word out at the source, bitmaps back at the receiver
static constexpr int MASK_MAXC = 4;  // the push scatter moves at most 4 words per row, the mask word included
static constexpr int GATHER_MAX_REGIONS = 8;

struct PackParams {
  int n_cols, key_col;
  DCol in[MASK_MAXC];
  const uint8_t *selected;
  int64_t n;
  uint64_t *mask;
  uint8_t *sel_out;
};

__global__ void __launch_bounds__(256) k_pack_null_mask(const PackParams p) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t m = 0;
    for (int c = 0; c < p.n_cols; c++) m |= (uint64_t)tqd::bm_not_null(p.in[c].bm, r) << c;
    p.mask[r] = m;
    const bool sel = p.selected ? p.selected[r] != 0 : true;
    p.sel_out[r] = (uint8_t)(sel && ((m >> p.key_col) & 1));
  }
}

int32_t pack_null_mask(const DCol *cols, int n_cols, int key_col, const uint8_t *selected, int64_t n, uint64_t *mask, uint8_t *sel_out,
                       cudaStream_t s) {
  if (n_cols < 1 || n_cols > MASK_MAXC || key_col < 0 || key_col >= n_cols || n < 1) { set_error("internal: pack_null_mask arguments"); return TQ_ERR_INVALID_ARG; }
  PackParams p{};
  p.n_cols = n_cols;
  p.key_col = key_col;
  for (int c = 0; c < n_cols; c++) p.in[c] = cols[c];
  p.selected = selected;
  p.n = n;
  p.mask = mask;
  p.sel_out = sel_out;
  const int64_t blocks = (n + 255) / 256, cap = (int64_t)rt().sm_count * 8;
  TQ_LAUNCH(k_pack_null_mask, (unsigned)(blocks < cap ? blocks : cap), 256, 0, s, p);
  count_launch();
  return check_launch("k_pack_null_mask");
}

struct GatherParams {
  int n_regions, n_cols, has_mask;  // region g holds n_cols (+ the mask word) columns
  const unsigned long long *slots;  // n_regions x {u64 rows, u64 epoch}
  unsigned long long region_cap, out_cap;
  const uint64_t *src[GATHER_MAX_REGIONS][MASK_MAXC];
  uint64_t *out[MASK_MAXC];
  uint32_t *out_bm[MASK_MAXC];
  unsigned long long *total;  // rows of all regions, ~0 when a slot reads more than region_cap (a region overflowed)
};

// Every thread reads the slots (through shared memory, once per CTA), so the kernel knows the row count before it writes:
// when a region overflowed or the rows exceed out_cap it writes nothing but *total.  Rows [0, rows) are the regions in order;
// bitmap words are written for the whole 64-row groups that hold them, with 0 for the rows past the end, so every output
// bitmap is a complete device bitmap of `rows` rows.  A warp covers 32 consecutive rows: one ballot = one bitmap word.
__global__ void __launch_bounds__(256) k_region_gather(const GatherParams p) {
  __shared__ unsigned long long s_off[GATHER_MAX_REGIONS + 1];
  __shared__ int s_ok;
  if (threadIdx.x == 0) {
    unsigned long long off = 0;
    bool ok = true;
    for (int g = 0; g < p.n_regions; g++) {
      const unsigned long long rows = p.slots[2 * g];
      s_off[g] = off;
      if (rows > p.region_cap) ok = false;
      else off += rows;
    }
    s_off[p.n_regions] = off;
    if (blockIdx.x == 0) *p.total = ok ? off : ~0ull;
    s_ok = ok && off <= p.out_cap;
  }
  __syncthreads();
  if (!s_ok) return;
  const unsigned long long rows = s_off[p.n_regions], padded = (rows + 63) & ~63ull;
  const int lane = threadIdx.x & 31;
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x; base < padded; base += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long r = base + threadIdx.x;
    const bool live = r < rows;
    int g = 0;
    if (live)
      while (r >= s_off[g + 1]) g++;
    const unsigned long long i = live ? r - s_off[g] : 0;
    const uint64_t m = (live && p.has_mask) ? p.src[g][p.n_cols][i] : ~0ull;
    for (int c = 0; c < p.n_cols; c++) {
      if (live) p.out[c][r] = p.src[g][c][i];
      if (p.out_bm[c]) {
        const unsigned w = __ballot_sync(0xffffffffu, live && ((m >> c) & 1));
        if (lane == 0 && r < padded) p.out_bm[c][r >> 5] = w;
      }
    }
  }
}

// ---- the GROUP BY push (tq_agg_push_partial, agg.cu): destination per partial row, scatter into the regions, mask expansion
struct GroupDestParams {
  int n_items, n_parts;
  uint32_t real_mask;  // bit g: item g is REAL
  DCol item[GROUP_MAX_ITEMS];
  const uint64_t *hash[GROUP_MAX_ITEMS];  // var-len item: the content hash of each dictionary id
  int64_t n;
  uint8_t *dest;
};

__global__ void __launch_bounds__(256) k_group_dest(const GroupDestParams p) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t h = 0;
    for (int g = 0; g < p.n_items; g++) {
      uint64_t v = GROUP_NULL_WORD;
      if (tqd::bm_not_null(p.item[g].bm, r)) {
        v = p.item[g].data[r];
        if (p.hash[g]) v = p.hash[g][v];                                      // a string id: its content hash
        else if (((p.real_mask >> g) & 1) && v == 0x8000000000000000ull) v = 0;  // -0.0 and +0.0 are one group
      }
      h = tqd::mix64(h ^ v);
    }
    p.dest[r] = (uint8_t)((h >> 40) % (uint64_t)p.n_parts);
  }
}

int32_t group_dest(const DCol *items, int n_items, uint32_t real_mask, int64_t n, int n_parts, uint8_t *dest, cudaStream_t s) {
  return group_dest(items, nullptr, n_items, real_mask, n, n_parts, dest, s);
}

int32_t group_dest(const DCol *items, const uint64_t *const *hashes, int n_items, uint32_t real_mask, int64_t n, int n_parts, uint8_t *dest,
                   cudaStream_t s) {
  if (n_items < 0 || n_items > GROUP_MAX_ITEMS || n_parts < 1 || n_parts > 8 || n < 1) { set_error("internal: group_dest arguments"); return TQ_ERR_INVALID_ARG; }
  GroupDestParams p{};
  p.n_items = n_items;
  p.n_parts = n_parts;
  p.real_mask = real_mask;
  for (int g = 0; g < n_items; g++) {
    p.item[g] = items[g];
    p.hash[g] = hashes ? hashes[g] : nullptr;
  }
  p.n = n;
  p.dest = dest;
  const int64_t blocks = (n + 255) / 256, cap = (int64_t)rt().sm_count * 8;
  TQ_LAUNCH(k_group_dest, (unsigned)(blocks < cap ? blocks : cap), 256, 0, s, p);
  count_launch();
  return check_launch("k_group_dest");
}

// rows[q] = rows destined to q (from the scanned histogram and its total), *overflow = some rows[q] > cap
__global__ void k_region_rows(const uint32_t *scanned, int64_t n_chunks, int n_parts, const uint64_t *total, uint32_t cap, uint32_t *rows,
                              unsigned long long *overflow) {
  if (threadIdx.x != 0) return;
  unsigned long long ovf = 0;
  for (int q = 0; q < n_parts; q++) {
    const uint64_t end = q + 1 < n_parts ? scanned[(int64_t)(q + 1) * n_chunks] : *total;
    rows[q] = (uint32_t)(end - scanned[(int64_t)q * n_chunks]);
    ovf |= rows[q] > cap ? 1ull : 0ull;
  }
  *overflow = ovf;
}

int32_t scatter_to_regions(const DCol *cols, int n_cols, const uint8_t *dest, int64_t n, int n_parts, uint64_t *const *out, int64_t cap,
                           uint32_t *rows, unsigned long long *overflow, RegionScratch &sc, cudaStream_t s) {
  return scatter_to_regions_var(cols, n_cols, nullptr, 0, dest, n, n_parts, out, cap, rows, overflow, sc, s);
}

struct ExpandParams {
  int n_cols;
  const uint64_t *mask;
  int64_t n;
  uint32_t *bm[REGION_MAXW];
};

// One warp covers 32 consecutive rows: one ballot per column = one bitmap word.  Words are written for the whole 64-row groups
// that hold the rows, 0 past the last row.
__global__ void __launch_bounds__(256) k_expand_mask(const ExpandParams p) {
  const int64_t padded = (p.n + 63) & ~63ll;
  const int lane = threadIdx.x & 31;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < padded; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = base + threadIdx.x;
    const uint64_t m = r < p.n ? p.mask[r] : 0;
    for (int c = 0; c < p.n_cols; c++) {
      const unsigned w = __ballot_sync(0xffffffffu, (m >> c) & 1);
      if (lane == 0 && r < padded) p.bm[c][r >> 5] = w;
    }
  }
}

int32_t expand_null_mask(const uint64_t *mask, int64_t n, int n_cols, uint32_t *const *bm, cudaStream_t s) {
  if (n_cols < 1 || n_cols > REGION_MAXW || n < 1) { set_error("internal: expand_null_mask arguments"); return TQ_ERR_INVALID_ARG; }
  ExpandParams p{};
  p.n_cols = n_cols;
  p.mask = mask;
  p.n = n;
  for (int c = 0; c < n_cols; c++) p.bm[c] = bm[c];
  const int64_t blocks = ((n + 63) / 64 * 64 + 255) / 256, cap = (int64_t)rt().sm_count * 8;
  TQ_LAUNCH(k_expand_mask, (unsigned)(blocks < cap ? blocks : cap), 256, 0, s, p);
  count_launch();
  return check_launch("k_expand_mask");
}

// ---- the broadcast push (tq_partition_push_broadcast, push.cu): every row to every destination, var-len columns included
struct BcastParams {
  int n_cols, n_parts, nullable;
  int64_t n;
  uint8_t is_bytes[BCAST_MAXC];
  const uint64_t *data[BCAST_MAXC];  // 8-byte values, or the n + 1 offsets of a BYTES column
  const uint8_t *cells[BCAST_MAXC];  // a BYTES column's cells
  const uint64_t *bm[BCAST_MAXC];    // 64-row bitmap words; null = no NULLs
  uint64_t byte_cap[BCAST_MAXC];
  uint64_t *dst_data[8][BCAST_MAXC];
  uint8_t *dst_cells[8][BCAST_MAXC];
  uint64_t *dst_bm[8][BCAST_MAXC];
  uint32_t *rows;
  unsigned long long *overflow;
};
static_assert(sizeof(BcastParams) <= 4096, "the broadcast's parameters fit the 4 KB kernel parameter space");

__device__ __forceinline__ void bcast_store16(uint64_t *d, uint64_t a, uint64_t b) {
  ulonglong2 v;
  v.x = a;
  v.y = b;
  *reinterpret_cast<ulonglong2 *>(d) = v;
}

// Word k of a copied word area: a value, an offset rebased to 0, or a bitmap word (all ones without a bitmap).
__device__ __forceinline__ uint64_t bcast_word(const uint64_t *src, int kind, uint64_t base, int64_t k) {
  if (kind == 2) return src ? src[k] : ~0ull;
  return src[k] - (kind == 1 ? base : 0);
}

// One 16-byte chunk per thread and step: two words are read once and stored to every destination, as one 16-byte store where
// the destination allows it.  kind 0 = values, 1 = offsets, 2 = bitmap words.
__device__ __forceinline__ void bcast_words(const BcastParams &p, int c, int kind, const uint64_t *src, uint64_t base, int64_t nw, int64_t t,
                                            int64_t stride) {
  for (int64_t i = t; 2 * i < nw; i += stride) {
    const int64_t k = 2 * i;
    const bool pair = k + 1 < nw;
    const uint64_t a = bcast_word(src, kind, base, k), b = pair ? bcast_word(src, kind, base, k + 1) : 0;
    for (int q = 0; q < p.n_parts; q++) {
      uint64_t *d = (kind == 2 ? p.dst_bm[q][c] : p.dst_data[q][c]) + k;
      if (pair && ((uintptr_t)d & 15) == 0) {
        bcast_store16(d, a, b);
      } else {
        d[0] = a;
        if (pair) d[1] = b;
      }
    }
  }
}

// Up to 16 bytes (cnt, 1..16) from s into x (bytes 0..7) and y (8..15), read as the aligned 8-byte words that hold them: each
// holds at least one of the bytes, so no read leaves the bytes' allocation.
__device__ __forceinline__ void load_chunk16(const uint8_t *s, uint64_t cnt, uint64_t &x, uint64_t &y) {
  const unsigned a = (unsigned)((uintptr_t)s & 7);
  const uint64_t *w = reinterpret_cast<const uint64_t *>(s - a);
  const unsigned last = (unsigned)((a + cnt - 1) >> 3);
  const uint64_t w0 = w[0], w1 = last >= 1 ? w[1] : 0, w2 = last >= 2 ? w[2] : 0;
  x = a ? (w0 >> (8 * a)) | (w1 << (64 - 8 * a)) : w0;
  y = a ? (w1 >> (8 * a)) | (w2 << (64 - 8 * a)) : w1;
}

// The cnt bytes of (x, y) to d: one 16-byte store where d is aligned and the chunk is whole, byte stores otherwise.
__device__ __forceinline__ void store_chunk16(uint8_t *d, uint64_t cnt, uint64_t x, uint64_t y) {
  if (cnt == 16 && ((uintptr_t)d & 15) == 0) {
    bcast_store16(reinterpret_cast<uint64_t *>(d), x, y);
  } else {
    for (unsigned b = 0; b < cnt; b++) d[b] = (uint8_t)((b < 8 ? x >> (8 * b) : y >> (8 * (b - 8))) & 0xFF);
  }
}

// The cells [off0, off0 + len) of a BYTES column to the start of each byte area: destination chunk i gets source bytes
// [16 i, 16 i + 16).
__device__ __forceinline__ void bcast_cells(const BcastParams &p, int c, const uint8_t *src, uint64_t len, int64_t t, int64_t stride) {
  for (uint64_t i = (uint64_t)t; 16 * i < len; i += (uint64_t)stride) {
    const uint64_t lo = 16 * i, cnt = len - lo < 16 ? len - lo : 16;
    uint64_t x, y;
    load_chunk16(src + lo, cnt, x, y);
    for (int q = 0; q < p.n_parts; q++) store_chunk16(p.dst_cells[q][c] + lo, cnt, x, y);
  }
}

__global__ void __launch_bounds__(256) k_broadcast(const BcastParams p) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  bool ovf = false;
  for (int c = 0; c < p.n_cols; c++) {
    if (p.is_bytes[c]) {
      const uint64_t off0 = p.data[c][0], len = p.data[c][p.n] - off0;
      bcast_words(p, c, 1, p.data[c], off0, p.n + 1, t, stride);
      if (len > p.byte_cap[c]) ovf = true;   // every thread sees it: none writes the cells
      else bcast_cells(p, c, p.cells[c] + off0, len, t, stride);
    } else {
      bcast_words(p, c, 0, p.data[c], 0, p.n, t, stride);
    }
    if (p.nullable) bcast_words(p, c, 2, p.bm[c], 0, (p.n + 63) >> 6, t, stride);
  }
  if (t < p.n_parts) p.rows[t] = (uint32_t)p.n;
  if (t == 0 && ovf) *p.overflow = 1;
}

int32_t broadcast_rows(int n_cols, const tq_column *cols, const int32_t *types, int nullable, int64_t n, int n_parts, void *const *dest_data,
                       const int64_t *byte_cap, uint32_t *rows, unsigned long long *overflow, cudaStream_t s) {
  if (n_cols < 1 || n_cols > BCAST_MAXC || n_parts < 1 || n_parts > 8 || n < 0 || n > 0xFFFFFFF0ll) {
    set_error("internal: broadcast_rows arguments");
    return TQ_ERR_INVALID_ARG;
  }
  BcastParams p{};
  p.n_cols = n_cols;
  p.n_parts = n_parts;
  p.nullable = nullable ? 1 : 0;
  p.n = n;
  p.rows = rows;
  p.overflow = overflow;
  const int n_wire = broadcast_wire_areas(n_cols, types, nullable);
  int64_t chunks = 0;   // 16-byte chunks of the largest area: every area is walked by the whole grid
  for (int c = 0; c < n_cols; c++) {
    const bool bytes = (types[c] & 0xFF) == TQ_TYPE_BYTES;
    p.is_bytes[c] = bytes;
    p.data[c] = reinterpret_cast<const uint64_t *>(bytes ? (const void *)cols[c].offsets : (const void *)cols[c].data);
    p.cells[c] = bytes ? cols[c].data : nullptr;
    p.bm[c] = reinterpret_cast<const uint64_t *>(cols[c].null_bitmap);
    p.byte_cap[c] = bytes ? (uint64_t)byte_cap[c] : 0;
    const int64_t area = bytes ? (byte_cap[c] + 15) / 16 : (n + 1) / 2;
    chunks = area > chunks ? area : chunks;
  }
  for (int q = 0; q < n_parts; q++) {
    int a = q * n_wire;
    for (int c = 0; c < n_cols; c++) {
      p.dst_data[q][c] = static_cast<uint64_t *>(dest_data[a++]);
      if (p.is_bytes[c]) p.dst_cells[q][c] = static_cast<uint8_t *>(dest_data[a++]);
      if (nullable) p.dst_bm[q][c] = static_cast<uint64_t *>(dest_data[a++]);
    }
  }
  const int64_t blocks = (chunks + 255) / 256, cap = (int64_t)rt().sm_count * 8;
  TQ_LAUNCH(k_broadcast, (unsigned)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap)), 256, 0, s, p);
  count_launch();
  return check_launch("k_broadcast");
}

// ---- the var-len wire columns of the GROUP BY push (scatter_to_regions_var): the cells follow their rows in the same stable
// order, each region's byte positions from a per-(column, destination, chunk) byte count and its scan

// One warp per chunk: the cell bytes each destination gets from it, per var-len column; also summed per region, exactly.
__global__ void __launch_bounds__(256) k_region_var_hist(const RegionParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (chunk >= p.n_chunks) return;
  const int64_t lo = chunk * PART_CHUNK;
  const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
  for (int v = 0; v < p.n_var; v++) {
    uint64_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t r = lo + lane; r < hi; r += 32) {
      const int q = p.dest[r];
      const uint64_t len = p.cell_len(v, r);
#pragma unroll
      for (int k = 0; k < 8; k++) acc[k] += k == q ? len : 0;
    }
#pragma unroll
    for (int q = 0; q < 8; q++) {
      if (q >= p.n_parts) break;
      uint64_t b = acc[q];
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) b += __shfl_xor_sync(0xffffffffu, b, d);
      if (lane == 0) {
        // a chunk's count past 32 bits means a region past its byte cap (< 2^32): the push publishes ~0 and writes no cell
        p.bcounts[((int64_t)v * p.n_parts + q) * p.n_chunks + chunk] = b > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)b;
        if (b) atomicAdd(p.btotal + v * p.n_parts + q, (unsigned long long)b);
      }
    }
  }
}

// After k_region_rows: a region past its byte cap sets the overflow; offsets entry 0 of every var-len area is 0.
__global__ void k_region_bytes(const RegionParams p, unsigned long long *overflow) {
  if (threadIdx.x != 0) return;
  bool ovf = false;
  for (int v = 0; v < p.n_var; v++)
    for (int q = 0; q < p.n_parts; q++) {
      ovf |= p.btotal[v * p.n_parts + q] > p.var[v].byte_cap;
      p.out[(int64_t)q * p.n_areas + p.var[v].col][0] = 0;
    }
  if (ovf) *overflow = 1;
}

// k_part_scatter with var-len columns: the row's words and mask as RegionParams::store, then per var-len column the row's
// byte position (the chunk's scanned base for its destination + the cells of the earlier rows of the same destination), its
// offset, and its cell, copied by the whole warp one cell at a time in 16-byte chunks.  Positions are exact modulo 2^32, so
// a region whose cells exceed its byte cap (< 2^32) gets no offset and no cell.
__global__ void __launch_bounds__(256) k_region_scatter_var(const RegionParams p) {
  __shared__ uint32_t s_base[8][8];
  __shared__ uint32_t s_bpos[8][REGION_MAXV][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)blockIdx.x * 8 + warp;
  if (chunk >= p.n_chunks) return;
  for (int i = lane; i < p.n_parts; i += 32) s_base[warp][i] = p.counts[(int64_t)i * p.n_chunks + chunk] - p.run_base(i);
  for (int k = lane; k < p.n_var * p.n_parts; k += 32)
    s_bpos[warp][k / p.n_parts][k % p.n_parts] = p.bcounts[(int64_t)k * p.n_chunks + chunk] - p.bcounts[(int64_t)k * p.n_chunks];
  __syncwarp();
  const int64_t lo = chunk * PART_CHUNK;
  const int64_t hi = lo + PART_CHUNK < p.n ? lo + PART_CHUNK : p.n;
  for (int64_t r0 = lo; r0 < hi; r0 += 32) {
    const int64_t r = r0 + lane;
    const bool active = r < hi;
    const int part = active ? p.dest_of(r) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, part);
    const unsigned rank = __popc(peers & ((1u << lane) - 1));
    const bool last = rank == (unsigned)__popc(peers) - 1;
    uint32_t pos = 0;
    if (active) pos = s_base[warp][part] + rank;
    __syncwarp();
    if (active && last) s_base[warp][part] = pos + 1;
    __syncwarp();
    if (active) p.store(r, part, pos);
    for (int v = 0; v < p.n_var; v++) {
      const uint64_t len = active ? p.cell_len(v, r) : 0;
      uint64_t pre = 0;   // cells of the earlier rows of this warp step that go to the same destination
      for (int d = 0; d < 32; d++) {
        const uint64_t l = __shfl_sync(0xffffffffu, len, d);
        if (d < lane && ((peers >> d) & 1)) pre += l;
      }
      uint32_t bpos = 0;
      if (active) bpos = s_bpos[warp][v][part] + (uint32_t)pre;
      __syncwarp();
      if (active && last) s_bpos[warp][v][part] = bpos + (uint32_t)len;
      __syncwarp();
      const bool fits = active && pos < p.cap && p.btotal[v * p.n_parts + part] <= p.var[v].byte_cap;
      unsigned long long src = 0, dst = 0;
      if (fits) {
        uint64_t *const *o = p.out + (int64_t)part * p.n_areas;
        o[p.var[v].col][pos + 1] = (uint64_t)bpos + len;
        dst = (unsigned long long)(reinterpret_cast<uint8_t *>(o[p.n_cols + 1 + v]) + bpos);
        if (len) src = (unsigned long long)(p.var[v].bytes + p.var[v].off[p.cell_id(v, r)]);
      }
      const unsigned todo = __ballot_sync(0xffffffffu, fits && len > 0);
      for (int j = 0; j < 32; j++) {
        if (!((todo >> j) & 1)) continue;
        const uint8_t *cs = reinterpret_cast<const uint8_t *>(__shfl_sync(0xffffffffu, src, j));
        uint8_t *cd = reinterpret_cast<uint8_t *>(__shfl_sync(0xffffffffu, dst, j));
        const uint64_t cl = __shfl_sync(0xffffffffu, len, j);
        for (uint64_t b = 16 * (uint64_t)lane; b < cl; b += 16 * 32) {
          const uint64_t cnt = cl - b < 16 ? cl - b : 16;
          uint64_t x, y;
          load_chunk16(cs + b, cnt, x, y);
          store_chunk16(cd + b, cnt, x, y);
        }
      }
    }
  }
}

int32_t scatter_to_regions_var(const DCol *cols, int n_cols, const RegionVar *var, int n_var, const uint8_t *dest, int64_t n, int n_parts,
                               uint64_t *const *out, int64_t cap, uint32_t *rows, unsigned long long *overflow, RegionScratch &sc,
                               cudaStream_t s) {
  if (n_cols < 1 || n_cols > REGION_MAXW || n_var < 0 || n_var > REGION_MAXV || (n_var && !var) || n_parts < 1 || n_parts > 8 || n < 1 ||
      n > 0xFFFFFFF0ll || cap < 1 || cap > 0xFFFFFFF0ll) {
    set_error("internal: scatter_to_regions arguments");
    return TQ_ERR_INVALID_ARG;
  }
  RegionParams p{};
  p.n_cols = n_cols;
  p.n_parts = n_parts;
  p.n = n;
  p.n_chunks = (n + PART_CHUNK - 1) / PART_CHUNK;
  for (int c = 0; c < n_cols; c++) p.in[c] = cols[c];
  p.dest = dest;
  p.out = out;
  p.cap = (uint32_t)cap;
  p.n_areas = n_cols + 1 + n_var;
  p.n_var = n_var;
  for (int v = 0; v < n_var; v++) {
    if (var[v].col < 0 || var[v].col >= n_cols || ((p.var_mask >> var[v].col) & 1) || var[v].byte_cap < 1 || var[v].byte_cap > 0xFFFFFFF0ull) {
      set_error("internal: scatter_to_regions var-len column %d", v);
      return TQ_ERR_INVALID_ARG;
    }
    p.var[v] = var[v];
    p.var_mask |= 1ull << var[v].col;
  }
  const int64_t n_counts = p.n_chunks * n_parts;
  TQ_TRY(sc.hist.reserve((size_t)n_counts * 4));
  TQ_TRY(sc.total.reserve(8));
  p.counts = sc.hist.as<uint32_t>();
  const unsigned blocks = (unsigned)((p.n_chunks + 7) / 8);
  TQ_LAUNCH(k_part_hist<RegionParams>, blocks, 256, 0, s, p);
  count_launch();
  TQ_TRY(check_launch("k_part_hist(regions)"));
  TQ_TRY(exclusive_scan_u32(p.counts, 1, p.counts, 1, n_counts, sc.total.as<uint64_t>(), sc.scan, s));
  TQ_LAUNCH(k_region_rows, 1, 32, 0, s, p.counts, p.n_chunks, n_parts, sc.total.as<uint64_t>(), p.cap, rows, overflow);
  count_launch();
  if (n_var == 0) {
    TQ_LAUNCH(k_part_scatter<RegionParams>, blocks, 256, 0, s, p);
    count_launch();
    return check_launch("k_part_scatter(regions)");
  }
  const int64_t n_bcounts = n_counts * n_var;
  TQ_TRY(sc.bhist.reserve((size_t)n_bcounts * 4));
  TQ_TRY(sc.btotal.reserve((size_t)n_var * n_parts * 8));
  p.bcounts = sc.bhist.as<uint32_t>();
  p.btotal = sc.btotal.as<unsigned long long>();
  TQ_CUDA(cudaMemsetAsync(p.btotal, 0, (size_t)n_var * n_parts * 8, s));
  TQ_LAUNCH(k_region_var_hist, blocks, 256, 0, s, p);
  count_launch();
  TQ_TRY(check_launch("k_region_var_hist"));
  TQ_TRY(exclusive_scan_u32(p.bcounts, 1, p.bcounts, 1, n_bcounts, nullptr, sc.bscan, s));
  TQ_LAUNCH(k_region_bytes, 1, 32, 0, s, p, overflow);
  TQ_LAUNCH(k_region_scatter_var, blocks, 256, 0, s, p);
  count_launch(2);
  return check_launch("k_region_scatter_var");
}

// ---- the range push of the multi-GPU ORDER BY (tq_partition_push_sample / _ranges, push.cu): the sample of a shard, and the
// destination of a row from the sorted sample's splitters, compared on the sort's own key words (sortkey.cuh)

struct SampleParams {
  int n_by;
  RangeBy by[RANGE_MAX_BY];
  SampleOut out;
  int64_t n, m;
  uint64_t seed;
  int src_rank;
};

// One CTA walks the m samples 256 at a time (a warp = 32 consecutive samples: one ballot = one bitmap word): positions, values,
// bits and tie words; cell lengths into the offsets, scanned in place by the block; then the cells, when they fit.
__global__ void __launch_bounds__(256) k_sample_gather(const SampleParams p) {
  __shared__ uint64_t s_scan[256];
  __shared__ uint64_t s_carry;
  const int lane = threadIdx.x & 31;
  const int64_t padded = (p.m + 255) & ~255ll;
  for (int64_t j = threadIdx.x; j < padded; j += 256) {
    const bool live = j < p.m;
    const uint64_t pos = live ? range_sample_pos(p.seed, p.src_rank, j, p.n, p.m) : 0;
    if (live) p.out.tie[j] = range_tie(p.src_rank, pos);
    for (int b = 0; b < p.n_by; b++) {
      const RangeBy &c = p.by[b];
      const bool nn = live && tqd::bm_not_null(c.bm, (int64_t)pos);
      if (live && c.type != TQ_TYPE_BYTES) p.out.data[b][j] = c.data[pos];
      if (live && c.type == TQ_TYPE_BYTES) p.out.off[b][j + 1] = nn ? c.off[pos + 1] - c.off[pos] : 0;   // lengths, scanned below
      if (p.out.bm[b]) {
        const unsigned w = __ballot_sync(0xffffffffu, nn);
        if (lane == 0) p.out.bm[b][j >> 5] = w;
      }
    }
  }
  for (int b = 0; b < p.n_by; b++) {
    if (p.by[b].type != TQ_TYPE_BYTES) continue;
    int64_t *off = p.out.off[b];
    if (threadIdx.x == 0) { off[0] = 0; s_carry = 0; }
    __syncthreads();
    for (int64_t j0 = 0; j0 < p.m; j0 += 256) {   // inclusive scan of off[1..m], 256 entries per round
      const int64_t j = j0 + threadIdx.x;
      uint64_t v = j < p.m ? (uint64_t)off[j + 1] : 0;
      s_scan[threadIdx.x] = v;
      __syncthreads();
      for (int d = 1; d < 256; d <<= 1) {
        const uint64_t add = threadIdx.x >= (unsigned)d ? s_scan[threadIdx.x - d] : 0;
        __syncthreads();
        v += add;
        s_scan[threadIdx.x] = v;
        __syncthreads();
      }
      if (j < p.m) off[j + 1] = (int64_t)(s_carry + v);
      __syncthreads();
      if (threadIdx.x == 255) s_carry += v;
      __syncthreads();
    }
    if ((uint64_t)off[p.m] > p.out.byte_cap[b]) continue;   // the broadcast finds the same total and publishes the overflow
    for (int64_t j = threadIdx.x; j < p.m; j += 256) {
      const uint64_t pos = range_sample_pos(p.seed, p.src_rank, j, p.n, p.m);
      const int64_t len = off[j + 1] - off[j];
      const uint8_t *src = p.by[b].bytes + (len ? p.by[b].off[pos] : 0);
      for (int64_t k = 0; k < len; k++) p.out.bytes[b][off[j] + k] = src[k];
    }
  }
}

int32_t sample_rows(const RangeBy *by, int n_by, int64_t n, int64_t m, uint64_t seed, int src_rank, const SampleOut &out, cudaStream_t s) {
  if (n_by < 0 || n_by > RANGE_MAX_BY || m < 1 || m > RANGE_MAX_SAMPLES || m > n || n > 0xFFFFFFF0ll) { set_error("internal: sample_rows arguments"); return TQ_ERR_INVALID_ARG; }
  SampleParams p{};
  p.n_by = n_by;
  for (int b = 0; b < n_by; b++) p.by[b] = by[b];
  p.out = out;
  p.n = n;
  p.m = m;
  p.seed = seed;
  p.src_rank = src_rank;
  TQ_LAUNCH(k_sample_gather, 1, 256, 0, s, p);
  count_launch();
  return check_launch("k_sample_gather");
}

struct RangeParams {
  int n_by, n_split, src_rank;
  RangeBy row[RANGE_MAX_BY], spl[RANGE_MAX_BY];
  const uint64_t *spl_tie;
  uint32_t pos[7];
  int64_t n;
  uint8_t *dest;
};

__device__ __forceinline__ KeySrc range_key(const RangeBy &c, int mode, int word) {
  KeySrc k{};
  k.mode = mode;
  k.type = c.type;
  k.word = word;
  k.desc = c.desc;
  k.d8 = c.data;
  k.off = c.off;
  k.bytes = c.bytes;
  k.base = 0;
  k.bm = c.bm;
  return k;
}

// -1 / 0 / +1: row r of the shard against splitter row s of the sorted sample, on the sort's key words most significant first
// (per ByItem the NULL flag, then the value word or the string's chunks and length), then the tie words
__device__ int range_cmp(const RangeParams &p, uint32_t r, uint32_t s) {
  for (int b = 0; b < p.n_by; b++) {
    const RangeBy &x = p.row[b], &y = p.spl[b];
    uint64_t a = key_word(range_key(x, KS_NULL_FLAG, 0), r), c = key_word(range_key(y, KS_NULL_FLAG, 0), s);
    if (a != c) return a < c ? -1 : 1;
    if (x.type != TQ_TYPE_BYTES) {
      a = key_word(range_key(x, KS_COL8, 0), r);
      c = key_word(range_key(y, KS_COL8, 0), s);
      if (a != c) return a < c ? -1 : 1;
      continue;
    }
    const bool nn = tqd::bm_not_null(x.bm, r);   // equal flags: both NULL (every word 0 or ~0) or both NOT NULL
    if (!nn) continue;
    const int64_t lx = x.off[r + 1] - x.off[r], ly = y.off[s + 1] - y.off[s];
    const int64_t chunks = ((lx > ly ? lx : ly) + 7) / 8;
    for (int64_t w = 0; w < chunks; w++) {
      a = key_word(range_key(x, KS_STR_CHUNK, (int)w), r);
      c = key_word(range_key(y, KS_STR_CHUNK, (int)w), s);
      if (a != c) return a < c ? -1 : 1;
    }
    a = key_word(range_key(x, KS_STR_LEN, 0), r);
    c = key_word(range_key(y, KS_STR_LEN, 0), s);
    if (a != c) return a < c ? -1 : 1;
  }
  const uint64_t t = range_tie(p.src_rank, r), u = p.spl_tie[s];
  return t == u ? 0 : (t < u ? -1 : 1);
}

// dest[r] = the splitters at or below row r: a binary search over the n_split (<= 7) splitters
__global__ void __launch_bounds__(256) k_range_dest(const RangeParams p) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = p.n_split;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (range_cmp(p, (uint32_t)r, p.pos[mid]) >= 0) lo = mid + 1;
      else hi = mid;
    }
    p.dest[r] = (uint8_t)lo;
  }
}

int32_t range_dest(const RangeBy *rows, const RangeBy *spl, int n_by, const uint64_t *spl_tie, const int64_t *pos, int n_split, int src_rank,
                   int64_t n, uint8_t *dest, cudaStream_t s) {
  if (n_by < 0 || n_by > RANGE_MAX_BY || n_split < 0 || n_split > 7 || n < 1 || n > 0xFFFFFFF0ll || (n_split && (!spl_tie || !pos))) {
    set_error("internal: range_dest arguments");
    return TQ_ERR_INVALID_ARG;
  }
  RangeParams p{};
  p.n_by = n_by;
  p.n_split = n_split;
  p.src_rank = src_rank;
  for (int b = 0; b < n_by; b++) {
    p.row[b] = rows[b];
    if (n_split) p.spl[b] = spl[b];
  }
  p.spl_tie = spl_tie;
  for (int k = 0; k < n_split; k++) p.pos[k] = (uint32_t)pos[k];
  p.n = n;
  p.dest = dest;
  const int64_t blocks = (n + 255) / 256, cap = (int64_t)rt().sm_count * 8;
  TQ_LAUNCH(k_range_dest, (unsigned)(blocks < cap ? blocks : cap), 256, 0, s, p);
  count_launch();
  return check_launch("k_range_dest");
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
  TQ_LAUNCH(k_part_hist<PartParams>, blocks, 256, 0, s, p);
  count_launch();
  TQ_TRY(check_launch("k_part_hist"));
  TQ_TRY(exclusive_scan_u32(p.counts, 1, p.counts, 1, n_counts, nullptr, scan_scratch, s));
  TQ_LAUNCH(k_part_offsets, (n_parts + 1 + 255) / 256, 256, 0, s, p.counts, p.n_chunks, n_parts, n, d_off.as<int64_t>());
  TQ_LAUNCH(k_part_scatter<PartParams>, blocks, 256, 0, s, p);
  count_launch(2);
  TQ_TRY(check_launch("k_part_scatter"));
  TQ_CUDA(cudaMemcpyAsync(h_off.p, d_off.p, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  memcpy(part_offsets, h_off.p, (size_t)(n_parts + 1) * 8);
  return TQ_OK;
}

extern "C" int32_t tq_region_gather(int32_t n_regions, const void *slots, int64_t region_cap, int32_t n_cols, int32_t has_mask,
                                    const tq_column *regions, tq_column *out_cols, int64_t out_cap, int64_t *n_rows) {
  TQ_TRY(ensure_init());
  if (n_regions < 1 || n_regions > GATHER_MAX_REGIONS || !slots || region_cap < 1 || n_cols < 1 || (has_mask != 0 && has_mask != 1) ||
      n_cols + has_mask > MASK_MAXC || !regions || !out_cols || out_cap < 0 || !n_rows) {
    set_error("tq_region_gather: 1..%d regions, 1..%d columns with the mask word, region_cap >= 1", GATHER_MAX_REGIONS, MASK_MAXC);
    return TQ_ERR_INVALID_ARG;
  }
  const int nw = n_cols + has_mask;
  GatherParams p{};
  p.n_regions = n_regions;
  p.n_cols = n_cols;
  p.has_mask = has_mask;
  p.slots = static_cast<const unsigned long long *>(slots);
  p.region_cap = (unsigned long long)region_cap;
  p.out_cap = (unsigned long long)out_cap;
  for (int g = 0; g < n_regions; g++)
    for (int c = 0; c < nw; c++) {
      p.src[g][c] = (const uint64_t *)regions[g * nw + c].data;
      if (!p.src[g][c]) { set_error("tq_region_gather: region %d column %d has no data", g, c); return TQ_ERR_INVALID_ARG; }
    }
  for (int c = 0; c < n_cols; c++) {
    p.out[c] = (uint64_t *)out_cols[c].data;
    p.out_bm[c] = (uint32_t *)out_cols[c].null_bitmap;
    if (!p.out[c]) { set_error("tq_region_gather: output column %d has no data", c); return TQ_ERR_INVALID_ARG; }
  }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.compute;
  static DevBuf d_total;
  static PinBuf h_total;
  TQ_TRY(d_total.reserve(8));
  TQ_TRY(h_total.reserve(8));
  p.total = d_total.as<unsigned long long>();
  const int64_t blocks = (out_cap + 255) / 256, cap = (int64_t)r.sm_count * 8;
  TQ_LAUNCH(k_region_gather, (unsigned)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap)), 256, 0, s, p);
  count_launch();
  TQ_TRY(check_launch("k_region_gather"));
  TQ_CUDA(cudaMemcpyAsync(h_total.p, d_total.p, 8, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  const unsigned long long total = *h_total.as<unsigned long long>();
  if (total == ~0ull) { set_error("tq_region_gather: a region overflowed (its slot reads more than %lld rows)", (long long)region_cap); return TQ_ERR_OOM; }
  if (total > (unsigned long long)out_cap) {
    set_error("tq_region_gather: %llu rows arrived, the output holds %lld", total, (long long)out_cap);
    return TQ_ERR_INVALID_ARG;
  }
  for (int c = 0; c < n_cols; c++) out_cols[c].length = (int64_t)total;
  *n_rows = (int64_t)total;
  return TQ_OK;
}
