// scatter.cuh — the radix scatter of join.cu (4096-row tiles counting-sorted in shared memory, full-sector stores into
// fixed per-partition slabs) exposed to the other operators.  Partition = top `pbits` bits of mix64(key).
#pragma once
#include <vector>

#include "common.cuh"

namespace tq {

// Scatters n rows of `n_cols` (1..4) NULL-free 8-byte columns by the hash of column `key_col` into 2^pbits slabs.
// out[c]: slab storage; lo / hi / lim (u32 per partition): first row, one past the last row written, slab end.
// *d_overflow (device u64, caller-zeroed) becomes non-zero when a slab was too small (skewed keys): the caller must
// then fall back to a path that does not depend on the slabs.
int32_t scatter_rows_by_hash(const DCol *cols, int n_cols, int key_col, int64_t n, int pbits, std::vector<DevBuf> &out, DevBuf &lo, DevBuf &hi, DevBuf &lim,
                             unsigned long long *d_overflow, cudaStream_t s);

// The streaming variant (join_stream.cuh: TMA-fed tiles, shared-atomic ranking): rows land as array-of-structs records of n_cols
// words in ONE slab buffer (`aos`), partition = top pbits (<= 9) bits of tqd::hash_key(key).  Same lo / hi / lim / overflow contract.
int32_t scatter_rows_by_hash_aos(const DCol *cols, int n_cols, int key_col, int64_t n, int pbits, DevBuf &aos, DevBuf &lo, DevBuf &hi, DevBuf &lim,
                                 unsigned long long *d_overflow, cudaStream_t s);
static constexpr int SCATTER_AOS_MAX_PBITS = 9;

// The wire format of a nullable side of the multi-GPU push (partition.cu, k_pack_null_mask): the push scatter moves 8-byte
// words only, so the NULL bitmaps of a row travel as one more column, mask[r] bit c = "column c of row r is NOT NULL".
// sel_out[r] = selected[r] (all 1 when selected is null) AND the key column of row r is NOT NULL: the push routes on it, so a
// row with a NULL key takes the path of an unselected row.  Enqueued on s; n >= 1.
int32_t pack_null_mask(const DCol *cols, int n_cols, int key_col, const uint8_t *selected, int64_t n, uint64_t *mask, uint8_t *sel_out,
                       cudaStream_t s);

// ---- the GROUP BY push (partition.cu; tq_agg_push_partial in agg.cu)
// Destination of a partial row, a pure function of its group: h = 0, then per GROUP BY item g  h = mix64(h ^ v_g), where v_g
// is the item's 8 bytes (a REAL item with -0.0 read as +0.0) or GROUP_NULL_WORD for a NULL item; destination = (h >> 40) %
// n_parts.  One NOT NULL item gives (mix64(v) >> 40) % n_parts, the join's rank of the same key; no item (a scalar aggregate)
// gives 0.  Only placement depends on the rule — equality of groups is decided by the merge — so a collision costs nothing.
static constexpr int GROUP_MAX_ITEMS = 8;
static constexpr uint64_t GROUP_NULL_WORD = 0x4E554C4C4E554C4Cull;
// dest[r] for n >= 1 rows; items: the n_items GROUP BY columns (device), real_mask bit g = item g is REAL.  Enqueued on s.
int32_t group_dest(const DCol *items, int n_items, uint32_t real_mask, int64_t n, int n_parts, uint8_t *dest, cudaStream_t s);
// The same with var-len items: where hashes[g] is not null, item g holds string-dictionary ids and v_g = hashes[g][id] (the
// dictionary's content hash of the cell, sd_warp_hash: the same bytes give the same word on every rank).
int32_t group_dest(const DCol *items, const uint64_t *const *hashes, int n_items, uint32_t real_mask, int64_t n, int n_parts, uint8_t *dest,
                   cudaStream_t s);
static constexpr int REGION_MAXW = 63;  // wire columns before the mask word: the mask's 64 bits cover them
struct RegionScratch {
  DevBuf hist, scan, total;
  DevBuf bhist, bscan, btotal;   // var-len wire columns: cell bytes per (column, destination, chunk) and per (column, destination)
};
// Scatters n >= 1 rows of n_cols (1..63) 8-byte columns to destination dest[r] < n_parts (<= 8): row i of destination q's run
// (input order) goes to out[q * (n_cols + 1) + c][i] for every column c, the mask word (bit c = column c is NOT NULL) to
// out[q * (n_cols + 1) + n_cols][i].  out is a DEVICE table of pointers.  rows[q] (device u32) = rows destined to q,
// *overflow (device u64) = 1 when some rows[q] > cap, 0 otherwise; rows at or past cap are not written.  Enqueued on s.
int32_t scatter_to_regions(const DCol *cols, int n_cols, const uint8_t *dest, int64_t n, int n_parts, uint64_t *const *out, int64_t cap,
                           uint32_t *rows, unsigned long long *overflow, RegionScratch &sc, cudaStream_t s);
// A var-len wire column of scatter_to_regions_var: column `col` holds ids into an arena of cells (id i = bytes
// [off[i], off[i + 1]) of `bytes`); a column whose DCol has no data is its own arena (row r's id is r: a device BYTES column,
// whose offsets may start anywhere).  On the wire its area is the region's cap + 1 offsets and its cells go to a byte area
// of byte_cap bytes.
static constexpr int REGION_MAXV = 16;
struct RegionVar {
  int col;
  const int64_t *off;
  const uint8_t *bytes;
  uint64_t byte_cap;
};
// scatter_to_regions with n_var (0..REGION_MAXV) var-len columns: destination q's areas are out[q * (n_cols + 1 + n_var) + a]:
// areas 0..n_cols - 1 as above except that var-len column var[v].col gets offsets (entry 0 = 0, entry i + 1 = end of row i's
// cell; a NULL cell is empty), the mask word at n_cols, then the n_var byte areas in var[] order holding the cells in row
// order.  *overflow = 1 also when some region's cells of var[v] exceed var[v].byte_cap; no byte is written past a byte cap
// and no offset past cap + 1 words.  1 <= byte_cap < 2^32.  Enqueued on s.
int32_t scatter_to_regions_var(const DCol *cols, int n_cols, const RegionVar *var, int n_var, const uint8_t *dest, int64_t n, int n_parts,
                               uint64_t *const *out, int64_t cap, uint32_t *rows, unsigned long long *overflow, RegionScratch &sc,
                               cudaStream_t s);
// The receiving side: bitmap bm[c] (a host array of n_cols <= 63 device bitmaps) gets bit c of mask[r] for the n >= 1 rows, whole 64-row
// groups, 0 past the last row.  Enqueued on s.
int32_t expand_null_mask(const uint64_t *mask, int64_t n, int n_cols, uint32_t *const *bm, cudaStream_t s);

// ---- the broadcast push (partition.cu; tq_partition_push_broadcast in push.cu)
// The areas of one column on the wire, in order: its values (8-byte types) or its rebased offsets (BYTES), then a BYTES
// column's cells, then, on a nullable side, its 64-row bitmap words.  Returns the areas per destination.
static constexpr int BCAST_MAXC = 16;
inline int broadcast_wire_areas(int n_cols, const int32_t *types, int nullable) {
  int a = 0;
  for (int c = 0; c < n_cols; c++) a += 1 + ((types[c] & 0xFF) == TQ_TYPE_BYTES) + (nullable ? 1 : 0);
  return a;
}
// Copies n rows (0 <= n < 2^32) of the n_cols (1..BCAST_MAXC) columns to each of the n_parts (1..8) destinations, whose areas
// are dest_data[q * n_areas + a] (broadcast_wire_areas).  Types and offsets are the caller's to check.  rows[q] (device u32)
// = n for every destination; *overflow (device u64, caller-zeroed) = 1 when a BYTES column's cells exceed byte_cap[c], and
// then no destination gets that column's cells.  One launch, enqueued on s.
int32_t broadcast_rows(int n_cols, const tq_column *cols, const int32_t *types, int nullable, int64_t n, int n_parts, void *const *dest_data,
                       const int64_t *byte_cap, uint32_t *rows, unsigned long long *overflow, cudaStream_t s);

// ---- the range push of the multi-GPU ORDER BY (partition.cu; tq_partition_push_sample / _ranges in push.cu)
// A ByItem of the range routing: an INT64 / UINT64 / FLOAT64 column (data) or a BYTES column (offsets into data, which may
// start anywhere), its NOT-NULL bitmap or null, and its Desc flag.
static constexpr int RANGE_MAX_BY = 8;
static constexpr int RANGE_MAX_SAMPLES = 1 << 16;
struct RangeBy {
  int type, desc;
  const uint64_t *data;
  const int64_t *off;
  const uint8_t *bytes;
  const uint32_t *bm;
};
// The tie word of row r of rank src_rank's shard: the last, ascending ByItem of the routing order, which makes it a total
// order that agrees with the global (rank-major, stable) sort order.
__host__ __device__ __forceinline__ uint64_t range_tie(int src_rank, uint64_t r) { return ((uint64_t)src_rank << 32) | r; }
// Row j (0 <= j < m = min(n, n_samples)) of the sample of a shard of n rows: a hashed position inside stratum
// [j n / m, (j + 1) n / m), so the m positions are distinct (the sampled cells never exceed the shard's) and a periodic input
// does not alias with the strata.
__host__ __device__ __forceinline__ uint64_t range_sample_pos(uint64_t seed, int src_rank, int64_t j, int64_t n, int64_t m) {
  const int64_t lo = (int64_t)((uint64_t)j * (uint64_t)n / (uint64_t)m);          // < 2^16 x 2^32: no overflow
  const int64_t hi = (int64_t)((uint64_t)(j + 1) * (uint64_t)n / (uint64_t)m);
  return (uint64_t)lo + tqd::mix64(seed ^ tqd::mix64(range_tie(src_rank, (uint64_t)j))) % (uint64_t)(hi - lo);
}
// The sample of a shard: for each sampled row j, every ByItem's value — out[b] = m words for an 8-byte item; for BYTES
// out_off[b] = m + 1 offsets from 0 and out_bytes[b] its cells, which are written only when they fit byte_cap[b] — its
// NOT-NULL bit (out_bm[b], 64-row words, written when the item has a bitmap) and its tie word (tie).  One CTA, enqueued on s;
// 1 <= m <= RANGE_MAX_SAMPLES.
struct SampleOut {
  uint64_t *data[RANGE_MAX_BY];
  int64_t *off[RANGE_MAX_BY];
  uint8_t *bytes[RANGE_MAX_BY];
  uint32_t *bm[RANGE_MAX_BY];
  uint64_t byte_cap[RANGE_MAX_BY];
  uint64_t *tie;
};
int32_t sample_rows(const RangeBy *by, int n_by, int64_t n, int64_t m, uint64_t seed, int src_rank, const SampleOut &out, cudaStream_t s);
// dest[r] for the n >= 1 rows of rank src_rank's shard: the number of splitters at or below (row r, its tie word) in the
// routing order.  The splitters are rows pos[0..n_split) (non-decreasing) of the sorted sample: its ByItem columns spl[] and
// its tie words spl_tie.  n_split = 0 sends every row to 0.  Enqueued on s.
int32_t range_dest(const RangeBy *rows, const RangeBy *spl, int n_by, const uint64_t *spl_tie, const int64_t *pos, int n_split, int src_rank,
                   int64_t n, uint8_t *dest, cudaStream_t s);

}  // namespace tq
