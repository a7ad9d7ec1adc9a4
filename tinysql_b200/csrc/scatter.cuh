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
// [off[i], off[i + 1]) of `bytes`); on the wire its area is the region's cap + 1 offsets and its cells go to a byte area of
// byte_cap bytes.
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

}  // namespace tq
