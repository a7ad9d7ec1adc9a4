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

}  // namespace tq
