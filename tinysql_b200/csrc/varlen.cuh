// varlen.cuh — FLOAT (4-byte) and var-len (offsets + bytes) payload columns of HashJoinExec.
//
// The join kernels move 8-byte slots.  A column of another width never takes part in key comparison (keys are the
// 8-byte types), so it is kept in a side store on the device and represented inside the join by its ROW ID (an INT64
// column carrying the original NULL bitmap).  After the probe the row ids of the result batch are gathered back into a
// column of the original layout — the device form of chunk.CopySelectedJoinRows' per-cell copy
// (util/chunk/chunk_util.go:38-66: fixed cells copy elemLen bytes, var-len cells copy data[offsets[i]:offsets[i+1]]).
#pragma once
#include <vector>

#include "common.cuh"

namespace tq {

struct SideStore {          // the cells of one column, device resident
  DevBuf offsets, bytes;    // var-len: int64 offsets[n+1] (relative to `base`) + bytes;  FLOAT: n 4-byte slots in `bytes`
  int64_t n = 0, base = 0;
  int64_t nbytes = 0;       // var-len: bytes held in `bytes`
  int elem = 0;             // 0 = var-len, 4 = FLOAT
};

struct VarOut {             // one gathered output column of a result batch
  DevBuf off, bytes;        // var-len: int64 off[n+1] starting at 0
  PinBuf h_off, h_bytes;
  int64_t total = 0;        // bytes in `bytes`
  int elem = 0;
  bool used = false, on_host = false;
};

// host staging of the cells of one FLOAT (elem 4) or var-len (elem 0) column
struct HostVarAccum {
  std::vector<int64_t> off{0};
  std::vector<uint8_t> bytes;
  int elem = 0;
  int64_t n = 0;
  void append(const tq_column &c, int64_t rows) {
    if (elem == 4) bytes.insert(bytes.end(), c.data, c.data + rows * 4);
    else {
      const int64_t base = c.offsets[0];
      for (int64_t i = 0; i < rows; i++) off.push_back(off.back() + (c.offsets[i + 1] - c.offsets[i]));
      bytes.insert(bytes.end(), c.data + base, c.data + c.offsets[rows]);
    }
    n += rows;
  }
  void reset() { off.assign(1, 0); bytes.clear(); n = 0; }
};

// Upload the staged cells of a FLOAT / var-len column into its device store (synchronises s: the source is pageable).
int32_t upload_store(const HostVarAccum &h, SideStore &st, cudaStream_t s);
int32_t iota_u64(uint64_t *dst, int64_t n, cudaStream_t s);
// dst[i] = bits of float64(src[i]) — how a FLOAT value enters key hashing / comparison (util/codec/codec.go:226-229,288-291)
int32_t widen_f32(const uint32_t *src, int64_t n, uint64_t *dst, cudaStream_t s);
// dst[i] (4-byte slot) = float32 of the float64 bits in src[i] (exact for values that came from widen_f32)
int32_t narrow_f64(const uint64_t *src, int64_t n, uint32_t *dst, cudaStream_t s);
// out = cells store[rowids[i]] for i in [0, n); a 0 bit in bm makes cell i NULL (empty).  Synchronises s.
int32_t gather_cells(const SideStore &st, const uint64_t *rowids, const uint32_t *bm, int64_t n, VarOut &out, DevBuf &lens, DevBuf &scan_scratch,
                     cudaStream_t s);

// Defined in sort.cu (the source the emulation build compiles).  Append the `rows` cells of a var-len column in DEVICE memory
// (offsets[0..rows], offsets[0] may be non-zero; data = the bytes the offsets index) to the device store st (var-len, base 0), growing its arrays by doubling.  *max_len =
// the longest appended cell.  One small read-back per call; synchronises s, so the caller may reuse its buffers on return.
// rows == 0 only makes sure an empty store has its offsets[0].  The NOT-NULL bitmap is the caller's business.
int32_t append_cells_device(SideStore &st, const int64_t *offsets, const uint8_t *data, int64_t rows, int64_t *max_len, DevBuf &meta,
                            cudaStream_t s);
// offsets[0] and offsets[rows] of a var-len column in DEVICE memory (one read-back; synchronises s)
int32_t device_cell_span(const int64_t *offsets, int64_t rows, int64_t *first, int64_t *last, cudaStream_t s);

}  // namespace tq
