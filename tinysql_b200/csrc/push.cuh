// push.cuh — what the region pushes share (push.cu): tq_partition_push_regions (join.cu), tq_agg_push_partial (agg.cu),
// tq_partition_push_broadcast, tq_partition_push_sample and tq_partition_push_ranges (push.cu)
// check their destinations with push_check_dests, set up their slot with push_begin, scatter into per-source regions of the
// peers' receive buffers on the push stream, then publish {rows, epoch} in each destination's slot with push_publish; the
// receiver waits on those slots with tq_region_wait.  Where the regions and slots sit is the caller's (dist.RegionLayout).
#pragma once
#include "scatter.cuh"

namespace tq {

static constexpr int PUSH_SLOTS = 16;

// The per-slot state of one push in flight: the device tables the scatter and k_publish_counts read, and the event the next
// push of the same slot (and tq_partition_push_sync) waits on before it rewrites them.
struct PushSlot {
  DevBuf cursor, lim, ovf, counts_ptrs, mask, sel;   // cursor: rows per destination (u32 x 16); ovf: u64, non-zero = overflow
  DevBuf dest, out_ptrs;                             // the GROUP BY and range pushes: destination per row, the region pointer table
  DevBuf sample[RANGE_MAX_BY][3], sample_tie;        // the sample push: per ByItem its values or offsets, cells, bitmap words; tie words
  RegionScratch region;
  PinBuf h_lim, h_ptrs, h_out_ptrs;
  cudaEvent_t ev = nullptr;
};

// The destinations of a push, checked before anything is enqueued: 1 <= n_parts <= 8, 0 <= slot < PUSH_SLOTS,
// 1 <= region_cap < 2^32, a count slot dest_counts[q] and a region dest_data[q * n_wire + c] for every destination q and wire
// column c.  A refusal sets the error text under the caller's name fn and returns TQ_ERR_INVALID_ARG.
int32_t push_check_dests(const char *fn, int n_parts, int n_wire, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                         int slot);
// Slot `slot` (checked by push_check_dests) once its previous push has finished, set up for a new push on s: its tables are
// reserved (cursor, lim, ovf, counts_ptrs, h_lim, h_ptrs), h_ptrs holds the n_parts count slots (then extra_count, when not
// null) that push_publish writes, and cursor / ovf are zeroed on s.
int32_t push_begin(int slot, int n_parts, void *const *dest_counts, void *extra_count, cudaStream_t s, PushSlot **out);
// Enqueues k_publish_counts on s — slot q (dest_counts[q], q < n_pub) gets {cursor[q] or ~0 when *ovf, epoch} — after copying
// the n_pub count-slot pointers of ps.h_ptrs to the device, and records ps.ev.
int32_t push_publish(PushSlot &ps, int n_pub, uint64_t epoch, cudaStream_t s);

// The rows word of a slot whose source failed after its arguments were checked: PUSH_FAILED | the status it returned.  Above
// every region cap, like ~0 (a region overflow), so a reader that only checks the cap refuses it too.
static constexpr uint64_t PUSH_FAILED = 0xFFFFFFFF00000000ull;
static inline bool push_failed(uint64_t rows) { return rows != ~0ull && (rows & PUSH_FAILED) == PUSH_FAILED; }
// Slot `slot` set up as push_begin does, then every count slot dest_counts[q] (q < n_parts) gets {PUSH_FAILED | status, epoch}
// on s, and ps.ev is recorded.  Writes no region.
int32_t push_publish_failure(int slot, int n_parts, void *const *dest_counts, int32_t status, uint64_t epoch, cudaStream_t s);

}  // namespace tq
