// push.cuh — the slot/epoch protocol the region pushes share (push.cu): tq_partition_push_regions (join.cu) and
// tq_agg_push_partial (agg.cu) scatter into per-source regions of the peers' receive buffers on the push stream, then publish
// {rows, epoch} in each destination's slot; the receiver waits on those slots with tq_region_wait.
#pragma once
#include "scatter.cuh"

namespace tq {

static constexpr int PUSH_SLOTS = 16;

// The per-slot state of one push in flight: the device tables the scatter and k_publish_counts read, and the event the next
// push of the same slot (and tq_partition_push_sync) waits on before it rewrites them.
struct PushSlot {
  DevBuf cursor, lim, ovf, counts_ptrs, mask, sel;   // cursor: rows per destination (u32 x 16); ovf: u64, non-zero = overflow
  DevBuf dest, out_ptrs;                             // the GROUP BY push: destination per row, the region pointer table
  RegionScratch region;
  PinBuf h_lim, h_ptrs, h_out_ptrs;
  cudaEvent_t ev = nullptr;
};

// Slot `slot` (0..PUSH_SLOTS-1, checked by the caller) once its previous push has finished: its event exists, its tables are
// reserved (cursor, lim, ovf, counts_ptrs, h_lim, h_ptrs) and the caller may rewrite them.
int32_t push_slot_acquire(int slot, PushSlot **out);
// Enqueues k_publish_counts on s — slot q (dest_counts[q], q < n_pub) gets {cursor[q] or ~0 when *ovf, epoch} — after copying
// the n_pub count-slot pointers of ps.h_ptrs to the device, and records ps.ev.
int32_t push_publish(PushSlot &ps, int n_pub, uint64_t epoch, cudaStream_t s);

}  // namespace tq
