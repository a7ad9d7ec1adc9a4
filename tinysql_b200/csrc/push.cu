// push.cu — the publish / wait halves of the region exchange (push.cuh), shared by the join's and the GROUP BY's pushes.
#include "push.cuh"

namespace tq {

// One 16-byte slot per (destination, table, source): {rows written, epoch}.  The count is stored first, the epoch flag after a
// system-scope fence: a receiver that sees the flag sees the count, and — the push kernel having completed before this
// kernel started — the rows.
__global__ void k_publish_counts(const uint32_t *cursor, const unsigned long long *overflow, int n_parts, unsigned long long *const *dest_slots,
                                 unsigned long long epoch) {
  const int q = threadIdx.x;
  if (q < n_parts) {
    volatile unsigned long long *slot = dest_slots[q];
    slot[0] = *overflow ? ~0ull : (unsigned long long)cursor[q];
    __threadfence_system();
    slot[1] = epoch;
  }
}

// A push that failed after its arguments were checked: every slot gets {PUSH_FAILED | status, epoch}, in the same order and
// with the same fence as k_publish_counts, so that no receiver waits for a count that will never come.
__global__ void k_publish_failure(int n_parts, unsigned long long *const *dest_slots, unsigned long long word, unsigned long long epoch) {
  const int q = threadIdx.x;
  if (q < n_parts) {
    volatile unsigned long long *slot = dest_slots[q];
    slot[0] = word;
    __threadfence_system();
    slot[1] = epoch;
  }
}

// Device-side wait for the peers: spins (bounded: ~4 s) until the n slots of this rank's table carry `epoch`.  Enqueued on the
// compute stream in front of the kernels that read the regions, so the exchange needs no host barrier.
__global__ void k_region_wait(const unsigned long long *slots, int n, unsigned long long epoch, unsigned *timed_out) {
  const int g = threadIdx.x;
  if (g >= n) return;
  const volatile unsigned long long *flag = slots + 2 * g + 1;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (*flag < epoch) {
    __nanosleep(500);
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > 4000000000ull) { atomicOr(timed_out, 1u << g); return; }
  }
}

static PushSlot g_push_slot[PUSH_SLOTS];

int32_t push_check_dests(const char *fn, int n_parts, int n_wire, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                         int slot) {
  if (!dest_data || !dest_counts || n_parts < 1 || n_parts > 8 || slot < 0 || slot >= PUSH_SLOTS || region_cap < 1 || region_cap > 0xFFFFFFF0ll) {
    set_error("%s: 1..8 destinations with their regions and count slots, slot 0..%d, 1 <= region_cap < 2^32", fn, PUSH_SLOTS - 1);
    return TQ_ERR_INVALID_ARG;
  }
  for (int q = 0; q < n_parts; q++) {
    if (!dest_counts[q]) { set_error("%s: destination %d has no count slot", fn, q); return TQ_ERR_INVALID_ARG; }
    for (int c = 0; c < n_wire; c++)
      if (!dest_data[q * n_wire + c]) { set_error("%s: destination %d has no region for wire column %d", fn, q, c); return TQ_ERR_INVALID_ARG; }
  }
  return TQ_OK;
}

int32_t push_begin(int slot, int n_parts, void *const *dest_counts, void *extra_count, cudaStream_t s, PushSlot **out) {
  PushSlot &ps = g_push_slot[slot];
  if (!ps.ev) TQ_CUDA(cudaEventCreateWithFlags(&ps.ev, cudaEventDisableTiming));
  TQ_TRY(ps.cursor.reserve(64));
  TQ_TRY(ps.lim.reserve(64));
  TQ_TRY(ps.ovf.reserve(8));
  TQ_TRY(ps.counts_ptrs.reserve(128));
  TQ_TRY(ps.h_lim.reserve(64));
  TQ_TRY(ps.h_ptrs.reserve(128));
  TQ_CUDA(cudaEventSynchronize(ps.ev));  // the previous push of this slot no longer reads the pinned tables or the scratch
  for (int q = 0; q < n_parts; q++) ps.h_ptrs.as<void *>()[q] = dest_counts[q];
  if (extra_count) ps.h_ptrs.as<void *>()[n_parts] = extra_count;
  TQ_CUDA(cudaMemsetAsync(ps.cursor.p, 0, 64, s));
  TQ_CUDA(cudaMemsetAsync(ps.ovf.p, 0, 8, s));
  *out = &ps;
  return TQ_OK;
}

int32_t push_publish(PushSlot &ps, int n_pub, uint64_t epoch, cudaStream_t s) {
  TQ_CUDA(cudaMemcpyAsync(ps.counts_ptrs.p, ps.h_ptrs.p, 128, cudaMemcpyHostToDevice, s));
  k_publish_counts<<<1, 32, 0, s>>>(ps.cursor.as<uint32_t>(), ps.ovf.as<unsigned long long>(), n_pub, ps.counts_ptrs.as<unsigned long long *>(), epoch);
  count_launch();
  TQ_TRY(check_launch("k_publish_counts"));
  TQ_CUDA(cudaEventRecord(ps.ev, s));
  return TQ_OK;
}

int32_t push_publish_failure(int slot, int n_parts, void *const *dest_counts, int32_t status, uint64_t epoch, cudaStream_t s) {
  PushSlot *ps = nullptr;
  TQ_TRY(push_begin(slot, n_parts, dest_counts, nullptr, s, &ps));
  TQ_CUDA(cudaMemcpyAsync(ps->counts_ptrs.p, ps->h_ptrs.p, 128, cudaMemcpyHostToDevice, s));
  k_publish_failure<<<1, 32, 0, s>>>(n_parts, ps->counts_ptrs.as<unsigned long long *>(), PUSH_FAILED | (uint32_t)status, epoch);
  count_launch();
  TQ_TRY(check_launch("k_publish_failure"));
  TQ_CUDA(cudaEventRecord(ps->ev, s));
  return TQ_OK;
}

}  // namespace tq

using namespace tq;

extern "C" {

int32_t tq_region_wait(const void *slots, int32_t n_sources, uint64_t epoch) {
  TQ_TRY(ensure_init());
  if (!slots || n_sources < 1 || n_sources > 32) return TQ_ERR_INVALID_ARG;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  static DevBuf timed_out;
  if (!timed_out.p) { TQ_TRY(timed_out.reserve(8)); TQ_CUDA(cudaMemsetAsync(timed_out.p, 0, 8, r.compute)); }
  k_region_wait<<<1, 32, 0, r.compute>>>(reinterpret_cast<const unsigned long long *>(slots), n_sources, epoch, timed_out.as<unsigned>());
  count_launch();
  return check_launch("k_region_wait");
}

int32_t tq_partition_push_broadcast(int32_t n_cols, const tq_column *cols, const int32_t *types, int32_t nullable, int64_t n, int32_t n_parts,
                                    void *const *dest_data, void *const *dest_counts, int64_t region_cap, const int64_t *byte_cap, int32_t slot,
                                    uint64_t epoch) {
  TQ_TRY(ensure_init());
  const char *fn = "tq_partition_push_broadcast";
  if (!cols || !types || n_cols < 1 || n_cols > BCAST_MAXC || n < 0 || n > 0xFFFFFFF0ll || n > region_cap) {
    set_error("%s: needs 1..%d columns with their types and 0 <= n <= region_cap rows", fn, BCAST_MAXC);
    return TQ_ERR_INVALID_ARG;
  }
  for (int c = 0; c < n_cols; c++) {
    const int t = types[c] & 0xFF;
    if (t != TQ_TYPE_INT64 && t != TQ_TYPE_UINT64 && t != TQ_TYPE_FLOAT64 && t != TQ_TYPE_BYTES) {
      set_error("%s: column %d has type %d: device columns are INT64, UINT64, FLOAT64 or BYTES", fn, c, types[c]);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
    const bool bytes = t == TQ_TYPE_BYTES;
    if (bytes != (cols[c].offsets != nullptr) || (n > 0 && !bytes && !cols[c].data)) {
      set_error("%s: column %d: offsets exactly on BYTES columns, data on every 8-byte column", fn, c);
      return TQ_ERR_INVALID_ARG;
    }
    if (bytes && (!byte_cap || byte_cap[c] < 0)) { set_error("%s: BYTES column %d needs byte_cap[%d] >= 0", fn, c, c); return TQ_ERR_INVALID_ARG; }
  }
  const int n_wire = broadcast_wire_areas(n_cols, types, nullable);
  TQ_TRY(push_check_dests(fn, n_parts, n_wire, dest_data, dest_counts, region_cap, slot));
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.h2d;   // the push stream, as tq_partition_push_regions
  PushSlot *ps = nullptr;
  TQ_TRY(push_begin(slot, n_parts, dest_counts, nullptr, s, &ps));
  TQ_TRY(broadcast_rows(n_cols, cols, types, nullable, n, n_parts, dest_data, byte_cap, ps->cursor.as<uint32_t>(), ps->ovf.as<unsigned long long>(), s));
  return push_publish(*ps, n_parts, epoch, s);
}

int32_t tq_partition_push_sync(int32_t slot) {
  TQ_TRY(ensure_init());
  if (slot < 0 || slot >= PUSH_SLOTS || !g_push_slot[slot].ev) return TQ_ERR_INVALID_ARG;
  TQ_CUDA(cudaEventSynchronize(g_push_slot[slot].ev));
  return TQ_OK;
}

}  // extern "C"
