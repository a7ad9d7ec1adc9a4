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

}  // extern "C"

// The columns of a range or sample push, checked before anything is enqueued: 1..63 columns of INT64 / UINT64 / FLOAT64 /
// BYTES (TQ_ERR_UNSUPPORTED_TYPE for any other type), offsets exactly on BYTES and data on every 8-byte column, at most
// REGION_MAXV BYTES columns with 1 <= byte_cap[c] < 2^32, 0..8 ByItems naming columns; 0 <= n < 2^32, 0 <= src_rank < 2^31.
static int32_t range_check_cols(const char *fn, int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by,
                                const int32_t *by_cols, int32_t src_rank, const int64_t *byte_cap, int *n_var) {
  if (!cols || !types || n_cols < 1 || n_cols > REGION_MAXW || n < 0 || n > 0xFFFFFFF0ll || n_by < 0 || n_by > RANGE_MAX_BY || (n_by && !by_cols) ||
      src_rank < 0) {
    set_error("%s: needs 1..%d columns with their types, 0 <= n < 2^32 rows, 0..%d ByItems and src_rank >= 0", fn, REGION_MAXW, RANGE_MAX_BY);
    return TQ_ERR_INVALID_ARG;
  }
  *n_var = 0;
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
    if (bytes && (!byte_cap || byte_cap[c] < 1 || byte_cap[c] > 0xFFFFFFF0ll)) {
      set_error("%s: BYTES column %d needs 1 <= byte_cap[%d] < 2^32", fn, c, c);
      return TQ_ERR_INVALID_ARG;
    }
    *n_var += bytes;
  }
  if (*n_var > REGION_MAXV) { set_error("%s: %d BYTES columns, at most %d", fn, *n_var, REGION_MAXV); return TQ_ERR_INVALID_ARG; }
  for (int b = 0; b < n_by; b++)
    if (by_cols[b] < 0 || by_cols[b] >= n_cols) { set_error("%s: ByItems[%d] is not an input column", fn, b); return TQ_ERR_INVALID_ARG; }
  return TQ_OK;
}

static RangeBy range_by(const tq_column &c, int32_t type, int32_t desc) {
  RangeBy b{};
  b.type = type & 0xFF;
  b.desc = desc ? 1 : 0;
  b.bm = reinterpret_cast<const uint32_t *>(c.null_bitmap);
  if (b.type == TQ_TYPE_BYTES) {
    b.off = c.offsets;
    b.bytes = c.data;
  } else {
    b.data = reinterpret_cast<const uint64_t *>(c.data);
  }
  return b;
}

// The sample push once its arguments are checked: gather the m sampled rows' ByItem values, bits and tie words into the slot's
// scratch, then broadcast them (broadcast_rows) and publish.
static int32_t sample_push_rows(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                                int32_t nullable, int32_t src_rank, int64_t m, uint64_t seed, int32_t n_parts, void *const *dest_data,
                                void *const *dest_counts, const int64_t *byte_cap, int32_t slot, uint64_t epoch, cudaStream_t s) {
  PushSlot *ps = nullptr;
  TQ_TRY(push_begin(slot, n_parts, dest_counts, nullptr, s, &ps));
  if (m > 0) {
    const int nw = n_by + 1;
    RangeBy by[RANGE_MAX_BY];
    SampleOut out{};
    tq_column wire[RANGE_MAX_BY + 1] = {};
    int32_t wtypes[RANGE_MAX_BY + 1];
    int64_t wcap[RANGE_MAX_BY + 1] = {};
    const size_t bm_bytes = (size_t)((m + 255) / 256) * 32;
    for (int b = 0; b < n_by; b++) {
      const int c = by_cols[b];
      by[b] = range_by(cols[c], types[c], 0);
      DevBuf *sb = ps->sample[b];
      wtypes[b] = types[c] & 0xFF;
      wire[b].length = m;
      if (by[b].type == TQ_TYPE_BYTES) {
        TQ_TRY(sb[0].reserve((size_t)(m + 1) * 8));
        TQ_TRY(sb[1].reserve((size_t)byte_cap[c] + 16));
        out.off[b] = sb[0].as<int64_t>();
        out.bytes[b] = sb[1].as<uint8_t>();
        out.byte_cap[b] = (uint64_t)byte_cap[c];
        wcap[b] = byte_cap[c];
        wire[b].offsets = sb[0].as<int64_t>();
        wire[b].data = sb[1].as<uint8_t>();
      } else {
        TQ_TRY(sb[0].reserve((size_t)m * 8));
        out.data[b] = sb[0].as<uint64_t>();
        wire[b].data = sb[0].as<uint8_t>();
      }
      if (by[b].bm) {
        TQ_TRY(sb[2].reserve(bm_bytes));
        out.bm[b] = sb[2].as<uint32_t>();
        wire[b].null_bitmap = sb[2].as<uint8_t>();
      }
    }
    TQ_TRY(ps->sample_tie.reserve((size_t)m * 8));
    out.tie = ps->sample_tie.as<uint64_t>();
    wtypes[n_by] = TQ_TYPE_UINT64;
    wire[n_by].length = m;
    wire[n_by].data = ps->sample_tie.as<uint8_t>();
    TQ_TRY(sample_rows(by, n_by, n, m, seed, src_rank, out, s));
    TQ_TRY(broadcast_rows(nw, wire, wtypes, nullable, m, n_parts, dest_data, wcap, ps->cursor.as<uint32_t>(), ps->ovf.as<unsigned long long>(), s));
  }
  return push_publish(*ps, n_parts, epoch, s);
}

// The range push once its arguments are checked: each row's destination (k_range_dest), then the GROUP BY push's scatter into
// the regions, a BYTES column as its own arena, and publish.
static int32_t range_push_rows(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                               const int32_t *by_desc, int32_t src_rank, int32_t n_parts, const tq_column *split_cols, int n_split,
                               const int64_t *split_pos, void *const *dest_data, void *const *dest_counts, int64_t region_cap, const int64_t *byte_cap,
                               int n_var, int32_t slot, uint64_t epoch, cudaStream_t s) {
  PushSlot *ps = nullptr;
  TQ_TRY(push_begin(slot, n_parts, dest_counts, nullptr, s, &ps));
  if (n > 0) {
    const size_t tab = (size_t)n_parts * (n_cols + 1 + n_var) * 8;
    TQ_TRY(ps->out_ptrs.reserve(tab));
    TQ_TRY(ps->h_out_ptrs.reserve(tab));
    TQ_TRY(ps->dest.reserve((size_t)n));
    memcpy(ps->h_out_ptrs.p, dest_data, tab);
    TQ_CUDA(cudaMemcpyAsync(ps->out_ptrs.p, ps->h_out_ptrs.p, tab, cudaMemcpyHostToDevice, s));
    RangeBy rows[RANGE_MAX_BY], spl[RANGE_MAX_BY];
    for (int b = 0; b < n_by; b++) {
      const int c = by_cols[b];
      rows[b] = range_by(cols[c], types[c], by_desc[b]);
      if (n_split) spl[b] = range_by(split_cols[b], types[c], by_desc[b]);
    }
    const uint64_t *tie = n_split ? reinterpret_cast<const uint64_t *>(split_cols[n_by].data) : nullptr;
    TQ_TRY(range_dest(rows, spl, n_by, tie, split_pos, n_split, src_rank, n, ps->dest.as<uint8_t>(), s));
    DCol dc[REGION_MAXW];
    RegionVar var[REGION_MAXV];
    for (int c = 0, v = 0; c < n_cols; c++) {
      const bool bytes = (types[c] & 0xFF) == TQ_TYPE_BYTES;
      dc[c] = DCol{bytes ? nullptr : reinterpret_cast<const uint64_t *>(cols[c].data), reinterpret_cast<const uint32_t *>(cols[c].null_bitmap)};
      if (bytes) var[v++] = RegionVar{c, cols[c].offsets, cols[c].data, (uint64_t)byte_cap[c]};
    }
    TQ_TRY(scatter_to_regions_var(dc, n_cols, var, n_var, ps->dest.as<uint8_t>(), n, n_parts, ps->out_ptrs.as<uint64_t *>(), region_cap,
                                  ps->cursor.as<uint32_t>(), ps->ovf.as<unsigned long long>(), ps->region, s));
  }
  return push_publish(*ps, n_parts, epoch, s);
}

extern "C" {

int32_t tq_partition_push_sample(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                                 int32_t nullable, int32_t src_rank, int32_t n_samples, uint64_t seed, int32_t n_parts, void *const *dest_data,
                                 void *const *dest_counts, int64_t region_cap, const int64_t *byte_cap, int32_t slot, uint64_t epoch) {
  TQ_TRY(ensure_init());
  const char *fn = "tq_partition_push_sample";
  int n_var = 0;
  TQ_TRY(range_check_cols(fn, n_cols, cols, types, n, n_by, by_cols, src_rank, byte_cap, &n_var));
  const int64_t m = n < n_samples ? n : n_samples;
  if (n_samples < 1 || n_samples > RANGE_MAX_SAMPLES || m > region_cap) {
    set_error("%s: 1 <= n_samples <= %d and min(n, n_samples) <= region_cap", fn, RANGE_MAX_SAMPLES);
    return TQ_ERR_INVALID_ARG;
  }
  int32_t wtypes[RANGE_MAX_BY + 1];
  for (int b = 0; b < n_by; b++) wtypes[b] = types[by_cols[b]];
  wtypes[n_by] = TQ_TYPE_UINT64;
  TQ_TRY(push_check_dests(fn, n_parts, broadcast_wire_areas(n_by + 1, wtypes, nullable), dest_data, dest_counts, region_cap, slot));
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.h2d;   // the push stream, as tq_partition_push_regions
  const int32_t st = sample_push_rows(n_cols, cols, types, n, n_by, by_cols, nullable, src_rank, m, seed, n_parts, dest_data, dest_counts, byte_cap,
                                      slot, epoch, s);
  if (st != TQ_OK) push_publish_failure(slot, n_parts, dest_counts, st, epoch, s);   // every destination refuses this step
  return st;
}

int32_t tq_partition_push_ranges(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                                 const int32_t *by_desc, int32_t src_rank, int32_t n_parts, const tq_column *split_cols, int64_t split_rows,
                                 const int64_t *split_pos, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                                 const int64_t *byte_cap, int32_t slot, uint64_t epoch) {
  TQ_TRY(ensure_init());
  const char *fn = "tq_partition_push_ranges";
  int n_var = 0;
  TQ_TRY(range_check_cols(fn, n_cols, cols, types, n, n_by, by_cols, src_rank, byte_cap, &n_var));
  if ((n_by && !by_desc) || n > region_cap || split_rows < 0) {
    set_error("%s: ByItems need their Desc flags, n <= region_cap, split_rows >= 0", fn);
    return TQ_ERR_INVALID_ARG;
  }
  TQ_TRY(push_check_dests(fn, n_parts, n_cols + 1 + n_var, dest_data, dest_counts, region_cap, slot));
  const int n_split = (n_parts > 1 && split_rows > 0) ? n_parts - 1 : 0;   // no splitters: every row to destination 0
  if (n_split) {
    if (!split_cols || !split_pos) { set_error("%s: %d destinations need the splitter columns and positions", fn, n_parts); return TQ_ERR_INVALID_ARG; }
    for (int k = 0; k < n_split; k++)
      if (split_pos[k] < 0 || split_pos[k] >= split_rows || (k && split_pos[k] < split_pos[k - 1])) {
        set_error("%s: splitter positions must be non-decreasing rows of the %lld splitter rows", fn, (long long)split_rows);
        return TQ_ERR_INVALID_ARG;
      }
    for (int b = 0; b <= n_by; b++) {
      const bool bytes = b < n_by && (types[by_cols[b]] & 0xFF) == TQ_TYPE_BYTES;
      if (!split_cols[b].data && !(bytes && split_cols[b].offsets) ) { set_error("%s: splitter column %d has no data", fn, b); return TQ_ERR_INVALID_ARG; }
      if (bytes != (split_cols[b].offsets != nullptr)) { set_error("%s: splitter column %d: offsets exactly on BYTES ByItems", fn, b); return TQ_ERR_INVALID_ARG; }
    }
  }
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.h2d;
  const int32_t st = range_push_rows(n_cols, cols, types, n, n_by, by_cols, by_desc, src_rank, n_parts, split_cols, n_split, split_pos, dest_data,
                                     dest_counts, region_cap, byte_cap, n_var, slot, epoch, s);
  if (st != TQ_OK) push_publish_failure(slot, n_parts, dest_counts, st, epoch, s);
  return st;
}

int32_t tq_partition_push_sync(int32_t slot) {
  TQ_TRY(ensure_init());
  if (slot < 0 || slot >= PUSH_SLOTS || !g_push_slot[slot].ev) return TQ_ERR_INVALID_ARG;
  TQ_CUDA(cudaEventSynchronize(g_push_slot[slot].ev));
  return TQ_OK;
}

}  // extern "C"
