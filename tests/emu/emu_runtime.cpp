// emu_runtime.cpp — the host pieces the emulated sources link against (TEST INFRASTRUCTURE, see include/cuda_runtime.h):
// the block / warp scheduler, "device" memory = malloc, and plain serial versions of the library helpers that live in
// runtime.cu / varlen.cu of the product (cell gather, bitmap copies) — those are exercised on the GPU by the existing parity
// tests; here they only have to be correct.  The exclusive scan is not stood in for: scan.cu is compiled in.
#include <cstdarg>
#include <cstdio>

#include "common.cuh"
#include "dict.cuh"
#include "strdict.cuh"
#include "varlen.cuh"

namespace tq_emu {
dim3 t_threadIdx, t_blockIdx, t_blockDim, t_gridDim;
int cur = 0;
uint64_t warp_slot[32][32];

namespace {
constexpr size_t STACK_BYTES = 128 * 1024;
struct Fiber { ucontext_t ctx; bool done; };
std::vector<Fiber> fibers;
std::vector<char> stacks;
ucontext_t sched_ctx;
unsigned n_threads = 0;
unsigned blk_arrived = 0, warp_arrived[32];
uint64_t blk_gen = 0, warp_gen[32];
const std::function<void()> *g_body = nullptr;

void fiber_main() {
  (*g_body)();
  fibers[(size_t)cur].done = true;
  swapcontext(&fibers[(size_t)cur].ctx, &sched_ctx);
}
void yield() { swapcontext(&fibers[(size_t)cur].ctx, &sched_ctx); }
}  // namespace

void block_sync() {
  const uint64_t g = blk_gen;
  if (++blk_arrived == n_threads) { blk_arrived = 0; blk_gen++; }
  else while (blk_gen == g) yield();
}
void warp_sync() {
  const int w = cur >> 5;
  const uint64_t g = warp_gen[w];
  if (++warp_arrived[w] == 32) { warp_arrived[w] = 0; warp_gen[w]++; }
  else while (warp_gen[w] == g) yield();
}

void launch(dim3 grid, dim3 block, const std::function<void()> &body) {
  const unsigned nt = block.x;
  if (nt == 0 || nt % 32 != 0 || nt > 1024 || block.y != 1 || block.z != 1) { fprintf(stderr, "emu: block of %u x %u threads is not supported\n", block.x, block.y); abort(); }
  n_threads = nt;
  g_body = &body;
  t_blockDim = block;
  t_gridDim = grid;
  fibers.resize(nt);
  stacks.resize((size_t)nt * STACK_BYTES);
  for (unsigned by = 0; by < grid.y; by++)
    for (unsigned bx = 0; bx < grid.x; bx++) {
      t_blockIdx = dim3(bx, by, 0);
      blk_arrived = 0;
      for (int w = 0; w < 32; w++) warp_arrived[w] = 0;
      for (unsigned t = 0; t < nt; t++) {
        getcontext(&fibers[t].ctx);
        fibers[t].ctx.uc_stack.ss_sp = stacks.data() + (size_t)t * STACK_BYTES;
        fibers[t].ctx.uc_stack.ss_size = STACK_BYTES;
        fibers[t].ctx.uc_link = nullptr;
        fibers[t].done = false;
        makecontext(&fibers[t].ctx, fiber_main, 0);
      }
      unsigned remaining = nt;
      uint64_t idle_sweeps = 0;
      while (remaining) {
        const unsigned before = remaining;
        for (unsigned t = 0; t < nt; t++) {
          if (fibers[t].done) continue;
          cur = (int)t;
          t_threadIdx = dim3(t, 0, 0);
          swapcontext(&sched_ctx, &fibers[t].ctx);
          if (fibers[t].done) remaining--;
        }
        // a block whose threads wait at a barrier that can never fill (a thread left early) would spin forever
        idle_sweeps = (remaining == before) ? idle_sweeps + 1 : 0;
        if (idle_sweeps > 100000000ull) { fprintf(stderr, "emu: block (%u, %u) does not make progress\n", bx, by); abort(); }
      }
    }
}
}  // namespace tq_emu

namespace tq {

static thread_local char g_err[512];
void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int32_t cuda_fail(cudaError_t, const char *what, const char *, int) { set_error("emulated CUDA call failed: %s", what); return TQ_ERR_CUDA; }
Runtime &rt() {
  static Runtime r;
  if (!r.inited) { r.inited = true; r.device = 0; r.sm_count = 2; }   // small grids: every block is 256 OS threads
  return r;
}
int32_t ensure_init() { rt(); return TQ_OK; }
int32_t check_launch(const char *) { return TQ_OK; }
int32_t DevBuf::reserve(size_t bytes) {
  if (bytes <= cap && p) return TQ_OK;
  release();
  p = malloc(bytes ? bytes : 1);   // exact size: an out-of-bounds access of a kernel is visible to AddressSanitizer / valgrind
  if (p) memset(p, 0xA5, bytes);   // device memory is not zeroed
  cap = bytes;
  return p ? TQ_OK : TQ_ERR_OOM;
}
void DevBuf::release() { free(p); p = nullptr; cap = 0; }
int32_t PinBuf::reserve(size_t bytes) {
  if (bytes <= cap && p) return TQ_OK;
  release();
  p = malloc(bytes ? bytes : 1);
  cap = bytes;
  return p ? TQ_OK : TQ_ERR_OOM;
}
void PinBuf::release() { free(p); p = nullptr; cap = 0; }
bool is_pinned_host(const void *) { return false; }

void host_bitmap_append(uint8_t *dst, int64_t dst_off, const uint8_t *src, int64_t n) {
  for (int64_t i = 0; i < n; i++) {
    const int bit = src ? (src[i >> 3] >> (i & 7)) & 1 : 1;
    const int64_t o = dst_off + i;
    if (bit) dst[o >> 3] |= (uint8_t)(1u << (o & 7)); else dst[o >> 3] &= (uint8_t)~(1u << (o & 7));
  }
  // like the product version: the bits of the last touched byte above the appended range are cleared
  const int64_t end = dst_off + n;
  if (n > 0 && (end & 7)) dst[end >> 3] &= (uint8_t)((1u << (end & 7)) - 1);
}
void host_bitmap_extract(uint8_t *dst, const uint8_t *src, int64_t src_off, int64_t n) {
  if (n <= 0) return;
  memset(dst, 0, (size_t)((n + 7) >> 3));
  for (int64_t i = 0; i < n; i++) {
    const int64_t o = src_off + i;
    if ((src[o >> 3] >> (o & 7)) & 1) dst[i >> 3] |= (uint8_t)(1u << (i & 7));
  }
}

int32_t upload_store(const HostVarAccum &h, SideStore &st, cudaStream_t) {
  st.elem = h.elem;
  st.n = h.n;
  st.base = 0;
  st.nbytes = (int64_t)h.bytes.size();
  TQ_TRY(st.bytes.reserve(h.bytes.size() + 16));
  if (!h.bytes.empty()) memcpy(st.bytes.p, h.bytes.data(), h.bytes.size());
  if (h.elem == 0) {
    TQ_TRY(st.offsets.reserve(h.off.size() * 8));
    memcpy(st.offsets.p, h.off.data(), h.off.size() * 8);
  }
  return TQ_OK;
}
int32_t iota_u64(uint64_t *dst, int64_t n, cudaStream_t) { for (int64_t i = 0; i < n; i++) dst[i] = (uint64_t)i; return TQ_OK; }
int32_t widen_f32(const uint32_t *src, int64_t n, uint64_t *dst, cudaStream_t) {
  for (int64_t i = 0; i < n; i++) { float f; memcpy(&f, &src[i], 4); const double d = (double)f; memcpy(&dst[i], &d, 8); }
  return TQ_OK;
}
int32_t narrow_f64(const uint64_t *src, int64_t n, uint32_t *dst, cudaStream_t) {
  for (int64_t i = 0; i < n; i++) { double d; memcpy(&d, &src[i], 8); const float f = (float)d; memcpy(&dst[i], &f, 4); }
  return TQ_OK;
}
int32_t gather_cells(const SideStore &st, const uint64_t *rowids, const uint32_t *bm, int64_t n, VarOut &out, DevBuf &, DevBuf &, cudaStream_t) {
  out.used = true;
  out.on_host = false;
  out.elem = st.elem;
  auto nn = [&](int64_t i) { return bm == nullptr || ((bm[i >> 5] >> (i & 31)) & 1u); };
  if (st.elem == 4) {
    TQ_TRY(out.bytes.reserve((size_t)(n ? n : 1) * 4));
    for (int64_t i = 0; i < n; i++) out.bytes.as<uint32_t>()[i] = nn(i) ? st.bytes.as<uint32_t>()[rowids[i]] : 0u;
    out.total = n * 4;
    return TQ_OK;
  }
  TQ_TRY(out.off.reserve((size_t)(n + 1) * 8));
  const int64_t *off = st.offsets.as<int64_t>();
  int64_t total = 0;
  for (int64_t i = 0; i < n; i++) if (nn(i)) total += off[rowids[i] + 1] - off[rowids[i]];
  TQ_TRY(out.bytes.reserve((size_t)total + 16));
  int64_t run = 0;
  for (int64_t i = 0; i < n; i++) {
    out.off.as<int64_t>()[i] = run;
    if (!nn(i)) continue;
    const int64_t s0 = off[rowids[i]], len = off[rowids[i] + 1] - s0;
    memcpy(out.bytes.as<uint8_t>() + run, st.bytes.as<uint8_t>() + (s0 - st.base), (size_t)len);
    run += len;
  }
  out.off.as<int64_t>()[n] = run;
  out.total = run;
  return TQ_OK;
}

}  // namespace tq

extern "C" int32_t tq_last_error(char *buf, int32_t buf_len) {
  if (!buf || buf_len <= 0) return TQ_ERR_INVALID_ARG;
  snprintf(buf, (size_t)buf_len, "%s", tq::g_err);
  return TQ_OK;
}

// The library's placement hashes themselves (common.cuh), for tests/test_hash_targets.py: the key-aiming edge tests restate
// them in Python, and this is what keeps the restatement honest.  Test-only exports, not part of the product ABI.
extern "C" uint64_t tq_emu_hash_key(uint64_t k) { return tqd::hash_key(k); }
extern "C" uint64_t tq_emu_mix64(uint64_t k) { return tqd::mix64(k); }

// "device" memory is host memory here
extern "C" int32_t tq_init(int32_t) { return TQ_OK; }
extern "C" int32_t tq_memcpy_d2h(void *dst, const void *src, size_t bytes) { if (bytes) memcpy(dst, src, bytes); return TQ_OK; }
extern "C" int32_t tq_memcpy_h2d(void *dst, const void *src, size_t bytes) { if (bytes) memcpy(dst, src, bytes); return TQ_OK; }
extern "C" int32_t tq_memcpy_d2d(void *dst, const void *src, size_t bytes) { if (bytes) memcpy(dst, src, bytes); return TQ_OK; }
extern "C" int32_t tq_memset_device(void *dst, int32_t v, size_t bytes) { if (bytes) memset(dst, v, bytes); return TQ_OK; }
extern "C" int32_t tq_device_alloc(size_t bytes, void **out) { *out = malloc(bytes ? bytes : 1); return *out ? TQ_OK : TQ_ERR_OOM; }
extern "C" int32_t tq_device_free(void *p) { free(p); return TQ_OK; }

// The key dictionaries (dict.cu, strdict.cu), for tests/test_emu_dicts.py: the string hash of one byte range through k_sd_hash,
// and thin handles that encode one batch of a StringDict / MultiKeyEncoder and report the table geometry it grew to.
// Test-only exports, not part of the product ABI.
namespace tq {
void k_sd_hash(const StrView v, const uint32_t *bm, int64_t n, uint64_t *row_hash);
}
extern "C" uint64_t tq_emu_sd_hash(const uint8_t *bytes, int64_t len) {
  const int64_t off[2] = {0, len};
  tq::StrView v;
  v.off = off;
  v.bytes = bytes;
  uint64_t h = 0;
  TQ_LAUNCH(tq::k_sd_hash, 1, 32, 0, nullptr, v, nullptr, 1, &h);
  return h;
}

extern "C" void *tq_emu_sd_new() { return new tq::StringDict(); }
extern "C" void tq_emu_sd_free(void *d) { delete static_cast<tq::StringDict *>(d); }
// cells r = bytes[off[r], off[r + 1]); bm: optional NOT-NULL bitmap (32-bit words).  out_geom = {count, n_slots}.
extern "C" int32_t tq_emu_sd_encode(void *d, const int64_t *off, const uint8_t *bytes, const uint32_t *bm, int64_t n, int32_t insert, uint64_t *ids_out,
                                    uint32_t *valid_out, uint64_t *out_geom) {
  auto *sd = static_cast<tq::StringDict *>(d);
  tq::StrView v;
  v.off = off;
  v.base = 0;
  v.bytes = bytes;
  const int32_t rc = sd->encode(v, bm, n, n > 0 ? off[n] - off[0] : 0, insert != 0, ids_out, valid_out, nullptr);
  out_geom[0] = sd->count;
  out_geom[1] = sd->n_slots;
  return rc;
}

extern "C" void *tq_emu_mk_new(int32_t k) {
  auto *e = new tq::MultiKeyEncoder();
  e->k = k;
  return e;
}
extern "C" void tq_emu_mk_free(void *e) { delete static_cast<tq::MultiKeyEncoder *>(e); }
// cols[i] / bms[i]: column i of the k key columns (bms[i] may be null).  out_geom = {count, n_slots} of col[0..k) followed by
// those of the pair dictionaries fold[1..k-1).
extern "C" int32_t tq_emu_mk_encode(void *h, const uint64_t *const *cols, const uint32_t *const *bms, const uint8_t *no_signbit, int64_t n, int32_t insert,
                                    int32_t null_is_value, uint64_t *out_comb, uint32_t *out_bm, uint64_t *out_geom) {
  auto *e = static_cast<tq::MultiKeyEncoder *>(h);
  tq::DCol kc[tq::MK_MAX_KEYS];
  bool ns[tq::MK_MAX_KEYS] = {};
  for (int i = 0; i < e->k && i < tq::MK_MAX_KEYS; i++) {
    kc[i].data = cols[i];
    kc[i].bm = bms ? bms[i] : nullptr;
    ns[i] = no_signbit && no_signbit[i];
  }
  const int32_t rc = e->encode(kc, ns, n, insert != 0, null_is_value != 0, out_comb, out_bm, nullptr);
  int g = 0;
  for (int i = 0; i < e->k; i++) { out_geom[g++] = e->col[i].count; out_geom[g++] = e->col[i].n_slots; }
  for (int i = 1; i < e->k - 1; i++) { out_geom[g++] = e->fold[i].count; out_geom[g++] = e->fold[i].n_slots; }
  return rc;
}
