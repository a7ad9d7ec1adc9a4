// expr.cu — vectorized builtin kernels (replaces expression/builtin_*_vec*.go vecEvalInt/vecEvalReal)
// and their C-ABI.  All kernels are HBM-streaming maps: 128-bit coalesced loads of the operand
// columns, null-bitmap words assembled with warp REDUX, 128-bit stores of the result column.
// No tensor cores: nothing here is a contraction.
#include <cstring>
#include <cstdint>

#include "expr_prog.cuh"

namespace tq {

static constexpr int MAP_THREADS = 256;
static constexpr int MAP_UNROLL = 4;        // independent 64-row groups in flight per warp
static constexpr int MAX_IN_LIST = 32;
static constexpr int64_t SLAB_ROWS = 1 << 22;  // host-path slab: 4M rows = 32 MiB per column

template <int NIN> struct InCols {
  const uint64_t *d[NIN];
  const uint32_t *bm[NIN];
};
template <int NOUT> struct OutCols {
  uint64_t *d[NOUT];
  uint32_t *bm[NOUT];
};

// Generic row-wise map.  A warp owns 64-row groups; lane l holds rows 2l, 2l+1 of the group, so every
// load/store instruction of the warp is one contiguous 512-byte run and the 64 result null bits are two
// REDUX.OR words written as a single 8-byte store.
template <int NIN, int NOUT, typename F>
__global__ void __launch_bounds__(MAP_THREADS) k_map(InCols<NIN> in, OutCols<NOUT> out, int64_t n, F f, unsigned *err,
                                                      unsigned long long *counter) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n_groups = (n + 63) >> 6;
  unsigned my_err = 0;
  unsigned my_cnt = 0;
  for (int64_t g0 = warp_global * MAP_UNROLL; g0 < n_groups; g0 += n_warps * MAP_UNROLL) {
    ulonglong2 v[MAP_UNROLL][NIN];
    uint32_t w[MAP_UNROLL][NIN];
#pragma unroll
    for (int u = 0; u < MAP_UNROLL; u++) {
      const int64_t g = g0 + u;
      const int64_t r0 = g * 64 + 2 * lane;
#pragma unroll
      for (int k = 0; k < NIN; k++) {
        v[u][k] = make_ulonglong2(0, 0);
        w[u][k] = 0xffffffffu;
        if (g < n_groups) {
          if (r0 + 1 < n) v[u][k] = tqd::ld_stream_u64x2(in.d[k] + r0);
          else if (r0 < n) v[u][k].x = in.d[k][r0];
          if (in.bm[k]) w[u][k] = in.bm[k][g * 2 + (lane >> 4)];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < MAP_UNROLL; u++) {
      const int64_t g = g0 + u;
      if (g >= n_groups) break;  // warp-uniform
      const int64_t r0 = g * 64 + 2 * lane;
      uint64_t o[2][NOUT];
      unsigned bits[NOUT];
#pragma unroll
      for (int q = 0; q < NOUT; q++) bits[q] = 0;
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const bool active = (r0 + e) < n;
        uint64_t iv[NIN];
        bool inn[NIN];
#pragma unroll
        for (int k = 0; k < NIN; k++) {
          iv[k] = e ? v[u][k].y : v[u][k].x;
          inn[k] = active && ((w[u][k] >> ((2 * lane + e) & 31)) & 1u);
        }
        bool onn[NOUT];
        f(iv, inn, o[e], onn, my_err, my_cnt, active);
#pragma unroll
        for (int q = 0; q < NOUT; q++) bits[q] |= (active && onn[q]) ? (1u << e) : 0u;
      }
#pragma unroll
      for (int q = 0; q < NOUT; q++) {
        if (r0 + 1 < n) tqd::st_stream_u64x2(out.d[q] + r0, make_ulonglong2(o[0][q], o[1][q]));
        else if (r0 < n) out.d[q][r0] = o[0][q];
        const unsigned sh = bits[q] << ((2 * lane) & 31);
        const unsigned lo = __reduce_or_sync(0xffffffffu, lane < 16 ? sh : 0u);
        const unsigned hi = __reduce_or_sync(0xffffffffu, lane >= 16 ? sh : 0u);
        if (lane == 0) *reinterpret_cast<uint2 *>(out.bm[q] + g * 2) = make_uint2(lo, hi);
      }
    }
  }
  if (my_err) atomicOr(err, my_err);
  if (counter) {
    unsigned c = __reduce_add_sync(0xffffffffu, my_cnt);
    if (lane == 0 && c) atomicAdd(counter, (unsigned long long)c);
  }
}

// ------------------------------------------------------------------ functors (the builtins are in expr_prog.cuh)
struct FLtPlus {  // config C2: (a < b, a + b) in one pass over a and b
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[2], bool (&onn)[2],
                                             unsigned &err, unsigned &, bool) const {
    const bool both = nn[0] && nn[1];
    onn[0] = both; onn[1] = both;
    o[0] = (uint64_t)((int64_t)v[0] < (int64_t)v[1]);
    o[1] = 0;
    if (both) {
      if (add_overflows_ss((int64_t)v[0], (int64_t)v[1])) err |= ERR_BIGINT;
      o[1] = v[0] + v[1];
    }
  }
};

// IN has a variable number of list columns: its own kernel, same row mapping.
struct InList {
  int n;
  bool ua;
  bool real;   // builtinInRealSig: operands are DOUBLE, equality is types.CompareFloat64 == 0 (builtin_other_vec_generated.go:151-204)
  const uint64_t *d[MAX_IN_LIST];
  const uint32_t *bm[MAX_IN_LIST];
  bool u[MAX_IN_LIST];
};
__global__ void __launch_bounds__(MAP_THREADS) k_in_int(const uint64_t *a, const uint32_t *abm, InList L, uint64_t *out, uint32_t *obm,
                                                         int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n_groups = (n + 63) >> 6;
  for (int64_t g = warp_global; g < n_groups; g += n_warps) {
    const int64_t r0 = g * 64 + 2 * lane;
    unsigned bits = 0;
    uint64_t res[2] = {0, 0};
    for (int e = 0; e < 2; e++) {                                   // builtin_other_vec_generated.go:42-94
      const int64_t r = r0 + e;
      if (r >= n) continue;
      const bool ann = tqd::bm_not_null(abm, r);
      const int64_t x = (int64_t)a[r];
      bool has_null = false, found = false;
      for (int j = 0; j < L.n; j++) {
        if (!ann || !tqd::bm_not_null(L.bm[j], r)) { has_null = true; continue; }
        const int64_t y = (int64_t)L.d[j][r];
        bool eq;
        if (L.real) eq = __longlong_as_double(x) == __longlong_as_double(y);
        else if (L.ua == L.u[j]) eq = (x == y);
        else if (!L.ua) eq = (x >= 0 && y == x);
        else eq = (y >= 0 && y == x);
        found |= eq;
      }
      res[e] = found ? 1 : 0;
      if (found || !has_null) bits |= 1u << e;
    }
    if (r0 + 1 < n) tqd::st_stream_u64x2(out + r0, make_ulonglong2(res[0], res[1]));
    else if (r0 < n) out[r0] = res[0];
    const unsigned sh = bits << ((2 * lane) & 31);
    const unsigned lo = __reduce_or_sync(0xffffffffu, lane < 16 ? sh : 0u);
    const unsigned hi = __reduce_or_sync(0xffffffffu, lane >= 16 ? sh : 0u);
    if (lane == 0) *reinterpret_cast<uint2 *>(obm + g * 2) = make_uint2(lo, hi);
  }
}

__global__ void k_filter_int(const uint64_t *a, const uint32_t *abm, uint8_t *sel, int64_t n, int real) {
  // VecEvalBool + toBool (expression/expression.go:205-326): selected = !isNull && value != 0;
  // ETReal: "zero" is types.RoundFloat(f) == 0 (types/helper.go:28-34), i.e. |f| < 0.5 — NaN rounds to NaN, which is not zero
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    bool nz;
    if (real) nz = !(fabs(__longlong_as_double((long long)a[i])) < 0.5);
    else nz = a[i] != 0;
    sel[i] = (uint8_t)(tqd::bm_not_null(abm, i) && nz);
  }
}

// ------------------------------------------------------------------ fused expression program
// Selection + Projection in one pass over the chunk (executor/executor.go SelectionExec.Next :463-499 →
// expression.VectorizedFilter chunk_executor.go:196-245, VecEvalBool expression.go:205-279; ProjectionExec →
// evalOneVec chunk_executor.go).  The host lowers the expression trees to a straight-line register program over
// the builtin functors, run per row by xp_run_row (expr_prog.cuh); every intermediate column the reference materialises (one chunk.Column per builtin,
// globalColumnAllocator) stays in a per-row register file here, so the HBM traffic is the input columns once and
// the output columns once.  Register k < n_in is input column k; register n_in + i is the result of op i.
struct ExprProg {
  int n_in, n_ops, n_out;
  const uint64_t *in_d[XP_MAX_IN];
  const uint32_t *in_bm[XP_MAX_IN];
  uint64_t *out_d[XP_MAX_OUT];
  uint32_t *out_bm[XP_MAX_OUT];
  int out_reg[XP_MAX_OUT];
  uint8_t *selected;
  XOp ops[XP_MAX_OPS];
};

__global__ void __launch_bounds__(MAP_THREADS) k_expr_prog(const __grid_constant__ ExprProg P, int64_t n, unsigned *err,
                                                            unsigned long long *counter) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n_groups = (n + 63) >> 6;
  unsigned my_err = 0, my_cnt = 0;
  for (int64_t g = warp_global; g < n_groups; g += n_warps) {
    const int64_t r0 = g * 64 + 2 * lane;
    ulonglong2 iv[XP_MAX_IN];
    uint32_t iw[XP_MAX_IN];
#pragma unroll
    for (int k = 0; k < XP_MAX_IN; k++) {
      iv[k] = make_ulonglong2(0, 0);
      iw[k] = 0xffffffffu;
      if (k < P.n_in) {
        if (r0 + 1 < n) iv[k] = tqd::ld_stream_u64x2(P.in_d[k] + r0);
        else if (r0 < n) iv[k].x = P.in_d[k][r0];
        if (P.in_bm[k]) iw[k] = P.in_bm[k][g * 2 + (lane >> 4)];
      }
    }
    uint64_t o[2][XP_MAX_OUT];
    unsigned bits[XP_MAX_OUT];
    unsigned selbits = 0;
#pragma unroll
    for (int q = 0; q < XP_MAX_OUT; q++) bits[q] = 0;
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const bool active = (r0 + e) < n;
      uint64_t rv[XP_REGS];
      uint64_t nn = 0;               // bit r: register r is not NULL
#pragma unroll
      for (int k = 0; k < XP_MAX_IN; k++) {
        rv[k] = e ? iv[k].y : iv[k].x;
        if (active && ((iw[k] >> ((2 * lane + e) & 31)) & 1u)) nn |= 1ull << k;
      }
      bool alive, sel;
      xp_run_row(P.ops, P.n_ops, P.n_in, rv, nn, active, alive, sel, my_err, my_cnt);
#pragma unroll
      for (int q = 0; q < XP_MAX_OUT; q++) {
        if (q < P.n_out) {
          o[e][q] = rv[P.out_reg[q]];
          bits[q] |= (active && ((nn >> P.out_reg[q]) & 1)) ? (1u << e) : 0u;
        }
      }
      selbits |= sel ? (1u << e) : 0u;
    }
#pragma unroll
    for (int q = 0; q < XP_MAX_OUT; q++) {
      if (q < P.n_out) {
        if (r0 + 1 < n) tqd::st_stream_u64x2(P.out_d[q] + r0, make_ulonglong2(o[0][q], o[1][q]));
        else if (r0 < n) P.out_d[q][r0] = o[0][q];
        const unsigned sh = bits[q] << ((2 * lane) & 31);
        const unsigned lo = __reduce_or_sync(0xffffffffu, lane < 16 ? sh : 0u);
        const unsigned hi = __reduce_or_sync(0xffffffffu, lane >= 16 ? sh : 0u);
        if (lane == 0) *reinterpret_cast<uint2 *>(P.out_bm[q] + g * 2) = make_uint2(lo, hi);
      }
    }
    if (P.selected) {
      if (r0 < n) P.selected[r0] = (uint8_t)(selbits & 1u);
      if (r0 + 1 < n) P.selected[r0 + 1] = (uint8_t)(selbits >> 1);
    }
  }
  if (my_err) atomicOr(err, my_err);
  if (counter) {
    unsigned c = __reduce_add_sync(0xffffffffu, my_cnt);
    if (lane == 0 && c) atomicAdd(counter, (unsigned long long)c);
  }
}

// ------------------------------------------------------------------ host driver
// Device scratch for the host (cgo) path: a ring of two slab sets so the H2D copy of slab i+1, the
// kernel of slab i and the D2H copy of slab i-1 overlap.
struct SlabSet {
  DevBuf in_d[3 + MAX_IN_LIST], in_bm[3 + MAX_IN_LIST], out_d[4], out_bm[4], sel_d;
  cudaEvent_t ev_h2d = nullptr, ev_k = nullptr, ev_d2h = nullptr;
  bool used = false;
};
struct ExprScratch {
  SlabSet set[2];
  DevBuf err;  // unsigned err[2] + u64 counter
  PinBuf err_host;
  bool ready = false;
};
static ExprScratch &scratch() {
  static ExprScratch s;
  return s;
}
static int32_t scratch_init() {
  ExprScratch &s = scratch();
  if (s.ready) return TQ_OK;
  for (int i = 0; i < 2; i++) {
    TQ_CUDA(cudaEventCreateWithFlags(&s.set[i].ev_h2d, cudaEventDisableTiming));
    TQ_CUDA(cudaEventCreateWithFlags(&s.set[i].ev_k, cudaEventDisableTiming));
    TQ_CUDA(cudaEventCreateWithFlags(&s.set[i].ev_d2h, cudaEventDisableTiming));
  }
  TQ_TRY(s.err.reserve(16));
  TQ_TRY(s.err_host.reserve(16));
  s.ready = true;
  return TQ_OK;
}

static inline int map_grid(int64_t n) {
  const int64_t groups = (n + 63) >> 6;
  const int64_t warps_needed = (groups + MAP_UNROLL - 1) / MAP_UNROLL;
  int64_t blocks = (warps_needed * 32 + MAP_THREADS - 1) / MAP_THREADS;
  const int64_t cap = (int64_t)rt().sm_count * 8;  // 8 resident 256-thread CTAs per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

struct ErrOut {
  unsigned err = 0;
  unsigned long long counter = 0;
};

// launch(ins, in_bms, outs, out_bms, rows, err*, counter*) enqueues the kernel on rt().compute.
// RunSel: an optional n-byte selection vector next to the output columns; run_map points .dev at the device bytes
// the current launch must write (the caller's own buffer in device mode, a per-slab buffer in host mode).
struct RunSel {
  uint8_t *user = nullptr;
  uint8_t *dev = nullptr;
};
template <typename Launch>
static int32_t run_map(int64_t n, int32_t mem, int nin, const tq_column *const *ins, int nout, tq_column *const *outs, Launch launch,
                       ErrOut *eo, RunSel *rs = nullptr) {
  TQ_TRY(ensure_init());
  if (n < 0) { set_error("negative row count"); return TQ_ERR_INVALID_ARG; }
  for (int k = 0; k < nin; k++)
    if (!ins[k] || (n > 0 && !ins[k]->data)) { set_error("input column %d missing", k); return TQ_ERR_INVALID_ARG; }
  for (int q = 0; q < nout; q++)
    if (!outs[q] || (n > 0 && (!outs[q]->data || !outs[q]->null_bitmap))) { set_error("output column %d needs data and null_bitmap buffers", q); return TQ_ERR_INVALID_ARG; }
  for (int q = 0; q < nout; q++) outs[q]->length = n;
  if (n == 0) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  TQ_TRY(scratch_init());
  ExprScratch &sc = scratch();
  unsigned *d_err = sc.err.as<unsigned>();
  unsigned long long *d_cnt = reinterpret_cast<unsigned long long *>(sc.err.as<unsigned>() + 2);
  TQ_CUDA(cudaMemsetAsync(d_err, 0, 16, r.compute));

  if (mem == TQ_MEM_DEVICE) {
    // device callers hand over raw HBM pointers: the kernels move two rows per lane (16-byte accesses) and whole 64-row
    // bitmap groups (one 8-byte store / 4-byte loads), so the buffers must be aligned and the bitmaps padded as the header says
    for (int k = 0; k < nin; k++)
      if (((uintptr_t)ins[k]->data & 15) || ((uintptr_t)ins[k]->null_bitmap & 3)) {
        set_error("device input column %d: data must be 16-byte aligned, null_bitmap 4-byte aligned and padded to ((n + 63) / 64) * 8 bytes", k);
        return TQ_ERR_INVALID_ARG;
      }
    for (int q = 0; q < nout; q++)
      if (((uintptr_t)outs[q]->data & 15) || ((uintptr_t)outs[q]->null_bitmap & 7)) {
        set_error("device output column %d: data must be 16-byte aligned, null_bitmap 8-byte aligned and padded to ((n + 63) / 64) * 8 bytes", q);
        return TQ_ERR_INVALID_ARG;
      }
    const uint64_t *id[3 + MAX_IN_LIST]; const uint32_t *ib[3 + MAX_IN_LIST]; uint64_t *od[4]; uint32_t *ob[4];
    if (rs) rs->dev = rs->user;
    for (int k = 0; k < nin; k++) { id[k] = (const uint64_t *)ins[k]->data; ib[k] = (const uint32_t *)ins[k]->null_bitmap; }
    for (int q = 0; q < nout; q++) { od[q] = (uint64_t *)outs[q]->data; ob[q] = (uint32_t *)outs[q]->null_bitmap; }
    launch(id, ib, od, ob, n, d_err, d_cnt);
    count_launch();
    TQ_TRY(check_launch("k_map"));
    TQ_CUDA(cudaMemcpyAsync(sc.err_host.p, d_err, 16, cudaMemcpyDeviceToHost, r.compute));
    TQ_CUDA(cudaStreamSynchronize(r.compute));
  } else {
    int slab = 0;
    for (int64_t row0 = 0; row0 < n; row0 += SLAB_ROWS, slab++) {
      const int64_t rows = (n - row0 < SLAB_ROWS) ? (n - row0) : SLAB_ROWS;
      SlabSet &ss = sc.set[slab & 1];
      const uint64_t *id[3 + MAX_IN_LIST]; const uint32_t *ib[3 + MAX_IN_LIST]; uint64_t *od[4]; uint32_t *ob[4];
      if (ss.used) TQ_CUDA(cudaStreamWaitEvent(r.h2d, ss.ev_d2h, 0));  // previous results of this set have left
      for (int k = 0; k < nin; k++) {
        TQ_TRY(ss.in_d[k].reserve((size_t)rows * 8));
        TQ_CUDA(cudaMemcpyAsync(ss.in_d[k].p, ins[k]->data + row0 * 8, (size_t)rows * 8, cudaMemcpyHostToDevice, r.h2d));
        id[k] = ss.in_d[k].as<uint64_t>();
        ib[k] = nullptr;
        if (ins[k]->null_bitmap) {
          TQ_TRY(ss.in_bm[k].reserve(bitmap_alloc_bytes(rows)));
          TQ_CUDA(cudaMemcpyAsync(ss.in_bm[k].p, ins[k]->null_bitmap + (row0 >> 3), bitmap_bytes(rows), cudaMemcpyHostToDevice, r.h2d));
          ib[k] = ss.in_bm[k].as<uint32_t>();
        }
      }
      for (int q = 0; q < nout; q++) {
        TQ_TRY(ss.out_d[q].reserve((size_t)rows * 8));
        TQ_TRY(ss.out_bm[q].reserve(bitmap_alloc_bytes(rows)));
        od[q] = ss.out_d[q].as<uint64_t>();
        ob[q] = ss.out_bm[q].as<uint32_t>();
      }
      if (rs && rs->user) {
        TQ_TRY(ss.sel_d.reserve((size_t)rows));
        rs->dev = ss.sel_d.as<uint8_t>();
      }
      TQ_CUDA(cudaEventRecord(ss.ev_h2d, r.h2d));
      TQ_CUDA(cudaStreamWaitEvent(r.compute, ss.ev_h2d, 0));
      launch(id, ib, od, ob, rows, d_err, d_cnt);
      count_launch();
      TQ_TRY(check_launch("k_map"));
      TQ_CUDA(cudaEventRecord(ss.ev_k, r.compute));
      TQ_CUDA(cudaStreamWaitEvent(r.d2h, ss.ev_k, 0));
      for (int q = 0; q < nout; q++) {
        TQ_CUDA(cudaMemcpyAsync(outs[q]->data + row0 * 8, od[q], (size_t)rows * 8, cudaMemcpyDeviceToHost, r.d2h));
        TQ_CUDA(cudaMemcpyAsync(outs[q]->null_bitmap + (row0 >> 3), ob[q], bitmap_bytes(rows), cudaMemcpyDeviceToHost, r.d2h));
      }
      if (rs && rs->user) TQ_CUDA(cudaMemcpyAsync(rs->user + row0, rs->dev, (size_t)rows, cudaMemcpyDeviceToHost, r.d2h));
      TQ_CUDA(cudaEventRecord(ss.ev_d2h, r.d2h));
      ss.used = true;
    }
    TQ_CUDA(cudaStreamSynchronize(r.d2h));
    TQ_CUDA(cudaMemcpyAsync(sc.err_host.p, d_err, 16, cudaMemcpyDeviceToHost, r.compute));
    TQ_CUDA(cudaStreamSynchronize(r.compute));
  }
  eo->err = sc.err_host.as<unsigned>()[0];
  eo->counter = *reinterpret_cast<unsigned long long *>(sc.err_host.as<unsigned>() + 2);
  return TQ_OK;
}

template <int NIN, int NOUT, typename F>
static int32_t map_call(int64_t n, int32_t mem, const tq_column *const *ins, tq_column *const *outs, F f, bool want_counter, ErrOut *eo) {
  auto launch = [&](const uint64_t **id, const uint32_t **ib, uint64_t **od, uint32_t **ob, int64_t rows, unsigned *d_err,
                    unsigned long long *d_cnt) {
    InCols<NIN> in;
    OutCols<NOUT> out;
    for (int k = 0; k < NIN; k++) { in.d[k] = id[k]; in.bm[k] = ib[k]; }
    for (int q = 0; q < NOUT; q++) { out.d[q] = od[q]; out.bm[q] = ob[q]; }
    k_map<NIN, NOUT, F><<<map_grid(rows), MAP_THREADS, 0, rt().compute>>>(in, out, rows, f, d_err, want_counter ? d_cnt : nullptr);
  };
  return run_map(n, mem, NIN, ins, NOUT, outs, launch, eo);
}

}  // namespace tq

using namespace tq;

extern "C" {

int32_t tq_vec_compare_int(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned, const tq_column *b, int32_t b_unsigned,
                           tq_column *out, int32_t mem) {
  if (op < TQ_CMP_LT || op > TQ_CMP_NE) { set_error("bad compare op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  return map_call<2, 1>(n, mem, ins, outs, FCompareInt{op, a_unsigned != 0, b_unsigned != 0}, false, &eo);
}

int32_t tq_vec_compare_real(int32_t op, int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem) {
  if (op < TQ_CMP_LT || op > TQ_CMP_NE) { set_error("bad compare op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  return map_call<2, 1>(n, mem, ins, outs, FCompareReal{op}, false, &eo);
}

int32_t tq_vec_arith_int(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned, const tq_column *b, int32_t b_unsigned,
                         tq_column *out, int32_t mem) {
  if (op < TQ_ARITH_PLUS || op > TQ_ARITH_MUL) { set_error("bad integer arithmetic op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  TQ_TRY((map_call<2, 1>(n, mem, ins, outs, FArithInt{op, a_unsigned != 0, b_unsigned != 0}, false, &eo)));
  static const char *names[] = {"(a + b)", "(a - b)", "(a * b)"};
  return err_to_status(eo.err, names[op]);
}

int32_t tq_vec_arith_real(int32_t op, int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int64_t *div_by_zero_warnings,
                          int32_t mem) {
  if (op < TQ_ARITH_PLUS || op > TQ_ARITH_DIV) { set_error("bad real arithmetic op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  TQ_TRY((map_call<2, 1>(n, mem, ins, outs, FArithReal{op}, true, &eo)));
  if (div_by_zero_warnings) *div_by_zero_warnings = (int64_t)eo.counter;
  static const char *names[] = {"(a + b)", "(a - b)", "(a * b)", "(a / b)"};
  return err_to_status(eo.err, names[op]);
}

int32_t tq_vec_logic(int32_t op, int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem) {
  if (op != TQ_LOGIC_AND && op != TQ_LOGIC_OR) { set_error("bad logic op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  return map_call<2, 1>(n, mem, ins, outs, FLogic{op}, false, &eo);
}

int32_t tq_vec_unary(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned, tq_column *out, int32_t mem) {
  if (op < TQ_UNARY_NOT_INT || op > TQ_UNARY_ISNULL) { set_error("bad unary op %d", op); return TQ_ERR_INVALID_ARG; }
  const tq_column *ins[1] = {a}; tq_column *outs[1] = {out};
  ErrOut eo;
  TQ_TRY((map_call<1, 1>(n, mem, ins, outs, FUnary{op, a_unsigned != 0}, false, &eo)));
  return err_to_status(eo.err, "-a");
}

int32_t tq_vec_if(int64_t n, const tq_column *cond, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem) {
  const tq_column *ins[3] = {cond, a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  return map_call<3, 1>(n, mem, ins, outs, FIf{}, false, &eo);
}

int32_t tq_vec_ifnull(int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem) {
  const tq_column *ins[2] = {a, b}; tq_column *outs[1] = {out};
  ErrOut eo;
  return map_call<2, 1>(n, mem, ins, outs, FIfNull{}, false, &eo);
}

int32_t tq_vec_lt_plus_int(int64_t n, const tq_column *a, const tq_column *b, tq_column *lt_out, tq_column *plus_out, int32_t mem) {
  const tq_column *ins[2] = {a, b}; tq_column *outs[2] = {lt_out, plus_out};
  ErrOut eo;
  TQ_TRY((map_call<2, 2>(n, mem, ins, outs, FLtPlus{}, false, &eo)));
  return err_to_status(eo.err, "(a + b)");
}

static int32_t vec_in(int64_t n, const tq_column *a, int32_t a_unsigned, int32_t n_list, const tq_column *list, const int32_t *list_unsigned, tq_column *out,
                      int32_t mem, bool real) {
  if (n_list < 0 || n_list > MAX_IN_LIST) { set_error("IN list of %d columns (max %d per call)", n_list, MAX_IN_LIST); return TQ_ERR_INVALID_ARG; }
  if (n_list > 0 && (!list || (!real && !list_unsigned))) return TQ_ERR_INVALID_ARG;
  const tq_column *ins[1 + MAX_IN_LIST];
  ins[0] = a;
  for (int j = 0; j < n_list; j++) ins[1 + j] = &list[j];
  tq_column *outs[1] = {out};
  ErrOut eo;
  auto launch = [&](const uint64_t **id, const uint32_t **ib, uint64_t **od, uint32_t **ob, int64_t rows, unsigned *, unsigned long long *) {
    InList L;
    L.n = n_list; L.ua = a_unsigned != 0; L.real = real;
    for (int j = 0; j < n_list; j++) { L.d[j] = id[1 + j]; L.bm[j] = ib[1 + j]; L.u[j] = !real && list_unsigned[j] != 0; }
    const int64_t groups = (rows + 63) >> 6;
    int64_t blocks = (groups * 32 + MAP_THREADS - 1) / MAP_THREADS;
    const int64_t cap = (int64_t)rt().sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    k_in_int<<<(int)blocks, MAP_THREADS, 0, rt().compute>>>(id[0], ib[0], L, od[0], ob[0], rows);
  };
  return run_map(n, mem, 1 + n_list, ins, 1, outs, launch, &eo);
}

int32_t tq_vec_in_int(int64_t n, const tq_column *a, int32_t a_unsigned, int32_t n_list, const tq_column *list, const int32_t *list_unsigned,
                      tq_column *out, int32_t mem) {
  return vec_in(n, a, a_unsigned, n_list, list, list_unsigned, out, mem, false);
}

int32_t tq_vec_in_real(int64_t n, const tq_column *a, int32_t n_list, const tq_column *list, tq_column *out, int32_t mem) {
  return vec_in(n, a, 0, n_list, list, nullptr, out, mem, true);
}

static int32_t vec_filter(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem, int real);
int32_t tq_vec_filter_int(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem) { return vec_filter(n, a, selected, mem, 0); }
int32_t tq_vec_filter_real(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem) { return vec_filter(n, a, selected, mem, 1); }

static int32_t vec_filter(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem, int real) {
  TQ_TRY(ensure_init());
  if (n < 0 || !a || (n > 0 && (!a->data || !selected))) return TQ_ERR_INVALID_ARG;
  if (n == 0) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  const int grid = (int)((n + 255) / 256 < (int64_t)r.sm_count * 8 ? (n + 255) / 256 : (int64_t)r.sm_count * 8);
  if (mem == TQ_MEM_DEVICE) {
    k_filter_int<<<grid, 256, 0, r.compute>>>((const uint64_t *)a->data, (const uint32_t *)a->null_bitmap, selected, n, real);
    count_launch();
    TQ_TRY(check_launch("k_filter_int"));
    TQ_CUDA(cudaStreamSynchronize(r.compute));
    return TQ_OK;
  }
  DevBuf d, bm, sel;
  TQ_TRY(d.reserve((size_t)n * 8));
  TQ_TRY(sel.reserve((size_t)n));
  TQ_CUDA(cudaMemcpyAsync(d.p, a->data, (size_t)n * 8, cudaMemcpyHostToDevice, r.compute));
  const uint32_t *dbm = nullptr;
  if (a->null_bitmap) {
    TQ_TRY(bm.reserve(bitmap_alloc_bytes(n)));
    TQ_CUDA(cudaMemcpyAsync(bm.p, a->null_bitmap, bitmap_bytes(n), cudaMemcpyHostToDevice, r.compute));
    dbm = bm.as<uint32_t>();
  }
  k_filter_int<<<grid, 256, 0, r.compute>>>(d.as<uint64_t>(), dbm, sel.as<uint8_t>(), n, real);
  count_launch();
  TQ_TRY(check_launch("k_filter_int"));
  TQ_CUDA(cudaMemcpyAsync(selected, sel.p, (size_t)n, cudaMemcpyDeviceToHost, r.compute));
  TQ_CUDA(cudaStreamSynchronize(r.compute));
  return TQ_OK;
}

int32_t tq_expr_eval(int64_t n, int32_t n_inputs, const tq_column *inputs, int32_t n_ops, const tq_expr_op *ops, int32_t n_outputs,
                     const int32_t *out_regs, tq_column *outs, uint8_t *selected, int64_t *div_by_zero_warnings, int32_t mem) {
  if (n_inputs < 0 || n_inputs > XP_MAX_IN || n_ops < 0 || n_ops > XP_MAX_OPS || n_outputs < 0 || n_outputs > XP_MAX_OUT) {
    set_error("expression program: at most %d inputs, %d ops, %d outputs", XP_MAX_IN, XP_MAX_OPS, XP_MAX_OUT);
    return TQ_ERR_INVALID_ARG;
  }
  if ((n_inputs && !inputs) || (n_ops && !ops) || (n_outputs && (!out_regs || !outs)) || (!n_outputs && !selected)) {
    set_error("expression program: missing argument");
    return TQ_ERR_INVALID_ARG;
  }
  ExprProg P;
  memset(&P, 0, sizeof(P));
  P.n_in = n_inputs; P.n_ops = n_ops; P.n_out = n_outputs;
  bool want_counter = false;
  TQ_TRY(xp_decode(n_inputs, n_ops, ops, P.ops, &want_counter));
  const tq_column *ins[XP_MAX_IN]; tq_column *op[XP_MAX_OUT];
  for (int k = 0; k < n_inputs; k++) ins[k] = &inputs[k];
  for (int q = 0; q < n_outputs; q++) {
    if (out_regs[q] < 0 || out_regs[q] >= n_inputs + n_ops) { set_error("expression program: output %d names register %d", q, out_regs[q]); return TQ_ERR_INVALID_ARG; }
    P.out_reg[q] = out_regs[q];
    op[q] = &outs[q];
  }
  RunSel rs;
  rs.user = selected;
  auto launch = [&](const uint64_t **id, const uint32_t **ib, uint64_t **od, uint32_t **ob, int64_t rows, unsigned *d_err,
                    unsigned long long *d_cnt) {
    for (int k = 0; k < n_inputs; k++) { P.in_d[k] = id[k]; P.in_bm[k] = ib[k]; }
    for (int q = 0; q < n_outputs; q++) { P.out_d[q] = od[q]; P.out_bm[q] = ob[q]; }
    P.selected = rs.dev;
    k_expr_prog<<<map_grid(rows), MAP_THREADS, 0, rt().compute>>>(P, rows, d_err, want_counter ? d_cnt : nullptr);
  };
  ErrOut eo;
  TQ_TRY(run_map(n, mem, n_inputs, ins, n_outputs, op, launch, &eo, &rs));
  if (div_by_zero_warnings) *div_by_zero_warnings = (int64_t)eo.counter;
  return xp_err_to_status(eo.err, P.ops, "expression program");
}

}  // extern "C"
