// othercond.cu — see othercond.cuh.  8-byte gathers / scatters over the result batch: HBM-bound.
#include "othercond.cuh"

namespace tq {

static int oc_grid(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// A comparison list (tq_join_set_other_conditions) lowers to [CONST] CMP FILTER per condition (join_prog_from_conds): each
// comparison reads an input register and either another input or the constant emitted just before it.  This walks that shape
// without xp_run_row's per-row register file: each operand is read from its column where the comparison needs it, and the
// first condition that fails ends the row.  The comparisons are the same functors, a NULL operand fails as the NULL result of
// the ETInt FILTER does, and comparisons raise nothing.  Measured reason (DESIGN.md §5): through the register file, which
// lives in local memory, the C3 join with a comparison list took 5 % longer.
__device__ __forceinline__ bool oc_cmp_list_passes(const OcPlan &pl, const OcCols &c, int64_t i) {
  uint64_t cval = 0;
  for (int k = 0; k < pl.prog.n_ops; k++) {
    const XOp x = pl.prog.ops[k];
    if (x.kind == TQ_X_CONST) { cval = x.imm; continue; }
    if (x.kind == TQ_X_FILTER) continue;
    const int ca = pl.prog.in_col[x.a];
    if (!tqd::bm_not_null(c.bm[ca], i)) return false;
    uint64_t v[2] = {c.data[ca][i], cval};
    if (x.b < pl.prog.n_in) {
      const int cb = pl.prog.in_col[x.b];
      if (!tqd::bm_not_null(c.bm[cb], i)) return false;
      v[1] = c.data[cb][i];
    }
    const bool nn[2] = {true, true};
    uint64_t o[1];
    bool on[1];
    unsigned e_ = 0, c_ = 0;
    if (x.kind == TQ_X_CMP_REAL) FCompareReal{x.op}(v, nn, o, on, e_, c_, true);
    else FCompareInt{x.op, (bool)(x.flags & 1), (bool)(x.flags & 2)}(v, nn, o, on, e_, c_, true);
    if (!o[0]) return false;
  }
  return true;
}

// flag: 0 = miss row of the outer join (kept as is), 1 = key match that passes, 2 = key match that fails.  Only key matches
// run the program, so miss rows raise no error and no warning (joiner.go:225-228,288-291 return before filter).
template <bool CMP_LIST>
__global__ void __launch_bounds__(256) k_oc_eval(const __grid_constant__ OcPlan pl, const __grid_constant__ OcCols c, int64_t n, uint8_t *flag,
                                                  uint32_t *surv, uint32_t *first, unsigned *d_err, unsigned long long *d_warn) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned my_err = 0, my_cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool match = pl.outer ? tqd::bm_not_null(c.bm[pl.build_key_col], i) : true;
    uint8_t f = 0;
    if (match) {
      bool pass;
      if (CMP_LIST) {
        pass = oc_cmp_list_passes(pl, c, i);
      } else {
        uint64_t rv[JP_REGS];
        uint64_t nn = 0;
        for (int k = 0; k < pl.prog.n_in; k++) {
          const int col = pl.prog.in_col[k];
          rv[k] = c.data[col][i];
          if (tqd::bm_not_null(c.bm[col], i)) nn |= 1ull << k;
        }
        bool alive;
        xp_run_row(pl.prog.ops, pl.prog.n_ops, pl.prog.n_in, rv, nn, true, alive, pass, my_err, my_cnt);
      }
      f = pass ? 1 : 2;
      if (pl.outer) {
        const uint32_t pid = (uint32_t)c.data[pl.rowid_col][i];
        if (pass) atomicAdd(&surv[pid], 1u);
        else atomicMin(&first[pid], (uint32_t)i);
      }
    }
    flag[i] = f;
  }
  if (CMP_LIST) return;
  my_err = __reduce_or_sync(0xffffffffu, my_err);
  my_cnt = __reduce_add_sync(0xffffffffu, my_cnt);
  if ((threadIdx.x & 31) == 0) {
    if (my_err) atomicOr(d_err, my_err);
    if (my_cnt) atomicAdd(d_warn, (unsigned long long)my_cnt);
  }
}

// keep[i] = 1 for rows that stay; flag 3 marks the ONE failed row of a survivor-less probe row that becomes its miss row
__global__ void __launch_bounds__(256) k_oc_decide(const OcPlan pl, const OcCols c, int64_t n, uint8_t *flag, const uint32_t *surv, const uint32_t *first,
                                                    uint32_t *keep) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint8_t f = flag[i];
    uint32_t k = (f == 0 || f == 1) ? 1u : 0u;
    if (f == 2 && pl.outer) {
      const uint32_t pid = (uint32_t)c.data[pl.rowid_col][i];
      if (surv[pid] == 0 && first[pid] == (uint32_t)i) { f = 3; k = 1; flag[i] = 3; }
    }
    keep[i] = k;
  }
}

__global__ void __launch_bounds__(256) k_oc_compact(const OcPlan pl, const OcCols c, int64_t n, const uint8_t *flag, const uint32_t *keep, const uint32_t *pos) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!keep[i]) continue;
    const uint32_t d = pos[i];
    const bool to_miss = flag[i] == 3;
    for (int col = 0; col < c.n; col++) {
      const bool build_side = col >= pl.build_lo && col < pl.build_hi;
      if (to_miss && build_side) {   // onMissMatch: the inner side becomes defaultInner
        const int bc = col - pl.build_lo;
        const bool dn = (pl.def_mask >> bc) & 1u;
        c.out_data[col][d] = dn ? pl.def_val[bc] : 0ull;
        if (dn) atomicOr(&c.out_bm[col][d >> 5], 1u << (d & 31));
        continue;
      }
      const bool nn = tqd::bm_not_null(c.bm[col], i);
      c.out_data[col][d] = nn ? c.data[col][i] : 0ull;
      if (nn) atomicOr(&c.out_bm[col][d >> 5], 1u << (d & 31));
    }
  }
}

int32_t oc_filter(const OcPlan &plan, const OcCols &cols, int64_t n, int64_t n_probe_rows, DevBuf &scratch, DevBuf &scan_scratch, int64_t *n_out,
                  unsigned *err, int64_t *div_by_zero, cudaStream_t s) {
  *n_out = 0;
  *err = 0;
  *div_by_zero = 0;
  if (n <= 0) return TQ_OK;
  if (n > 0xFFFFFFF0ll || n_probe_rows > 0xFFFFFFF0ll) { set_error("OtherConditions: result batch too large"); return TQ_ERR_INVALID_ARG; }
  // scratch: keep u32[n] | pos u32[n] | surv u32[np] | first u32[np] | {total u64, warnings u64, err u32} | flag u8[n]
  const size_t np = plan.outer ? (size_t)n_probe_rows : 0;
  const size_t words = (size_t)n * 2 + np * 2;
  const size_t total_off = (words * 4 + 7) & ~(size_t)7;
  TQ_TRY(scratch.reserve(total_off + 24 + (size_t)n + 16));
  uint32_t *keep = scratch.as<uint32_t>(), *pos = keep + n, *surv = pos + n, *first = surv + np;
  uint64_t *d_total = reinterpret_cast<uint64_t *>(scratch.as<uint8_t>() + total_off);
  unsigned long long *d_warn = reinterpret_cast<unsigned long long *>(d_total + 1);
  unsigned *d_err = reinterpret_cast<unsigned *>(d_total + 2);
  uint8_t *flag = scratch.as<uint8_t>() + total_off + 24;
  if (!plan.cmp_list) TQ_CUDA(cudaMemsetAsync(d_warn, 0, 16, s));   // comparisons raise no errors and no warnings
  if (np) {
    TQ_CUDA(cudaMemsetAsync(surv, 0, np * 4, s));
    TQ_CUDA(cudaMemsetAsync(first, 0xFF, np * 4, s));
  }
  if (plan.cmp_list) k_oc_eval<true><<<oc_grid(n), 256, 0, s>>>(plan, cols, n, flag, surv, first, d_err, d_warn);
  else k_oc_eval<false><<<oc_grid(n), 256, 0, s>>>(plan, cols, n, flag, surv, first, d_err, d_warn);
  k_oc_decide<<<oc_grid(n), 256, 0, s>>>(plan, cols, n, flag, surv, first, keep);
  count_launch(2);
  TQ_TRY(check_launch("k_oc_decide"));
  TQ_TRY(exclusive_scan_u32(keep, 1, pos, 1, n, d_total, scan_scratch, s));
  for (int c = 0; c < cols.n; c++) TQ_CUDA(cudaMemsetAsync(cols.out_bm[c], 0, bitmap_alloc_bytes(n), s));
  k_oc_compact<<<oc_grid(n), 256, 0, s>>>(plan, cols, n, flag, keep, pos);
  count_launch();
  TQ_TRY(check_launch("k_oc_compact"));
  uint64_t back[3] = {0, 0, 0};   // total, warnings, err
  TQ_CUDA(cudaMemcpyAsync(back, d_total, 24, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  *n_out = (int64_t)back[0];
  if (!plan.cmp_list) {
    *div_by_zero = (int64_t)back[1];
    *err = (unsigned)back[2];
  }
  return TQ_OK;
}

}  // namespace tq
