// sort.cu — SortExec / TopNExec / MergeJoinExec (SURVEY §8 f3) as radix-sort / sorted-search operators.
//
//   SortExec   executor/sort.go:28-157   fetch every child chunk, sort row pointers with the ByItems comparator, emit in order
//   TopNExec   executor/sort.go:159-318  the rows [Offset, Offset + Count) of that order
//   MergeJoin  executor/merge_join.go    both children arrive sorted by the join keys; per outer row the group of inner rows
//                                        with the same key is joined in inner order, a miss emits the joiner's miss row
//
// Device design.  Rows are accumulated per column (host chunks -> one upload at eof).  Sorting never moves rows: a u32
// permutation is sorted by ONE 64-bit key word at a time with a stable LSD radix sort (8-bit digits; digit passes whose digit is
// constant over the whole input are skipped — found with one OR / AND reduction), least significant word first, so that any
// ByItems list — several columns, ASC / DESC, NULLs, strings — is a sequence of the same three kernels:
//     k_sort_keys     keys[i] = order-preserving word of row perm[i]   (int: sign flip, double: IEEE total-order map with
//                     -0 == +0, string: 8 big-endian bytes at a time + the length, NULL: a flag word; DESC: bitwise NOT)
//     k_radix_count   per-tile digit histogram (shared-memory atomics)          -> exclusive scan (digit-major)
//     k_radix_scatter stable scatter: rank inside a 256-row round = match.any peers below me in my warp + the warp prefix
// The comparator restated: chunk.GetCompareFunc (util/chunk/compare.go:27-110): NULL < everything, cmpInt64 / cmpUint64 /
// cmpFloat32 / cmpFloat64 / cmpString (bytes); SortExec.lessRow flips the sign for Desc (sort.go:115-129), which puts NULLs
// last.  sort.Slice is not stable (ties come out in any order); this sort IS stable (ties keep child order), one of the
// orders the reference may produce.
// The merge join needs no merge loop: the inner side's rows with non-NULL keys form a sorted array, every outer row finds its
// group [lower_bound, upper_bound) by binary search (k_mj_bounds), an exclusive scan of the group sizes gives each outer row
// its output range, and k_mj_expand writes (outer row, inner row) pairs — output order = outer order, inner order inside a
// group, exactly the order MergeJoinExec.joinToChunk produces (merge_join.go:246-321).
// Result columns of every chunk layout are gathered by row id (8-byte / FLOAT slots here, var-len cells by varlen.cu).
#include <algorithm>
#include <memory>
#include <vector>

#include "common.cuh"
#include "expr_prog.cuh"
#include "varlen.cuh"

using namespace tq;

namespace {

constexpr uint32_t ROW_MISS = 0xFFFFFFFFu;
constexpr int SORT_MAX_BY = 8;
constexpr int MJ_MAX_KEYS = 8;
constexpr int RADIX_THREADS = 256;
constexpr int RADIX_ITEMS = 16;
constexpr int RADIX_TILE = RADIX_THREADS * RADIX_ITEMS;

int grid_for(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// ------------------------------------------------------------------------------------------------ order-preserving words
// types.CompareInt64 / CompareUint64 / CompareFloat64 (types/compare.go) as unsigned comparisons of one word
__device__ __forceinline__ uint64_t enc_word(uint64_t v, int type) {
  if (type == TQ_TYPE_INT64) return v ^ 0x8000000000000000ull;
  if (type == TQ_TYPE_FLOAT64) {
    if ((v << 1) == 0) return 0x8000000000000000ull;          // -0.0 == +0.0
    return (v >> 63) ? ~v : (v | 0x8000000000000000ull);
  }
  return v;  // BIGINT UNSIGNED
}

enum { KS_COL8 = 0, KS_F32 = 1, KS_STR_CHUNK = 2, KS_STR_LEN = 3, KS_NULL_FLAG = 4, KS_MIX_CLASS = 5, KS_MIX_VALUE = 6 };
struct KeySrc {
  int mode;             // KS_*
  int type;             // KS_COL8 / KS_MIX_*: TQ_TYPE_* of the column
  int word;             // KS_STR_CHUNK: which 8-byte chunk of the cell
  int desc;             // ByItems.Desc: the word is inverted
  const uint64_t *d8;   // 8-byte slots
  const uint32_t *d4;   // FLOAT slots
  const int64_t *off;   // var-len: offsets[n + 1] (relative to `base`) and bytes
  const uint8_t *bytes;
  int64_t base;
  const uint32_t *bm;   // NOT-NULL bitmap or nullptr
};

__device__ __forceinline__ uint64_t key_word(const KeySrc &k, uint32_t r) {
  const bool nn = tqd::bm_not_null(k.bm, r);
  uint64_t w = 0;
  switch (k.mode) {
    case KS_COL8: if (nn) w = enc_word(k.d8[r], k.type); break;
    case KS_F32: if (nn) w = enc_word((uint64_t)__double_as_longlong((double)__uint_as_float(k.d4[r])), TQ_TYPE_FLOAT64); break;
    case KS_STR_CHUNK:
      if (nn) {
        const int64_t s0 = k.off[r] - k.base, len = k.off[r + 1] - k.off[r];
        const int64_t b0 = (int64_t)k.word * 8;
#pragma unroll
        for (int j = 0; j < 8; j++) w = (w << 8) | (uint64_t)((b0 + j < len) ? k.bytes[s0 + b0 + j] : 0);
      }
      break;
    case KS_STR_LEN: if (nn) w = (uint64_t)(k.off[r + 1] - k.off[r]); break;
    case KS_NULL_FLAG: w = nn ? 1 : 0; break;
    // a BIGINT compared with a BIGINT UNSIGNED (types.CompareInt with mixed flags): (class, value) pairs order and
    // equate the two domains exactly — negative < [0, 2^63) < unsigned >= 2^63
    case KS_MIX_CLASS:
      if (nn) { const uint64_t v = k.d8[r]; w = (k.type == TQ_TYPE_INT64) ? ((v >> 63) ? 0 : 1) : ((v >> 63) ? 2 : 1); }
      break;
    default: if (nn) w = k.d8[r]; break;   // KS_MIX_VALUE: inside a class the raw two's-complement word orders both domains
  }
  return k.desc ? ~w : w;
}

__global__ void __launch_bounds__(256) k_sort_keys(const KeySrc k, const uint32_t *__restrict__ perm, int64_t n, uint64_t *__restrict__ keys) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) keys[i] = key_word(k, perm ? perm[i] : (uint32_t)i);
}

__global__ void __launch_bounds__(256) k_iota_u32(uint32_t *dst, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = (uint32_t)i;
}

// out[0] |= every key, out[1] &= every key: a digit whose bits agree in both is constant and its pass can be skipped
__global__ void __launch_bounds__(256) k_or_and(const uint64_t *__restrict__ keys, int64_t n, unsigned long long *out) {
  uint64_t o = 0, a = ~0ull;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) { const uint64_t k = keys[i]; o |= k; a &= k; }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { o |= __shfl_xor_sync(0xffffffffu, o, d); a &= __shfl_xor_sync(0xffffffffu, a, d); }
  if ((threadIdx.x & 31) == 0) { atomicOr(out, (unsigned long long)o); atomicAnd(out + 1, (unsigned long long)a); }
}

// counts[digit * n_blocks + block] = rows of the block's tile with that digit
__global__ void __launch_bounds__(RADIX_THREADS) k_radix_count(const uint64_t *__restrict__ keys, int64_t n, int shift, uint32_t *counts, int n_blocks) {
  __shared__ uint32_t sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * RADIX_TILE;
  for (int r = 0; r < RADIX_ITEMS; r++) {
    const int64_t i = base + (int64_t)r * RADIX_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&sh[(unsigned)(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  counts[(int64_t)threadIdx.x * n_blocks + blockIdx.x] = sh[threadIdx.x];
}

// Stable scatter of one tile.  Rows are taken 256 at a time in input order; inside a round the rank of a row among the rows
// with its digit = (rows of earlier warps) + (peer lanes below it in its own warp), so equal digits keep their input order.
__global__ void __launch_bounds__(RADIX_THREADS) k_radix_scatter(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ perm, int64_t n, int shift,
                                                                 const uint32_t *__restrict__ offsets, int n_blocks, uint64_t *__restrict__ keys_out,
                                                                 uint32_t *__restrict__ perm_out) {
  __shared__ uint32_t warp_cnt[RADIX_THREADS / 32][256];
  __shared__ uint32_t run[256];   // next free output slot of each digit for this tile
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  run[tid] = offsets[(int64_t)tid * n_blocks + blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * RADIX_TILE;
  for (int r = 0; r < RADIX_ITEMS; r++) {
    if (base + (int64_t)r * RADIX_THREADS >= n) break;   // uniform over the block
#pragma unroll
    for (int ww = 0; ww < RADIX_THREADS / 32; ww++) warp_cnt[ww][tid] = 0;
    __syncthreads();
    const int64_t i = base + (int64_t)r * RADIX_THREADS + tid;
    const bool valid = i < n;
    uint64_t k = 0;
    uint32_t p = 0;
    unsigned d = 256u + (unsigned)lane;   // rows past the end match nobody
    if (valid) { k = keys[i]; p = perm[i]; d = (unsigned)(k >> shift) & 255u; }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) warp_cnt[w][d] = __popc(peers);
    __syncthreads();
    {  // thread t owns digit t: turn the per-warp counts into per-warp start slots
      uint32_t acc = run[tid];
#pragma unroll
      for (int ww = 0; ww < RADIX_THREADS / 32; ww++) { const uint32_t c = warp_cnt[ww][tid]; warp_cnt[ww][tid] = acc; acc += c; }
      run[tid] = acc;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = warp_cnt[w][d] + rank;
      keys_out[pos] = k;
      perm_out[pos] = p;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ gathers by row id
__global__ void __launch_bounds__(256) k_gather_u64(const uint64_t *__restrict__ src, const uint32_t *__restrict__ rows, int64_t m, uint64_t dflt, uint64_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) { const uint32_t r = rows[i]; out[i] = r == ROW_MISS ? dflt : src[r]; }
}
__global__ void __launch_bounds__(256) k_gather_u32(const uint32_t *__restrict__ src, const uint32_t *__restrict__ rows, int64_t m, uint32_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) { const uint32_t r = rows[i]; out[i] = r == ROW_MISS ? 0u : src[r]; }
}
// out bitmap word w = NOT-NULL bits of result rows [32w, 32w + 32): a miss row takes dflt_nn (joiner.go:139-143 defaultInner)
__global__ void __launch_bounds__(256) k_gather_bm(const uint32_t *__restrict__ src_bm, const uint32_t *__restrict__ rows, int64_t m, int dflt_nn, uint32_t *__restrict__ out, int64_t out_words) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t limit = out_words * 32;   // whole warps stay converged for the ballot
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < limit; i += stride) {
    bool nn = false;
    if (i < m) { const uint32_t r = rows[i]; nn = r == ROW_MISS ? (dflt_nn != 0) : tqd::bm_not_null(src_bm, r); }
    const unsigned word = __ballot_sync(0xffffffffu, nn);
    if ((threadIdx.x & 31) == 0) out[i >> 5] = word;
  }
}
__global__ void __launch_bounds__(256) k_rows_to_u64(const uint32_t *__restrict__ rows, int64_t m, uint64_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) { const uint32_t r = rows[i]; out[i] = r == ROW_MISS ? 0ull : (uint64_t)r; }
}

// ------------------------------------------------------------------------------------------------ merge join kernels
struct MJKeyCol {
  int is_str;
  const uint64_t *enc[2];     // [0] inner, [1] outer: order-preserving words
  const int64_t *off[2];      // strings: offsets / bytes of each side
  const uint8_t *bytes[2];
};
struct MJKeys {
  int k;
  MJKeyCol c[2 * MJ_MAX_KEYS];
};

// compareChunkRow (merge_join.go:200-208) over prepared key columns: row ra of side sa against row rb of side sb
__device__ int mj_cmp(const MJKeys &K, int sa, uint32_t ra, int sb, uint32_t rb) {
  for (int c = 0; c < K.k; c++) {
    const MJKeyCol &kc = K.c[c];
    if (!kc.is_str) {
      const uint64_t a = kc.enc[sa][ra], b = kc.enc[sb][rb];
      if (a != b) return a < b ? -1 : 1;
    } else {   // types.CompareString: bytes.Compare
      const int64_t a0 = kc.off[sa][ra], la = kc.off[sa][ra + 1] - a0, b0 = kc.off[sb][rb], lb = kc.off[sb][rb + 1] - b0;
      const uint8_t *pa = kc.bytes[sa] + a0, *pb = kc.bytes[sb] + b0;
      const int64_t m = la < lb ? la : lb;
      for (int64_t i = 0; i < m; i++) if (pa[i] != pb[i]) return pa[i] < pb[i] ? -1 : 1;
      if (la != lb) return la < lb ? -1 : 1;
    }
  }
  return 0;
}

struct BmList { int n; const uint32_t *bm[MJ_MAX_KEYS]; };
// flags[i] = 1 iff no key column of row i is NULL (hasNullInJoinKey, merge_join.go:154-162) and, outer side, the row passed
// the outer filter (selected[], merge_join.go:262)
__global__ void __launch_bounds__(256) k_mj_valid(const BmList b, const uint8_t *__restrict__ selected, int64_t n, uint32_t *__restrict__ flags) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    bool ok = selected ? selected[i] != 0 : true;
    for (int c = 0; c < b.n; c++) ok = ok && tqd::bm_not_null(b.bm[c], i);
    flags[i] = ok ? 1u : 0u;
  }
}
__global__ void __launch_bounds__(256) k_compact(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ offs, int64_t n, uint32_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) if (flags[i]) out[offs[i]] = (uint32_t)i;
}
// inner rows with usable keys must be non-decreasing (the reference relies on its children for this, merge_join.go:28-30)
__global__ void __launch_bounds__(256) k_mj_check_sorted(const MJKeys K, const uint32_t *__restrict__ ivalid, int64_t iv, unsigned *bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < iv; i += stride)
    if (mj_cmp(K, 0, ivalid[i], 0, ivalid[i + 1]) > 0) atomicAdd(bad, 1u);
}
// per outer row: its group of inner rows [lo, lo + cnt) in the compacted inner list, and how many rows it emits
__global__ void __launch_bounds__(256) k_mj_bounds(const MJKeys K, const uint32_t *__restrict__ ivalid, int64_t iv, const uint32_t *__restrict__ oflags, int64_t n_outer,
                                                   int outer_join, uint32_t *__restrict__ lo_out, uint32_t *__restrict__ cnt_out, uint32_t *__restrict__ emit_out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_outer; o += stride) {
    uint32_t lo = 0, cnt = 0;
    if (oflags[o]) {
      int64_t a = 0, b = iv;                  // lower bound: first inner >= outer
      while (a < b) { const int64_t mid = (a + b) >> 1; if (mj_cmp(K, 1, (uint32_t)o, 0, ivalid[mid]) > 0) a = mid + 1; else b = mid; }
      const int64_t lb = a;
      b = iv;                                 // upper bound: first inner > outer
      while (a < b) { const int64_t mid = (a + b) >> 1; if (mj_cmp(K, 1, (uint32_t)o, 0, ivalid[mid]) >= 0) a = mid + 1; else b = mid; }
      lo = (uint32_t)lb;
      cnt = (uint32_t)(a - lb);
    }
    lo_out[o] = lo;
    cnt_out[o] = cnt;
    emit_out[o] = cnt ? cnt : (outer_join ? 1u : 0u);   // onMissMatch emits one row for outer joins, none for inner (joiner.go)
  }
}
// result row t belongs to the last outer row whose first result row is <= t
__global__ void __launch_bounds__(256) k_mj_expand(const uint32_t *__restrict__ emit_off, const uint32_t *__restrict__ lo, const uint32_t *__restrict__ cnt,
                                                   const uint32_t *__restrict__ ivalid, int64_t n_outer, int64_t total, uint32_t *__restrict__ out_outer,
                                                   uint32_t *__restrict__ out_inner) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    int64_t a = 0, b = n_outer;               // first o with emit_off[o] > t
    while (a < b) { const int64_t mid = (a + b) >> 1; if ((int64_t)emit_off[mid] <= t) a = mid + 1; else b = mid; }
    const int64_t o = a - 1;
    const uint32_t j = (uint32_t)(t - (int64_t)emit_off[o]);
    out_outer[t] = (uint32_t)o;
    out_inner[t] = cnt[o] ? ivalid[lo[o] + j] : ROW_MISS;
  }
}

// OtherConditions of the joiner (baseJoiner.filter, executor/joiner.go:155-167) over the expanded pairs: the condition program
// (expr_prog.cuh) with input register k gathered by row id from the inner or the outer row store.  flags[t] = 1 iff pair t
// joins an inner row and the program selects it.  A ROW_MISS pair (no key match, a NULL key, an outer row the outer filter
// dropped) never runs the program, so it raises no error and no warning (joiner.go:225-228,288-291 return before filter).
struct MJProg {
  int n_in = 0, n_ops = 0;
  const uint64_t *data[JP_MAX_IN] = {};
  const uint32_t *bm[JP_MAX_IN] = {};
  int inner[JP_MAX_IN] = {};   // 1: register k comes from the inner row, 0: from the outer row
  XOp ops[XP_MAX_OPS] = {};
};
// err_warn[0] |= ERR_* bits, err_warn[1] += division-by-zero warnings of the evaluated pairs
__global__ void __launch_bounds__(256) k_mj_prog(const __grid_constant__ MJProg P, const uint32_t *__restrict__ out_outer, const uint32_t *__restrict__ out_inner,
                                                 int64_t m, uint32_t *__restrict__ flags, unsigned long long *err_warn) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned my_err = 0, my_cnt = 0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += stride) {
    const uint32_t ir = out_inner[t], orow = out_outer[t];
    bool pass = false;
    if (ir != ROW_MISS) {
      uint64_t rv[JP_REGS];
      uint64_t nn = 0;
      for (int k = 0; k < P.n_in; k++) {
        const uint32_t r = P.inner[k] ? ir : orow;
        rv[k] = P.data[k][r];
        if (tqd::bm_not_null(P.bm[k], r)) nn |= 1ull << k;
      }
      bool alive;
      xp_run_row(P.ops, P.n_ops, P.n_in, rv, nn, true, alive, pass, my_err, my_cnt);
    }
    flags[t] = pass ? 1u : 0u;
  }
  if (my_err) atomicOr(&err_warn[0], (unsigned long long)my_err);
  if (my_cnt) atomicAdd(&err_warn[1], (unsigned long long)my_cnt);
}
// rows each outer row emits once its pairs are filtered: the survivors, or the miss row of an outer join when none survived
__global__ void __launch_bounds__(256) k_mj_survivors(const uint32_t *__restrict__ emit_off, const uint32_t *__restrict__ fscan, int64_t n_outer, int64_t m, uint32_t n_pass,
                                                      int outer_join, uint32_t *__restrict__ emit2) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_outer; o += stride) {
    const int64_t lo = emit_off[o], hi = o + 1 < n_outer ? (int64_t)emit_off[o + 1] : m;
    const uint32_t s0 = lo < m ? fscan[lo] : n_pass, s1 = hi < m ? fscan[hi] : n_pass;
    const uint32_t surv = s1 - s0;
    emit2[o] = surv ? surv : (outer_join ? 1u : 0u);
  }
}
// surviving pairs keep their order inside the outer row's new range; an outer row without survivors writes its miss row
__global__ void __launch_bounds__(256) k_mj_refill_pairs(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ fscan, const uint32_t *__restrict__ emit_off,
                                                         const uint32_t *__restrict__ emit2_off, const uint32_t *__restrict__ out_outer, const uint32_t *__restrict__ out_inner,
                                                         int64_t m, uint32_t *__restrict__ new_outer, uint32_t *__restrict__ new_inner) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += stride) {
    if (!flags[t]) continue;
    const uint32_t o = out_outer[t];
    const uint32_t pos = emit2_off[o] + (fscan[t] - fscan[emit_off[o]]);
    new_outer[pos] = o;
    new_inner[pos] = out_inner[t];
  }
}
__global__ void __launch_bounds__(256) k_mj_refill_misses(const uint32_t *__restrict__ emit_off, const uint32_t *__restrict__ fscan, const uint32_t *__restrict__ emit2_off,
                                                          int64_t n_outer, int64_t m, uint32_t n_pass, int64_t m2, uint32_t *__restrict__ new_outer,
                                                          uint32_t *__restrict__ new_inner) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_outer; o += stride) {
    const int64_t lo = emit_off[o], hi = o + 1 < n_outer ? (int64_t)emit_off[o + 1] : m;
    const uint32_t s0 = lo < m ? fscan[lo] : n_pass, s1 = hi < m ? fscan[hi] : n_pass;
    const int64_t p0 = emit2_off[o], p1 = o + 1 < n_outer ? (int64_t)emit2_off[o + 1] : m2;
    if (s1 == s0 && p1 > p0) { new_outer[p0] = (uint32_t)o; new_inner[p0] = ROW_MISS; }   // only outer joins have p1 > p0 here
  }
}

// ------------------------------------------------------------------------------------------------ host side: row store
struct StoreCol {
  int type = 0;
  int kind = 0;                 // 0: 8-byte slots, 1: FLOAT slots, 2: var-len
  std::vector<uint8_t> h_data;  // kind 0 / 1
  HostVarAccum h_var;           // kind 2
  int64_t max_len = 0;          // kind 2: longest cell
  std::vector<uint8_t> h_bm;
  bool has_bm = false;
  DevBuf d_data, d_bm;
  SideStore store;
  const uint32_t *bm() const { return has_bm ? d_bm.as<uint32_t>() : nullptr; }
};

struct RowStore {
  std::vector<StoreCol> cols;
  int64_t n = 0;
  bool uploaded = false;
  bool host_mode = false, device_mode = false;   // a handle takes host chunks or device chunks, not both
  int64_t dev_cap = 0;                           // device mode: rows the columns' device arrays can hold

  int32_t init(int n_cols, const int32_t *types) {
    cols.resize((size_t)n_cols);
    for (int c = 0; c < n_cols; c++) {
      const int t = types[c] & 0xFF;
      if (t < TQ_TYPE_INT64 || t > TQ_TYPE_BYTES) { set_error("unsupport column type %d of column %d", t, c); return TQ_ERR_UNSUPPORTED_TYPE; }
      cols[c].type = t;
      cols[c].kind = t == TQ_TYPE_FLOAT32 ? 1 : (t == TQ_TYPE_BYTES ? 2 : 0);
      cols[c].h_var.elem = 0;
    }
    return TQ_OK;
  }

  // one child chunk (host memory)
  int32_t append(const tq_column *in) {
    if (cols.empty()) return TQ_OK;
    const int64_t rows = in[0].length;
    if (rows < 0) return TQ_ERR_INVALID_ARG;
    for (size_t c = 0; c < cols.size(); c++) {
      if (in[c].length != rows) { set_error("ragged input chunk"); return TQ_ERR_INVALID_ARG; }
      if (cols[c].kind == 2 && !in[c].offsets) { set_error("var-len column %d needs offsets", (int)c); return TQ_ERR_INVALID_ARG; }
      if (cols[c].kind != 2 && in[c].offsets) { set_error("unsupport column type for encode (var-len data in fixed-width column %d)", (int)c); return TQ_ERR_UNSUPPORTED_TYPE; }
      if (rows && !in[c].data && !(cols[c].kind == 2 && in[c].offsets[rows] == in[c].offsets[0])) return TQ_ERR_INVALID_ARG;
    }
    if (device_mode) { set_error("one handle takes either host chunks or device chunks"); return TQ_ERR_STATE; }
    host_mode = true;
    if (rows == 0) return TQ_OK;
    if (n + rows > 0xFFFFFFF0ll) { set_error("more than 2^32 rows in one sort / merge-join input"); return TQ_ERR_INVALID_ARG; }
    for (size_t c = 0; c < cols.size(); c++) {
      StoreCol &sc = cols[c];
      if (sc.kind == 2) {
        sc.h_var.append(in[c], rows);
        for (int64_t i = 0; i < rows; i++) sc.max_len = std::max(sc.max_len, in[c].offsets[i + 1] - in[c].offsets[i]);
      } else {
        const size_t w = sc.kind == 1 ? 4 : 8;
        sc.h_data.insert(sc.h_data.end(), in[c].data, in[c].data + (size_t)rows * w);
      }
      append_bitmap(sc, in[c].null_bitmap, rows);
    }
    n += rows;
    return TQ_OK;
  }

  // NOT-NULL bits of `rows` more rows of column sc (host bytes, bit 0 = first new row; nullptr = no NULLs)
  void append_bitmap(StoreCol &sc, const uint8_t *bits, int64_t rows) {
    if (bits && !sc.has_bm) {   // first chunk with NULL information: everything before it was NOT NULL
      sc.h_bm.assign(bitmap_alloc_bytes(n + rows), 0);
      host_bitmap_append(sc.h_bm.data(), 0, nullptr, n);
      sc.has_bm = true;
    }
    if (sc.has_bm) {
      if (sc.h_bm.size() < bitmap_alloc_bytes(n + rows)) sc.h_bm.resize(std::max(bitmap_alloc_bytes(n + rows), sc.h_bm.size() * 2), 0);
      host_bitmap_append(sc.h_bm.data(), n, bits, rows);
    }
  }

  // One chunk whose columns live in HBM (TQ_MEM_DEVICE: e.g. rows lent by tq_join_next_device).  8-byte columns only; the data
  // never leaves the device: it is appended to the column's device array (grown by doubling), only the NOT-NULL bitmap — one
  // bit per row — is read back so that chunks can be concatenated at any bit offset.  The call returns after the copies, so
  // the caller may recycle its buffers.
  int32_t append_device(const tq_column *in, cudaStream_t s) {
    if (cols.empty()) return TQ_OK;
    if (host_mode) { set_error("one handle takes either host chunks or device chunks"); return TQ_ERR_STATE; }
    const int64_t rows = in[0].length;
    if (rows < 0) return TQ_ERR_INVALID_ARG;
    for (size_t c = 0; c < cols.size(); c++) {
      if (cols[c].kind != 0 || in[c].offsets) { set_error("device chunks: 8-byte columns only (column %d)", (int)c); return TQ_ERR_UNSUPPORTED_TYPE; }
      if (in[c].length != rows) { set_error("ragged input chunk"); return TQ_ERR_INVALID_ARG; }
      if (rows && !in[c].data) return TQ_ERR_INVALID_ARG;
    }
    device_mode = true;
    if (rows == 0) return TQ_OK;
    if (n + rows > 0xFFFFFFF0ll) { set_error("more than 2^32 rows in one sort / merge-join input"); return TQ_ERR_INVALID_ARG; }
    if (n + rows > dev_cap) {
      const int64_t new_cap = std::max<int64_t>(std::max<int64_t>(n + rows, dev_cap * 2), 1 << 16);
      for (StoreCol &sc : cols) {
        DevBuf bigger;
        TQ_TRY(bigger.reserve((size_t)new_cap * 8 + 16));
        if (n) TQ_CUDA(cudaMemcpyAsync(bigger.p, sc.d_data.p, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
        TQ_CUDA(cudaStreamSynchronize(s));   // the old array goes back to the allocator's cache: nothing may still read it
        sc.d_data = std::move(bigger);
      }
      dev_cap = new_cap;
    }
    std::vector<uint8_t> bits;
    for (size_t c = 0; c < cols.size(); c++) {
      StoreCol &sc = cols[c];
      TQ_CUDA(cudaMemcpyAsync(sc.d_data.as<uint8_t>() + (size_t)n * 8, in[c].data, (size_t)rows * 8, cudaMemcpyDeviceToDevice, s));
      if (in[c].null_bitmap) {
        bits.assign(bitmap_bytes(rows), 0);
        TQ_CUDA(cudaMemcpyAsync(bits.data(), in[c].null_bitmap, bitmap_bytes(rows), cudaMemcpyDeviceToHost, s));
        TQ_CUDA(cudaStreamSynchronize(s));
        append_bitmap(sc, bits.data(), rows);
      } else append_bitmap(sc, nullptr, rows);
    }
    TQ_CUDA(cudaStreamSynchronize(s));
    n += rows;
    return TQ_OK;
  }

  int32_t upload(cudaStream_t s) {
    if (uploaded) return TQ_OK;
    for (StoreCol &sc : cols) {
      if (sc.kind == 2) TQ_TRY(upload_store(sc.h_var, sc.store, s));
      else if (!device_mode) {   // device mode: the data is in d_data already
        TQ_TRY(sc.d_data.reserve(sc.h_data.size() + 16));
        if (!sc.h_data.empty()) TQ_CUDA(cudaMemcpyAsync(sc.d_data.p, sc.h_data.data(), sc.h_data.size(), cudaMemcpyHostToDevice, s));
      }
      if (sc.has_bm) {
        const size_t nb = bitmap_alloc_bytes(n);
        sc.h_bm.resize(std::max(nb, sc.h_bm.size()), 0);
        TQ_TRY(sc.d_bm.reserve(nb));
        TQ_CUDA(cudaMemcpyAsync(sc.d_bm.p, sc.h_bm.data(), nb, cudaMemcpyHostToDevice, s));
      }
    }
    TQ_CUDA(cudaStreamSynchronize(s));   // pageable sources
    for (StoreCol &sc : cols) { std::vector<uint8_t>().swap(sc.h_data); sc.h_var.reset(); }
    uploaded = true;
    return TQ_OK;
  }
};

KeySrc key_src(const StoreCol &sc, int mode, int word, int desc) {
  KeySrc k{};
  k.mode = mode;
  k.type = sc.type;
  k.word = word;
  k.desc = desc;
  k.d8 = sc.d_data.as<uint64_t>();
  k.d4 = sc.d_data.as<uint32_t>();
  k.off = sc.store.offsets.as<int64_t>();
  k.bytes = sc.store.bytes.as<uint8_t>();
  k.base = sc.store.base;
  k.bm = sc.bm();
  return k;
}

// ------------------------------------------------------------------------------------------------ host side: result
struct ResultCol {
  int kind = 0;
  std::vector<uint8_t> data;    // 8-byte / 4-byte slots, or the cells' bytes
  std::vector<int64_t> off;     // var-len: n + 1 offsets starting at 0
  std::vector<uint8_t> bm;      // NOT-NULL bits of the n rows
};
struct ResultHost {
  std::vector<ResultCol> cols;
  int64_t n = 0, pos = 0;
};
struct GatherScratch { DevBuf out, obm, rowid64, lens, scan; VarOut var; };

// Append to `res` the columns of `st` gathered at d_rows[0, m) (ROW_MISS = the joiner's miss row: dflt / NULL)
int32_t gather_columns(const RowStore &st, const uint32_t *d_rows, int64_t m, const uint64_t *dflt_bits, const uint8_t *dflt_nn, ResultHost &res,
                       GatherScratch &g, cudaStream_t s) {
  for (size_t c = 0; c < st.cols.size(); c++) {
    const StoreCol &sc = st.cols[c];
    res.cols.emplace_back();
    ResultCol &rc = res.cols.back();
    rc.kind = sc.kind;
    const int64_t words = (m + 31) >> 5;
    rc.bm.assign(bitmap_alloc_bytes(m), 0);
    if (sc.kind == 2) rc.off.assign((size_t)m + 1, 0);
    if (m == 0) continue;
    const int nn_dflt = (sc.kind == 0 && dflt_nn) ? dflt_nn[c] : 0;
    TQ_TRY(g.obm.reserve(bitmap_alloc_bytes(m)));
    TQ_LAUNCH(k_gather_bm, grid_for(words * 32), 256, 0, s, sc.bm(), d_rows, m, nn_dflt, g.obm.as<uint32_t>(), words);
    count_launch();
    TQ_TRY(check_launch("k_gather_bm"));
    TQ_CUDA(cudaMemcpyAsync(rc.bm.data(), g.obm.p, (size_t)words * 4, cudaMemcpyDeviceToHost, s));
    if (sc.kind == 0) {
      TQ_TRY(g.out.reserve((size_t)m * 8));
      TQ_LAUNCH(k_gather_u64, grid_for(m), 256, 0, s, sc.d_data.as<uint64_t>(), d_rows, m, (dflt_bits && nn_dflt) ? dflt_bits[c] : 0ull, g.out.as<uint64_t>());
      count_launch();
      TQ_TRY(check_launch("k_gather_u64"));
      rc.data.resize((size_t)m * 8);
      TQ_CUDA(cudaMemcpyAsync(rc.data.data(), g.out.p, (size_t)m * 8, cudaMemcpyDeviceToHost, s));
    } else if (sc.kind == 1) {
      TQ_TRY(g.out.reserve((size_t)m * 4));
      TQ_LAUNCH(k_gather_u32, grid_for(m), 256, 0, s, sc.d_data.as<uint32_t>(), d_rows, m, g.out.as<uint32_t>());
      count_launch();
      TQ_TRY(check_launch("k_gather_u32"));
      rc.data.resize((size_t)m * 4);
      TQ_CUDA(cudaMemcpyAsync(rc.data.data(), g.out.p, (size_t)m * 4, cudaMemcpyDeviceToHost, s));
    } else {
      TQ_TRY(g.rowid64.reserve((size_t)m * 8));
      TQ_LAUNCH(k_rows_to_u64, grid_for(m), 256, 0, s, d_rows, m, g.rowid64.as<uint64_t>());
      count_launch();
      TQ_TRY(check_launch("k_rows_to_u64"));
      TQ_TRY(gather_cells(sc.store, g.rowid64.as<uint64_t>(), g.obm.as<uint32_t>(), m, g.var, g.lens, g.scan, s));
      rc.data.resize((size_t)g.var.total);
      TQ_CUDA(cudaMemcpyAsync(rc.off.data(), g.var.off.p, (size_t)(m + 1) * 8, cudaMemcpyDeviceToHost, s));
      if (g.var.total) TQ_CUDA(cudaMemcpyAsync(rc.data.data(), g.var.bytes.p, (size_t)g.var.total, cudaMemcpyDeviceToHost, s));
    }
    TQ_CUDA(cudaStreamSynchronize(s));   // the scratch buffers are reused by the next column
  }
  return TQ_OK;
}

// The same result kept in HBM (tq_sort_next_device / tq_mjoin_next_device): one device array per column, lent to the caller
struct ResultDev {
  std::vector<DevBuf> data, bm;
  std::vector<VarOut> var;      // var-len columns: offsets + bytes (indexed like data)
  std::vector<int> kind;
  DevBuf rowid64, lens, scan;
  bool ready = false, lent = false;
};

int32_t gather_columns_device(const RowStore &st, const uint32_t *d_rows, int64_t m, const uint64_t *dflt_bits, const uint8_t *dflt_nn, ResultDev &rd, cudaStream_t s) {
  for (size_t c = 0; c < st.cols.size(); c++) {
    const StoreCol &sc = st.cols[c];
    rd.data.emplace_back();
    rd.bm.emplace_back();
    rd.var.emplace_back();
    rd.kind.push_back(sc.kind);
    DevBuf &od = rd.data.back(), &ob = rd.bm.back();
    VarOut &ov = rd.var.back();
    const int64_t words = (m + 31) >> 5;
    const int nn_dflt = (sc.kind == 0 && dflt_nn) ? dflt_nn[c] : 0;
    TQ_TRY(ob.reserve(bitmap_alloc_bytes(m)));
    TQ_CUDA(cudaMemsetAsync(ob.p, 0, bitmap_alloc_bytes(m), s));   // the pad words consumers of 64-row groups may touch
    TQ_TRY(od.reserve((size_t)(m ? m : 1) * 8 + 16));
    if (m == 0) continue;
    TQ_LAUNCH(k_gather_bm, grid_for(words * 32), 256, 0, s, sc.bm(), d_rows, m, nn_dflt, ob.as<uint32_t>(), words);
    count_launch();
    TQ_TRY(check_launch("k_gather_bm"));
    if (sc.kind == 0) {
      TQ_LAUNCH(k_gather_u64, grid_for(m), 256, 0, s, sc.d_data.as<uint64_t>(), d_rows, m, (dflt_bits && nn_dflt) ? dflt_bits[c] : 0ull, od.as<uint64_t>());
      count_launch();
      TQ_TRY(check_launch("k_gather_u64"));
    } else if (sc.kind == 1) {
      TQ_LAUNCH(k_gather_u32, grid_for(m), 256, 0, s, sc.d_data.as<uint32_t>(), d_rows, m, od.as<uint32_t>());
      count_launch();
      TQ_TRY(check_launch("k_gather_u32"));
    } else {
      TQ_TRY(rd.rowid64.reserve((size_t)m * 8));
      TQ_LAUNCH(k_rows_to_u64, grid_for(m), 256, 0, s, d_rows, m, rd.rowid64.as<uint64_t>());
      count_launch();
      TQ_TRY(check_launch("k_rows_to_u64"));
      TQ_TRY(gather_cells(sc.store, rd.rowid64.as<uint64_t>(), ob.as<uint32_t>(), m, ov, rd.lens, rd.scan, s));
    }
  }
  TQ_CUDA(cudaStreamSynchronize(s));
  rd.ready = true;
  return TQ_OK;
}

// lend the device result: everything in one batch, then eof
void result_lend(ResultDev &rd, int64_t m, int first_col, int n_cols, tq_column *out) {
  for (int c = 0; c < n_cols; c++) {
    const size_t i = (size_t)(first_col + c);
    out[c].length = m;
    out[c].null_bitmap = rd.bm[i].as<uint8_t>();
    out[c].offsets = nullptr;
    out[c].data = rd.data[i].as<uint8_t>();
    if (rd.kind[i] == 2) { out[c].offsets = rd.var[i].off.as<int64_t>(); out[c].data = rd.var[i].bytes.as<uint8_t>(); }
  }
}

int32_t result_next_bytes(const ResultHost &res, int64_t max_rows, int64_t *bytes_per_col) {
  const int64_t take = std::min(max_rows, res.n - res.pos);
  for (size_t c = 0; c < res.cols.size(); c++) {
    const ResultCol &rc = res.cols[c];
    if (take <= 0) bytes_per_col[c] = 0;
    else if (rc.kind == 0) bytes_per_col[c] = take * 8;
    else if (rc.kind == 1) bytes_per_col[c] = take * 4;
    else bytes_per_col[c] = rc.off[(size_t)(res.pos + take)] - rc.off[(size_t)res.pos];
  }
  return TQ_OK;
}

// the next <= max_rows rows in chunk.Column layout (offsets rebased to 0, NOT-NULL bits from bit 0)
int32_t result_next(ResultHost &res, int64_t max_rows, tq_column *out, int64_t *n_rows, int32_t *eof) {
  const int64_t take = std::min(max_rows, res.n - res.pos);
  *n_rows = 0;
  if (take <= 0) {
    *eof = 1;
    for (size_t c = 0; c < res.cols.size(); c++) out[c].length = 0;
    return TQ_OK;
  }
  for (size_t c = 0; c < res.cols.size(); c++) {
    const ResultCol &rc = res.cols[c];
    if (!out[c].null_bitmap || (!out[c].data && rc.kind != 2) || (rc.kind == 2 && !out[c].offsets)) {
      set_error("output column %d needs data and null_bitmap buffers (and offsets for a var-len column)", (int)c);
      return TQ_ERR_INVALID_ARG;
    }
  }
  for (size_t c = 0; c < res.cols.size(); c++) {
    const ResultCol &rc = res.cols[c];
    if (rc.kind == 2) {
      const int64_t *off = rc.off.data() + res.pos;
      const int64_t b0 = off[0];
      for (int64_t i = 0; i <= take; i++) out[c].offsets[i] = off[i] - b0;
      if (off[take] > b0) {
        if (!out[c].data) { set_error("output column %d needs a data buffer", (int)c); return TQ_ERR_INVALID_ARG; }
        memcpy(out[c].data, rc.data.data() + b0, (size_t)(off[take] - b0));
      }
    } else {
      const size_t w = rc.kind == 1 ? 4 : 8;
      memcpy(out[c].data, rc.data.data() + (size_t)res.pos * w, (size_t)take * w);
    }
    host_bitmap_extract(out[c].null_bitmap, rc.bm.data(), res.pos, take);
    out[c].length = take;
  }
  res.pos += take;
  *n_rows = take;
  *eof = 0;
  return TQ_OK;
}

// ------------------------------------------------------------------------------------------------ host side: the sort
struct SortBufs {
  DevBuf keys[2], perm[2], counts, scan, meta;
  int cur = 0;
  int64_t passes = 0;   // radix digit passes that ran
};

// stable sort of (keys[cur], perm[cur]) by the 64-bit keys: LSD over the digits that are not constant
int32_t radix_sort_word(SortBufs &b, int64_t n, cudaStream_t s) {
  TQ_TRY(b.meta.reserve(64));
  const unsigned long long init[2] = {0ull, ~0ull};
  TQ_CUDA(cudaMemcpyAsync(b.meta.p, init, 16, cudaMemcpyHostToDevice, s));
  TQ_LAUNCH(k_or_and, grid_for(n), 256, 0, s, b.keys[b.cur].as<uint64_t>(), n, b.meta.as<unsigned long long>());
  count_launch();
  TQ_TRY(check_launch("k_or_and"));
  unsigned long long oa[2] = {0, 0};
  TQ_CUDA(cudaMemcpyAsync(oa, b.meta.p, 16, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));
  const uint64_t diff = oa[0] ^ oa[1];
  const int64_t n_blocks = (n + RADIX_TILE - 1) / RADIX_TILE;
  for (int d = 0; d < 8; d++) {
    if (((diff >> (8 * d)) & 0xFFull) == 0) continue;
    const int nxt = b.cur ^ 1;
    TQ_TRY(b.counts.reserve((size_t)n_blocks * 256 * 4));
    TQ_LAUNCH(k_radix_count, (unsigned)n_blocks, RADIX_THREADS, 0, s, b.keys[b.cur].as<uint64_t>(), n, 8 * d, b.counts.as<uint32_t>(), (int)n_blocks);
    count_launch();
    TQ_TRY(check_launch("k_radix_count"));
    TQ_TRY(exclusive_scan_u32(b.counts.as<uint32_t>(), 1, b.counts.as<uint32_t>(), 1, n_blocks * 256, nullptr, b.scan, s));
    TQ_LAUNCH(k_radix_scatter, (unsigned)n_blocks, RADIX_THREADS, 0, s, b.keys[b.cur].as<uint64_t>(), b.perm[b.cur].as<uint32_t>(), n, 8 * d, b.counts.as<uint32_t>(),
                                                                 (int)n_blocks, b.keys[nxt].as<uint64_t>(), b.perm[nxt].as<uint32_t>());
    count_launch();
    TQ_TRY(check_launch("k_radix_scatter"));
    b.cur = nxt;
    b.passes++;
  }
  return TQ_OK;
}

// order perm by one ByItem (column + Desc), stable with respect to the order it already has
int32_t sort_by_column(const StoreCol &sc, int desc, SortBufs &b, int64_t n, cudaStream_t s) {
  std::vector<KeySrc> words;   // least significant first
  if (sc.kind == 0) words.push_back(key_src(sc, KS_COL8, 0, desc));
  else if (sc.kind == 1) words.push_back(key_src(sc, KS_F32, 0, desc));
  else {
    // bytes.Compare = the first differing byte decides, a proper prefix is smaller: zero-padded 8-byte big-endian chunks
    // compared first to last, then the length
    words.push_back(key_src(sc, KS_STR_LEN, 0, desc));
    const int64_t chunks = (sc.max_len + 7) / 8;
    for (int64_t w = chunks - 1; w >= 0; w--) words.push_back(key_src(sc, KS_STR_CHUNK, (int)w, desc));
  }
  if (sc.has_bm) words.push_back(key_src(sc, KS_NULL_FLAG, 0, desc));   // cmpNull: NULL before everything (after, when Desc)
  for (const KeySrc &k : words) {
    TQ_LAUNCH(k_sort_keys, grid_for(n), 256, 0, s, k, b.perm[b.cur].as<uint32_t>(), n, b.keys[b.cur].as<uint64_t>());
    count_launch();
    TQ_TRY(check_launch("k_sort_keys"));
    TQ_TRY(radix_sort_word(b, n, s));
  }
  return TQ_OK;
}

}  // namespace

// ================================================================================================ C ABI: SortExec / TopNExec
struct tq_sort {
  RowStore rows;
  int n_by = 0;
  int by_col[SORT_MAX_BY] = {}, by_desc[SORT_MAX_BY] = {};
  int64_t limit_offset = 0, limit_count = -1;
  bool eof = false;
  ResultHost res;
  bool host_ready = false;     // res holds the rows (device-chunk handles materialise the host copy only if tq_sort_next asks)
  DevBuf keep_rows;            // device-chunk handles: row ids of the result window, kept for the lazy gathers
  ResultDev dev;
  int64_t launches = 0, passes = 0, sort_ns = 0;   // tq_sort_stats
};

struct tq_mjoin {
  int join_type = 0, outer_is_right = 0, n_keys = 0;
  int inner_keys[MJ_MAX_KEYS] = {}, outer_keys[MJ_MAX_KEYS] = {};
  RowStore inner, outer;
  std::vector<uint8_t> selected;   // one byte per outer row once a filter result was passed
  bool has_selected = false;
  std::vector<uint64_t> dflt_bits;
  std::vector<uint8_t> dflt_nn;
  int oc_form = 0;                   // OtherConditions: 0 none, 1 tq_mjoin_set_other_conditions, 2 tq_mjoin_set_other_program
  JoinProg oc;                       // input registers name output columns (left ++ right)
  unsigned oc_err = 0;               // ERR_* bits the program raised: the calls that deliver the result report them
  int64_t oc_warnings = 0;
  bool finished = false;
  ResultHost res;
  bool host_ready = false;
  DevBuf keep_o, keep_i;             // device-chunk handles: (outer row, inner row) of every result row
  ResultDev dev;
};

extern "C" {

int32_t tq_sort_create(const tq_sort_desc *d, tq_sort **out) {
  if (!d || !out) return TQ_ERR_INVALID_ARG;
  *out = nullptr;
  TQ_TRY(ensure_init());
  if (d->n_cols <= 0 || d->n_cols > 64 || !d->types || d->n_by < 0 || d->n_by > SORT_MAX_BY || (d->n_by && (!d->by_cols || !d->by_desc)) || d->limit_offset < 0) {
    set_error("bad sort descriptor");
    return TQ_ERR_INVALID_ARG;
  }
  std::unique_ptr<tq_sort> h(new tq_sort());
  TQ_TRY(h->rows.init(d->n_cols, d->types));
  h->n_by = d->n_by;
  for (int i = 0; i < d->n_by; i++) {
    if (d->by_cols[i] < 0 || d->by_cols[i] >= d->n_cols) { set_error("ByItems[%d] is not an input column", i); return TQ_ERR_INVALID_ARG; }
    h->by_col[i] = d->by_cols[i];
    h->by_desc[i] = d->by_desc[i] ? 1 : 0;
  }
  h->limit_offset = d->limit_offset;
  h->limit_count = d->limit_count;
  *out = h.release();
  return TQ_OK;
}

int32_t tq_sort_put(tq_sort *h, const tq_column *cols, int32_t mem) {
  if (!h || !cols) return TQ_ERR_INVALID_ARG;
  if (h->eof) { set_error("put after eof"); return TQ_ERR_STATE; }
  if (mem == TQ_MEM_DEVICE) {
    TQ_TRY(ensure_init());
    Runtime &r = rt();
    std::lock_guard<std::recursive_mutex> lk(r.mu);
    return h->rows.append_device(cols, r.compute);
  }
  if (mem != TQ_MEM_HOST) return TQ_ERR_INVALID_ARG;
  return h->rows.append(cols);
}

// fetchRowChunks is done: sort (sort.go:58-70) and materialise the rows the parent may ask for
int32_t tq_sort_eof(tq_sort *h) {
  if (!h) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (h->eof) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.compute;
  const int64_t n = h->rows.n;
  h->eof = true;
  const int64_t launches0 = r.launches.load();
  // TopN window (sort.go:210-214: Idx starts at Offset, totalLimit = Offset + Count); SortExec = everything
  const int64_t lo = std::min(h->limit_offset, n);
  const int64_t m = h->limit_count >= 0 ? std::min(h->limit_count, n - lo) : n - lo;
  h->res.n = m;
  if (n == 0 || m == 0) {
    GatherScratch g;
    h->host_ready = true;
    return gather_columns(h->rows, nullptr, 0, nullptr, nullptr, h->res, g, s);
  }
  TQ_TRY(h->rows.upload(s));
  SortBufs b;
  for (int i = 0; i < 2; i++) { TQ_TRY(b.keys[i].reserve((size_t)n * 8)); TQ_TRY(b.perm[i].reserve((size_t)n * 4 + 16)); }
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // device time of the sort phase (upload and result gather excluded)
  TQ_CUDA(cudaEventCreate(&ev0));
  TQ_CUDA(cudaEventCreate(&ev1));
  TQ_CUDA(cudaEventRecord(ev0, s));
  TQ_LAUNCH(k_iota_u32, grid_for(n), 256, 0, s, b.perm[0].as<uint32_t>(), n);
  count_launch();
  int32_t st = check_launch("k_iota_u32");
  if (st == TQ_OK && n > 1)
    for (int i = h->n_by - 1; i >= 0 && st == TQ_OK; i--) st = sort_by_column(h->rows.cols[(size_t)h->by_col[i]], h->by_desc[i], b, n, s);
  if (st == TQ_OK && cudaEventRecord(ev1, s) == cudaSuccess && cudaEventSynchronize(ev1) == cudaSuccess) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) h->sort_ns = (int64_t)(ms * 1e6);
  }
  cudaEventDestroy(ev0);
  cudaEventDestroy(ev1);
  TQ_TRY(st);
  h->passes = b.passes;
  if (h->rows.device_mode) {
    // device chunks in: the result stays in HBM until somebody asks for it (tq_sort_next_device lends it, tq_sort_next copies it)
    TQ_TRY(h->keep_rows.reserve((size_t)m * 4 + 16));
    TQ_CUDA(cudaMemcpyAsync(h->keep_rows.p, b.perm[b.cur].as<uint32_t>() + lo, (size_t)m * 4, cudaMemcpyDeviceToDevice, s));
    TQ_CUDA(cudaStreamSynchronize(s));
  } else {
    GatherScratch g;
    TQ_TRY(gather_columns(h->rows, b.perm[b.cur].as<uint32_t>() + lo, m, nullptr, nullptr, h->res, g, s));
    h->host_ready = true;
  }
  h->launches = r.launches.load() - launches0;
  return TQ_OK;
}

// device-chunk handles: the host copy of the result is made on the first tq_sort_next / tq_sort_next_bytes
static int32_t sort_host_result(tq_sort *h) {
  if (h->host_ready) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  GatherScratch g;
  TQ_TRY(gather_columns(h->rows, h->keep_rows.as<uint32_t>(), h->res.n, nullptr, nullptr, h->res, g, r.compute));
  h->host_ready = true;
  return TQ_OK;
}

int32_t tq_sort_next_bytes(tq_sort *h, int64_t max_rows, int64_t *bytes_per_col) {
  if (!h || !bytes_per_col || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  if (!h->eof) { set_error("next before eof"); return TQ_ERR_STATE; }
  TQ_TRY(sort_host_result(h));
  return result_next_bytes(h->res, max_rows, bytes_per_col);
}

int32_t tq_sort_next(tq_sort *h, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!h || !out_cols || !n_rows || !eof || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  if (!h->eof) { set_error("next before eof"); return TQ_ERR_STATE; }
  TQ_TRY(sort_host_result(h));
  return result_next(h->res, max_rows, out_cols, n_rows, eof);
}

// The whole result (the TopN window) as DEVICE columns, lent until the handle is destroyed: first call = all rows, then eof.
int32_t tq_sort_next_device(tq_sort *h, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!h || !out_cols || !n_rows || !eof) return TQ_ERR_INVALID_ARG;
  if (!h->eof) { set_error("next before eof"); return TQ_ERR_STATE; }
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  *n_rows = 0;
  *eof = 0;
  if (h->dev.lent || h->res.n == 0) { *eof = 1; return TQ_OK; }
  if (!h->rows.device_mode) { set_error("tq_sort_next_device needs a handle fed with device chunks"); return TQ_ERR_STATE; }
  if (!h->dev.ready) TQ_TRY(gather_columns_device(h->rows, h->keep_rows.as<uint32_t>(), h->res.n, nullptr, nullptr, h->dev, r.compute));
  result_lend(h->dev, h->res.n, 0, (int)h->rows.cols.size(), out_cols);
  h->dev.lent = true;
  *n_rows = h->res.n;
  return TQ_OK;
}

int32_t tq_sort_stats(tq_sort *h, int64_t *stats4) {
  if (!h || !stats4) return TQ_ERR_INVALID_ARG;
  stats4[0] = h->rows.n;
  stats4[1] = h->sort_ns;
  stats4[2] = h->launches;
  stats4[3] = h->passes;
  return TQ_OK;
}

int32_t tq_sort_destroy(tq_sort *h) {
  if (!h) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  delete h;
  return TQ_OK;
}

// ================================================================================================ C ABI: MergeJoinExec
int32_t tq_mjoin_create(const tq_mjoin_desc *d, tq_mjoin **out) {
  if (!d || !out) return TQ_ERR_INVALID_ARG;
  *out = nullptr;
  TQ_TRY(ensure_init());
  if (d->n_inner_cols <= 0 || d->n_outer_cols <= 0 || d->n_inner_cols > 64 || d->n_outer_cols > 64 || !d->inner_types || !d->outer_types || d->n_keys < 0 ||
      d->n_keys > MJ_MAX_KEYS || (d->n_keys && (!d->inner_keys || !d->outer_keys)) || d->join_type < TQ_JOIN_INNER || d->join_type > TQ_JOIN_RIGHT_OUTER) {
    set_error("bad merge-join descriptor");
    return TQ_ERR_INVALID_ARG;
  }
  std::unique_ptr<tq_mjoin> h(new tq_mjoin());
  TQ_TRY(h->inner.init(d->n_inner_cols, d->inner_types));
  TQ_TRY(h->outer.init(d->n_outer_cols, d->outer_types));
  h->join_type = d->join_type;
  h->outer_is_right = d->outer_is_right ? 1 : 0;
  h->n_keys = d->n_keys;
  for (int k = 0; k < d->n_keys; k++) {
    const int ik = d->inner_keys[k], ok = d->outer_keys[k];
    if (ik < 0 || ik >= d->n_inner_cols || ok < 0 || ok >= d->n_outer_cols) { set_error("join key %d is not an input column", k); return TQ_ERR_INVALID_ARG; }
    const int ti = h->inner.cols[(size_t)ik].type, to = h->outer.cols[(size_t)ok].type;
    auto cls = [](int t) { return t == TQ_TYPE_BYTES ? 2 : ((t == TQ_TYPE_FLOAT64 || t == TQ_TYPE_FLOAT32) ? 1 : 0); };
    // the planner casts both sides of an equality to one evaluation type (int / real / string) before it builds the join
    if (cls(ti) != cls(to)) { set_error("join key %d compares columns of different evaluation types", k); return TQ_ERR_UNSUPPORTED_TYPE; }
    h->inner_keys[k] = ik;
    h->outer_keys[k] = ok;
  }
  if (d->default_inner_not_null) {
    h->dflt_nn.assign(d->default_inner_not_null, d->default_inner_not_null + d->n_inner_cols);
    h->dflt_bits.assign((size_t)d->n_inner_cols, 0);
    if (d->default_inner_bits) h->dflt_bits.assign(d->default_inner_bits, d->default_inner_bits + d->n_inner_cols);
    for (int c = 0; c < d->n_inner_cols; c++)
      if (h->dflt_nn[(size_t)c] && h->inner.cols[(size_t)c].kind != 0) { set_error("defaultInner values are supported for 8-byte columns"); return TQ_ERR_UNSUPPORTED_TYPE; }
  }
  *out = h.release();
  return TQ_OK;
}

}  // extern "C"

// output column c of left ++ right
static const StoreCol &mjoin_col(const tq_mjoin *h, int c) {
  const int n_first = (int)(h->outer_is_right ? h->inner.cols.size() : h->outer.cols.size());
  const bool in_first = c < n_first;
  const RowStore &st = (in_first == (h->outer_is_right != 0)) ? h->inner : h->outer;
  return st.cols[(size_t)(in_first ? c : c - n_first)];
}
// the comparison list may be set again (the last call counts); the program once, and never both forms on one handle
static int32_t mjoin_oc_settable(const tq_mjoin *h, int form) {
  if (h->finished || h->inner.n || h->outer.n) { set_error("other conditions must be set right after tq_mjoin_create"); return TQ_ERR_STATE; }
  if (h->oc_form && (h->oc_form != form || form == 2)) { set_error("the handle has other conditions already"); return TQ_ERR_STATE; }
  return TQ_OK;
}

extern "C" {

// OtherConditions: comparisons over the joined row (left ++ right), as tq_join_set_other_conditions takes them
int32_t tq_mjoin_set_other_conditions(tq_mjoin *h, int32_t n_conds, const tq_join_cond *conds) {
  if (!h || n_conds < 0 || n_conds > JP_MAX_CONDS || (n_conds && !conds)) { set_error("at most %d other conditions", JP_MAX_CONDS); return TQ_ERR_INVALID_ARG; }
  TQ_TRY(mjoin_oc_settable(h, 1));
  const int n_all = (int)(h->inner.cols.size() + h->outer.cols.size());
  for (int k = 0; k < n_conds; k++) {
    const tq_join_cond &c = conds[k];
    if (c.op < TQ_CMP_LT || c.op > TQ_CMP_NE || c.lhs_col < 0 || c.lhs_col >= n_all || c.rhs_col >= n_all) { set_error("bad other condition %d", k); return TQ_ERR_INVALID_ARG; }
    const StoreCol &a = mjoin_col(h, c.lhs_col);
    const int tb = c.rhs_col >= 0 ? mjoin_col(h, c.rhs_col).type : (c.const_type & 0xFF);
    const bool b_fixed8 = c.rhs_col >= 0 ? mjoin_col(h, c.rhs_col).kind == 0 : (tb >= TQ_TYPE_INT64 && tb <= TQ_TYPE_FLOAT64);
    if (a.kind != 0 || !b_fixed8 || ((a.type == TQ_TYPE_FLOAT64) != (tb == TQ_TYPE_FLOAT64))) {
      set_error("other condition %d: BIGINT with BIGINT (any sign mix) or DOUBLE with DOUBLE", k);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
  }
  h->oc_form = 0;
  if (n_conds == 0) return TQ_OK;
  join_prog_from_conds(n_conds, conds, [&](int c) { return mjoin_col(h, c).type; }, &h->oc);
  h->oc_form = 1;
  return TQ_OK;
}

int32_t tq_mjoin_set_other_program(tq_mjoin *h, int32_t n_inputs, const int32_t *input_cols, int32_t n_ops, const tq_expr_op *ops) {
  if (!h) return TQ_ERR_INVALID_ARG;
  TQ_TRY(mjoin_oc_settable(h, 2));
  const int n_all = (int)(h->inner.cols.size() + h->outer.cols.size());
  TQ_TRY(join_prog_from_ops(n_inputs, input_cols, n_ops, ops, n_all, [&](int c) { return mjoin_col(h, c).type; }, &h->oc));
  h->oc_form = 2;
  return TQ_OK;
}

int32_t tq_mjoin_warnings(tq_mjoin *h, int64_t *div_by_zero) {
  if (!h || !div_by_zero) return TQ_ERR_INVALID_ARG;
  *div_by_zero = h->oc_warnings;
  return TQ_OK;
}

int32_t tq_mjoin_put_inner(tq_mjoin *h, const tq_column *cols, int32_t mem) {
  if (!h || !cols) return TQ_ERR_INVALID_ARG;
  if (h->finished) { set_error("put after finish"); return TQ_ERR_STATE; }
  if (mem == TQ_MEM_DEVICE) {
    TQ_TRY(ensure_init());
    Runtime &r = rt();
    std::lock_guard<std::recursive_mutex> lk(r.mu);
    return h->inner.append_device(cols, r.compute);
  }
  if (mem != TQ_MEM_HOST) return TQ_ERR_INVALID_ARG;
  return h->inner.append(cols);
}

int32_t tq_mjoin_put_outer(tq_mjoin *h, const tq_column *cols, const uint8_t *selected, int32_t mem) {
  if (!h || !cols) return TQ_ERR_INVALID_ARG;
  if (h->finished) { set_error("put after finish"); return TQ_ERR_STATE; }
  if (mem != TQ_MEM_HOST && mem != TQ_MEM_DEVICE) return TQ_ERR_INVALID_ARG;
  const int64_t before = h->outer.n;
  if (mem == TQ_MEM_DEVICE) {   // `selected` stays a host []bool either way
    TQ_TRY(ensure_init());
    Runtime &r = rt();
    std::lock_guard<std::recursive_mutex> lk(r.mu);
    TQ_TRY(h->outer.append_device(cols, r.compute));
  } else TQ_TRY(h->outer.append(cols));
  const int64_t rows = h->outer.n - before;
  if (selected && !h->has_selected) { h->selected.assign((size_t)before, 1); h->has_selected = true; }
  if (h->has_selected) {
    if (selected) h->selected.insert(h->selected.end(), selected, selected + rows);
    else h->selected.insert(h->selected.end(), (size_t)rows, 1);
  }
  return TQ_OK;
}

// both children are exhausted: join
int32_t tq_mjoin_finish(tq_mjoin *h) {
  if (!h) return TQ_ERR_INVALID_ARG;
  TQ_TRY(ensure_init());
  if (h->finished) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  cudaStream_t s = r.compute;
  h->finished = true;
  const int64_t ni = h->inner.n, no = h->outer.n;
  const bool outer_join = h->join_type != TQ_JOIN_INNER;
  GatherScratch g;
  RowStore *first = h->outer_is_right ? &h->inner : &h->outer, *second = h->outer_is_right ? &h->outer : &h->inner;
  auto dflt_b = [&](RowStore *st) { return (st == &h->inner && !h->dflt_nn.empty()) ? h->dflt_bits.data() : nullptr; };
  auto dflt_n = [&](RowStore *st) { return (st == &h->inner && !h->dflt_nn.empty()) ? h->dflt_nn.data() : nullptr; };
  if (no == 0) {
    h->res.n = 0;
    h->host_ready = true;
    TQ_TRY(gather_columns(*first, nullptr, 0, nullptr, nullptr, h->res, g, s));
    return gather_columns(*second, nullptr, 0, nullptr, nullptr, h->res, g, s);
  }
  TQ_TRY(h->inner.upload(s));
  TQ_TRY(h->outer.upload(s));
  // key columns as comparable words (strings are compared in place)
  MJKeys K{};
  std::vector<DevBuf> enc_bufs;
  enc_bufs.reserve(4 * MJ_MAX_KEYS);
  BmList ibm{}, obm{};
  for (int k = 0; k < h->n_keys; k++) {
    const StoreCol &ci = h->inner.cols[(size_t)h->inner_keys[k]], &co = h->outer.cols[(size_t)h->outer_keys[k]];
    if (ci.has_bm) ibm.bm[ibm.n++] = ci.bm();
    if (co.has_bm) obm.bm[obm.n++] = co.bm();
    if (ci.kind == 2) {
      MJKeyCol &kc = K.c[K.k++];
      kc.is_str = 1;
      kc.off[0] = ci.store.offsets.as<int64_t>(); kc.bytes[0] = ci.store.bytes.as<uint8_t>();
      kc.off[1] = co.store.offsets.as<int64_t>(); kc.bytes[1] = co.store.bytes.as<uint8_t>();
      continue;
    }
    const bool mixed = ci.kind == 0 && co.kind == 0 && ci.type != co.type && ci.type != TQ_TYPE_FLOAT64 && co.type != TQ_TYPE_FLOAT64;
    const int modes[2] = {mixed ? KS_MIX_CLASS : -1, mixed ? KS_MIX_VALUE : -1};
    for (int part = mixed ? 0 : 1; part < 2; part++) {
      MJKeyCol &kc = K.c[K.k++];
      kc.is_str = 0;
      for (int side = 0; side < 2; side++) {
        const StoreCol &sc = side == 0 ? ci : co;
        const int64_t n = side == 0 ? ni : no;
        enc_bufs.emplace_back();
        DevBuf &eb = enc_bufs.back();
        TQ_TRY(eb.reserve((size_t)(n ? n : 1) * 8));
        if (n > 0) {
          KeySrc ks = key_src(sc, mixed ? modes[part] : (sc.kind == 1 ? KS_F32 : KS_COL8), 0, 0);
          ks.bm = nullptr;   // NULL keys never reach a comparison (k_mj_valid)
          TQ_LAUNCH(k_sort_keys, grid_for(n), 256, 0, s, ks, nullptr, n, eb.as<uint64_t>());
          count_launch();
          TQ_TRY(check_launch("k_sort_keys"));
        }
        kc.enc[side] = eb.as<uint64_t>();
      }
    }
  }
  // inner rows that can match, in child order
  DevBuf iflags, ioffs, ivalid, scan, meta, oflags, d_sel, lo, cnt, emit, out_o, out_i;
  TQ_TRY(meta.reserve(64));
  TQ_CUDA(cudaMemsetAsync(meta.p, 0, 64, s));
  int64_t iv = 0;
  TQ_TRY(ivalid.reserve((size_t)(ni ? ni : 1) * 4));
  if (ni > 0) {
    TQ_TRY(iflags.reserve((size_t)ni * 4));
    TQ_TRY(ioffs.reserve((size_t)ni * 4));
    TQ_LAUNCH(k_mj_valid, grid_for(ni), 256, 0, s, ibm, nullptr, ni, iflags.as<uint32_t>());
    count_launch();
    TQ_TRY(check_launch("k_mj_valid"));
    TQ_TRY(exclusive_scan_u32(iflags.as<uint32_t>(), 1, ioffs.as<uint32_t>(), 1, ni, meta.as<uint64_t>(), scan, s));
    TQ_LAUNCH(k_compact, grid_for(ni), 256, 0, s, iflags.as<uint32_t>(), ioffs.as<uint32_t>(), ni, ivalid.as<uint32_t>());
    count_launch();
    TQ_TRY(check_launch("k_compact"));
    uint64_t total = 0;
    TQ_CUDA(cudaMemcpyAsync(&total, meta.p, 8, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    iv = (int64_t)total;
    if (iv > 1) {
      TQ_LAUNCH(k_mj_check_sorted, grid_for(iv), 256, 0, s, K, ivalid.as<uint32_t>(), iv, meta.as<unsigned>() + 4);
      count_launch();
      TQ_TRY(check_launch("k_mj_check_sorted"));
      unsigned bad = 0;
      TQ_CUDA(cudaMemcpyAsync(&bad, meta.as<unsigned>() + 4, 4, cudaMemcpyDeviceToHost, s));
      TQ_CUDA(cudaStreamSynchronize(s));
      if (bad) { set_error("merge join: the inner child is not sorted by the join keys (%u inversions)", bad); return TQ_ERR_STATE; }
    }
  }
  // outer rows: filter + NULL keys, group bounds, output ranges
  TQ_TRY(oflags.reserve((size_t)no * 4));
  const uint8_t *dsel = nullptr;
  if (h->has_selected) {
    TQ_TRY(d_sel.reserve((size_t)no));
    TQ_CUDA(cudaMemcpyAsync(d_sel.p, h->selected.data(), (size_t)no, cudaMemcpyHostToDevice, s));
    dsel = d_sel.as<uint8_t>();
  }
  TQ_LAUNCH(k_mj_valid, grid_for(no), 256, 0, s, obm, dsel, no, oflags.as<uint32_t>());
  count_launch();
  TQ_TRY(check_launch("k_mj_valid"));
  TQ_TRY(lo.reserve((size_t)no * 4));
  TQ_TRY(cnt.reserve((size_t)no * 4));
  TQ_TRY(emit.reserve((size_t)no * 4));
  TQ_LAUNCH(k_mj_bounds, grid_for(no), 256, 0, s, K, ivalid.as<uint32_t>(), iv, oflags.as<uint32_t>(), no, outer_join ? 1 : 0, lo.as<uint32_t>(), cnt.as<uint32_t>(),
                                           emit.as<uint32_t>());
  count_launch();
  TQ_TRY(check_launch("k_mj_bounds"));
  TQ_TRY(exclusive_scan_u32(emit.as<uint32_t>(), 1, emit.as<uint32_t>(), 1, no, meta.as<uint64_t>() + 1, scan, s));
  uint64_t total = 0;
  TQ_CUDA(cudaMemcpyAsync(&total, meta.as<uint64_t>() + 1, 8, cudaMemcpyDeviceToHost, s));
  TQ_CUDA(cudaStreamSynchronize(s));   // also: the pageable `selected` source is done
  if (total > 0xFFFFFFF0ull) { set_error("merge join result of %llu rows exceeds 2^32", (unsigned long long)total); return TQ_ERR_INVALID_ARG; }
  const int64_t m = (int64_t)total;
  h->res.n = m;
  TQ_TRY(out_o.reserve((size_t)(m ? m : 1) * 4));
  TQ_TRY(out_i.reserve((size_t)(m ? m : 1) * 4));
  if (m > 0) {
    TQ_LAUNCH(k_mj_expand, grid_for(m), 256, 0, s, emit.as<uint32_t>(), lo.as<uint32_t>(), cnt.as<uint32_t>(), ivalid.as<uint32_t>(), no, m, out_o.as<uint32_t>(),
                                            out_i.as<uint32_t>());
    count_launch();
    TQ_TRY(check_launch("k_mj_expand"));
  }
  const uint32_t *rows_o = out_o.as<uint32_t>(), *rows_i = out_i.as<uint32_t>();
  int64_t m_out = m;
  DevBuf flags, fscan, emit2, new_o, new_i;
  if (h->oc_form) {
    // tryToMatchInners filters the joined rows of an outer row with the OtherConditions; when none survives the outer row
    // takes the miss path (merge_join.go:290-305, joiner.go:225-248,288-311,351-378)
    MJProg P;
    P.n_in = h->oc.n_in;
    P.n_ops = h->oc.n_ops;
    for (int i = 0; i < P.n_ops; i++) P.ops[i] = h->oc.ops[i];
    const int n_first = (int)first->cols.size();
    for (int k = 0; k < P.n_in; k++) {
      const int c = h->oc.in_col[k];
      const bool in_first = c < n_first;
      const RowStore *st = in_first ? first : second;
      const StoreCol &sc = st->cols[(size_t)(in_first ? c : c - n_first)];
      P.inner[k] = st == &h->inner ? 1 : 0;
      P.data[k] = sc.d_data.as<uint64_t>();
      P.bm[k] = sc.bm();
    }
    TQ_TRY(flags.reserve((size_t)(m ? m : 1) * 4));
    TQ_TRY(fscan.reserve((size_t)(m ? m : 1) * 4));
    TQ_TRY(emit2.reserve((size_t)no * 4));
    uint64_t n_pass = 0;
    if (m > 0) {
      // meta[5] / meta[6]: the program's error bits and warnings, read back with n_pass (meta[3])
      TQ_LAUNCH(k_mj_prog, grid_for(m), 256, 0, s, P, out_o.as<uint32_t>(), out_i.as<uint32_t>(), m, flags.as<uint32_t>(),
                reinterpret_cast<unsigned long long *>(meta.as<uint64_t>() + 5));
      count_launch();
      TQ_TRY(check_launch("k_mj_prog"));
      TQ_TRY(exclusive_scan_u32(flags.as<uint32_t>(), 1, fscan.as<uint32_t>(), 1, m, meta.as<uint64_t>() + 3, scan, s));
      uint64_t back[4] = {0, 0, 0, 0};   // n_pass, (meta[4]), error bits, warnings
      TQ_CUDA(cudaMemcpyAsync(back, meta.as<uint64_t>() + 3, 32, cudaMemcpyDeviceToHost, s));
      TQ_CUDA(cudaStreamSynchronize(s));
      n_pass = back[0];
      h->oc_err = (unsigned)back[2];
      h->oc_warnings += (int64_t)back[3];
    }
    TQ_LAUNCH(k_mj_survivors, grid_for(no), 256, 0, s, emit.as<uint32_t>(), fscan.as<uint32_t>(), no, m, (uint32_t)n_pass, outer_join ? 1 : 0, emit2.as<uint32_t>());
    count_launch();
    TQ_TRY(check_launch("k_mj_survivors"));
    TQ_TRY(exclusive_scan_u32(emit2.as<uint32_t>(), 1, emit2.as<uint32_t>(), 1, no, meta.as<uint64_t>() + 4, scan, s));
    uint64_t total2 = 0;
    TQ_CUDA(cudaMemcpyAsync(&total2, meta.as<uint64_t>() + 4, 8, cudaMemcpyDeviceToHost, s));
    TQ_CUDA(cudaStreamSynchronize(s));
    const int64_t m2 = (int64_t)total2;
    TQ_TRY(new_o.reserve((size_t)(m2 ? m2 : 1) * 4));
    TQ_TRY(new_i.reserve((size_t)(m2 ? m2 : 1) * 4));
    if (m > 0 && m2 > 0) {
      TQ_LAUNCH(k_mj_refill_pairs, grid_for(m), 256, 0, s, flags.as<uint32_t>(), fscan.as<uint32_t>(), emit.as<uint32_t>(), emit2.as<uint32_t>(), out_o.as<uint32_t>(),
                out_i.as<uint32_t>(), m, new_o.as<uint32_t>(), new_i.as<uint32_t>());
      count_launch();
      TQ_TRY(check_launch("k_mj_refill_pairs"));
    }
    if (m2 > 0 && outer_join) {
      TQ_LAUNCH(k_mj_refill_misses, grid_for(no), 256, 0, s, emit.as<uint32_t>(), fscan.as<uint32_t>(), emit2.as<uint32_t>(), no, m, (uint32_t)n_pass, m2,
                new_o.as<uint32_t>(), new_i.as<uint32_t>());
      count_launch();
      TQ_TRY(check_launch("k_mj_refill_misses"));
    }
    rows_o = new_o.as<uint32_t>();
    rows_i = new_i.as<uint32_t>();
    m_out = m2;
    h->res.n = m2;
  }
  if (h->inner.device_mode || h->outer.device_mode) {
    // device chunks in: keep the (outer row, inner row) lists; the columns are gathered when a next call asks for them
    TQ_TRY(h->keep_o.reserve((size_t)(m_out ? m_out : 1) * 4));
    TQ_TRY(h->keep_i.reserve((size_t)(m_out ? m_out : 1) * 4));
    if (m_out) {
      TQ_CUDA(cudaMemcpyAsync(h->keep_o.p, rows_o, (size_t)m_out * 4, cudaMemcpyDeviceToDevice, s));
      TQ_CUDA(cudaMemcpyAsync(h->keep_i.p, rows_i, (size_t)m_out * 4, cudaMemcpyDeviceToDevice, s));
    }
    TQ_CUDA(cudaStreamSynchronize(s));
    h->res.n = m_out;
    return TQ_OK;
  }
  // output schema = left child columns ++ right child columns (executor/builder.go: the joiner's makeJoinRowToChunk)
  TQ_TRY(gather_columns(*first, first == &h->inner ? rows_i : rows_o, m_out, dflt_b(first), dflt_n(first), h->res, g, s));
  TQ_TRY(gather_columns(*second, second == &h->inner ? rows_i : rows_o, m_out, dflt_b(second), dflt_n(second), h->res, g, s));
  h->host_ready = true;
  return TQ_OK;
}

}  // extern "C"

// gathers of a device-chunk merge join: left child columns ++ right child columns from the kept row lists
template <typename Gather>
static int32_t mjoin_gather(tq_mjoin *h, Gather &&gather) {
  RowStore *first = h->outer_is_right ? &h->inner : &h->outer, *second = h->outer_is_right ? &h->outer : &h->inner;
  for (RowStore *st : {first, second}) {
    const bool is_inner = st == &h->inner;
    const uint64_t *db = (is_inner && !h->dflt_nn.empty()) ? h->dflt_bits.data() : nullptr;
    const uint8_t *dn = (is_inner && !h->dflt_nn.empty()) ? h->dflt_nn.data() : nullptr;
    TQ_TRY(gather(*st, is_inner ? h->keep_i.as<uint32_t>() : h->keep_o.as<uint32_t>(), db, dn));
  }
  return TQ_OK;
}
static int32_t mjoin_host_result(tq_mjoin *h) {
  if (h->host_ready) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  GatherScratch g;
  TQ_TRY(mjoin_gather(h, [&](const RowStore &st, const uint32_t *rows, const uint64_t *db, const uint8_t *dn) {
    return gather_columns(st, rows, h->res.n, db, dn, h->res, g, r.compute);
  }));
  h->host_ready = true;
  return TQ_OK;
}

extern "C" {

int32_t tq_mjoin_next_bytes(tq_mjoin *h, int64_t max_rows, int64_t *bytes_per_col) {
  if (!h || !bytes_per_col || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  if (!h->finished) { set_error("next before finish"); return TQ_ERR_STATE; }
  if (h->oc_err) return err_to_status(h->oc_err, "other conditions");
  TQ_TRY(mjoin_host_result(h));
  return result_next_bytes(h->res, max_rows, bytes_per_col);
}

int32_t tq_mjoin_next(tq_mjoin *h, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!h || !out_cols || !n_rows || !eof || max_rows <= 0) return TQ_ERR_INVALID_ARG;
  if (!h->finished) { set_error("next before finish"); return TQ_ERR_STATE; }
  if (h->oc_err) return err_to_status(h->oc_err, "other conditions");
  TQ_TRY(mjoin_host_result(h));
  return result_next(h->res, max_rows, out_cols, n_rows, eof);
}

// The whole join result as DEVICE columns, lent until the handle is destroyed: first call = all rows, then eof.
int32_t tq_mjoin_next_device(tq_mjoin *h, tq_column *out_cols, int64_t *n_rows, int32_t *eof) {
  if (!h || !out_cols || !n_rows || !eof) return TQ_ERR_INVALID_ARG;
  if (!h->finished) { set_error("next before finish"); return TQ_ERR_STATE; }
  if (h->oc_err) return err_to_status(h->oc_err, "other conditions");
  TQ_TRY(ensure_init());
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  *n_rows = 0;
  *eof = 0;
  if (h->dev.lent || h->res.n == 0) { *eof = 1; return TQ_OK; }
  if (!h->inner.device_mode && !h->outer.device_mode) { set_error("tq_mjoin_next_device needs a handle fed with device chunks"); return TQ_ERR_STATE; }
  if (!h->dev.ready)
    TQ_TRY(mjoin_gather(h, [&](const RowStore &st, const uint32_t *rows, const uint64_t *db, const uint8_t *dn) {
      return gather_columns_device(st, rows, h->res.n, db, dn, h->dev, r.compute);
    }));
  result_lend(h->dev, h->res.n, 0, (int)(h->inner.cols.size() + h->outer.cols.size()), out_cols);
  h->dev.lent = true;
  *n_rows = h->res.n;
  return TQ_OK;
}

int32_t tq_mjoin_destroy(tq_mjoin *h) {
  if (!h) return TQ_OK;
  Runtime &r = rt();
  std::lock_guard<std::recursive_mutex> lk(r.mu);
  delete h;
  return TQ_OK;
}

}  // extern "C"
