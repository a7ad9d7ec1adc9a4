// nlj.cu — kernels of the key-less hash join (see nlj.cuh).  Plain CUDA C++.
#include "nlj.cuh"

namespace tq {

static int nlj_grid(int64_t threads, int per_sm) {
  const int64_t blocks = (threads + 255) / 256;
  const int64_t cap = (int64_t)rt().sm_count * per_sm;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

__device__ __forceinline__ bool nlj_not_null(const uint32_t *bm, int64_t i) { return bm == nullptr || ((bm[i >> 5] >> (i & 31)) & 1u); }

// One warp per survivor word: lane l evaluates the pair (probe row r0 + r, build row 32 w + l) with the condition program and
// the warp's ballot is the word.  The probe row's inputs are the same address for the whole warp (one broadcast load), the build
// rows' inputs are 32 consecutive rows (coalesced).  Pairs of an unselected probe row are not evaluated: the reference returns
// before filter for it (joiner.go:225-228,288-291), so they raise nothing.
__global__ void __launch_bounds__(256) k_nlj_eval(const __grid_constant__ NljEvalParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t n_words = p.rows * (int64_t)p.words;
  const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5);
  unsigned err = 0, cnt = 0;
  for (int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < n_words; g += wstride) {
    const int64_t r = g / p.words;
    const uint32_t w = (uint32_t)(g - r * p.words);
    const int64_t i = p.r0 + r;
    const uint32_t b = w * 32 + lane;
    bool pass = false;
    if ((!p.selected || p.selected[i]) && b < p.n_build) {
      uint64_t rv[JP_REGS];
      uint64_t nn = 0;
      for (int k = 0; k < p.prog.n_in; k++) {
        const int64_t row = p.in_build[k] ? (int64_t)b : i;
        rv[k] = p.in[k].data[row];
        if (nlj_not_null(p.in[k].bm, row)) nn |= 1ull << k;
      }
      bool alive;
      xp_run_row(p.prog.ops, p.prog.n_ops, p.prog.n_in, rv, nn, true, alive, pass, err, cnt);
    }
    const unsigned word = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) p.mask[g] = word;
  }
  err = __reduce_or_sync(0xffffffffu, err);
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) {
    if (err) atomicOr(p.err, err);
    if (cnt) atomicAdd(p.warn, (unsigned long long)cnt);
  }
}

// One warp per probe row: rows it emits, whether that is its miss row, and (with conditions) the set bits of its earlier words.
__global__ void __launch_bounds__(256) k_nlj_count(const NljCountParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < p.rows; r += wstride) {
    const int64_t i = p.r0 + r;
    uint64_t c;
    bool miss = false;
    if ((p.selected && !p.selected[i]) || p.n_build == 0) {   // unselected, or an empty build side: onMissMatch (outer) or nothing
      c = p.outer ? 1 : 0;
      miss = p.outer != 0;
    } else if (!p.mask) {
      c = p.n_build;
    } else {
      const uint32_t *m = p.mask + r * p.words;
      uint32_t *pre = p.wpre + r * p.words;
      uint32_t run = 0;
      for (uint32_t w0 = 0; w0 < p.words; w0 += 32) {
        const uint32_t w = w0 + lane;
        const uint32_t pc = w < p.words ? __popc(m[w]) : 0u;
        uint32_t inc = pc;
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
          if (lane >= d) inc += v;
        }
        if (w < p.words) pre[w] = run + inc - pc;
        run += __shfl_sync(0xffffffffu, inc, 31);
      }
      c = run;
      if (run == 0 && p.outer) { c = 1; miss = true; }   // no joined row survives: the probe row's miss row
    }
    if (lane == 0) {
      p.cnt[r] = c;
      p.miss[r] = miss ? 1 : 0;
    }
  }
}

// ---- exclusive scan of u64 counts: per-tile sums -> one CTA scans the tile sums -> rescan with the tile offsets
static constexpr int NS_THREADS = 256, NS_ITEMS = 8, NS_TILE = NS_THREADS * NS_ITEMS;

__device__ __forceinline__ uint64_t nlj_block_scan(uint64_t v, uint64_t *s_warp) {   // exclusive; s_warp[8] = block total
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t inc = v;
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const uint64_t w = lane < NS_THREADS / 32 ? s_warp[lane] : 0;
    uint64_t winc = w;
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += t;
    }
    if (lane < NS_THREADS / 32) s_warp[lane] = winc - w;
    if (lane == NS_THREADS / 32 - 1) s_warp[NS_THREADS / 32] = winc;
  }
  __syncthreads();
  return inc - v + s_warp[warp];
}

__global__ void __launch_bounds__(NS_THREADS) k_nlj_scan_sums(const uint64_t *in, int64_t n, uint64_t *tile_sums) {
  __shared__ uint64_t s_warp[NS_THREADS / 32 + 1];
  const int64_t base = (int64_t)blockIdx.x * NS_TILE + (int64_t)threadIdx.x * NS_ITEMS;
  uint64_t sum = 0;
  for (int k = 0; k < NS_ITEMS; k++)
    if (base + k < n) sum += in[base + k];
  nlj_block_scan(sum, s_warp);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = s_warp[NS_THREADS / 32];
}

__global__ void __launch_bounds__(1024) k_nlj_scan_tiles(uint64_t *tile_sums, int64_t n_tiles, uint64_t *total_out) {
  __shared__ uint64_t s_part[1024];
  const int t = threadIdx.x;
  const int64_t per = (n_tiles + 1023) / 1024;
  const int64_t lo = t * per, hi = lo + per < n_tiles ? lo + per : n_tiles;
  uint64_t sum = 0;
  for (int64_t i = lo; i < hi; i++) sum += tile_sums[i];
  s_part[t] = sum;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const uint64_t v = t >= d ? s_part[t - d] : 0;
    __syncthreads();
    s_part[t] += v;
    __syncthreads();
  }
  uint64_t run = s_part[t] - sum;
  for (int64_t i = lo; i < hi; i++) {
    const uint64_t v = tile_sums[i];
    tile_sums[i] = run;
    run += v;
  }
  if (t == 1023) *total_out = s_part[1023];
}

__global__ void __launch_bounds__(NS_THREADS) k_nlj_scan_final(const uint64_t *in, uint64_t *out, int64_t n, const uint64_t *tile_off) {
  __shared__ uint64_t s_warp[NS_THREADS / 32 + 1];
  const int64_t base = (int64_t)blockIdx.x * NS_TILE + (int64_t)threadIdx.x * NS_ITEMS;
  uint64_t v[NS_ITEMS], sum = 0;
  for (int k = 0; k < NS_ITEMS; k++) {
    v[k] = base + k < n ? in[base + k] : 0;
    sum += v[k];
  }
  uint64_t run = nlj_block_scan(sum, s_warp) + tile_off[blockIdx.x];
  for (int k = 0; k < NS_ITEMS; k++) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
}

// Largest r in [lo, hi] with off[r] <= g (off is non-decreasing and off[hi + 1] > g): the probe row whose output holds g.
// Rows that emit nothing share their offset with the next row, so the search lands on the row that does emit g.
__device__ __forceinline__ int64_t nlj_row_of(const uint64_t *off, uint64_t g, int64_t lo, int64_t hi) {
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (off[mid] <= g) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Thread per output row.  A CTA takes 256 consecutive positions and first finds the range of probe rows they come from, so each
// thread's search covers one or two rows when a probe row emits hundreds of rows.  The 256 positions start on a 32-row boundary
// of the batch, so each warp's ballot is one whole NOT-NULL bitmap word (tail bits past len are 0).
__global__ void __launch_bounds__(256) k_nlj_materialize(const __grid_constant__ NljOutParams p) {
  __shared__ int64_t s_rows[2];
  const int lane = threadIdx.x & 31;
  for (int64_t t0 = (int64_t)blockIdx.x * blockDim.x; t0 < p.len; t0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t last = (t0 + blockDim.x < p.len ? t0 + blockDim.x : p.len) - 1;
    if (threadIdx.x == 0) s_rows[0] = nlj_row_of(p.off, p.q0 + (uint64_t)t0, 0, p.rows - 1);
    if (threadIdx.x == 32) s_rows[1] = nlj_row_of(p.off, p.q0 + (uint64_t)last, 0, p.rows - 1);
    __syncthreads();
    const int64_t lo = s_rows[0], hi = s_rows[1];
    __syncthreads();
    const int64_t q = t0 + threadIdx.x;
    const bool active = q < p.len;
    int64_t i = 0;
    uint32_t b = 0;
    bool miss = false;
    if (active) {
      const uint64_t g = p.q0 + (uint64_t)q;
      const int64_t r = nlj_row_of(p.off, g, lo, hi);
      const uint64_t k = g - p.off[r];
      i = p.r0 + r;
      miss = p.miss[r] != 0;
      if (!miss && p.mask) {
        // the k-th surviving build row: the word whose prefix holds k, then the bit inside it
        const uint32_t *pre = p.wpre + r * p.words;
        uint32_t wlo = 0, whi = p.words - 1;
        while (wlo < whi) {
          const uint32_t mid = (wlo + whi + 1) >> 1;
          if (pre[mid] <= (uint32_t)k) wlo = mid;
          else whi = mid - 1;
        }
        uint32_t m = p.mask[r * p.words + wlo];
        for (uint32_t s = (uint32_t)k - pre[wlo]; s; s--) m &= m - 1;
        b = wlo * 32 + (uint32_t)(__ffs(m) - 1);
      } else if (!miss) {
        b = (uint32_t)k;
      }
    }
    const int64_t word = q >> 5;
    for (int c = 0; c < p.n_probe_cols; c++) {
      bool nn = false;
      if (active) {
        p.out_probe[c].data[q] = p.probe[c].data[i];
        nn = nlj_not_null(p.probe[c].bm, i);
      }
      const unsigned bits = __ballot_sync(0xffffffffu, nn);
      if (lane == 0) p.out_probe[c].bm[word] = bits;
    }
    for (int c = 0; c < p.n_build_cols; c++) {
      bool nn = false;
      if (active) {
        if (miss) {   // onMissMatch: the inner side is defaultInner (joiner.go:139-143), NULL unless the descriptor gave a value
          nn = (p.def_mask >> c) & 1u;
          p.out_build[c].data[q] = nn ? p.def_val[c] : 0ull;
        } else {
          p.out_build[c].data[q] = p.build[c].data[b];
          nn = nlj_not_null(p.build[c].bm, b);
        }
      }
      const unsigned bits = __ballot_sync(0xffffffffu, nn);
      if (lane == 0) p.out_build[c].bm[word] = bits;
    }
  }
}

int32_t nlj_eval(const NljEvalParams &p, cudaStream_t s) {
  const int64_t n_words = p.rows * (int64_t)p.words;
  if (n_words <= 0) return TQ_OK;
  k_nlj_eval<<<nlj_grid(n_words * 32, 16), 256, 0, s>>>(p);
  count_launch();
  return check_launch("k_nlj_eval");
}

int32_t nlj_count(const NljCountParams &p, cudaStream_t s) {
  if (p.rows <= 0) return TQ_OK;
  k_nlj_count<<<nlj_grid(p.rows * 32, 16), 256, 0, s>>>(p);
  count_launch();
  return check_launch("k_nlj_count");
}

int32_t nlj_scan_u64(const uint64_t *in, uint64_t *out, int64_t n, DevBuf &scratch, cudaStream_t s) {
  if (n <= 0) {
    TQ_CUDA(cudaMemsetAsync(out, 0, 8, s));
    return TQ_OK;
  }
  const int64_t n_tiles = (n + NS_TILE - 1) / NS_TILE;
  TQ_TRY(scratch.reserve((size_t)n_tiles * 8));
  uint64_t *sums = scratch.as<uint64_t>();
  k_nlj_scan_sums<<<(unsigned)n_tiles, NS_THREADS, 0, s>>>(in, n, sums);
  k_nlj_scan_tiles<<<1, 1024, 0, s>>>(sums, n_tiles, out + n);
  k_nlj_scan_final<<<(unsigned)n_tiles, NS_THREADS, 0, s>>>(in, out, n, sums);
  count_launch(3);
  return check_launch("nlj_scan_u64");
}

int32_t nlj_materialize(const NljOutParams &p, cudaStream_t s) {
  if (p.len <= 0) return TQ_OK;
  k_nlj_materialize<<<nlj_grid(p.len, 8), 256, 0, s>>>(p);
  count_launch();
  return check_launch("k_nlj_materialize");
}

}  // namespace tq
