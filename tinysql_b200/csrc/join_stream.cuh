// join_stream.cuh — the streaming PK-FK pipeline of HashJoinExec (included by join.cu, which defines ScatterParams,
// ProbeParams, JoinTable, ld_pair and the TMA / mbarrier helpers it uses).
//
// The kernels, all HBM/L2-bound integer work (no tensor cores: nothing here is a contraction):
//
//   k_scatter_aos<NC>   radix scatter of NC 8-byte columns into array-of-structs partition slabs (the build side, and the
//                       aggregation's pre-pass).  Input tiles arrive in shared memory by TMA bulk copies (cp.async.bulk +
//                       mbarrier, SASS UBLKCP) one tile ahead; a row's rank inside its partition is the return value of one
//                       shared-memory histogram atomic; rows leave through an AoS staging area as full-sector 16-byte stores.
//   k_scatter_cols<NC>  the probe side's scatter: k_scatter_aos's tiles and ranking, but every column is written straight into
//                       its RESULT column.  The result is cut into pages of page_rows slots, each owned by one partition and
//                       handed out while the scatter runs (a page table maps a partition's virtual pages to physical ones), so
//                       no pass has to count the partitions first.  k_pos_reset clears the cursors before it, k_pos_pages
//                       turns the final cursors into the span and the probe's work list after it.
//   k_probe_pos<NB>     probe of one partition against its L2-resident table.  Tiles of the result's probe KEY column are
//                       TMA-streamed through a ring of shared-memory stages by a producer warp that takes each tile's address
//                       from the page table; every consumer warp is independent (no CTA barrier, no output cursor): the probe
//                       columns are already in place, so a warp's 32 rows write 32 consecutive slots of every BUILD column,
//                       and a ballot word records which slots are real.  The holes (misses, and the unfilled tail of each
//                       partition's last page) are filled afterwards from the tail of the result (k_hole_*): for a
//                       foreign-key join that is about P * page_rows / 2 rows.  The contract is the result MULTISET (SURVEY
//                       Appendix B); order is not.
//   k_build_cta<NB>     build of the partition tables from build-side AoS slabs: one CTA per sub-table builds it in its own
//                       shared memory and writes it out once (the 2^lbits CTAs of a slab read it once from DRAM, then from L2).
//   k_build_cluster<NB> the same for sub-tables too large for one CTA: one 8-CTA cluster per slab builds its sub-tables in
//                       distributed shared memory.
#pragma once

#include <cooperative_groups.h>

namespace tq {

__device__ __forceinline__ bool mbar_try_wait(uint64_t *mbar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(mbar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_spin(uint64_t *mbar, uint32_t parity) {
  while (!mbar_try_wait(mbar, parity)) {}
}
__device__ __forceinline__ void mbar_arrive(uint64_t *mbar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(mbar)) : "memory");
}

// ------------------------------------------------------------------------------------------------ AoS scatter
static constexpr int SA_WARPS = 16;
static constexpr int SA_THREADS = SA_WARPS * 32;
static constexpr int SA_MAX_PBITS = 9;                       // 512 partitions (+ outer bin + trash bin)
static constexpr int SA_MAX_BINS = (1 << SA_MAX_PBITS) + 2;

static constexpr int SA_MAX_SEGS = 8;
struct ScatterAosParams {
  ScatterParams sp;        // columns, key, selected, pbits, cursors, slab limits; sp.out: the result columns of k_scatter_cols
  uint64_t *out;           // AoS slabs of k_scatter_aos: row r = out[r * NC .. r * NC + NC)
  int use_tma;             // every input column is 16-byte aligned: whole tiles are fetched by TMA bulk copies
  // Segmented input (multi-GPU receive buffers: one region per source rank, filled by the peers' push kernels): the batch is
  // the concatenation of n_segs regions of `seg_tiles` tiles each; region g holds *seg_cnt[g] rows (a DEVICE value the
  // pushing rank publishes), its columns start at seg_in[g][c].  n_segs == 0: one range, sp.in / sp.n.
  int n_segs, seg_tiles;
  const unsigned long long *seg_cnt[SA_MAX_SEGS];
  const uint64_t *seg_in[SA_MAX_SEGS][4];
};

// q.use_tma: whether every input column (of every segment) is 16-byte aligned, as the TMA bulk copies of whole tiles require.
static void set_use_tma(ScatterAosParams &q) {
  auto aligned = [](const void *ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  q.use_tma = 1;
  for (int c = 0; c < q.sp.n_cols; c++) {
    if (!aligned(q.sp.in[c].data)) q.use_tma = 0;
    for (int g = 0; g < q.n_segs; g++)
      if (!aligned(q.seg_in[g][c])) q.use_tma = 0;
  }
}

template <int T>
__host__ __device__ constexpr int sa_smem_bytes(int nc, int bins) {
  // 2 input stages + AoS staging + destination row per sorted position + 4 bin tables (4 bytes per bin each) + 2 mbarriers
  return 2 * nc * T * 8 + nc * T * 8 + T * 4 + 4 * ((bins * 4 + 15) & ~15) + 64;
}
template <int T>
__host__ __device__ constexpr int sa_occ(int nc) {  // resident CTAs per SM the shared-memory image allows (at most 3)
  return sa_smem_bytes<T>(nc, 130) <= 72 * 1024 ? 3 : (sa_smem_bytes<T>(nc, 130) <= 110 * 1024 ? 2 : 1);
}

// One tile = T rows.  Ranking a row inside its bin with a shared-memory atomicAdd-with-return costs about as much as
// reading the key, warp ballots over the bin bits or match.any several times that (scripts/ub/rank.cu measures the three)
// — so the rank is the atomic's return value.
// PLAIN: no outerSideFilter bytes and every key can match (same key type on both sides) — the foreign-key join; the general
// instantiation pays a few runtime-uniform branches per row for `selected`, the signed/unsigned rule and the outer-join bin.
template <int NC, int T, bool PLAIN>
__global__ void __launch_bounds__(SA_THREADS, sa_occ<T>(NC)) k_scatter_aos(const ScatterAosParams q) {
  constexpr int R = T / SA_THREADS;  // rows per thread per tile
  extern __shared__ __align__(128) unsigned char s_raw[];
  const ScatterParams &p = q.sp;
  const int n_part_bins = scatter_bins(p);      // partitions + the outer-join bin
  const int n_bins = n_part_bins + 1;           // + trash (rows that produce nothing)
  const int trash = n_bins - 1;
  const int bstride = (n_bins + 3) & ~3;
  uint64_t *s_in = reinterpret_cast<uint64_t *>(s_raw);                       // [2][NC][T]
  uint64_t *s_sorted = s_in + 2 * NC * T;                                      // [T][NC]
  uint32_t *s_dst = reinterpret_cast<uint32_t *>(s_sorted + NC * T);           // [T] slab row of sorted position i (0xFFFFFFFF: slab full)
  uint32_t *s_hist = s_dst + T;                                                // [n_bins] tile histogram (zero between tiles)
  uint2 *s_bin = reinterpret_cast<uint2 *>(s_hist + bstride);                  // [n_bins] {first sorted position of the bin, slab row of its first row}
  uint32_t *s_fit = reinterpret_cast<uint32_t *>(s_bin + bstride);             // [n_bins] rows of the bin that still fit its slab (read only when s_ovf)
  uint64_t *s_mbar = reinterpret_cast<uint64_t *>(s_fit + bstride);            // [2]
  __shared__ uint32_t s_warp[SA_WARPS + 1];
  __shared__ uint32_t s_ovf;                                                   // some bin of this tile overflowed its slab

  const int tid = threadIdx.x;
  const int kc = p.key_col;
  const int64_t n_tiles = q.n_segs ? (int64_t)q.n_segs * q.seg_tiles : (p.n + T - 1) / T;
  const int bpt = (n_bins + SA_THREADS - 1) / SA_THREADS;
  // where tile `tile` starts: column pointers + the rows it holds
  auto tile_src = [&](int64_t tile, const uint64_t *(&src)[NC]) -> int {
    if (q.n_segs == 0) {
#pragma unroll
      for (int c = 0; c < NC; c++) src[c] = p.in[c].data + tile * T;
      const int64_t left = p.n - tile * T;
      return (int)(left < T ? left : T);
    }
    const int g = (int)(tile / q.seg_tiles);
    const int64_t r0 = (tile % q.seg_tiles) * (int64_t)T;
    const unsigned long long cnt = *q.seg_cnt[g];
    int64_t left = cnt > (unsigned long long)q.seg_tiles * T ? 0 : (int64_t)cnt - r0;  // (an overflowed / unpublished region reads as empty)
    if (left < 0) left = 0;
#pragma unroll
    for (int c = 0; c < NC; c++) src[c] = q.seg_in[g][c] + r0;
    return (int)(left < T ? left : T);
  };

  for (int i = tid; i < n_bins; i += SA_THREADS) s_hist[i] = 0;
  if (tid == 0) {
    s_ovf = 0;
    mbar_init(&s_mbar[0], 1);
    mbar_init(&s_mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto tile_is_tma = [&](int64_t tile) {
    if (!q.use_tma) return false;
    const uint64_t *src[NC];
    return tile_src(tile, src) == T;
  };
  auto issue = [&](int64_t tile, int stage) {  // thread 0 only
    const uint64_t *src[NC];
    tile_src(tile, src);
    mbar_expect_tx(&s_mbar[stage], (uint32_t)(NC * T * 8));
#pragma unroll
    for (int c = 0; c < NC; c++) tma_load_1d(s_in + (stage * NC + c) * T, src[c], (uint32_t)(T * 8), &s_mbar[stage]);
  };
  if (tid == 0) {
    const int64_t t0 = blockIdx.x, t1 = t0 + gridDim.x;
    if (t0 < n_tiles && tile_is_tma(t0)) issue(t0, 0);
    if (t1 < n_tiles && tile_is_tma(t1)) issue(t1, 1);
  }
  int it = 0;
  int uses0 = 0, uses1 = 0;  // TMA fills consumed per stage = the mbarrier phase to wait for (ragged tiles do not use the barrier)
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
    const int stage = it & 1;
    const int64_t tile_base = tile * T;  // (row index for `selected`: single-range batches only)
    const uint64_t *tsrc[NC];
    const int rows = tile_src(tile, tsrc);
    uint64_t *in_s = s_in + stage * NC * T;
    if (q.use_tma && rows == T) {
      mbar_spin(&s_mbar[stage], (uint32_t)((stage ? uses1 : uses0) & 1));
      if (stage) uses1++; else uses0++;
    } else {  // unaligned caller buffers or a ragged / empty tile: plain loads
#pragma unroll
      for (int c = 0; c < NC; c++)
        for (int i = tid; i < rows; i += SA_THREADS) in_s[c * T + i] = tqd::ld_stream_u64(tsrc[c] + i);
      __syncthreads();
    }
    // ---- bin + rank of every row (rank = the histogram atomic's return value)
    uint16_t pid[R], rank[R];
#pragma unroll
    for (int k = 0; k < R; k++) {
      const int row = k * SA_THREADS + tid;
      uint32_t b = (uint32_t)trash;
      if (row < rows) {
        const uint64_t key = in_s[kc * T + row];
        if constexpr (PLAIN) {
          b = (uint32_t)part_of_hash(tqd::hash_key(key), p.pbits);
        } else {
          const bool sel = p.selected ? (p.selected[tile_base + row] != 0) : true;
          if (sel && key_valid(key, true, p.key_mode)) b = (uint32_t)part_of_hash(tqd::hash_key(key), p.pbits);
          else if (p.is_outer) b = (uint32_t)(n_part_bins - 1);
        }
      }
      pid[k] = (uint16_t)b;
      rank[k] = (uint16_t)atomicAdd(&s_hist[b], 1u);
    }
    __syncthreads();
    // ---- exclusive scan over the bins; every non-empty bin claims its slab run with ONE global atomic
    uint32_t tsum = 0;
    for (int j = 0; j < bpt; j++) {
      const int b = tid * bpt + j;
      if (b < n_bins) tsum += s_hist[b];
    }
    uint32_t run = block_excl_scan<SA_THREADS>(tsum, s_warp);
    for (int j = 0; j < bpt; j++) {
      const int b = tid * bpt + j;
      if (b < n_bins) {
        const uint32_t c = s_hist[b];
        s_hist[b] = 0;  // ready for the next tile (its ranking starts behind two more barriers)
        uint32_t g = 0;
        if (c && b != trash) {
          g = atomicAdd(&p.part_cursor[b], c);
          uint32_t fit = c;
          if (p.part_lim) {
            const uint32_t lim = p.part_lim[b];
            if (g + c > lim) { fit = (g < lim) ? (lim - g) : 0u; atomicOr(p.overflow, 1ull); s_ovf = 1; }
          }
          s_fit[b] = fit;
        }
        s_bin[b] = make_uint2(run, g);
        run += c;
      }
    }
    __syncthreads();
    const uint32_t total = s_bin[trash].x;  // rows that go somewhere
    const bool ovf = s_ovf != 0;            // (sticky: the whole batch is re-run on the exact path anyway)
    // ---- place the rows at their sorted positions (AoS) together with their slab row
#pragma unroll
    for (int k = 0; k < R; k++) {
      const uint32_t b = pid[k];
      if (b == (uint32_t)trash) continue;
      const int row = k * SA_THREADS + tid;
      const uint2 bin = s_bin[b];
      const uint32_t sp = bin.x + rank[k];
      s_dst[sp] = (ovf && rank[k] >= s_fit[b]) ? 0xFFFFFFFFu : bin.y + rank[k];
      if constexpr (NC == 2) {
        *reinterpret_cast<ulonglong2 *>(s_sorted + (size_t)sp * 2) = make_ulonglong2(in_s[row], in_s[T + row]);
      } else {
#pragma unroll
        for (int c = 0; c < NC; c++) s_sorted[(size_t)sp * NC + c] = in_s[c * T + row];
      }
    }
    __syncthreads();
    // the input stage is free again: fetch the tile this CTA handles two iterations from now
    if (tid == 0) {
      const int64_t nt = tile + 2 * (int64_t)gridDim.x;
      if (nt < n_tiles && tile_is_tma(nt)) issue(nt, stage);
    }
    // ---- stream the sorted tile out: consecutive threads write consecutive slab rows (full sectors inside a run)
    if constexpr (NC % 2 == 0) {
      constexpr int V = NC / 2;  // 16-byte pieces per row
      for (uint32_t i = tid; i < total * V; i += SA_THREADS) {
        const uint32_t r = i / V, piece = i % V;
        const uint32_t d = s_dst[r];
        if (d == 0xFFFFFFFFu) continue;  // slab full (the batch is re-run on the exact path)
        tqd::st_stream_u64x2(q.out + (uint64_t)d * NC + piece * 2, *reinterpret_cast<const ulonglong2 *>(s_sorted + (size_t)r * NC + piece * 2));
      }
    } else {
      for (uint32_t i = tid; i < total * NC; i += SA_THREADS) {
        const uint32_t r = i / NC, w = i % NC;
        const uint32_t d = s_dst[r];
        if (d == 0xFFFFFFFFu) continue;
        tqd::st_stream_u64(q.out + (uint64_t)d * NC + w, s_sorted[(size_t)r * NC + w]);
      }
    }
    __syncthreads();  // the staging area and the bin tables are rewritten by the next tile
  }
}

typedef void (*ScatterAosKernel)(const ScatterAosParams);
template <int T, bool PLAIN>
static ScatterAosKernel scatter_aos_kernel_t(int nc) {
  switch (nc) {
    case 1: return k_scatter_aos<1, T, PLAIN>;
    case 2: return k_scatter_aos<2, T, PLAIN>;
    case 3: return k_scatter_aos<3, T, PLAIN>;
    case 4: return k_scatter_aos<4, T, PLAIN>;
  }
  return nullptr;
}
// tile size: 2048 rows if that shared-memory image fits an SM, else 1024
static int scatter_aos_tile(int nc, int bins) {
  return sa_smem_bytes<2048>(nc, bins) <= 220 * 1024 ? 2048 : 1024;
}
static int32_t launch_scatter_aos(const ScatterAosParams &q, int nc, cudaStream_t s) {
  const int bins = scatter_bins(q.sp) + 1;
  const int T = scatter_aos_tile(nc, bins);
  const bool plain = !q.sp.selected && q.sp.key_mode == KEYMODE_RAW;
  ScatterAosKernel k;
  int smem, per_sm;
  if (T == 2048) { k = plain ? scatter_aos_kernel_t<2048, true>(nc) : scatter_aos_kernel_t<2048, false>(nc); smem = sa_smem_bytes<2048>(nc, bins); per_sm = sa_occ<2048>(nc); }
  else { k = plain ? scatter_aos_kernel_t<1024, true>(nc) : scatter_aos_kernel_t<1024, false>(nc); smem = sa_smem_bytes<1024>(nc, bins); per_sm = sa_occ<1024>(nc); }
  if (!k || smem > 227 * 1024) { set_error("internal: AoS scatter of %d columns into %d bins does not fit shared memory", nc, bins); return TQ_ERR_INVALID_ARG; }
  TQ_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int64_t tiles = (q.sp.n + T - 1) / T;
  while (per_sm > 1 && (int64_t)smem * per_sm > 224 * 1024) per_sm--;   // (more bins than the occupancy estimate assumed)
  const int64_t cap = (int64_t)rt().sm_count * per_sm;
  k<<<(int)(tiles < cap ? tiles : cap), SA_THREADS, smem, s>>>(q);
  count_launch();
  return check_launch("k_scatter_aos");
}

// ------------------------------------------------------------------------------------------------ positional probe
// The paged result of a positional batch.  The result's slots are cut into pages of page_rows slots (whole probe tiles); a
// page belongs to one partition.  Partition q's rows take VIRTUAL slots 0, 1, ... (cursor[q] counts them); its virtual page k
// is physical page pt[q * kmax + k], and physical page i holds result slots [i * page_rows, (i + 1) * page_rows).
//   cursor  [n_parts + 1]  rows of each partition so far; cursor[n_parts] = physical pages handed out
//   chunk   [n_parts + 1]  first probe CTA of each partition (k_pos_pages); chunk[n_parts] = the probe CTAs in all
//   pt      [n_parts * kmax]  page table: (epoch << 32) | physical page.  An entry with another epoch belongs to an earlier
//                          batch, so the table is never cleared: each batch only writes the entries it uses.
//   err     set when a page id did not appear in time (the batch fails with an internal error instead of hanging)
struct PosPages {
  uint32_t *cursor, *chunk;
  unsigned long long *pt;
  uint32_t page_rows, kmax, epoch;
  unsigned long long *err;
};
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Rows of tile `tile` of a batch (T rows per tile) and where its column c starts: one range (sp.in / sp.n), or the segmented
// regions as k_scatter_aos reads them (region g = tiles [g * seg_tiles, (g + 1) * seg_tiles)).
__device__ __forceinline__ int stream_tile_rows(const ScatterAosParams &q, int T, int64_t tile) {
  if (q.n_segs == 0) {
    const int64_t left = q.sp.n - tile * T;
    return (int)(left < T ? left : T);
  }
  const int g = (int)(tile / q.seg_tiles);
  const int64_t r0 = (tile % q.seg_tiles) * (int64_t)T;
  const unsigned long long cnt = *q.seg_cnt[g];
  int64_t left = cnt > (unsigned long long)q.seg_tiles * T ? 0 : (int64_t)cnt - r0;  // (an overflowed / unpublished region reads as empty)
  if (left < 0) left = 0;
  return (int)(left < T ? left : T);
}
__device__ __forceinline__ const uint64_t *stream_tile_col(const ScatterAosParams &q, int T, int64_t tile, int c) {
  if (q.n_segs == 0) return q.sp.in[c].data + tile * T;
  return q.seg_in[tile / q.seg_tiles][c] + (tile % q.seg_tiles) * (int64_t)T;
}
// The partition of a probe row on the positional path (an inner join), or -1 for a row that produces nothing: k_scatter_aos's
// bin rule.  `row` indexes `selected` (single-range batches only).
template <bool PLAIN>
__device__ __forceinline__ int stream_part(const ScatterParams &p, uint64_t key, int64_t row) {
  if constexpr (!PLAIN) {
    const bool sel = p.selected ? (p.selected[row] != 0) : true;
    if (!sel || !key_valid(key, true, p.key_mode)) return -1;
  }
  return (int)part_of_hash(tqd::hash_key(key), p.pbits);
}

// ---- batch start (one CTA): every partition's cursor and the page counter back to zero.
static constexpr int POS_BASES_THREADS = 512;   // >= partitions of the streaming path (SA_MAX_PBITS)
__global__ void __launch_bounds__(POS_BASES_THREADS) k_pos_reset(uint32_t *cursor, int n) {
  for (int i = threadIdx.x; i < n; i += POS_BASES_THREADS) cursor[i] = 0;
}

// ---- after the scatter (one CTA): from the final cursors (rows per partition) the span S = pages * page_rows (*span) and the
// probe's work list: ceil(cursor[q] / tile_rows) tiles per partition, PP_CHUNK_TILES tiles per CTA, consecutive CTAs on one
// partition (so its table stays in L2 while they run).
static constexpr int PP_CHUNK_TILES = 11;       // probe tiles per CTA (~8K rows): enough CTAs per partition that only a handful of partitions are live at once
__global__ void __launch_bounds__(POS_BASES_THREADS) k_pos_pages(const PosPages m, int n_parts, int tile_rows, unsigned long long *span) {
  __shared__ uint32_t s_warp[POS_BASES_THREADS / 32 + 1];
  const int q = threadIdx.x;
  const uint32_t c = q < n_parts ? m.cursor[q] : 0u;
  const uint32_t tiles = (c + (uint32_t)tile_rows - 1) / (uint32_t)tile_rows;
  const uint32_t first = block_excl_scan<POS_BASES_THREADS>((tiles + PP_CHUNK_TILES - 1) / PP_CHUNK_TILES, s_warp);
  if (q < n_parts) m.chunk[q] = first;
  if (q == 0) {
    m.chunk[n_parts] = s_warp[POS_BASES_THREADS / 32];
    *span = (unsigned long long)m.cursor[n_parts] * m.page_rows;
  }
}

// ---- column-wise scatter into the result: k_scatter_aos's TMA-fed tiles and shared-memory ranking; a row's virtual slot is
// the run its tile claims on cursor[q] plus its rank.  Pages are handed out as the claims reach them: the claim whose run
// contains the first slot of virtual page k allocates a physical page (one atomic on the page counter) and publishes its id in
// pt.  A page is at least one tile, so a run crosses at most one page boundary: it lies in the page its first slot falls in
// (allocated by this claim when the run starts it, else by an earlier claim) and, past the boundary, in the page it opens.
// An earlier claim's page id is loaded right after the claim and only needed once the rows are placed; a thread makes all its
// claims and allocations before it waits on any id, so every id it waits for belongs to a claim that has nothing left to
// wait for (no deadlock), and the wait is bounded besides.  Rows are placed as (bin, rank) and mapped to physical slots in
// the write-out loop through a per-bin record.  Every page is whole tiles of the probe, so nothing can overflow and a skewed
// batch stays on this path.  The staging area is column-major, so each column leaves as runs of consecutive 8-byte stores
// (consecutive threads, consecutive slots).  k_scatter_aos's shared-memory image plus one more per-bin table (sc_smem_bytes),
// and the same segmented-region geometry.
template <int T>
__host__ __device__ constexpr int sc_smem_bytes(int nc, int bins) { return sa_smem_bytes<T>(nc, bins) + ((bins * 4 + 15) & ~15); }
static constexpr uint32_t PAGE_WAIT_SPINS = 1u << 20;   // ~0.1 s of polling for a page id before the batch is failed
template <int NC, int T, bool PLAIN>
__global__ void __launch_bounds__(SA_THREADS, sa_occ<T>(NC)) k_scatter_cols(const ScatterAosParams q, const PosPages pg) {
  constexpr int R = T / SA_THREADS;  // rows per thread per tile
  constexpr int BPT = (SA_MAX_BINS + SA_THREADS - 1) / SA_THREADS;  // bins per thread, at most
  extern __shared__ __align__(128) unsigned char s_raw[];
  const ScatterParams &p = q.sp;
  const int n_parts = 1 << p.pbits;
  const int trash = n_parts;                    // rows that produce nothing
  const int n_bins = n_parts + 1;
  const int bstride = (n_bins + 3) & ~3;
  const uint32_t PG = pg.page_rows;
  uint64_t *s_in = reinterpret_cast<uint64_t *>(s_raw);                       // [2][NC][T]
  uint64_t *s_sorted = s_in + 2 * NC * T;                                      // [NC][T]
  uint32_t *s_dst = reinterpret_cast<uint32_t *>(s_sorted + NC * T);           // [T] (bin << 16) | rank of sorted position i
  uint32_t *s_hist = s_dst + T;                                                // [n_bins] tile histogram (zero between tiles)
  uint2 *s_bin = reinterpret_cast<uint2 *>(s_hist + bstride);                  // [n_bins] {first sorted position of the bin, rows of its run before the page boundary}
  uint2 *s_map = s_bin + bstride;                                              // [n_bins] {physical slot of rank 0, physical slot of rank e minus e}
  uint64_t *s_mbar = reinterpret_cast<uint64_t *>(s_map + bstride);            // [2]
  __shared__ uint32_t s_warp[SA_WARPS + 1];

  const int tid = threadIdx.x;
  const int kc = p.key_col;
  const int64_t n_tiles = q.n_segs ? (int64_t)q.n_segs * q.seg_tiles : (p.n + T - 1) / T;
  const int bpt = (n_bins + SA_THREADS - 1) / SA_THREADS;

  for (int i = tid; i < n_bins; i += SA_THREADS) s_hist[i] = 0;
  if (tid == 0) {
    mbar_init(&s_mbar[0], 1);
    mbar_init(&s_mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto tile_is_tma = [&](int64_t tile) { return q.use_tma && stream_tile_rows(q, T, tile) == T; };
  auto issue = [&](int64_t tile, int stage) {  // thread 0 only
    mbar_expect_tx(&s_mbar[stage], (uint32_t)(NC * T * 8));
#pragma unroll
    for (int c = 0; c < NC; c++) tma_load_1d(s_in + (stage * NC + c) * T, stream_tile_col(q, T, tile, c), (uint32_t)(T * 8), &s_mbar[stage]);
  };
  // a new physical page for virtual page slot `e` of the page table: its id
  auto alloc_page = [&](unsigned long long *e) {
    const uint32_t id = atomicAdd(&pg.cursor[n_parts], 1u);
    st_relaxed_u64(e, ((unsigned long long)pg.epoch << 32) | id);  // (the id is the only datum: nothing else to release)
    return id;
  };
  if (tid == 0) {
    const int64_t t0 = blockIdx.x, t1 = t0 + gridDim.x;
    if (t0 < n_tiles && tile_is_tma(t0)) issue(t0, 0);
    if (t1 < n_tiles && tile_is_tma(t1)) issue(t1, 1);
  }
  int it = 0;
  int uses0 = 0, uses1 = 0;  // TMA fills consumed per stage = the mbarrier phase to wait for (ragged tiles do not use the barrier)
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
    const int stage = it & 1;
    const int rows = stream_tile_rows(q, T, tile);
    uint64_t *in_s = s_in + stage * NC * T;
    if (q.use_tma && rows == T) {
      mbar_spin(&s_mbar[stage], (uint32_t)((stage ? uses1 : uses0) & 1));
      if (stage) uses1++; else uses0++;
    } else {  // unaligned caller buffers or a ragged / empty tile: plain loads
#pragma unroll
      for (int c = 0; c < NC; c++) {
        const uint64_t *src = stream_tile_col(q, T, tile, c);
        for (int i = tid; i < rows; i += SA_THREADS) in_s[c * T + i] = tqd::ld_stream_u64(src + i);
      }
      __syncthreads();
    }
    // ---- bin + rank of every row (rank = the histogram atomic's return value)
    uint16_t pid[R], rank[R];
#pragma unroll
    for (int k = 0; k < R; k++) {
      const int row = k * SA_THREADS + tid;
      int b = trash;
      if (row < rows) {
        b = stream_part<PLAIN>(p, in_s[kc * T + row], tile * T + row);
        if (b < 0) b = trash;
      }
      pid[k] = (uint16_t)b;
      rank[k] = (uint16_t)atomicAdd(&s_hist[b], 1u);
    }
    __syncthreads();
    // ---- exclusive scan over the bins; every non-empty partition claims its run of virtual slots with ONE global atomic
    uint32_t tsum = 0;
    for (int j = 0; j < bpt; j++) {
      const int b = tid * bpt + j;
      if (b < n_bins) tsum += s_hist[b];
    }
    uint32_t run = block_excl_scan<SA_THREADS>(tsum, s_warp);
    // a run that starts inside a page an earlier claim opened: that page's table entry (loaded now, awaited after placement)
    const unsigned long long *wait_e[BPT];
    unsigned long long wait_v[BPT];
    uint32_t wait_o[BPT], wait_d1[BPT];
#pragma unroll
    for (int j = 0; j < BPT; j++) {
      const int b = tid * bpt + j;
      wait_e[j] = nullptr;
      if (j < bpt && b < n_bins) {
        const uint32_t c = s_hist[b];
        s_hist[b] = 0;  // ready for the next tile (its ranking starts behind two more barriers)
        uint32_t e = 0;
        if (c && b != trash) {
          const uint32_t g = atomicAdd(&pg.cursor[b], c);
          unsigned long long *row = pg.pt + (uint64_t)b * pg.kmax;
          const uint32_t k0 = g / PG, o = g - k0 * PG;
          e = PG - o;                                              // rows of the run inside its first page
          const uint32_t d1 = c > e ? alloc_page(row + k0 + 1) * PG - e : 0u;   // (rank r >= e lands at d1 + r)
          if (o == 0) {
            s_map[b] = make_uint2(alloc_page(row + k0) * PG, d1);
          } else {
            wait_e[j] = row + k0;
            wait_v[j] = ld_relaxed_u64(row + k0);
            wait_o[j] = o;
            wait_d1[j] = d1;
          }
        }
        s_bin[b] = make_uint2(run, e);
        run += c;
      }
    }
    __syncthreads();
    const uint32_t total = s_bin[trash].x;  // rows that go somewhere
    // ---- place the rows at their sorted positions (column-major) together with their bin and rank
#pragma unroll
    for (int k = 0; k < R; k++) {
      const uint32_t b = pid[k];
      if (b == (uint32_t)trash) continue;
      const int row = k * SA_THREADS + tid;
      const uint32_t sp = s_bin[b].x + rank[k];
      s_dst[sp] = (b << 16) | rank[k];
#pragma unroll
      for (int c = 0; c < NC; c++) s_sorted[c * T + sp] = in_s[c * T + row];
    }
    // ---- the page ids of runs that started inside an earlier claim's page
#pragma unroll
    for (int j = 0; j < BPT; j++) {
      if (!wait_e[j]) continue;
      unsigned long long v = wait_v[j];
      for (uint32_t spins = 0; (uint32_t)(v >> 32) != pg.epoch; spins++) {
        if (spins == PAGE_WAIT_SPINS) { atomicOr(pg.err, 1ull); v = 0; break; }   // (page 0: writes stay in bounds)
        __nanosleep(64);
        v = ld_relaxed_u64(wait_e[j]);
      }
      s_map[tid * bpt + j] = make_uint2((uint32_t)v * PG + wait_o[j], wait_d1[j]);
    }
    __syncthreads();
    // the input stage is free again: fetch the tile this CTA handles two iterations from now
    if (tid == 0) {
      const int64_t nt = tile + 2 * (int64_t)gridDim.x;
      if (nt < n_tiles && tile_is_tma(nt)) issue(nt, stage);
    }
    // ---- stream the sorted tile out: consecutive threads write consecutive slots of every result column
    for (uint32_t i = tid; i < total; i += SA_THREADS) {
      const uint32_t u = s_dst[i], b = u >> 16, r = u & 0xFFFFu;
      const uint2 m = s_map[b];
      const uint32_t d = (r < s_bin[b].y ? m.x : m.y) + r;
#pragma unroll
      for (int c = 0; c < NC; c++) tqd::st_stream_u64(p.out[c].data + d, s_sorted[c * T + i]);
    }
    __syncthreads();  // the staging area and the bin tables are rewritten by the next tile
  }
}

typedef void (*ScatterColsKernel)(const ScatterAosParams, const PosPages);
template <int T, bool PLAIN>
static ScatterColsKernel scatter_cols_kernel_t(int nc) {
  if (T == 4096) return nc == 1 ? k_scatter_cols<1, 4096, PLAIN> : (nc == 2 ? k_scatter_cols<2, 4096, PLAIN> : nullptr);
  switch (nc) {  // (one column always takes 4096-row tiles: that image fits at every partition count)
    case 2: return k_scatter_cols<2, 2048, PLAIN>;
    case 3: return k_scatter_cols<3, 2048, PLAIN>;
    case 4: return k_scatter_cols<4, 2048, PLAIN>;
  }
  return nullptr;
}
// Rows per tile of the column scatter: 4096 where that shared-memory image fits an SM (one or two columns), else 2048.  A run
// a tile claims in one partition is then ~T / P rows of every column: at C3 (128 partitions) 4096-row tiles write runs of
// 256 bytes per column, which measured 1.39 ms against 1.65 ms for 2048-row tiles (H100 80GB HBM3, 700 W).
static int scatter_cols_tile(int nc, int bins) { return sc_smem_bytes<4096>(nc, bins) <= 220 * 1024 ? 4096 : 2048; }
// Segmented regions are read in whole scatter tiles, so a region's rows are a multiple of the largest.
static constexpr int POS_SEG_ROWS_ALIGN = 4096;
static constexpr int PP_TILE_ROWS = 12 * 32 * 2;  // rows per tile of k_probe_pos (probe_pos_variant)

// Rows per page of the positional result.  Whole probe tiles, so ballot words and the probe's bulk copies stay inside a page;
// at least one scatter tile, so a run a tile claims crosses at most one page boundary; past that, the most tiles that keep
// P * page_rows -- the rows the partitions' last pages can leave unfilled, hence the room the result needs beyond n and the
// holes to fill -- within 1 % of the batch.  At C3 (1e8 rows, 128 partitions) that is 10 tiles = 7,680 rows; a batch of 8M
// rows gets the 6-tile minimum.
static uint32_t pos_page_rows(int64_t n, int P, int nc) {
  const int64_t min_tiles = (scatter_cols_tile(nc, P + 1) + PP_TILE_ROWS - 1) / PP_TILE_ROWS;
  const int64_t tiles = n / (100ll * P * PP_TILE_ROWS);
  return (uint32_t)((tiles > min_tiles ? tiles : min_tiles) * PP_TILE_ROWS);
}

// reset -> column-wise scatter -> page bases of one positional batch into the result columns q.sp.out[c] (every slot of
// [0, S) belongs to exactly one page).  q describes the input as for k_scatter_aos (columns, key, key_mode, selected, pbits,
// n, segments of seg_rows rows each, a multiple of POS_SEG_ROWS_ALIGN); m's words are reserved by the caller.
static int32_t launch_pos_scatter(ScatterAosParams &q, int64_t seg_rows, const PosPages &m, unsigned long long *span, cudaStream_t s) {
  const int nc = q.sp.n_cols, P = 1 << q.sp.pbits;
  const bool plain = !q.sp.selected && q.sp.key_mode == KEYMODE_RAW;
  const int T = scatter_cols_tile(nc, P + 1);
  ScatterColsKernel k = T == 4096 ? (plain ? scatter_cols_kernel_t<4096, true>(nc) : scatter_cols_kernel_t<4096, false>(nc))
                                  : (plain ? scatter_cols_kernel_t<2048, true>(nc) : scatter_cols_kernel_t<2048, false>(nc));
  const int smem = T == 4096 ? sc_smem_bytes<4096>(nc, P + 1) : sc_smem_bytes<2048>(nc, P + 1);
  int per_sm = T == 4096 ? sa_occ<4096>(nc) : sa_occ<2048>(nc);
  if (!k || smem > 227 * 1024) { set_error("internal: column scatter of %d columns into %d partitions does not fit shared memory", nc, P); return TQ_ERR_INVALID_ARG; }
  TQ_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  while (per_sm > 1 && (int64_t)smem * per_sm > 224 * 1024) per_sm--;
  // (launched after the host-side set-up above, so that the scatter follows the tiny reset without a gap)
  k_pos_reset<<<1, POS_BASES_THREADS, 0, s>>>(m.cursor, P + 1);
  TQ_TRY(check_launch("k_pos_reset"));
  const int64_t tiles = q.n_segs ? (int64_t)q.n_segs * (seg_rows / T) : (q.sp.n + T - 1) / T, cap = (int64_t)rt().sm_count * per_sm;
  q.seg_tiles = (int)(seg_rows / T);
  set_use_tma(q);
  k<<<(int)(tiles < cap ? (tiles < 1 ? 1 : tiles) : cap), SA_THREADS, smem, s>>>(q, m);
  TQ_TRY(check_launch("k_scatter_cols"));
  k_pos_pages<<<1, POS_BASES_THREADS, 0, s>>>(m, P, PP_TILE_ROWS, span);
  count_launch(3);
  return check_launch("k_pos_pages");
}

static constexpr int PP_STAGES = 4;

struct ProbePosParams {
  const uint64_t *keys;              // the result's probe key column
  const uint32_t *cnt, *chunk;       // PosPages: rows per partition (the final cursors), the work list
  const unsigned long long *pt;      // PosPages: the page table, kmax entries per partition
  uint32_t page_rows, kmax;
  int n_parts;
  uint64_t *out_build[4];
  int build_word[4];                 // word of build column c inside a table entry
  uint32_t *valid;                   // one bit per output slot
  unsigned long long *cursor;        // [0] += matched rows
  int dbg_no_tma, dbg_late_release;  // diagnostics (TQ_JOIN_PP_DEBUG bit 0 / bit 1): plain copies by the producer warp; release a stage only after the step
};

// Find `key` in its partition table starting at its home entry.  SHIFT == 1: 16-byte entries fetched as 32-byte aligned
// PAIRS (one sector tests two slots); SHIFT == 2: 32-byte entries.  loc is the entry index in the whole table (the home
// entry, already loaded into a / b); past it the walk wraps inside the key's table of `cap` entries (table index = its top
// `pbits` hash bits).  Returns hit; w1 = word 1 of the matched entry, loc = its index.  The common case — the key sits in
// its home pair — is straight-line code.
template <int SHIFT>
__device__ __forceinline__ bool probe_find(const uint64_t *words, uint32_t cap, int pbits, uint64_t key, uint32_t &loc, uint64_t &w1, ulonglong2 a, ulonglong2 b) {
  // 1: hit at loc (+ 1 for the pair's second entry), 0: miss, -1: the walk goes on
  auto test = [&](ulonglong2 x, ulonglong2 y) -> int {
    if (x.x == key) { w1 = x.y; return 1; }
    if constexpr (SHIFT == 1) {
      if (y.x == key) { w1 = y.y; loc += 1; return 1; }
      if (y.x == EMPTY_KEY) return 0;
    }
    return x.x == EMPTY_KEY ? 0 : -1;
  };
  int r = test(a, b);
  if (r >= 0) return r != 0;
  const uint32_t base = (uint32_t)part_of_hash(tqd::hash_key(key), pbits) * cap;
  uint32_t i = loc - base;
  for (;;) {
    i = next_slot(i, SHIFT == 1 ? 2 : 1, cap);
    loc = base + i;
    if constexpr (SHIFT == 1) {
      const EntryPair pr = ld_pair(words, loc, false);
      r = test(pr.a, pr.b);
    } else {
      r = test(ld_entry(words, loc, SHIFT), b);
    }
    if (r >= 0) return r != 0;
  }
}

// R rows per lane per step, CW consumer warps (+ 1 producer warp), OCC resident CTAs per SM asked of the compiler.
// One tile = CW * 32 * R rows, and a page is whole tiles: the producer maps each tile of the partition to its physical slots
// through the page table and hands that slot to the consumers with the stage.  The probe columns are already in their result
// slots (k_scatter_cols): this kernel reads the key column back and writes the build columns and the validity ballots.
template <int NB, int R, int CW, int OCC>
__global__ void __launch_bounds__((CW + 1) * 32, OCC) k_probe_pos(const ProbePosParams p, const JoinTable t) {
  constexpr int PP_TILE = CW * 32 * R;
  constexpr int PP_CONSUMER_WARPS = CW;
  constexpr int SHIFT = NB > 2 ? 2 : 1;  // words per entry = 1 << SHIFT (the host builds the table the same way)
  extern __shared__ __align__(128) unsigned char s_raw[];
  uint64_t *s_tile = reinterpret_cast<uint64_t *>(s_raw);  // [PP_STAGES][PP_TILE] probe keys
  __shared__ __align__(8) uint64_t s_full[PP_STAGES], s_empty[PP_STAGES];
  __shared__ uint64_t s_sink[CW];
  __shared__ uint32_t s_slot[PP_STAGES];  // physical slot of the first row of the tile in each stage
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // this CTA's partition and tiles, from the work list of k_pos_pages: chunk[part] <= blockIdx.x < chunk[part + 1]
  const uint32_t cta = blockIdx.x;
  if (cta >= p.chunk[p.n_parts]) return;  // (the grid is sized for the worst case)
  uint32_t part = 0, hi = (uint32_t)p.n_parts;
  while (hi - part > 1) {
    const uint32_t mid = (part + hi) >> 1;
    if (p.chunk[mid] <= cta) part = mid;
    else hi = mid;
  }
  const int64_t p_rows = p.cnt[part];
  const int64_t p_tiles = (p_rows + PP_TILE - 1) / PP_TILE;
  const int64_t t_lo = (int64_t)(cta - p.chunk[part]) * PP_CHUNK_TILES;
  const int64_t t_hi = t_lo + PP_CHUNK_TILES < p_tiles ? t_lo + PP_CHUNK_TILES : p_tiles;
  const unsigned long long *pages = p.pt + (uint64_t)part * p.kmax;
  const uint32_t PG = p.page_rows;
  auto tile_slot = [&](int64_t tile) {  // physical slot of the tile's first row: a multiple of 32 (256-byte aligned keys)
    const uint32_t r0 = (uint32_t)(tile * PP_TILE), k = r0 / PG;
    return (uint32_t)pages[k] * PG + (r0 - k * PG);
  };
  if (tid == 0) {
    for (int s = 0; s < PP_STAGES; s++) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], PP_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == PP_CONSUMER_WARPS && p.dbg_no_tma) {
    int it = 0;
    for (int64_t tile = t_lo; tile < t_hi; tile++, it++) {
      const int s = it % PP_STAGES;
      if (it >= PP_STAGES) mbar_spin(&s_empty[s], (uint32_t)(((it / PP_STAGES) - 1) & 1));
      const int64_t r0 = tile * PP_TILE;
      const int64_t rows = (p_rows - r0) < PP_TILE ? (p_rows - r0) : PP_TILE;
      const uint32_t slot = tile_slot(tile);
      uint64_t *dst = s_tile + (size_t)s * PP_TILE;
      for (int64_t i = lane; i < rows; i += 32) dst[i] = p.keys[slot + i];
      __syncwarp();
      if (lane == 0) {
        s_slot[s] = slot;
        mbar_arrive(&s_full[s]);
      }
    }
    return;
  }
  if (warp == PP_CONSUMER_WARPS) {
    // ---- producer: keeps PP_STAGES key tiles in flight (TMA bulk copies; bytes rounded up to 16: an odd row count ends
    // inside the tile's page)
    if (lane == 0) {
      int it = 0;
      for (int64_t tile = t_lo; tile < t_hi; tile++, it++) {
        const int s = it % PP_STAGES;
        if (it >= PP_STAGES) mbar_spin(&s_empty[s], (uint32_t)(((it / PP_STAGES) - 1) & 1));
        const int64_t r0 = tile * PP_TILE;
        const int64_t rows = (p_rows - r0) < PP_TILE ? (p_rows - r0) : PP_TILE;
        const uint32_t bytes = (uint32_t)((rows * 8 + 15) & ~15ll);
        const uint32_t slot = tile_slot(tile);
        s_slot[s] = slot;  // (published to the consumers by the arrive below)
        mbar_expect_tx(&s_full[s], bytes);
        tma_load_1d(s_tile + (size_t)s * PP_TILE, p.keys + slot, bytes, &s_full[s]);
      }
    }
    return;
  }
  // ---- consumers: warp w owns rows [w * 32 * R, (w + 1) * 32 * R) of every tile.  The table may be split finer than the
  // probe partitions (k_build_cluster's sub-tables), so a row's table comes from its own hash.
  const uint32_t cap = t.cap;
  const int woff = warp * (32 * R) + lane;                      // this lane's first row inside a tile
  uint64_t *ob[NB];
  int bw[NB];
#pragma unroll
  for (int c = 0; c < NB; c++) { ob[c] = p.out_build[c] + woff; bw[c] = p.build_word[c]; }
  unsigned matched = 0;
  int it = 0;
  for (int64_t tile = t_lo; tile < t_hi; tile++, it++) {
    const int s = it % PP_STAGES;
    mbar_spin(&s_full[s], (uint32_t)((it / PP_STAGES) & 1));
    const int64_t t0 = tile * PP_TILE;                              // first row of the tile inside the partition
    const uint64_t *src = s_tile + (size_t)s * PP_TILE + woff;
    const uint32_t oslot = s_slot[s];                               // ... and its physical slot
    uint64_t key[R];
#pragma unroll
    for (int k = 0; k < R; k++) key[k] = src[k * 32];
    // The stage may be refilled (a TMA write) as soon as every warp has released it, so the values must have LEFT shared
    // memory first.  An issued LDS is not a completed one: SASS showed LDS.128 x4, WARPSYNC, SYNCS.ARRIVE with no scoreboard
    // wait in between, and the refill then tore rows (first 16 bytes of one tile, last 16 of another).  The register scoreboard is per warp, so ONE instruction that reads every loaded
    // register waits for the whole warp's loads: lane 0 stores their XOR to a sink word before it arrives on the barrier.
    uint64_t dep = oslot;
#pragma unroll
    for (int k = 0; k < R; k++) dep ^= key[k];
    __syncwarp();
    if (lane == 0) {
      *reinterpret_cast<volatile uint64_t *>(&s_sink[warp]) = dep;
      if (!p.dbg_late_release) mbar_arrive(&s_empty[s]);  // the stage can be refilled while this warp probes
    }
    uint32_t loc[R];  // entry index in the whole table (probe_find)
    bool inb[R];
    ulonglong2 ea[R], eb[R];
#pragma unroll
    for (int k = 0; k < R; k++) {  // R independent sector loads in flight
      inb[k] = (t0 + woff + k * 32) < p_rows;
      const uint64_t h = tqd::hash_key(key[k]);
      loc[k] = (uint32_t)part_of_hash(h, t.pbits) * cap + home_slot(h, cap, SHIFT);
      ea[k] = make_ulonglong2(EMPTY_KEY, 0);
      eb[k] = ea[k];
      if (inb[k] && key[k] != EMPTY_KEY) {
        if constexpr (SHIFT == 1) { const EntryPair pr = ld_pair(t.words, loc[k], false); ea[k] = pr.a; eb[k] = pr.b; }
        else ea[k] = ld_entry(t.words, loc[k], SHIFT);
      }
    }
    uint32_t *vword = p.valid + ((oslot + warp * (32 * R)) >> 5);   // output slot of this lane's k-th row = ob[c] + oslot + k * 32
#pragma unroll
    for (int k = 0; k < R; k++) {
      uint64_t w1 = 0;
      bool hit = false;
      if (inb[k]) {
        if (key[k] != EMPTY_KEY) hit = probe_find<SHIFT>(t.words, cap, t.pbits, key[k], loc[k], w1, ea[k], eb[k]);
        else if (t.sent_cnt) {  // a probe key equal to the empty marker: its row is the table's side entry
          loc[k] = t.sent_off;
          w1 = t.words[((uint64_t)t.sent_off << SHIFT) + 1];
          hit = true;
        }
      }
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      // only groups that start inside the partition are recorded (the words past them in its last page are cleared below)
      if (lane == 0 && (t0 + woff + k * 32) < p_rows) {
        vword[k] = bal;
        matched += __popc(bal);
      }
      if (hit) {
#pragma unroll
        for (int c = 0; c < NB; c++) {
          uint64_t x;
          if (bw[c] == 0) x = key[k];
          else if (bw[c] == 1) x = w1;
          else x = t.words[((uint64_t)loc[k] << SHIFT) + bw[c]];  // words 2..3 of a 32-byte entry: same sector as the key
          tqd::st_stream_u64(ob[c] + oslot + k * 32, x);
        }
      }
    }
    if (p.dbg_late_release) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_empty[s]);
    }
  }
  // the CTA with the partition's last tile clears the ballot words past it in its last page (no row ever lands there), so the
  // validity bitmap is exact over the whole span
  if (t_hi == p_tiles && p_rows > 0) {
    const uint32_t kl = (uint32_t)((p_rows - 1) / PG), fill = (uint32_t)p_rows - kl * PG;
    uint32_t *pw = p.valid + (((uint32_t)pages[kl] * PG) >> 5);
    for (uint32_t w = (fill + 31) / 32 + warp * 32 + lane; w < PG / 32; w += CW * 32) pw[w] = 0;
  }
  if (lane == 0 && matched) atomicAdd(p.cursor, (unsigned long long)matched);
}

typedef void (*ProbePosKernel)(const ProbePosParams, const JoinTable);
struct ProbePosVariant {
  ProbePosKernel k;
  int tile, threads;
};
template <int NB>
static ProbePosVariant probe_pos_variant() {
  // 2 rows per lane x 12 consumer warps x 3 CTAs per SM: more warps in flight hide the L2 latency of the table gathers better
  // than more loads per warp (4 rows per lane spills at 3 CTAs per SM).
  static_assert(PP_TILE_ROWS == 12 * 32 * 2, "page sizes are whole probe tiles");
  return {k_probe_pos<NB, 2, 12, 3>, PP_TILE_ROWS, 13 * 32};
}
static ProbePosVariant probe_pos_kernel(int nb) {
  switch (nb) {
    case 1: return probe_pos_variant<1>();
    case 2: return probe_pos_variant<2>();
    case 3: return probe_pos_variant<3>();
    case 4: return probe_pos_variant<4>();
  }
  return {nullptr, 0, 0};
}

// ---- hole filling: the k-th empty slot below M takes the k-th real row at or above M (M = rows of the result)
__global__ void __launch_bounds__(256) k_hole_popc(const uint32_t *valid, int64_t n_words, uint32_t *cnt) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) cnt[w] = __popc(valid[w]);
}
__device__ __forceinline__ uint32_t valid_rank(const uint32_t *valid, const uint32_t *vpre, uint64_t pos, int64_t n_words) {
  const uint64_t w = pos >> 5;
  if ((int64_t)w >= n_words) return vpre[n_words];  // vpre has n_words + 1 entries (the last = total)
  return vpre[w] + __popc(valid[w] & ((1u << (pos & 31)) - 1u));
}
__global__ void __launch_bounds__(256) k_hole_lists(const uint32_t *valid, const uint32_t *vpre, int64_t n_words, uint64_t M, uint32_t *hole_pos, uint32_t *tail_src) {
  const uint32_t below = valid_rank(valid, vpre, M, n_words);  // real rows in [0, M)
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
    const uint32_t bits = valid[w];
    const uint64_t p0 = (uint64_t)w << 5;
    if (p0 + 32 <= M && bits == 0xFFFFFFFFu) continue;
    if (p0 >= M && bits == 0) continue;
    const uint32_t pre = vpre[w];
    for (int b = 0; b < 32; b++) {
      const uint64_t pos = p0 + b;
      const bool v = (bits >> b) & 1u;
      const uint32_t vr = pre + __popc(bits & ((1u << b) - 1u));
      if (pos < M && !v) hole_pos[pos - vr] = (uint32_t)pos;             // holes before pos = pos - (real rows before pos)
      else if (pos >= M && v) tail_src[vr - below] = (uint32_t)pos;
    }
  }
}
struct HoleMoveParams {
  int n_cols;
  uint64_t *col[8];
  const uint32_t *hole_pos, *tail_src;
  const uint32_t *valid, *vpre;
  int64_t n_words;
  uint64_t M;
};
__global__ void __launch_bounds__(256) k_hole_move(const HoleMoveParams h) {
  const uint64_t H = h.M - valid_rank(h.valid, h.vpre, h.M, h.n_words);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < H; k += stride) {
    const uint32_t d = h.hole_pos[k], s = h.tail_src[k];
    for (int c = 0; c < h.n_cols; c++) h.col[c][d] = h.col[c][s];
  }
}

// ------------------------------------------------------------------------------------------------ cluster build
// Only where a sub-table does not fit one CTA (k_build_cta below otherwise).  One cluster of BC_CLUSTER CTAs builds the
// sub-tables of one scatter bin in distributed shared memory.  A partition's table is split into 2^sbits sub-tables (the next
// sbits hash bits below the partition bits), each small enough to live in the cluster's shared memory, CTA r holding entries
// [r * slice, (r + 1) * slice).  The build side is scattered into one slab per sub-table (2^lbits sub-tables per slab only
// past SA_MAX_PBITS scatter bits).  Per sub-table: initialise the slices, insert the slab's rows of that sub-table with
// atomicCAS on the owning CTA's shared memory, then stream every slice to its place in the table with coalesced 16-byte
// stores.  Each table line is written to DRAM once, with no initialisation pass and no L2 atomics.  With one sub-table per
// slab the write-back follows the last cluster barrier, so no CTA waits for it.
static constexpr int BC_CLUSTER = 8;
static constexpr int BC_THREADS = 512;
static constexpr int BC_MAX_SLICE_BYTES = 112 << 10;  // one CTA's share of a sub-table: two CTAs fit an SM's 228 KB
// shared::cluster addresses: the same shared-memory offset in the CTA of the given rank, and accesses through them
__device__ __forceinline__ uint32_t dsmem_map(uint32_t local, uint32_t rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local), "r"(rank));
  return a;
}
__device__ __forceinline__ uint64_t dsmem_cas_u64(uint32_t a, uint64_t cmp, uint64_t val) {
  uint64_t prev;
  asm volatile("atom.shared::cluster.cas.b64 %0, [%1], %2, %3;" : "=l"(prev) : "r"(a), "l"(cmp), "l"(val) : "memory");
  return prev;
}
__device__ __forceinline__ void dsmem_st_u64(uint32_t a, uint64_t v) { asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ void dsmem_add_u32(uint32_t a, uint32_t v) { asm volatile("red.shared::cluster.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// The parameters of both streaming builds (k_build_cluster, k_build_cta).
struct BuildParams {
  const uint64_t *slab;              // AoS build rows (NB words each), one slab per scatter bin
  const uint32_t *lo, *hi, *lim;     // a slab that overflowed (hi > lim) holds lim - lo rows; the caller discards the build anyway
  uint64_t *words;                   // the table: sub-table t (top tbits hash bits) starts at entry t * cap
  uint32_t cap;                      // entries per sub-table (a multiple of 16: every slice holds whole entry pairs)
  uint32_t max_rows;                 // rows a sub-table may hold at the configured load factor
  int tbits, lbits, key_col;         // 2^tbits sub-tables in all, 2^lbits of them per scatter bin
  int word_of_col[4];
  unsigned *flags;                   // |= 1: duplicate key, |= 2: the empty-marker key appeared, |= 4: a sub-table is over the load limit  -> the caller rebuilds on the general path
  unsigned long long *rows;          // += rows inserted into every sub-table
};
template <int NB>
__global__ void __launch_bounds__(BC_THREADS, 2) k_build_cluster(const BuildParams b) {
  namespace cg = cooperative_groups;
  constexpr int SHIFT = NB > 2 ? 2 : 1;  // words per entry = 1 << SHIFT (the probers read the table the same way)
  constexpr int BC_UNROLL = 4;  // slab rows loaded ahead of their inserts, per thread
  extern __shared__ __align__(16) uint64_t s_tbl[];  // this CTA's slice of the current sub-table
  __shared__ uint32_t s_rows;                         // rank 0: rows of the current sub-table, counted by the whole cluster
  cg::cluster_group cluster = cg::this_cluster();
  const int tid = threadIdx.x;
  const uint32_t rank = cluster.block_rank();
  const uint32_t bin = blockIdx.x / BC_CLUSTER;
  const uint32_t cap = b.cap, slice = cap / BC_CLUSTER;
  const uint32_t n_vec = (slice << SHIFT) / 2;        // 16-byte pieces of a slice
  const int64_t p_lo = b.lo[bin];
  int64_t p_hi = b.hi[bin];
  if (p_hi > (int64_t)b.lim[bin]) p_hi = b.lim[bin];
  const uint32_t s_base = smem_u32(s_tbl), rows0 = dsmem_map(smem_u32(&s_rows), 0);
  ulonglong2 *s_vec = reinterpret_cast<ulonglong2 *>(s_tbl);
  const uint32_t n_sub = 1u << b.lbits;
  for (uint32_t sub = 0; sub < n_sub; sub++) {
    for (uint32_t i = tid; i < n_vec; i += BC_THREADS)
      s_vec[i] = (SHIFT == 1 || (i & 1) == 0) ? make_ulonglong2(EMPTY_KEY, 0) : make_ulonglong2(0, 0);
    if (rank == 0 && tid == 0) s_rows = 0;
    cluster.sync();  // every slice is empty before any CTA inserts into it
    uint32_t mine = 0;
    for (int64_t r0 = p_lo + (int64_t)rank * BC_THREADS * BC_UNROLL + tid; r0 < p_hi; r0 += (int64_t)BC_CLUSTER * BC_THREADS * BC_UNROLL) {
      uint64_t w[BC_UNROLL][NB];
#pragma unroll
      for (int u = 0; u < BC_UNROLL; u++) {
        const int64_t r = r0 + u * BC_THREADS;
        if (r >= p_hi) continue;
        if constexpr (NB == 2) {
          const ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 2);
          w[u][0] = x.x;
          w[u][1] = x.y;
        } else if constexpr (NB == 4) {
          const ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 4), y = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 4 + 2);
          w[u][0] = x.x; w[u][1] = x.y; w[u][2] = y.x; w[u][3] = y.y;
        } else {
#pragma unroll
          for (int c = 0; c < NB; c++) w[u][c] = b.slab[r * NB + c];
        }
      }
      // (Issuing the home-slot CAS of all BC_UNROLL rows before awaiting any measured slower on the H100: 1.33 vs 0.74 ms.)
#pragma unroll
      for (int u = 0; u < BC_UNROLL; u++) {
        if (r0 + u * BC_THREADS >= p_hi) continue;
        uint64_t key = 0;  // (selected by masks: an index by key_col would put w in local memory)
#pragma unroll
        for (int c = 0; c < NB; c++) key |= w[u][c] & (c == b.key_col ? ~0ull : 0ull);
        if (key == EMPTY_KEY) { if (sub == 0) atomicOr(b.flags, 2u); continue; }
        const uint64_t h = tqd::hash_key(key);
        // (n_sub == 1, every slab a single sub-table: the mask is 0 and every row passes)
        if (((uint32_t)part_of_hash(h, b.tbits) & (n_sub - 1)) != sub) continue;
        mine++;
        uint32_t loc = home_slot(h, cap, SHIFT);
        for (uint32_t probes = 0;; probes++) {
          if (probes >= cap) { atomicOr(b.flags, 4u); break; }  // the sub-table is full (far over the load limit)
          const uint32_t owner = loc / slice;
          const uint32_t ent = dsmem_map(s_base + ((loc - owner * slice) << (SHIFT + 3)), owner);
          const uint64_t prev = dsmem_cas_u64(ent, EMPTY_KEY, key);
          if (prev == EMPTY_KEY) {
#pragma unroll
            for (int c = 0; c < NB; c++) if (c != b.key_col) dsmem_st_u64(ent + 8 * b.word_of_col[c], w[u][c]);
            break;
          }
          if (prev == key) { atomicOr(b.flags, 1u); break; }
          loc = next_slot(loc, 1, cap);
        }
      }
    }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((tid & 31) == 0 && mine) dsmem_add_u32(rows0, mine);
    // Every insert into every slice is complete and visible.  This is also the last access of any peer's shared memory in
    // this iteration, so after the last sub-table it is the barrier that lets every CTA exit.
    cluster.sync();
    if (rank == 0 && tid == 0) {
      if (s_rows > b.max_rows) atomicOr(b.flags, 4u);
      if (s_rows) atomicAdd(b.rows, (unsigned long long)s_rows);
    }
    uint64_t *dst = b.words + (((((uint64_t)bin << b.lbits) | (uint64_t)sub) * cap + (uint64_t)rank * slice) << SHIFT);
    for (uint32_t i = tid; i < n_vec; i += BC_THREADS) tqd::st_stream_u64x2(dst + 2 * (uint64_t)i, s_vec[i]);
    if (sub + 1 < n_sub) __syncthreads();  // the slice is re-initialised for the next sub-table
  }
}
typedef void (*BuildKernel)(const BuildParams);
static BuildKernel build_cluster_kernel(int nb) {
  switch (nb) {
    case 1: return k_build_cluster<1>;
    case 2: return k_build_cluster<2>;
    case 3: return k_build_cluster<3>;
    case 4: return k_build_cluster<4>;
  }
  return nullptr;
}

// ------------------------------------------------------------------------------------------------ CTA build
// Where a sub-table fits one CTA's shared memory, one CTA builds it alone: inserts are local 64-bit atomicCAS with no remote
// round trips and no cluster barriers.  CTA blockIdx.x builds sub-table blockIdx.x = (slab << lbits) | sub, so the 2^lbits
// CTAs of one slab are adjacent: each reads the whole slab and keeps the rows of its own sub-table, the first read of a slab
// comes from DRAM and the others hit L2.  Same parameters, table layout, flags and write-back as k_build_cluster.
// 1024 threads and up to 200 KB of table per CTA, one CTA per SM: at C3 (1e7 build rows of 16-byte entries) that is 2^11
// sub-tables of 176 KB, 4 per slab.  512 threads with 2^12 sub-tables of 93 KB (2 CTAs per SM, 8 per slab) read every slab
// twice as often from L2 and measured 0.377 ms against 0.293 ms (H100 80GB HBM3, 700 W).
static constexpr int BT_THREADS = 1024;
static constexpr int BT_MAX_BYTES = 200 << 10;
template <int NB>
__global__ void __launch_bounds__(BT_THREADS, 1) k_build_cta(const BuildParams b) {
  constexpr int SHIFT = NB > 2 ? 2 : 1;  // words per entry = 1 << SHIFT (the probers read the table the same way)
  constexpr int BT_UNROLL = 4;           // slab rows loaded ahead of their inserts, per thread
  extern __shared__ __align__(16) uint64_t s_tbl[];
  __shared__ uint32_t s_rows;
  const int tid = threadIdx.x;
  const uint32_t n_sub = 1u << b.lbits;
  const uint32_t bin = blockIdx.x >> b.lbits, sub = blockIdx.x & (n_sub - 1);
  const uint32_t cap = b.cap;
  const uint32_t n_vec = (cap << SHIFT) / 2;  // 16-byte pieces of the sub-table
  ulonglong2 *s_vec = reinterpret_cast<ulonglong2 *>(s_tbl);
  for (uint32_t i = tid; i < n_vec; i += BT_THREADS)
    s_vec[i] = (SHIFT == 1 || (i & 1) == 0) ? make_ulonglong2(EMPTY_KEY, 0) : make_ulonglong2(0, 0);
  if (tid == 0) s_rows = 0;
  __syncthreads();
  const int64_t p_lo = b.lo[bin];
  int64_t p_hi = b.hi[bin];
  if (p_hi > (int64_t)b.lim[bin]) p_hi = b.lim[bin];
  uint32_t mine = 0;
  for (int64_t r0 = p_lo + tid; r0 < p_hi; r0 += (int64_t)BT_THREADS * BT_UNROLL) {
    uint64_t w[BT_UNROLL][NB];
#pragma unroll
    for (int u = 0; u < BT_UNROLL; u++) {
      const int64_t r = r0 + u * BT_THREADS;
      if (r >= p_hi) continue;
      if constexpr (NB == 2) {
        const ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 2);
        w[u][0] = x.x;
        w[u][1] = x.y;
      } else if constexpr (NB == 4) {
        const ulonglong2 x = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 4);
        const ulonglong2 y = *reinterpret_cast<const ulonglong2 *>(b.slab + r * 4 + 2);
        w[u][0] = x.x; w[u][1] = x.y; w[u][2] = y.x; w[u][3] = y.y;
      } else {
#pragma unroll
        for (int c = 0; c < NB; c++) w[u][c] = b.slab[r * NB + c];
      }
    }
#pragma unroll
    for (int u = 0; u < BT_UNROLL; u++) {
      if (r0 + u * BT_THREADS >= p_hi) continue;
      uint64_t key = 0;  // (selected by masks: an index by key_col would put w in local memory)
#pragma unroll
      for (int c = 0; c < NB; c++) key |= w[u][c] & (c == b.key_col ? ~0ull : 0ull);
      if (key == EMPTY_KEY) { if (sub == 0) atomicOr(b.flags, 2u); continue; }
      const uint64_t h = tqd::hash_key(key);
      if (((uint32_t)part_of_hash(h, b.tbits) & (n_sub - 1)) != sub) continue;
      mine++;
      uint32_t loc = home_slot(h, cap, SHIFT);
      for (uint32_t probes = 0;; probes++) {
        if (probes >= cap) { atomicOr(b.flags, 4u); break; }  // the sub-table is full (far over the load limit)
        uint64_t *ent = s_tbl + ((size_t)loc << SHIFT);
        const uint64_t prev =
            atomicCAS(reinterpret_cast<unsigned long long *>(ent), (unsigned long long)EMPTY_KEY, (unsigned long long)key);
        if (prev == EMPTY_KEY) {
#pragma unroll
          for (int c = 0; c < NB; c++) if (c != b.key_col) ent[b.word_of_col[c]] = w[u][c];
          break;
        }
        if (prev == key) { atomicOr(b.flags, 1u); break; }
        loc = next_slot(loc, 1, cap);
      }
    }
  }
  mine = __reduce_add_sync(0xffffffffu, mine);
  if ((tid & 31) == 0 && mine) atomicAdd(&s_rows, mine);
  __syncthreads();  // every insert is complete and visible
  if (tid == 0) {
    if (s_rows > b.max_rows) atomicOr(b.flags, 4u);
    if (s_rows) atomicAdd(b.rows, (unsigned long long)s_rows);
  }
  uint64_t *dst = b.words + (((uint64_t)blockIdx.x * cap) << SHIFT);
  for (uint32_t i = tid; i < n_vec; i += BT_THREADS) tqd::st_stream_u64x2(dst + 2 * (uint64_t)i, s_vec[i]);
}
static BuildKernel build_cta_kernel(int nb) {
  switch (nb) {
    case 1: return k_build_cta<1>;
    case 2: return k_build_cta<2>;
    case 3: return k_build_cta<3>;
    case 4: return k_build_cta<4>;
  }
  return nullptr;
}

}  // namespace tq
