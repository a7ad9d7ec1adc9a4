// nlj.cuh — the key-less hash join (tq_join_desc.n_keys == 0): cross joins and joins whose ON holds no equality.
//
// Reference: with no key columns hashRowContainer.PutChunk puts every build row into ONE chain in insertion order and every
// selected probe row finds that chain (executor/hash_table.go:146-169,259-272, join.go:325-362), so the joined rows of a probe
// row are all build rows in insertion order, filtered by the OtherConditions (joiner.go:155-167).  The pair space
// |probe| x |build| is never built: a probe batch is walked in sub-ranges of whole probe rows.  Per sub-range
//   k_nlj_eval   (conditions only) survivor bits, one 32-bit word per probe row and 32 build rows;
//   k_nlj_count  rows each probe row emits (popcount; B without conditions; 1 for a miss row of an outer join) + the word
//                prefix inside the row;
//   scan_u64     exclusive 64-bit scan of the counts: the output position of every probe row;
//   k_nlj_materialize  any slice [q0, q0 + len) of the sub-range's output, written at its final positions.
#pragma once
#include "expr_prog.cuh"

namespace tq {

static constexpr int NLJ_MAXC = 16;   // columns per join side (= join.cu's MAXC)

struct NljEvalParams {
  JoinProg prog;               // prog.in_col is not read: in[k] is the column input register k reads
  DCol in[JP_MAX_IN];
  int in_build[JP_MAX_IN];     // 1: input k is a build column (indexed by build row), 0: a probe column (indexed by probe row)
  const uint8_t *selected;     // probe rows' outerSideFilter result or nullptr
  int64_t r0, rows;            // the sub-range: probe rows [r0, r0 + rows)
  uint32_t n_build, words;     // B, ceil(B / 32)
  uint32_t *mask;              // [rows * words] survivor bits
  unsigned *err;               // ops that raised on a pair of the evaluation set (bit i: op i)
  unsigned long long *warn;    // division-by-zero warnings of those pairs
};

struct NljCountParams {
  const uint8_t *selected;
  int64_t r0, rows;
  uint32_t n_build, words;
  const uint32_t *mask;        // nullptr: no conditions (a selected probe row emits all B build rows)
  uint32_t *wpre;              // [rows * words] set bits in the row's earlier words
  int outer;
  uint64_t *cnt;               // [rows] output rows per probe row
  uint8_t *miss;               // [rows] 1: the row is emitted once as a miss row (NULL / defaultInner inner side)
};

struct NljOutParams {
  int n_probe_cols, n_build_cols;
  DCol probe[NLJ_MAXC], build[NLJ_MAXC];
  DColMut out_probe[NLJ_MAXC], out_build[NLJ_MAXC];
  uint64_t def_val[NLJ_MAXC];  // defaultInner of a miss row (+ its NOT-NULL bits)
  uint32_t def_mask;
  const uint64_t *off;         // [rows + 1] output position of each probe row of the sub-range; off[rows] = its total
  const uint8_t *miss;
  const uint32_t *mask, *wpre; // nullptr: no conditions
  uint32_t words;
  int64_t r0, rows;
  uint64_t q0;                 // first output position of the slice (within the sub-range)
  int64_t len;                 // rows of the slice (= rows of the result batch)
};

int32_t nlj_eval(const NljEvalParams &p, cudaStream_t s);
int32_t nlj_count(const NljCountParams &p, cudaStream_t s);
// out[0, n] = exclusive scan of in[0, n), out[n] = the total
int32_t nlj_scan_u64(const uint64_t *in, uint64_t *out, int64_t n, DevBuf &scratch, cudaStream_t s);
int32_t nlj_materialize(const NljOutParams &p, cudaStream_t s);

}  // namespace tq
