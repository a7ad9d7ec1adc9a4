// othercond.cuh — HashJoinExec OtherConditions on the device.
//
// Reference: joiner.tryToMatchInners builds the joined rows of one outer row, baseJoiner.filter keeps those for which every
// condition is true (expression.VectorizedFilter), and an outer row none of whose joined rows survive is emitted once with a
// NULL / defaultInner inner side by onMissMatch (executor/joiner.go:155-167,225-248,274-277,337-340).  Here the conditions
// are applied to a finished result batch: run the condition program (expr_prog.cuh) per joined row, count survivors per
// probe row (outer joins carry a hidden probe-row-id column), turn one failed row of every survivor-less probe row into its
// miss row, compact.
#pragma once
#include "expr_prog.cuh"

namespace tq {

static constexpr int OC_MAX_COLS = 34;

struct OcPlan {
  JoinProg prog;           // input registers name result-batch columns
  int cmp_list = 0;        // prog is a lowered tq_join_cond list: evaluated by oc_cmp_list_passes
  int outer = 0;           // left / right outer join
  int build_key_col = -1;  // result column of the build-side key: NOT NULL <=> the row is a key match
  int rowid_col = -1;      // outer joins: result column holding the probe row id within the batch
  int build_lo = 0, build_hi = 0;  // result columns [build_lo, build_hi) belong to the build (inner) side
  uint64_t def_val[16] = {};       // defaultInner: what the inner side of a miss row holds (joiner.go:139-143)
  uint32_t def_mask = 0;
};

struct OcCols {
  int n = 0;
  const uint64_t *data[OC_MAX_COLS];
  const uint32_t *bm[OC_MAX_COLS];
  uint64_t *out_data[OC_MAX_COLS];
  uint32_t *out_bm[OC_MAX_COLS];
};

// Filters n joined rows into the out_* columns (caller-allocated for n rows, bitmaps zeroed here); *n_out = rows kept,
// *err = the ERR_* bits and *div_by_zero = the division-by-zero warnings the key-matched rows raised.
int32_t oc_filter(const OcPlan &plan, const OcCols &cols, int64_t n, int64_t n_probe_rows, DevBuf &scratch, DevBuf &scan_scratch, int64_t *n_out,
                  unsigned *err, int64_t *div_by_zero, cudaStream_t s);

}  // namespace tq
