/*
 * oracle.h — CPU restatement of the TinySQL hot path (TEST INFRASTRUCTURE ONLY).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library; the product (libtinysql_b200.so) never links or calls it.
 * Each function cites the reference file:line it restates (paths relative to
 * the reference repository).  Parity status: pinned against the reference's own known-answer
 * tests re-expressed in tests/test_oracle_golden.py, test_oracle_sort_merge.py (+ sort_cases.py),
 * test_oracle_final_agg.py and test_oracle_strnum.py (+ strnum_cases.py) (the Go reference cannot be
 * built here: no Go toolchain, and the join/agg hot functions are course stubs).
 */
#ifndef TQ_ORACLE_H
#define TQ_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

/* identical layout to tq_column (include/tinysql_b200.h) */
typedef struct orc_column {
  int64_t length;
  uint8_t *null_bitmap;
  int64_t *offsets;
  uint8_t *data;
} orc_column;

enum { ORC_OK = 0, ORC_ERR_INVALID = 1, ORC_ERR_UNSUPPORTED = 2, ORC_ERR_OVERFLOW_BIGINT = 3,
       ORC_ERR_OVERFLOW_BIGINT_UNSIGNED = 4, ORC_ERR_OVERFLOW_DOUBLE = 5, ORC_ERR_DIV_ZERO = 6 };
enum { ORC_TYPE_INT64 = 1, ORC_TYPE_UINT64 = 2, ORC_TYPE_FLOAT64 = 3,
       ORC_TYPE_FLOAT32 = 4 /* 4-byte slots */, ORC_TYPE_BYTES = 5 /* offsets + data; join payload columns only */ };

/* FNV-1 64 over flag||raw8 per key column — executor/hash_table.go:55-72 (fnv.New64),
 * util/codec/codec.go:249-276.  Exposed for the codec known-answer tests. */
uint64_t orc_hash_row(int n_keys, const int *types, const orc_column *cols, const int *key_idx,
                      int64_t row, int *has_null);
/* util/codec/codec.go:363-382 EqualChunkRow */
int orc_equal_row(int n_keys, const int *types1, const orc_column *cols1, const int *idx1, int64_t row1,
                  const int *types2, const orc_column *cols2, const int *idx2, int64_t row2);

/* rowHashMap Put/Get — executor/hash_table.go:221-272; for the TestRowHashMap golden. */
typedef struct orc_rowmap orc_rowmap;
orc_rowmap *orc_rowmap_new(void);
void orc_rowmap_put(orc_rowmap *m, uint64_t hash_key, uint32_t chk_idx, uint32_t row_idx);
/* returns count; fills up to cap (chk_idx,row_idx) pairs in INSERTION order */
int64_t orc_rowmap_get(orc_rowmap *m, uint64_t hash_key, uint32_t *pairs, int64_t cap);
int64_t orc_rowmap_len(orc_rowmap *m);
void orc_rowmap_free(orc_rowmap *m);

/* HashJoinExec — executor/join.go:125-362 + Appendix B of SURVEY.md for the stubs.
 * The inner side is given as one concatenated column set (chunking does not affect
 * results: RowPtr order == row order).  Output columns are malloc'ed by the oracle in
 * (probe row asc, build insertion asc) order; free with orc_free_columns. */
int orc_hash_join(int join_type, int outer_is_right,
                  int n_build_cols, const int *build_types, const orc_column *build_cols,
                  int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                  int n_keys, const int *build_key_idx, const int *probe_key_idx,
                  const uint8_t *selected, orc_column *out_cols, int64_t *n_out);
/* The same with OtherConditions (HashJoinExec.joiners' filter, joiner.go:155-167): every condition compares output column
 * lhs_col (index into lhs ++ rhs) with output column rhs_col, or with a constant when rhs_col < 0. */
typedef struct orc_join_cond { int32_t op, lhs_col, rhs_col, const_type; uint64_t const_bits; } orc_join_cond;
int orc_hash_join_cond(int join_type, int outer_is_right,
                       int n_build_cols, const int *build_types, const orc_column *build_cols,
                       int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                       int n_keys, const int *build_key_idx, const int *probe_key_idx,
                       const uint8_t *selected, int n_conds, const orc_join_cond *conds, orc_column *out_cols, int64_t *n_out);
void orc_free_columns(int n, orc_column *cols);

/* HashAggExec — executor/aggregate.go:332-457,559-588; aggfuncs/ sources.  n_partial_workers
 * >= 1 reproduces the partial -> shuffle -> final split: input is dealt in 1024-row chunks
 * round-robin to the partial workers, partials are merged in worker order with
 * MergePartialResult.  Output rows are in first-seen group order of the merge. */
typedef struct orc_agg_func { int32_t func; int32_t arg_col; } orc_agg_func;
int orc_hash_agg(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                 int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_func *funcs,
                 int n_partial_workers, orc_column *out_cols, int64_t *n_out);

/* The coprocessor's partial aggregation (store/mockstore/mocktikv/aggregate.go) and the FinalMode HashAggExec that consumes
 * its rows (aggfuncs/builder.go Partial2Mode / FinalMode).  orc_cop_partial_agg writes, per group in first-seen order, the
 * GetPartialResult columns of every function (AVG: count then sum) followed by the GROUP BY columns; out_types receives the
 * column types (n_group_by + n_funcs + number of AVGs entries). */
typedef struct orc_agg_final_func { int32_t func; int32_t arg_col; int32_t arg_col2; } orc_agg_final_func;
int orc_cop_partial_agg(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                        int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_func *funcs,
                        orc_column *out_cols, int *out_types, int64_t *n_out);
int orc_hash_agg_final(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                       int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_final_func *funcs,
                       orc_column *out_cols, int64_t *n_out);

/* SortExec / TopNExec (executor/sort.go) and MergeJoinExec (executor/merge_join.go).  orc_sort keeps rows that compare equal
 * in child order (one of the outcomes sort.Slice may produce); limit_count < 0 = SortExec, else the rows
 * [limit_offset, limit_offset + limit_count) of the order.  orc_merge_join expects both inputs sorted ascending by their keys. */
int orc_sort(int n_cols, const int *types, const orc_column *cols, int64_t n_rows, int n_by, const int *by_cols, const int *by_desc,
             int64_t limit_offset, int64_t limit_count, orc_column *out_cols, int64_t *n_out);
int orc_merge_join(int join_type, int outer_is_right,
                   int n_inner_cols, const int *inner_types, const orc_column *inner_cols,
                   int n_outer_cols, const int *outer_types, const orc_column *outer_cols,
                   int n_keys, const int *inner_keys, const int *outer_keys, const uint8_t *selected,
                   int n_conds, const orc_join_cond *conds,
                   const uint64_t *default_bits, const uint8_t *default_nn, orc_column *out_cols, int64_t *n_out);

/* types.StrToInt in a SELECT statement (types/convert.go:224-232) and toBool for ETString (expression/expression.go:308-322):
 * *overflow_err = ParseInt failed (ErrOverflow "BIGINT"); orc_vec_filter_string reports the error of the LAST non-NULL row. */
int orc_str_to_int(const uint8_t *bytes, int64_t len, int64_t *ival, int *overflow_err);
int orc_vec_filter_string(int64_t n, const orc_column *a, uint8_t *selected, int *err_overflow);

/* vectorized builtins — restated statement by statement from expression/builtin_*_vec*.go */
int orc_vec_compare_int(int op, int64_t n, const orc_column *a, int a_unsigned, const orc_column *b,
                        int b_unsigned, orc_column *out);
int orc_vec_compare_real(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_arith_int(int op, int64_t n, const orc_column *a, int a_unsigned, const orc_column *b,
                      int b_unsigned, orc_column *out);
int orc_vec_arith_real(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out,
                       int64_t *div_by_zero);
int orc_vec_logic(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_unary(int op, int64_t n, const orc_column *a, int a_unsigned, orc_column *out);
int orc_vec_if(int64_t n, const orc_column *c, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_ifnull(int64_t n, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_in_int(int64_t n, const orc_column *a, int a_unsigned, int n_list, const orc_column *list,
                   const int *list_unsigned, orc_column *out);
int orc_vec_filter_int(int64_t n, const orc_column *a, uint8_t *selected);

/* ---- multi-threaded CPU restatement of the reference *design* (cpu_ref.c): the baseline
 * timed beside the GPU path.  Serial build + `workers` probe goroutine-equivalents over
 * 1024-row chunks with private result chunks (join.go:194-362); returns joined rows and
 * writes elapsed seconds (build+probe) — results are checksummed, not returned. */
int64_t orc_mt_join_bench(int64_t n_build, const int64_t *bk, const int64_t *bv,
                          int64_t n_probe, const int64_t *pk, const int64_t *pv,
                          int workers, double *build_seconds, double *probe_seconds,
                          uint64_t *checksum);
/* P partial workers + F final workers, SUM(f64)+COUNT(*) GROUP BY int64 (aggregate.go:96-133) */
int64_t orc_mt_agg_bench(int64_t n, const int64_t *k, const double *x, int partial_workers,
                         int final_workers, double *seconds, double *sum_of_sums, int64_t *sum_of_counts);
/* 1024-row-chunk LT + Plus loops (builtin_compare_vec.go:186-223, builtin_arithmetic_vec.go:389-495) */
int64_t orc_mt_lt_plus_bench(int64_t n, const int64_t *a, const int64_t *b, int64_t *lt_out,
                             int64_t *plus_out, int workers, double *seconds);

/* string builtins over var-len columns (offsets + data) */
int orc_vec_compare_string(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_string_unary(int op, int64_t n, const orc_column *a, orc_column *out);

int orc_hash_join_full(int join_type, int outer_is_right,
                       int n_build_cols, const int *build_types, const orc_column *build_cols,
                       int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                       int n_keys, const int *build_key_idx, const int *probe_key_idx,
                       const uint8_t *selected, int n_conds, const orc_join_cond *conds,
                       const uint64_t *default_bits, const uint8_t *default_nn, orc_column *out_cols, int64_t *n_out);
/* the rest of the vectorized signatures (builtin_other_vec_generated.go:97-204, builtin_control_vec_generated.go:81-112,209-262) */
int orc_vec_in_real(int64_t n, const orc_column *a, int n_list, const orc_column *list, orc_column *out);
int orc_vec_in_string(int64_t n, const orc_column *a, int n_list, const orc_column *list, orc_column *out);
int orc_vec_pick_string(int mode, int64_t n, const orc_column *cond, const orc_column *a, const orc_column *b, orc_column *out);
int orc_vec_filter_real(int64_t n, const orc_column *a, uint8_t *selected);
#ifdef __cplusplus
}
#endif
#endif
