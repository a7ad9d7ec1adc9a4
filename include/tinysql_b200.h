/*
 * tinysql_b200.h — C-ABI of the H100-native vectorized execution path for TinySQL.
 *
 * This is the drop-in boundary: exactly the calls a cgo shim inside TinySQL's
 * `executor`, `expression` and `util/chunk` packages would bind (see INTEGRATION.md
 * for the Go side).  Plain pointers and sizes only; no C++/torch types.
 *
 * Every entry point returns an int32 status (TQ_OK == 0).  On failure a
 * thread-local message is available through tq_last_error().  The library is
 * re-entrant across handles; one handle must be driven by one thread at a time
 * (the reference calls Next from a single goroutine per operator instance,
 * executor/executor.go:155-162).
 *
 * Reference citations are relative to the root of pingcap-incubator/tinysql.
 */
#ifndef TINYSQL_B200_H
#define TINYSQL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ status */
enum {
  TQ_OK = 0,
  TQ_ERR_INVALID_ARG = 1,
  TQ_ERR_UNSUPPORTED_TYPE = 2,      /* "unsupport column type for encode" util/codec/codec.go:235,335 */
  TQ_ERR_OVERFLOW_BIGINT = 3,       /* types.ErrOverflow "BIGINT"           expression/builtin_arithmetic_vec.go:489 */
  TQ_ERR_OVERFLOW_BIGINT_UNSIGNED = 4, /* types.ErrOverflow "BIGINT UNSIGNED" builtin_arithmetic_vec.go:441 */
  TQ_ERR_OVERFLOW_DOUBLE = 5,       /* types.ErrOverflow "DOUBLE"           builtin_arithmetic_vec.go:52 */
  TQ_ERR_DIVISION_BY_ZERO = 6,      /* handleDivisionByZeroError in strict mode, builtin_arithmetic_vec.go:369-375 */
  TQ_ERR_CUDA = 7,                  /* device fault / launch failure (generic internal error) */
  TQ_ERR_NO_DEVICE = 8,             /* no usable sm_90 device: there is NO CPU fallback */
  TQ_ERR_OOM = 9,
  TQ_ERR_STATE = 10                 /* call out of protocol order (e.g. probe before finalize_build) */
};

/* ------------------------------------------------------------------ types  */
/* util/chunk/codec.go:171-181: every SQL integer / DOUBLE is an 8-byte slot;
 * signedness comes from mysql.UnsignedFlag on the FieldType. */
enum {
  TQ_TYPE_INT64 = 1,   /* TINY..LONGLONG, YEAR (signed)            */
  TQ_TYPE_UINT64 = 2,  /* same, with mysql.UnsignedFlag            */
  TQ_TYPE_FLOAT64 = 3, /* DOUBLE                                   */
  TQ_TYPE_FLOAT32 = 4, /* FLOAT (4-byte slots).  HashJoin key or payload column, HashAgg GROUP BY item or argument; as a key /
                        *   group item / argument it counts as float64(f) (util/codec/codec.go:226-229).  Host memory only. */
  TQ_TYPE_BYTES = 5,   /* var-len (VARCHAR, BLOB, ...): offsets = length+1 int64 (Go's Column.offsets), data = the cells' bytes.
                        *   HashJoin key or payload, HashAgg GROUP BY item or COUNT / MAX / MIN / FIRSTROW argument; compared
                        *   byte-wise (compactBytesFlag, codec.go:230-233).  Host or device memory (TQ_MEM_DEVICE rules at
                        *   tq_column below).                                                                               */
  /* OR-ed into a tq_agg_desc.input_types entry: the column's FieldType carries mysql.NotNullFlag.  Lets HashAgg
   * drop the per-group "saw a non-NULL input" word of SUM / MAX / MIN (16-byte instead of 32-byte group records
   * for SUM + COUNT); any null bitmap passed for such a column is ignored. */
  TQ_TYPE_NOT_NULL = 0x100
};

/* Where the buffers of a tq_column live. */
enum {
  TQ_MEM_HOST = 0,   /* ordinary or pinned host memory (the cgo path)                 */
  TQ_MEM_DEVICE = 1  /* device memory on the library's device (bench / multi-GPU path) */
};

/* One chunk.Column exactly as Go holds it (util/chunk/column.go:28-34):
 *   data        = length * 8 bytes, little-endian values (NULL slots are don't-care)
 *   null_bitmap = ceil(length/8) bytes; bit (i&7) of byte (i>>3); 1 = NOT NULL.
 *                 May be NULL meaning "no NULLs". High bits of the last byte are ignored.
 * For outputs the caller provides both buffers (capacity >= the rows it asks for).
 * TQ_MEM_DEVICE columns (not Go memory) have stricter rules, checked by the vectorized-builtin calls: data
 * 16-byte aligned; null_bitmap 8-byte aligned and allocated as ((length + 63) / 64) * 8 bytes — the kernels move
 * whole 64-row bitmap groups.
 * A var-len TQ_MEM_DEVICE column given to tq_join_put_build / _put_probe, tq_agg_put, tq_sort_put or tq_mjoin_put_*:
 * offsets = length + 1 int64 in device memory, 8-byte aligned, non-decreasing; offsets[0] may be non-zero (a sliced column,
 * a cell range of a lent result) and cell i is data[offsets[i], offsets[i + 1]); data has any alignment (may be NULL when
 * every cell is empty); null_bitmap as for the other device columns.  The offsets are never read on the host: a put reads
 * back offsets[0], offsets[length] and the longest cell once, and refuses offsets that go backwards (TQ_ERR_INVALID_ARG).
 * Every such put copies (join, sort, merge join) or encodes (aggregation) the cells before it returns, so the caller may
 * reuse offsets and data right away; the null_bitmap follows the rule of the operator's 8-byte device columns (sort, merge
 * join, aggregation: copied too; join build: borrowed until tq_join_finalize_build; join probe: borrowed until the batch is
 * finished — the next tq_join_put_probe, tq_join_probe_eof or the tq_join_next* call that returns its rows).
 * FLOAT columns (TQ_TYPE_FLOAT32) come from host memory only: a TQ_MEM_DEVICE put refuses them (TQ_ERR_UNSUPPORTED_TYPE). */
typedef struct tq_column {
  int64_t length;
  uint8_t *null_bitmap;
  int64_t *offsets; /* var-len only; must be NULL for fixed-width columns */
  uint8_t *data;
} tq_column;

/* ------------------------------------------------------------------ library */
/* Select the CUDA device for this process (one process per GPU).  Fails with
 * TQ_ERR_NO_DEVICE when no sm_90 GPU is visible. */
int32_t tq_init(int32_t device_ordinal);
int32_t tq_shutdown(void);
/* Copies the calling thread's last error text (NUL-terminated) into buf. */
int32_t tq_last_error(char *buf, int32_t buf_len);
const char *tq_version(void);

/* util/chunk bridge: page-locked host memory so chunk.Column buffers are DMA-able
 * (SURVEY §8b "Ownership" option ii). */
int32_t tq_pinned_alloc(size_t bytes, void **out);
int32_t tq_pinned_free(void *p);

/* Device memory helpers used by the benchmark / multi-GPU drivers. */
int32_t tq_device_alloc(size_t bytes, void **out);
int32_t tq_device_free(void *p);
int32_t tq_memcpy_h2d(void *dst_dev, const void *src_host, size_t bytes);
int32_t tq_memcpy_d2h(void *dst_host, const void *src_dev, size_t bytes);
int32_t tq_memcpy_d2d(void *dst_dev, const void *src_dev, size_t bytes); /* e.g. keep rows lent by *_next_device / export_partial */
int32_t tq_memset_device(void *dst_dev, int32_t byte_value, size_t bytes);
int32_t tq_device_synchronize(void);
/* waits for the library's compute stream only (kernels of the operators): copies and peer pushes on the other streams go on */
int32_t tq_compute_synchronize(void);

/* Device-side timing on the library's compute stream (the stream every kernel of
 * this library is launched on).  tq_timer_stop returns elapsed milliseconds. */
int32_t tq_timer_start(void);
int32_t tq_timer_stop(float *elapsed_ms);
/* Number of kernels this library has launched since process start. */
int64_t tq_kernel_launch_count(void);
/* Writes `bytes` of a scratch buffer to evict L2 between timed iterations. */
int32_t tq_flush_l2(void);

/* ------------------------------------------------------- vectorized builtins
 * Replaces expression.vecEvalInt / vecEvalReal of the builtin signatures
 * (expression/builtin.go:256-263).  `n` rows; a/b/out are columns of n rows in
 * memory space `mem`; `out` buffers are caller-allocated (data n*8 bytes,
 * null_bitmap ceil(n/8) bytes).  The callee fills data and null bitmap (all bits
 * beyond n in the last byte are written as 0).  Error statuses follow the
 * reference: any non-NULL row overflowing fails the whole call. */

enum { TQ_CMP_LT = 0, TQ_CMP_LE = 1, TQ_CMP_GT = 2, TQ_CMP_GE = 3, TQ_CMP_EQ = 4, TQ_CMP_NE = 5 };
/* builtin{LT,LE,GT,GE,EQ,NE}IntSig.vecEvalInt — expression/builtin_compare_vec.go:22-292,
 * types.VecCompare{II,UU,IU,UI} types/compare.go:44-100.  Result int64 0/1. */
int32_t tq_vec_compare_int(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned,
                           const tq_column *b, int32_t b_unsigned, tq_column *out, int32_t mem);
/* builtin{LT..NE}RealSig.vecEvalInt — expression/builtin_compare_vec_generated.go:23-473. */
int32_t tq_vec_compare_real(int32_t op, int64_t n, const tq_column *a, const tq_column *b,
                            tq_column *out, int32_t mem);
/* String (var-len column) builtins.  a / b: offsets + data (+ bitmap); out: int64 column.
 *   op TQ_CMP_LT..TQ_CMP_NE  builtin{LT..NE}StringSig.vecEvalInt — expression/builtin_compare_vec_generated.go:65-555
 *   op TQ_STR_STRCMP         builtinStrcmpSig.vecEvalInt (-1 / 0 / 1) — expression/builtin_string_vec.go:52-83
 * Order is types.CompareString (types/compare.go:115-123): byte-wise.  NULL iff either argument is NULL. */
enum { TQ_STR_STRCMP = 6 };
int32_t tq_vec_compare_string(int32_t op, int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem);
/*   TQ_STR_LENGTH  builtinLengthSig: byte length (expression/builtin_string.go:75-81; the vectorized body is a course stub)
 *   TQ_STR_ISNULL  builtinStringIsNullSig.vecEvalInt — expression/builtin_string_vec.go:21-42 (never NULL) */
enum { TQ_STR_LENGTH = 0, TQ_STR_ISNULL = 1 };
int32_t tq_vec_string_unary(int32_t op, int64_t n, const tq_column *a, tq_column *out, int32_t mem);

enum { TQ_ARITH_PLUS = 0, TQ_ARITH_MINUS = 1, TQ_ARITH_MUL = 2, TQ_ARITH_DIV = 3 };
/* builtinArithmetic{Plus,Minus,Multiply}IntSig / MultiplyIntUnsignedSig.vecEvalInt —
 * expression/builtin_arithmetic_vec.go:88-340,389-532.  MUL with EITHER unsigned flag set
 * is MultiplyIntUnsigned (both operands read as uint64), otherwise MultiplyInt — the choice
 * multiplyFunctionClass.getFunction makes (expression/builtin_arithmetic.go:344-352). */
int32_t tq_vec_arith_int(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned,
                         const tq_column *b, int32_t b_unsigned, tq_column *out, int32_t mem);
/* builtinArithmetic{Plus,Minus,Multiply,Divide}RealSig.vecEvalReal —
 * builtin_arithmetic_vec.go:25-86,282-387.  Division by zero yields NULL and bumps
 * *div_by_zero_warnings (may be NULL) — the non-strict-mode behaviour of
 * handleDivisionByZeroError; the Go shim turns the count into warnings/errors. */
int32_t tq_vec_arith_real(int32_t op, int64_t n, const tq_column *a, const tq_column *b,
                          tq_column *out, int64_t *div_by_zero_warnings, int32_t mem);

enum { TQ_LOGIC_AND = 0, TQ_LOGIC_OR = 1 };
/* builtinLogic{And,Or}Sig.vecEvalInt — expression/builtin_op_vec.go:29-68,173-215. */
int32_t tq_vec_logic(int32_t op, int64_t n, const tq_column *a, const tq_column *b,
                     tq_column *out, int32_t mem);

enum {
  TQ_UNARY_NOT_INT = 0,   /* builtinUnaryNotIntSig   builtin_op_vec.go:249-267 */
  TQ_UNARY_NOT_REAL = 1,  /* builtinUnaryNotRealSig  builtin_op_vec.go:141-167 */
  TQ_UNARY_MINUS_INT = 2, /* builtinUnaryMinusIntSig builtin_op_vec.go:221-243 */
  TQ_UNARY_MINUS_REAL = 3,/* builtinUnaryMinusRealSig builtin_op_vec.go:74-86  */
  TQ_UNARY_ISNULL = 4     /* builtin{Int,Real}IsNullSig builtin_op_vec.go:92-135 */
};
int32_t tq_vec_unary(int32_t op, int64_t n, const tq_column *a, int32_t a_unsigned,
                     tq_column *out, int32_t mem);

/* builtinIf{Int,Real}Sig — expression/builtin_control_vec_generated.go:117-207.
 * cond is an int column; a/b/out share one 8-byte type (bits are moved verbatim). */
int32_t tq_vec_if(int64_t n, const tq_column *cond, const tq_column *a, const tq_column *b,
                  tq_column *out, int32_t mem);
/* builtinIfNull{Int,Real}Sig — builtin_control_vec_generated.go:23-79. */
int32_t tq_vec_ifnull(int64_t n, const tq_column *a, const tq_column *b, tq_column *out,
                      int32_t mem);
/* builtinInIntSig — expression/builtin_other_vec_generated.go:24-96.  list has n_list
 * columns; list_unsigned[j] is the unsigned flag of list element j. */
int32_t tq_vec_in_int(int64_t n, const tq_column *a, int32_t a_unsigned, int32_t n_list,
                      const tq_column *list, const int32_t *list_unsigned, tq_column *out,
                      int32_t mem);

/* builtinInRealSig — expression/builtin_other_vec_generated.go:151-204 (DOUBLE operands, types.CompareFloat64 == 0). */
int32_t tq_vec_in_real(int64_t n, const tq_column *a, int32_t n_list, const tq_column *list, tq_column *out, int32_t mem);
/* builtinInStringSig — builtin_other_vec_generated.go:97-149 (var-len operands, byte-wise equality); n_list <= 8 per call. */
int32_t tq_vec_in_string(int64_t n, const tq_column *a, int32_t n_list, const tq_column *list, tq_column *out, int32_t mem);
/* builtinIfStringSig / builtinIfNullStringSig.vecEvalString — builtin_control_vec_generated.go:209-262, 81-112.  a / b / out are
 * var-len columns; out needs offsets for n + 1 entries, a null_bitmap, and a data buffer of at least bytes(a) + bytes(b). */
int32_t tq_vec_if_string(int64_t n, const tq_column *cond, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem);
int32_t tq_vec_ifnull_string(int64_t n, const tq_column *a, const tq_column *b, tq_column *out, int32_t mem);

/* The BASELINE config-2 pair in one pass: lt_out = (a < b), plus_out = a + b, both
 * signed BIGINT — one read of a and b instead of two (32 B/row instead of 48). */
int32_t tq_vec_lt_plus_int(int64_t n, const tq_column *a, const tq_column *b,
                           tq_column *lt_out, tq_column *plus_out, int32_t mem);

/* expression.VectorizedFilter over an already-evaluated boolean-ish int column
 * (expression/chunk_executor.go:196-245, toBool expression.go:281-326): selected[i] =
 * (not NULL && value != 0).  selected is n bytes (Go []bool). */
int32_t tq_vec_filter_int(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem);
/* the same for an ETReal expression: toBool's zero test is types.RoundFloat(f) == 0, i.e. |f| < 0.5 (expression.go:296-307). */
int32_t tq_vec_filter_real(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem);

/* the same for an ETString expression: toBool's zero test is types.StrToInt(cell) == 0 in the statement context of a SELECT
 * (expression.go:308-322; types/convert.go:224-232: white space trimmed, longest valid numeric prefix, rounded to an integer —
 * "0.5" is 1, "abc" is 0).  Returns TQ_ERR_OVERFLOW_BIGINT when the LAST non-NULL row's integer does not fit BIGINT — the
 * error VecEvalBool keeps (`err = err1` per row).  `a` is a var-len column (offsets + data). */
int32_t tq_vec_filter_string(int64_t n, const tq_column *a, uint8_t *selected, int32_t mem);

/* ---- fused Selection + Projection (SURVEY §8 f1) -------------------------------------
 * One pass over a chunk for a whole list of filters and projection expressions: replaces
 * SelectionExec.Next → expression.VectorizedFilter (executor/executor.go:463-499,
 * expression/chunk_executor.go:196-245, VecEvalBool expression/expression.go:205-279) followed by
 * ProjectionExec's per-expression VecEval (expression/chunk_executor.go evalOneVec).  The planner-side
 * shim lowers the expression trees of fixed-width (ETInt / ETReal) builtins to a straight-line program:
 * register k < n_inputs is input column k, register n_inputs + i is the result of ops[i]; an op may read
 * only inputs and earlier results.  IN (a, l0, l1 …) lowers to a chain of EQ + LOGIC_OR, which has the
 * same three-valued result as builtinInIntSig / builtinInRealSig.
 *   TQ_X_FILTER a      : one CNF item of the filter list; op = 0 for an ETInt item, 1 for ETReal (toBool,
 *                        expression.go:281-326).  A row whose item is zero (or, ETReal, NULL) leaves the
 *                        evaluation set exactly as VecEvalBool narrows input.Sel(): overflow errors and
 *                        division-by-zero warnings of LATER ops do not count for it.  An ETInt NULL keeps the
 *                        row in the set (nulls[] quirk, expression.go:249-259) but it is not selected.
 *   TQ_X_COMPACT       : the Selection → Projection boundary: only selected rows remain in the set.
 * Outputs are dense (all n rows; values of unselected rows are unspecified); selected (n bytes, may be
 * NULL when no FILTER op is present) is Go's []bool.  The error is the error of the first op, in program
 * order, that raises on an in-set row (same codes as tq_vec_arith_*): the reference evaluates children
 * before parents, CNF items and projections in order, and returns at the first op that raises. */
enum { TQ_X_CONST = 0, TQ_X_CMP_INT, TQ_X_CMP_REAL, TQ_X_ARITH_INT, TQ_X_ARITH_REAL, TQ_X_LOGIC, TQ_X_UNARY,
       TQ_X_IF, TQ_X_IFNULL, TQ_X_FILTER, TQ_X_COMPACT };
#define TQ_EXPR_MAX_INPUTS 8
#define TQ_EXPR_MAX_OPS 32
#define TQ_EXPR_MAX_OUTPUTS 4
typedef struct tq_expr_op {
  int32_t kind;        /* TQ_X_* */
  int32_t op;          /* TQ_CMP_* / TQ_ARITH_* / TQ_LOGIC_* / TQ_UNARY_* for the kind; FILTER: 0 int, 1 real */
  int32_t a, b, c;     /* operand registers (IF: a = condition, b = then, c = else) */
  int32_t a_unsigned;  /* mysql.UnsignedFlag of operand a / b (CMP_INT, ARITH_INT, UNARY minus) */
  int32_t b_unsigned;
  int32_t is_null;     /* CONST: the constant is NULL */
  uint64_t imm;        /* CONST: the 8 value bytes (int64 / uint64 / float64 bits) */
} tq_expr_op;
int32_t tq_expr_eval(int64_t n, int32_t n_inputs, const tq_column *inputs, int32_t n_ops,
                     const tq_expr_op *ops, int32_t n_outputs, const int32_t *out_regs, tq_column *outs,
                     uint8_t *selected, int64_t *div_by_zero_warnings, int32_t mem);

/* ------------------------------------------------------------------ hash join
 * Replaces HashJoinExec (executor/join.go:31-146), hashRowContainer / rowHashMap
 * (executor/hash_table.go), joiner (executor/joiner.go).  Protocol (= the reference's
 * Open / fetchAndBuildHashTable / fetchAndProbeHashTable / Next / Close):
 *
 *   tq_join_create
 *   tq_join_put_build   xN   one inner-side chunk each   (hashRowContainer.PutChunk)
 *   tq_join_finalize_build
 *   loop { tq_join_put_probe (one outer-side chunk)  |  tq_join_probe_eof }
 *        interleaved with tq_join_next until it reports eof
 *   tq_join_destroy                                  (Close; legal at any point)
 *
 * Output schema = left child columns ++ right child columns (executor/builder.go:443);
 * with outer_is_right != 0 the build (inner) side is the left child.
 *
 * Key-less join (n_keys == 0: cross joins, ON conditions without an equality, outer joins whose ON names one side only).
 * With no key columns the reference puts every build row into one chain in insertion order (hash_table.go:146-169) and every
 * selected probe row finds it (join.go:325-362, rowHashMap.Get hash_table.go:259-272), so:
 *  - the candidates of a probe row are all build rows in insertion order; the OtherConditions filter the pairs
 *    (joiner.go:155-167);
 *  - an outer join emits a probe row once as its miss row (NULL / defaultInner inner side) when no pair survives, when
 *    selected[i] == 0, or when the build side is empty; the conditions never run for the last two (joiner.go:225-228,288-291),
 *    so those rows raise no error and no warning;
 *  - the output is exactly the reference's row sequence: probe rows in input order, build rows in insertion order inside one.
 * Same protocol, column layouts, selected[], defaultInner and conditions as the keyed join.  A probe batch is owned by the
 * handle once put (device chunks are copied) and produces no rows by itself: result batches of at most probe_batch_rows rows
 * are built only when tq_join_next / _next_bytes / _next_device needs rows (at most one ahead), so memory does not depend
 * on |probe| x |build|, and tq_join_destroy mid-stream is cheap.  An overflow of a pair in the evaluation set is returned by
 * the call that would deliver the first row of the probe-row sub-range it belongs to (DESIGN.md §3).
 * tq_join_put_probe_segments answers a key-less handle with TQ_ERR_UNSUPPORTED_TYPE. */
enum { TQ_JOIN_INNER = 0, TQ_JOIN_LEFT_OUTER = 1, TQ_JOIN_RIGHT_OUTER = 2 }; /* planner/core/logical_plans.go:52-57 */

typedef struct tq_join_desc {
  int32_t join_type;          /* TQ_JOIN_*                                                    */
  int32_t outer_is_right;     /* 1 iff InnerChildIdx == 0 (builder.go:451-477, joiner.go:93-95) */
  int32_t n_build_cols;       /* inner-side schema                                            */
  const int32_t *build_types; /* TQ_TYPE_* per inner column                                   */
  int32_t n_probe_cols;       /* outer-side schema                                            */
  const int32_t *probe_types;
  int32_t n_keys;             /* len(innerKeys) == len(outerKeys), 0..8; any supported column type (codec.go:216-236).
                               * 0 = the key-less join below: build_key_idx / probe_key_idx may be NULL */
  const int32_t *build_key_idx; /* innerKeys[i].Index                                         */
  const int32_t *probe_key_idx; /* outerKeys[i].Index                                         */
  int64_t probe_batch_rows;   /* device batch size the ≤1024-row chunks are accumulated into; 0 = default */
  int32_t flags;              /* TQ_JOIN_STABLE_INPUT or 0                                    */
  /* defaultInner of an outer join — PhysicalHashJoin.DefaultValues (executor/joiner.go:139-143, builder.go:449-465; set by
   * the aggregation push-down, planner/core/rule_aggregation_push_down.go:211-214, e.g. COUNT -> 0): the inner side of a miss
   * row.  default_inner_not_null[c] != 0 gives inner column c the value default_inner_bits[c] (8-byte column types);
   * both NULL = the usual all-NULL inner side. */
  const uint64_t *default_inner_bits;
  const uint8_t *default_inner_not_null;
} tq_join_desc;

/* tq_join_desc.flags.  STABLE_INPUT: every host buffer passed to tq_join_put_build / tq_join_put_probe stays valid and
 * unmodified until the handle is destroyed (the util/chunk bridge hands out C-owned pinned columns and does not recycle
 * them while the join runs).  Large host columns are then uploaded asynchronously: the call returns while the DMA is in
 * flight, so the upload of batch i+1 overlaps the result download of batch i.  Without the flag every call finishes
 * reading its arguments before it returns (the cgo pointer rule). */
enum { TQ_JOIN_STABLE_INPUT = 1 };

typedef struct tq_join tq_join;

int32_t tq_join_create(const tq_join_desc *desc, tq_join **out);
/* OtherConditions of the joiners (executor/joiner.go:155-167: baseJoiner.filter over the joined rows; an outer row whose
 * joined rows all fail is emitted once with a NULL / defaultInner inner side).  Two forms, one per handle:
 *
 * tq_join_set_other_conditions: each condition compares output column lhs_col (index into lhs ++ rhs) with output column
 * rhs_col, or with the constant when rhs_col < 0: BIGINT with BIGINT (any sign mix) or DOUBLE with DOUBLE; all conditions
 * are ANDed, a NULL operand fails.  At most 8 conditions.  The library runs them as the program below (one CMP + FILTER
 * item per condition).
 *
 * tq_join_set_other_program: the conditions as a tq_expr_op program over the joined row (left ++ right).  Input register
 * k = output column input_cols[k], which must be an INT64 / UINT64 / FLOAT64 column.  ops: kinds TQ_X_CONST .. TQ_X_FILTER
 * (no TQ_X_COMPACT), at least one TQ_X_FILTER, with the operand rules of tq_expr_eval.  A joined row passes iff every
 * FILTER item selects it.
 *
 * Rules.  Call either setter once, right after tq_join_create; a handle that has conditions of one form answers a call
 * for the other with TQ_ERR_STATE.  A malformed program (a bad register or operator, TQ_X_COMPACT, no FILTER, more than
 * TQ_EXPR_MAX_INPUTS inputs or TQ_EXPR_MAX_OPS ops) is TQ_ERR_INVALID_ARG, an input column of type FLOAT or var-len
 * TQ_ERR_UNSUPPORTED_TYPE; both before any device work.
 *
 * Semantics (joiner.go:155-167,225-340).
 *  - Inner join: a joined row survives iff the conditions select it.
 *  - Outer join: a probe row with key matches none of which passes is emitted once as its miss row, defaultInner on the
 *    inner side, at the position of one of its failed joined rows.
 *  - The conditions never run for probe rows without a key match, with a NULL key or with selected[i] == 0: the reference
 *    returns before filter when inners.Len() == 0 (joiner.go:225-228,288-291).  Such rows raise no error and no warning.
 *  - Errors: a joined row in the evaluation set (tq_expr_eval's narrowing: a row an earlier FILTER item dropped does not
 *    raise) that overflows makes the call that would deliver its batch return TQ_ERR_OVERFLOW_BIGINT / _UNSIGNED /
 *    _DOUBLE — tq_join_next, tq_join_next_device or tq_join_next_bytes, whichever takes up the batch.  After that the
 *    handle only supports tq_join_destroy.  The reference reports the first error in its per-chunk order; here any in-set
 *    row of the batch may be the one reported (DESIGN.md §3).
 *  - Result order is unchanged: compaction is stable, so the one-table path (build side below 2^18 rows) still yields
 *    (probe row ascending, build insertion ascending).
 * tq_join_warnings: division-by-zero warnings raised so far by joined rows in the evaluation set (handleDivisionByZeroError,
 * builtin_arithmetic_vec.go:369-375), counted as their batches are finished. */
typedef struct tq_join_cond {
  int32_t op;         /* TQ_CMP_*                                   */
  int32_t lhs_col;    /* output column                              */
  int32_t rhs_col;    /* output column, or -1: the constant below   */
  int32_t const_type; /* TQ_TYPE_* of the constant                  */
  uint64_t const_bits;
} tq_join_cond;
int32_t tq_join_set_other_conditions(tq_join *j, int32_t n_conds, const tq_join_cond *conds);
int32_t tq_join_set_other_program(tq_join *j, int32_t n_inputs, const int32_t *input_cols, int32_t n_ops, const tq_expr_op *ops);
int32_t tq_join_warnings(tq_join *j, int64_t *div_by_zero);
int32_t tq_join_put_build(tq_join *j, const tq_column *cols, int32_t mem);
int32_t tq_join_finalize_build(tq_join *j);
/* selected: outerSideFilter result (join.go:328), n bytes of 0/1 in HOST memory, or NULL = all selected. */
int32_t tq_join_put_probe(tq_join *j, const tq_column *cols, const uint8_t *selected, int32_t mem);
int32_t tq_join_probe_eof(tq_join *j);
/* Multi-GPU variant of put_probe: the batch is the concatenation of n_segs DEVICE regions (one per source rank, filled by the
 * peers' tq_partition_push_regions kernels).  cols[g * n_probe_cols + c] = column c of region g (NOT NULL 8-byte columns,
 * `length` ignored); *seg_counts[g] = the rows region g holds — a DEVICE value, read by the kernels, never by the host, so no
 * host synchronisation sits between the exchange and the join; seg_cap = rows a region can hold.  Inner PK-FK joins on the
 * streaming path only (TQ_ERR_UNSUPPORTED_TYPE otherwise: read the regions with tq_region_gather and use tq_join_put_probe,
 * which is also how outer joins and nullable columns pushed by tq_partition_push_regions are joined).
 * The call only enqueues the batch: the regions and their counts must stay unchanged until the batch is finalised, i.e.
 * until the next tq_join_put_probe / _put_probe_segments, tq_join_probe_eof, or the tq_join_next* call that returns its
 * rows.  Skewed probe keys that overflow a partition slab are still joined: the batch is then re-run on the exact
 * (histogram) path, which costs one host read of the counts, a device copy of every region's rows into one buffer, and a
 * second probe pass.  Later segmented batches on the handle start on the streaming path again. */
int32_t tq_join_put_probe_segments(tq_join *j, int32_t n_segs, const tq_column *cols, const uint64_t *const *seg_counts, int64_t seg_cap);
/* Fills at most max_rows joined rows into out_cols (n_build_cols + n_probe_cols caller-
 * allocated columns, host memory).  *n_rows == 0 with *eof == 0 means "feed more probe
 * chunks"; *n_rows == 0 with *eof != 0 is the reference's end of stream. */
int32_t tq_join_next(tq_join *j, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* Data bytes each output column of the NEXT tq_join_next(j, max_rows, ...) call will carry (8 * rows for the 8-byte
 * types, 4 * rows for FLOAT, the cells' total length for var-len columns), so the caller can size out_cols[c].data —
 * the "*_next_size query" of the ownership contract.  All zero when that call would return no rows. */
int32_t tq_join_next_bytes(tq_join *j, int64_t max_rows, int64_t *bytes_per_col);
int32_t tq_join_destroy(tq_join *j);

/* Benchmark / multi-GPU variant of Next: pops the oldest finished device result batch and
 * lends its device-resident columns (valid until the next call on this handle). */
int32_t tq_join_next_device(tq_join *j, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* Statistics of the handle: [0] build rows inserted, [1] distinct build keys, [2] partitions,
 * [3] probe rows consumed, [4] joined rows produced, [5] last probe kernel time in ns,
 * [6] last build time in ns, [7] probe kernel launches.
 * Key-less handles: [0] build rows stored, [1] = [2] = 0, [4] rows of the result batches built so far, [5] device time of
 * the last result batch's kernels.  */
int32_t tq_join_stats(tq_join *j, int64_t *stats8);
/* Which build made the handle's hash table (after tq_join_finalize_build): the general build, or the streaming build of a
 * large unique NOT NULL build side with each sub-table built in one thread-block cluster's or in one CTA's shared memory. */
#define TQ_JOIN_BUILD_GENERAL 0
#define TQ_JOIN_BUILD_CLUSTER 1
#define TQ_JOIN_BUILD_CTA 2
int32_t tq_join_build_path(tq_join *j, int32_t *path);

/* ------------------------------------------------------------------ chunk wire codec
 * chunk.Codec.Encode / DecodeToChunk (util/chunk/codec.go:42-143) — the bytes child readers hand up.  Decoding fills
 * tq_column VIEWS into the buffer (zero copy; null_bitmap == NULL for a column without NULLs), ready for
 * tq_join_put_* / tq_agg_put.  No device is needed for these three calls. */
int32_t tq_chunk_encoded_size(int32_t n_cols, const int32_t *types, const tq_column *cols, int64_t *bytes);
int32_t tq_chunk_encode(int32_t n_cols, const int32_t *types, const tq_column *cols, uint8_t *buffer, int64_t capacity, int64_t *written);
int32_t tq_chunk_decode(const uint8_t *buffer, int64_t len, int32_t n_cols, const int32_t *types, tq_column *out, int64_t *consumed);

/* Decoder for the device: the wire bytes cross PCIe once, as they are, and ONE kernel launch lays every column out in HBM
 * (util/chunk/codec.go:92-143,246-353; distsql/select_result.go:102-141 is where the reference decodes on the CPU).
 * out[c] receives DEVICE pointers — data (8-byte slots; 4-byte slots for FLOAT; the cells' bytes for var-len columns),
 * offsets (var-len only) and null_bitmap (NULL when the column has no NULLs; otherwise 8-byte aligned words, tail bits 0) —
 * which the TQ_MEM_DEVICE entry points accept as they are (tq_join_put_build / put_probe, tq_agg_put, tq_sort_put,
 * tq_mjoin_put_*: 8-byte and var-len columns, FLOAT columns are refused; tq_vec_*, tq_expr_eval: their operand types).
 * *chunk == NULL creates a handle; passing the same handle again reuses its device memory (the
 * previous columns become invalid).  The call returns after the bytes have left `buffer` and the columns are complete. */
typedef struct tq_chunk_device tq_chunk_device;
int32_t tq_chunk_decode_device(const uint8_t *buffer, int64_t len, int32_t n_cols, const int32_t *types, tq_chunk_device **chunk,
                               tq_column *out, int64_t *consumed);
int32_t tq_chunk_device_free(tq_chunk_device *chunk);

/* ------------------------------------------------------------------ hash agg
 * Replaces HashAggExec + workers (executor/aggregate.go) and the aggfuncs it drives
 * (executor/aggfuncs/ sources).  GROUP BY items and aggregate arguments are column
 * references into the input chunk (the shim pre-projects expressions with tq_vec_*). */
enum {
  TQ_AGG_COUNT = 0,    /* aggfuncs/func_count.go      */
  TQ_AGG_SUM = 1,      /* aggfuncs/func_sum.go        */
  TQ_AGG_AVG = 2,      /* aggfuncs/func_avg.go        */
  TQ_AGG_MAX = 3,      /* aggfuncs/func_max_min.go    */
  TQ_AGG_MIN = 4,
  TQ_AGG_FIRSTROW = 5  /* aggfuncs/func_first_row.go  */
};

typedef struct tq_agg_func {
  int32_t func;    /* TQ_AGG_*                                                          */
  int32_t arg_col; /* input column index; -1 = constant non-NULL argument (COUNT(*) == count(1)) */
} tq_agg_func;

typedef struct tq_agg_desc {
  int32_t n_input_cols;
  const int32_t *input_types;   /* TQ_TYPE_* per input column */
  int32_t n_group_by;           /* 0 = scalar aggregate       */
  const int32_t *group_by_cols; /* input column indices       */
  int32_t n_funcs;
  const tq_agg_func *funcs;     /* output column i = funcs[i] (builder.go:523-535) */
  int64_t est_groups;           /* hint; 0 = unknown          */
} tq_agg_desc;

typedef struct tq_agg tq_agg;

int32_t tq_agg_create(const tq_agg_desc *desc, tq_agg **out);
/* Output type (TQ_TYPE_*) of aggregate i: COUNT → INT64; SUM/AVG keep the argument's eval
 * type (AVG(int) is the truncating integer division of func_avg.go:53). */
int32_t tq_agg_output_type(tq_agg *a, int32_t func_idx, int32_t *type_out);
int32_t tq_agg_put(tq_agg *a, const tq_column *cols, int32_t mem);
int32_t tq_agg_eof(tq_agg *a);
int32_t tq_agg_next(tq_agg *a, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* Data bytes each output column of the NEXT tq_agg_next(a, max_rows, ...) call will carry (8 * rows; 4 * rows for a FLOAT
 * result; the cells' total length for a var-len result), so the caller can size out_cols[c].data. */
int32_t tq_agg_next_bytes(tq_agg *a, int64_t max_rows, int64_t *bytes_per_col);
int32_t tq_agg_next_device(tq_agg *a, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
int32_t tq_agg_destroy(tq_agg *a);
/* [0] input rows, [1] groups, [2] last update-kernel time ns, [3] kernel launches */
int32_t tq_agg_stats(tq_agg *a, int64_t *stats4);

/* Partial → shuffle → final (aggregate.go:96-133,352-356,424-427), used across GPUs:
 * tq_agg_export_partial lends device arrays holding one row per local group —
 * n_group_by key columns followed by the partial-state columns (COUNT: count; SUM: sum
 * [NULL = no value yet]; AVG: count then sum; MAX/MIN/FIRSTROW: value) — and
 * tq_agg_merge_partial consumes rows of that layout with MergePartialResult semantics. */
int32_t tq_agg_partial_width(tq_agg *a, int32_t *n_cols);
int32_t tq_agg_export_partial(tq_agg *a, tq_column *out_cols, int64_t *n_rows);
int32_t tq_agg_merge_partial(tq_agg *a, const tq_column *cols, int32_t mem);
/* The same partial -> shuffle -> final over the region exchange (tq_partition_push_regions, below): no count exchange, no
 * staging copy, nullable columns and GROUP BYs of any number of items.  Wire format: with w = tq_agg_partial_width(a), a partial
 * row (the layout of tq_agg_export_partial: key columns, then states) travels as w + 1 8-byte words, the last the NULL mask
 * (bit c = column c is NOT NULL); w + 1 > 64 is TQ_ERR_INVALID_ARG.
 *
 * tq_agg_push_partial, after the raw rows of a tq_agg_create handle (tq_agg_eof is implied): exports the partial rows (one
 * host read of the group count) and scatters them on the push stream — dest_data[q * (w + 1) + c] = THIS rank's region for
 * wire column c on rank q (local or PEER pointer), region_cap rows; dest_counts[q] = its 16-byte {u64 rows, u64 epoch} slot
 * there — then publishes the slots as tq_partition_push_regions does (same slots 0..15, waited for with
 * tq_partition_push_sync(slot); overflow of any region makes every slot read ~0).  The handle's partial rows are read until
 * the push has finished.  A row goes to the rank its group names, a pure function of the group: h = 0, then per GROUP BY item
 * g  h = mix64(h ^ v_g), v_g = the item's 8 bytes (REAL: -0.0 read as +0.0) or 0x4E554C4C4E554C4C for NULL; rank =
 * (h >> 40) % n_parts.  One NOT NULL item: (mix64(v) >> 40) % n_parts, the rank tq_partition_push_regions sends that key to;
 * a scalar aggregate (no GROUP BY) sends its row to rank 0.  n_parts 1..8, 1 <= region_cap < 2^32.
 *
 * tq_agg_merge_regions, on a handle created with the same desc that has taken no raw rows (queue tq_region_wait first):
 * reads the n_regions (1..8) consecutive slots at `slots` (one host read) and merges regions[g * (w + 1) + c] (wire column c
 * of region g) with tq_agg_merge_partial's semantics, reading the regions in place.  A slot reading 0xFFFFFFFF00000000 | s
 * (a failed push, below) returns status s and merges nothing, so every rank refuses a step one source could not push; any
 * other slot above region_cap (or ~0) is TQ_ERR_OOM and merges nothing.  Then tq_agg_eof / next as usual: a merged total
 * that leaves int64 is TQ_ERR_OVERFLOW_BIGINT from next / next_device on the rank that finishes the group.
 *
 * Both refuse what tq_agg_export_partial / tq_agg_merge_partial refuse (var-len columns: TQ_ERR_UNSUPPORTED_TYPE; a FinalMode
 * handle, or raw and partial rows on one handle: TQ_ERR_STATE), and check every argument before anything is enqueued: a
 * refused push writes no region and publishes no slot.  A push that fails after those checks — a group's partial SUM / AVG
 * total on this rank leaves int64 (TQ_ERR_OVERFLOW_BIGINT, as tq_agg_export_partial), more than 2^32 - 16 partial rows, a
 * failed allocation — writes no region row but still publishes {0xFFFFFFFF00000000 | status, epoch} in every destination's
 * slot (waited for with tq_partition_push_sync(slot) as usual), so no tq_region_wait waits for it and every merge of the
 * step returns that status.  tq_region_gather and dist.RegionLayout.counts refuse the marker as a count past the cap. */
int32_t tq_agg_push_partial(tq_agg *a, int32_t n_parts, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                            int32_t slot, uint64_t epoch);
int32_t tq_agg_merge_regions(tq_agg *a, int32_t n_regions, const void *slots, int64_t region_cap, const tq_column *regions);
/* The same pair for handles with var-len (string) partial columns; on a handle without them both behave exactly as the pair
 * above, wire format included.  A partial column is var-len when it is a GROUP BY item on a BYTES input column or the state
 * of MAX / MIN / FIRSTROW over a BYTES argument; V = their number (at most 16).  Per source region the wire areas are:
 *   0 .. w - 1   the partial columns as above, except that a var-len column's area holds region_cap + 1 int64 OFFSETS:
 *                entry 0 = 0, entry i + 1 = the end of row i's cell in that column's byte area (a NULL cell is empty and its
 *                mask bit is 0)
 *   w            the NULL mask word
 *   w + 1 + v    byte area v of byte_cap[v] bytes: the cells of the v-th var-len column (partial-column order), in row order
 * tq_agg_push_partial_var: dest_data[q * (w + 1 + V) + a] = this rank's area a on rank q; byte_cap: V entries,
 * 1 <= byte_cap[v] < 2^32 (may be NULL when V = 0).  A string GROUP BY item routes by the 64-bit content hash of its bytes
 * (the one its string dictionary keeps), the same on every rank, so the empty string and NULL are different groups; 8-byte
 * items route as above.  Rows keep the handle's partial-row order in every region, and each cell is copied from the handle's
 * dictionary.  A region past region_cap rows or a byte area past byte_cap makes every slot read ~0; nothing is written past
 * either cap.  No host synchronisation beyond the group-count read.
 * tq_agg_merge_regions_var: regions[g * (w + 1) + c]; a var-len column c has .offsets = its offsets area and .data = its
 * byte area, every other column .data only.  Each var-len column is encoded into this handle's dictionary of the input
 * column it came from (GROUP BY s and MAX(s) share one), then merged as tq_agg_merge_regions does.  Refusals as above, less
 * the var-len one; a var-len column without offsets is TQ_ERR_INVALID_ARG. */
int32_t tq_agg_push_partial_var(tq_agg *a, int32_t n_parts, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                                const int64_t *byte_cap, int32_t slot, uint64_t epoch);
int32_t tq_agg_merge_regions_var(tq_agg *a, int32_t n_regions, const void *slots, int64_t region_cap, const tq_column *regions);

/* FinalMode HashAgg over pushed-down partial results (SURVEY §8 f4).  The planner splits an aggregation into a Partial1
 * half that runs inside the coprocessor (planner/core/task.go:564-625, store/mockstore/mocktikv/aggregate.go:81-124: each row
 * it returns = the GetPartialResult columns of every function — COUNT: count; SUM / MAX / MIN / FIRSTROW: value; AVG: count
 * then sum — followed by the GROUP BY columns) and a FinalMode HashAggExec whose AggFuncDesc.Args are column references into
 * that partial schema (expression/aggregation/descriptor.go:52-75, aggfuncs/builder.go:50-62,86-109: countPartial,
 * avgPartial4Int64 / avgPartial4Float64; SUM / MAX / MIN / FIRSTROW merge with their ordinary functions).
 * tq_agg_create_final builds that executor: tq_agg_put then takes the child's chunks of PARTIAL rows (any column order; all
 * three chunk layouts), and eof / next / next_bytes / destroy behave as for tq_agg_create.  arg_col = the partial column the
 * function reads (for AVG: the partial COUNT), arg_col2 = AVG's partial SUM column (ignored otherwise).  A partial row whose
 * COUNT or SUM is NULL is skipped by AVG (func_avg.go:93-103), NULL partial values are skipped by SUM / MAX / MIN / COUNT. */
typedef struct tq_agg_final_func {
  int32_t func;     /* TQ_AGG_* */
  int32_t arg_col;
  int32_t arg_col2;
} tq_agg_final_func;

typedef struct tq_agg_final_desc {
  int32_t n_input_cols;
  const int32_t *input_types;   /* TQ_TYPE_* per column of the partial schema */
  int32_t n_group_by;
  const int32_t *group_by_cols;
  int32_t n_funcs;
  const tq_agg_final_func *funcs;
  int64_t est_groups;
} tq_agg_final_desc;

int32_t tq_agg_create_final(const tq_agg_final_desc *desc, tq_agg **out);

/* ------------------------------------------------------------------ sort / top-n / merge join (SURVEY §8 f3)
 * SortExec and TopNExec (executor/sort.go:28-157, 159-318): put every child chunk, eof, then next until eof.
 * ByItems are column references (the shim pre-projects expressions) with a Desc flag; the comparator is
 * chunk.GetCompareFunc (util/chunk/compare.go:27-110): NULL first, then signed / unsigned / float / byte-string order; Desc
 * reverses the whole comparison (NULLs last).  Rows that compare equal keep child order (sort.Slice promises no order for
 * them).  limit_count >= 0 makes it a TopNExec returning rows [limit_offset, limit_offset + limit_count) of the order
 * (sort.go:210-214); limit_count < 0 is a SortExec.  All three chunk layouts, as keys and as payload. */
typedef struct tq_sort_desc {
  int32_t n_cols;
  const int32_t *types;     /* TQ_TYPE_* per child column */
  int32_t n_by;             /* 0..8 ByItems */
  const int32_t *by_cols;   /* column index of ByItems[i].Expr */
  const int32_t *by_desc;   /* ByItems[i].Desc */
  int64_t limit_offset;
  int64_t limit_count;
} tq_sort_desc;
typedef struct tq_sort tq_sort;
int32_t tq_sort_create(const tq_sort_desc *desc, tq_sort **out);
/* Chunks come from host memory (all chunk layouts) or, for 8-byte and var-len column types, from HBM (TQ_MEM_DEVICE: e.g. the
 * rows tq_join_next_device lends; FLOAT columns come from host memory only) — one or the other per handle.  With device chunks the rows never leave the GPU: tq_sort_next_device
 * lends the result (the TopN window) as device columns, and tq_sort_next copies it to the host only if it is called. */
int32_t tq_sort_put(tq_sort *s, const tq_column *cols, int32_t mem);
int32_t tq_sort_eof(tq_sort *s);
int32_t tq_sort_next_bytes(tq_sort *s, int64_t max_rows, int64_t *bytes_per_col);
int32_t tq_sort_next(tq_sort *s, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* device-chunk handles: the whole result at once as DEVICE columns, lent until tq_sort_destroy; then eof */
int32_t tq_sort_next_device(tq_sort *s, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* The receiving side of the multi-GPU ORDER BY (tq_partition_push_ranges): puts the n_regions (1..8) regions that arrived on
 * this rank, in source order, each as one device chunk.  Queue tq_region_wait first; slots = the n_regions consecutive
 * {u64 rows, u64 epoch} slots, read once on the host.  regions[g * (n_cols + 1) + c] = wire column c of region g: an 8-byte
 * column's values in .data; a BYTES column's offsets area (rows + 1 offsets from 0) in .offsets and its byte area in .data;
 * the mask word (bit c = column c is NOT NULL) at c = n_cols, in .data.  A slot past region_cap (~0: an overflowed push) is
 * TQ_ERR_OOM and a source that failed its push returns that push's status; either way nothing is put.  FLOAT32 columns are
 * TQ_ERR_UNSUPPORTED_TYPE (the push carries none).  After it, tq_sort_eof and tq_sort_next_device run as for any device put. */
int32_t tq_sort_put_regions(tq_sort *s, int32_t n_regions, const void *slots, int64_t region_cap, const tq_column *regions);
/* [0] rows sorted, [1] device time of the sort phase in ns (CUDA events; upload and result gather excluded),
 * [2] kernel launches of tq_sort_eof, [3] radix digit passes that ran (constant digits are skipped) */
int32_t tq_sort_stats(tq_sort *s, int64_t *stats4);
int32_t tq_sort_destroy(tq_sort *s);

/* MergeJoinExec (executor/merge_join.go:31-373).  Both children deliver rows sorted ascending by their join keys (the planner
 * guarantees it, exhaust_physical_plans.go:281-295; an unsorted inner child is reported as TQ_ERR_STATE).  Inner rows with a
 * NULL key are skipped (merge_join.go:154-162); an outer row that fails the outer filter (`selected`), has a NULL key or finds
 * no inner row with an equal key takes the joiner's miss path: outer joins emit it padded with NULLs / defaultInner
 * (joiner.go:139-143), inner joins drop it.  Output order = outer child order, inner child order inside a key group —
 * the order joinToChunk produces (merge_join.go:246-321).  Output schema = left child columns ++ right child columns.
 * Key pairs must share an evaluation type (int incl. signed/unsigned mixes, real incl. FLOAT, string). */
typedef struct tq_mjoin_desc {
  int32_t join_type;        /* TQ_JOIN_* */
  int32_t outer_is_right;   /* 1: the inner child is the left child */
  int32_t n_inner_cols;
  const int32_t *inner_types;
  int32_t n_outer_cols;
  const int32_t *outer_types;
  int32_t n_keys;
  const int32_t *inner_keys;
  const int32_t *outer_keys;
  const uint64_t *default_inner_bits;       /* per inner column, may be NULL: the 8 value bytes of its default */
  const uint8_t *default_inner_not_null;    /* per inner column, may be NULL (= all NULL): 1 = the default is a value */
} tq_mjoin_desc;
typedef struct tq_mjoin tq_mjoin;
int32_t tq_mjoin_create(const tq_mjoin_desc *desc, tq_mjoin **out);
/* OtherConditions of the joiner (baseJoiner.filter, joiner.go:155-167; tryToMatchInners in merge_join.go:290-305): the two forms
 * of the hash join (tq_join_cond comparisons or a tq_expr_op program), over the joined row left ++ right, with the same rules
 * and semantics; an outer row whose joined rows all fail takes the miss path, in its place in the output.  Set them right
 * after tq_mjoin_create; the comparison list may be set again, the program once.  The result is computed by
 * tq_mjoin_finish; an overflow of an in-set joined row is returned by every tq_mjoin_next / _next_device / _next_bytes
 * call after it.  The output order stays exactly the reference's. */
int32_t tq_mjoin_set_other_conditions(tq_mjoin *j, int32_t n_conds, const tq_join_cond *conds);
int32_t tq_mjoin_set_other_program(tq_mjoin *j, int32_t n_inputs, const int32_t *input_cols, int32_t n_ops, const tq_expr_op *ops);
/* division-by-zero warnings raised by joined rows in the evaluation set (handleDivisionByZeroError, builtin_arithmetic_vec.go:369-375) */
int32_t tq_mjoin_warnings(tq_mjoin *j, int64_t *div_by_zero);
/* host chunks (all layouts) or, for 8-byte and var-len column types, device chunks (TQ_MEM_DEVICE) — per child one or the other */
int32_t tq_mjoin_put_inner(tq_mjoin *j, const tq_column *cols, int32_t mem);
int32_t tq_mjoin_put_outer(tq_mjoin *j, const tq_column *cols, const uint8_t *selected, int32_t mem); /* selected: HOST Go []bool or NULL */
int32_t tq_mjoin_finish(tq_mjoin *j);   /* both children exhausted */
int32_t tq_mjoin_next_bytes(tq_mjoin *j, int64_t max_rows, int64_t *bytes_per_col);
int32_t tq_mjoin_next(tq_mjoin *j, int64_t max_rows, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
/* handles with a device-chunk child: the whole result at once as DEVICE columns, lent until tq_mjoin_destroy; then eof */
int32_t tq_mjoin_next_device(tq_mjoin *j, tq_column *out_cols, int64_t *n_rows, int32_t *eof);
int32_t tq_mjoin_destroy(tq_mjoin *j);

/* ------------------------------------------------------------- radix exchange
 * The shard boundary of the multi-GPU path: splits rows into n_parts partitions by
 * the key's hash (the moral equivalent of shuffleIntermData, aggregate.go:352-356).
 * All buffers are device memory.  out_cols must hold `n` rows each; rows of partition p
 * occupy [offsets[p], offsets[p+1]) of every output column, stable within a partition.
 * part_offsets is a HOST array of n_parts+1 entries.  Rows whose key is NULL go to
 * partition (row % n_parts): they never match but outer joins still emit them.
 * Every column is moved as 8-byte words: types[c] & 0xFF must be TQ_TYPE_INT64, _UINT64 or
 * _FLOAT64 and `offsets` NULL; a FLOAT32 or BYTES column is refused with
 * TQ_ERR_UNSUPPORTED_TYPE before anything is written. */
int32_t tq_partition_device(int32_t n_cols, const tq_column *cols, const int32_t *types,
                            int32_t key_col, int64_t n, int32_t n_parts, tq_column *out_cols,
                            int64_t *part_offsets);

/* Kernel-level load/store access from this process's device to `peer_device` (cudaDeviceEnablePeerAccess): required
 * before tq_partition_push_regions is handed PEER pointers. */
int32_t tq_enable_peer_access(int32_t peer_device);
/* CUDA IPC (cudaIpcGetMemHandle / OpenMemHandle / CloseMemHandle) for buffers from tq_device_alloc: a rank exports its
 * receive buffer as a 64-byte handle; peers open it under THEIR device and push rows into it over NVLink. */
int32_t tq_ipc_get_handle(void *dev_ptr, void *handle64);
int32_t tq_ipc_open_handle(const void *handle64, void **dev_ptr);
int32_t tq_ipc_close_handle(void *dev_ptr);
/* Fused scatter + exchange over NVLink peer memory (one process per GPU, buffers shared through CUDA IPC): the push into
 * per-source REGIONS, with no count exchange before it.  Destination q reserves `region_cap` rows per source rank and wire
 * column; this rank scatters each of its n rows straight into its region on rank (mix64(key) >> 40) % n_parts and then
 * publishes, per destination, how many rows it wrote there.
 *  - n_parts 1..8, n < 2^32, 0 <= key_col < n_cols, 1 <= region_cap < 2^32.
 *  - cols may carry NULL bitmaps (SURVEY §8(e): NULL-key rows never match; an inner join drops them before the exchange,
 *    an outer join emits their miss rows on the rank that holds them).  If any does, the side travels with one more column,
 *    the mask word: bit c of a row's word = column c is NOT NULL.  Wire columns per row: n_wire = n_cols (+ 1 with the mask,
 *    which comes last).  At most 4 wire columns: 3 nullable or 4 NOT NULL columns; a wider side is TQ_ERR_UNSUPPORTED_TYPE.
 *  - dest_data[q * n_wire + c] = the start of THIS rank's region for wire column c on rank q (local or PEER pointer).
 *  - dest_counts[q] points at a 16-byte slot {u64 rows, u64 epoch} on rank q: the count is published first (~0 = overflow),
 *    the epoch after a system-scope fence.
 *  - selected: n DEVICE bytes of 0/1 (the outer-side filter) or NULL = all selected.
 *  - A row can match when its key is NOT NULL and it is selected.  Any other row is dropped, or with keep_misses != 0 (the
 *    probe side of an outer join) written to this rank's miss_data[c] (n_wire local device columns of miss_cap rows, 0 <=
 *    miss_cap < 2^32), whose count is published at the 16-byte slot miss_count like a peer's; such a row never crosses a link.
 *  - Overflow of any region or of the miss columns makes every slot this push publishes read ~0.
 * A NOT NULL inner-join push passes selected = NULL, keep_misses = 0 and no miss buffers.  This signature replaced a
 * 10-argument NOT NULL-only form; against it two refusals changed: NULL bitmaps are accepted (were TQ_ERR_UNSUPPORTED_TYPE),
 * and more than 4 wire columns is TQ_ERR_UNSUPPORTED_TYPE (was TQ_ERR_INVALID_ARG).
 * Every argument is checked before anything is enqueued: a refused push writes no region and publishes no slot.  The push is
 * enqueued on the library's push stream; tq_partition_push_sync(slot) waits for it (slots 0..15 may be in flight together).
 * The receiver waits with tq_region_wait, then joins an inner join of NOT NULL columns in place with
 * tq_join_put_probe_segments, and everything else by copying the regions out with tq_region_gather and joining them with
 * tq_join_put_build / tq_join_put_probe (TQ_MEM_DEVICE): the kept miss rows as one more probe batch whose host `selected` is
 * all zeros. */
int32_t tq_partition_push_regions(int32_t n_cols, const tq_column *cols, int32_t key_col, int64_t n, int32_t n_parts,
                                  const uint8_t *selected, int32_t keep_misses, void *const *dest_data, void *const *dest_counts,
                                  int64_t region_cap, void *const *miss_data, void *miss_count, int64_t miss_cap, int32_t slot,
                                  uint64_t epoch);
/* The broadcast push (the other classic distributed join: replicate the build side, keep the probe side in place): copies
 * this rank's n rows into its region on each of the n_parts destinations, this rank included, then publishes {n, epoch} in
 * each destination's slot as tq_partition_push_regions does.  Every destination receives the rows in input order.
 *  - n_parts 1..8, 1..16 columns, 0 <= n <= region_cap < 2^32.
 *  - types[c] & 0xFF: INT64, UINT64 and FLOAT64 travel as 8-byte values; BYTES as its offsets, rebased to start at 0 (n + 1
 *    entries), and its cells [offsets[0], offsets[n]) copied to the start of a byte area of byte_cap[c] bytes.  FLOAT32 (and
 *    any other type) is TQ_ERR_UNSUPPORTED_TYPE: device puts refuse FLOAT columns.  offsets must be set exactly on the BYTES
 *    columns (TQ_ERR_INVALID_ARG otherwise), and may start anywhere, as for a TQ_MEM_DEVICE put.
 *  - nullable != 0: every column also travels as its ceil(n / 64) 64-row NULL bitmap words, all ones for a column without a
 *    bitmap, so the layout depends only on the declaration.  The receiver hands the words to tq_join_put_build as they are.
 *  - Areas per destination q, column by column: dest_data[q * n_areas + a] with, for each column c in order, its values (n
 *    words) or offsets (n + 1 words), then for BYTES its byte area, then on a nullable side its bitmap words.  n_areas =
 *    n_cols + (BYTES columns) + (nullable ? n_cols : 0).  Each area is stored with 16-byte stores where it is 16-byte aligned.
 *  - dest_counts[q]: the 16-byte slot {u64 rows, u64 epoch} on rank q.
 * Every argument is checked before anything is enqueued: a refused push writes no region and publishes no slot.  Cells that
 * exceed byte_cap[c] are found on the device: that column's cells are not copied and every slot this push publishes reads
 * ~0, so the receiver fails (tq_region_gather: TQ_ERR_OOM; dist.RegionLayout.counts: RuntimeError).  The push is enqueued
 * on the push stream; tq_partition_push_sync(slot) waits for it.  The receiver waits with tq_region_wait, reads the slots
 * and puts each source's region as one device build chunk (tq_join_put_build, TQ_MEM_DEVICE). */
int32_t tq_partition_push_broadcast(int32_t n_cols, const tq_column *cols, const int32_t *types, int32_t nullable, int64_t n, int32_t n_parts,
                                    void *const *dest_data, void *const *dest_counts, int64_t region_cap, const int64_t *byte_cap, int32_t slot,
                                    uint64_t epoch);
/* The two pushes of the multi-GPU ORDER BY (dist.RegionSort): rank src_rank routes each row of its shard to the rank whose
 * slice of the global order holds it.  The routing order is the ByItems' order followed by one more, ascending, word per
 * row, the tie word (src_rank << 32) | row: a total order that agrees with the rank-major stable sort, so a run of equal
 * keys may be split between ranks anywhere.  Both take 1..63 columns of TQ_TYPE_INT64, _UINT64, _FLOAT64 or _BYTES (any
 * other type, FLOAT32 included, is TQ_ERR_UNSUPPORTED_TYPE), device memory, offsets exactly on the BYTES columns (they may
 * start anywhere, as for a TQ_MEM_DEVICE put), NULL bitmaps where a column has NULLs; 0..8 ByItems by_cols[i] (Desc
 * by_desc[i]: NULL first ascending, last descending, as tq_sort); 0 <= n < 2^32, src_rank >= 0; byte_cap[c], for each BYTES
 * column c, the byte area of its cells per region, 1 <= byte_cap[c] < 2^32.  Every argument is checked before anything is
 * enqueued: a refused push writes no region and publishes no slot.  A failure after the checks publishes that status in
 * every slot, so every receiver refuses the step.  Both are enqueued on the push stream; tq_partition_push_sync(slot)
 * waits for them.
 * tq_partition_push_sample: the splitter sample.  m = min(n, n_samples) rows (1 <= n_samples <= 65536), row j taken at a
 *   hashed position of (seed, src_rank, j) inside the stratum [j n / m, (j + 1) n / m) — distinct rows, and no aliasing
 *   with a periodic input.  Their ByItem columns and their tie word (UINT64) are broadcast to the n_parts destinations in
 *   tq_partition_push_broadcast's wire format with n_by + 1 columns (the nullable flag, byte_cap of each BYTES ByItem
 *   column); m <= region_cap.  Each received sample region is a device chunk for tq_sort_put (TQ_MEM_DEVICE).
 * tq_partition_push_ranges: the rows.  split_cols = the sorted sample's n_by + 1 device columns (ByItems, then the tie
 *   word), split_rows its rows, split_pos the n_parts - 1 non-decreasing splitter rows; row r goes to the number of
 *   splitters at or below it, comparing the sort's own key words most significant first (per ByItem the NULL flag, then the
 *   value word or the 8-byte big-endian chunks and the length of a string, each inverted when Desc; the tie word last).
 *   n_parts == 1 or split_rows == 0 reads no splitter and sends every row to destination 0.  The rows go out in the GROUP BY
 *   push's wire format, in input order per destination: dest_data[q * (n_cols + 1 + n_bytes) + a] = n_cols word areas (a
 *   BYTES column's is its region_cap + 1 offsets from 0), the mask word, then the byte area of each BYTES column in column
 *   order.  n <= region_cap, so no region overflows on rows; a byte area past its cap makes every slot read ~0.  The
 *   receiver is tq_sort_put_regions. */
int32_t tq_partition_push_sample(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                                 int32_t nullable, int32_t src_rank, int32_t n_samples, uint64_t seed, int32_t n_parts, void *const *dest_data,
                                 void *const *dest_counts, int64_t region_cap, const int64_t *byte_cap, int32_t slot, uint64_t epoch);
int32_t tq_partition_push_ranges(int32_t n_cols, const tq_column *cols, const int32_t *types, int64_t n, int32_t n_by, const int32_t *by_cols,
                                 const int32_t *by_desc, int32_t src_rank, int32_t n_parts, const tq_column *split_cols, int64_t split_rows,
                                 const int64_t *split_pos, void *const *dest_data, void *const *dest_counts, int64_t region_cap,
                                 const int64_t *byte_cap, int32_t slot, uint64_t epoch);
int32_t tq_partition_push_sync(int32_t slot);
/* Enqueues, on the compute stream, a kernel that waits (bounded) until the n_sources consecutive slots at `slots` (this rank's
 * own table) carry `epoch` — the device-side barrier between the peers' pushes and the kernels that read the regions; no host
 * synchronisation, no NCCL call on the data path. */
int32_t tq_region_wait(const void *slots, int32_t n_sources, uint64_t epoch);
/* Receives n_regions (1..8) regions into one set of contiguous DEVICE columns, on the compute stream (queue tq_region_wait
 * first).  slots: the n_regions consecutive published {u64 rows, u64 epoch} slots, read on the device; regions[g * n_wire + c]
 * = wire column c of region g (n_wire = n_cols + has_mask; the mask word, when has_mask, is the last).  out_cols[c].data
 * holds out_cap rows; out_cols[c].null_bitmap, when not NULL, is a device bitmap for out_cap rows and receives the mask's bit
 * c (whole 64-row groups, bits past the last row 0), or all ones without a mask.  Rows keep region order.  Returns the rows in
 * *n_rows and every out_cols[c].length (one host read).  A slot reading more than region_cap (~0: an overflowed push) is
 * TQ_ERR_OOM, more rows than out_cap TQ_ERR_INVALID_ARG; either way nothing is written to the outputs. */
int32_t tq_region_gather(int32_t n_regions, const void *slots, int64_t region_cap, int32_t n_cols, int32_t has_mask, const tq_column *regions,
                         tq_column *out_cols, int64_t out_cap, int64_t *n_rows);

#ifdef __cplusplus
}
#endif
#endif /* TINYSQL_B200_H */
