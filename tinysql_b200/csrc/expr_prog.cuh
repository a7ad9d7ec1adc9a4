// expr_prog.cuh — the builtin functors of the vectorized expressions and the one interpreter of the tq_expr_op register
// program, shared by the fused Selection + Projection (expr.cu: k_expr_prog) and the OtherConditions of the hash join
// (othercond.cu) and the merge join (sort.cu).  Plain CUDA C++ without inline PTX: tests/emu compiles sort.cu with g++, so the
// few CUDA intrinsics used here go through helpers that fall back to standard C++ outside a device compilation pass.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>

#include "common.cuh"

namespace tq {

enum : unsigned { ERR_BIGINT = 1u, ERR_UBIGINT = 2u, ERR_DOUBLE = 4u };

static constexpr int XP_MAX_IN = TQ_EXPR_MAX_INPUTS;
static constexpr int XP_MAX_OPS = TQ_EXPR_MAX_OPS;
static constexpr int XP_MAX_OUT = TQ_EXPR_MAX_OUTPUTS;
static constexpr int XP_REGS = XP_MAX_IN + XP_MAX_OPS;

// one decoded tq_expr_op
struct XOp {
  int8_t kind, op, a, b, c, flags;   // flags: 1 a_unsigned, 2 b_unsigned, 4 constant is NULL
  uint64_t imm;
};

// The first overflow error of the bits an evaluation raised, in the order the reference's checks would name them.
static inline int32_t err_to_status(unsigned e, const char *what) {
  if (e & ERR_UBIGINT) { set_error("BIGINT UNSIGNED value is out of range in '%s'", what); return TQ_ERR_OVERFLOW_BIGINT_UNSIGNED; }
  if (e & ERR_BIGINT) { set_error("BIGINT value is out of range in '%s'", what); return TQ_ERR_OVERFLOW_BIGINT; }
  if (e & ERR_DOUBLE) { set_error("DOUBLE value is out of range in '%s'", what); return TQ_ERR_OVERFLOW_DOUBLE; }
  return TQ_OK;
}

// Checks a tq_expr_op program over n_inputs input registers and decodes it into out[0, n_ops).  *want_counter: the program
// has a real arithmetic op, which may count division-by-zero warnings.
static inline int32_t xp_decode(int32_t n_inputs, int32_t n_ops, const tq_expr_op *ops, XOp *out, bool *want_counter) {
  *want_counter = false;
  for (int i = 0; i < n_ops; i++) {
    const tq_expr_op &s = ops[i];
    const int avail = n_inputs + i;   // an op reads inputs and earlier results only
    int arity = 2, lo = 0, hi = 0;
    switch (s.kind) {
      case TQ_X_CONST: arity = 0; break;
      case TQ_X_CMP_INT: case TQ_X_CMP_REAL: lo = TQ_CMP_LT; hi = TQ_CMP_NE; break;
      case TQ_X_ARITH_INT: lo = TQ_ARITH_PLUS; hi = TQ_ARITH_MUL; break;
      case TQ_X_ARITH_REAL: lo = TQ_ARITH_PLUS; hi = TQ_ARITH_DIV; *want_counter = true; break;
      case TQ_X_LOGIC: lo = TQ_LOGIC_AND; hi = TQ_LOGIC_OR; break;
      case TQ_X_UNARY: arity = 1; lo = TQ_UNARY_NOT_INT; hi = TQ_UNARY_ISNULL; break;
      case TQ_X_IF: arity = 3; break;
      case TQ_X_IFNULL: break;
      case TQ_X_FILTER: arity = 1; lo = 0; hi = 1; break;
      case TQ_X_COMPACT: arity = 0; break;
      default: set_error("expression program: op %d has unknown kind %d", i, s.kind); return TQ_ERR_INVALID_ARG;
    }
    if (s.op < lo || s.op > hi) { set_error("expression program: op %d (kind %d) has bad operator %d", i, s.kind, s.op); return TQ_ERR_INVALID_ARG; }
    const int regs[3] = {s.a, s.b, s.c};
    for (int k = 0; k < arity; k++)
      if (regs[k] < 0 || regs[k] >= avail) { set_error("expression program: op %d reads register %d before it is written", i, regs[k]); return TQ_ERR_INVALID_ARG; }
    XOp &x = out[i];
    x.kind = (int8_t)s.kind; x.op = (int8_t)s.op;
    x.a = (int8_t)(arity > 0 ? s.a : 0); x.b = (int8_t)(arity > 1 ? s.b : 0); x.c = (int8_t)(arity > 2 ? s.c : 0);
    x.flags = (int8_t)((s.a_unsigned ? 1 : 0) | (s.b_unsigned ? 2 : 0) | (s.is_null ? 4 : 0));
    x.imm = s.imm;
  }
  return TQ_OK;
}

// ------------------------------------------------------------------ intrinsics with a host fallback
__device__ __forceinline__ uint64_t xp_umulhi(uint64_t a, uint64_t b) {   // high 64 bits of the unsigned product
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
__device__ __forceinline__ int64_t xp_mulhi(int64_t a, int64_t b) {       // high 64 bits of the signed product
#ifdef __CUDA_ARCH__
  return __mul64hi(a, b);
#else
  return (int64_t)(((__int128)a * b) >> 64);
#endif
}
__device__ __forceinline__ bool xp_isinf(double x) {
#ifdef __CUDA_ARCH__
  return isinf(x);
#else
  return std::isinf(x);
#endif
}

// ------------------------------------------------------------------ functors
__device__ __forceinline__ int cmp_int_dev(bool ua, bool ub, int64_t x, int64_t y) {
  // types.VecCompare{UU,II,UI,IU}  types/compare.go:44-100
  if (ua && ub) { uint64_t a = (uint64_t)x, b = (uint64_t)y; return a < b ? -1 : (a == b ? 0 : 1); }
  if (!ua && !ub) return x < y ? -1 : (x == y ? 0 : 1);
  if (ua) { if (y < 0 || x < 0) return 1; return x < y ? -1 : (x == y ? 0 : 1); }   // x<0 <=> uint64(x) > MaxInt64
  if (x < 0 || y < 0) return -1;
  return x < y ? -1 : (x == y ? 0 : 1);
}
__device__ __forceinline__ uint64_t cmp_res_dev(int op, int c) {
  // vecResOf{LT,LE,GT,GE,EQ,NE}  expression/builtin_compare_vec.go:214-279
  switch (op) {
    case TQ_CMP_LT: return c < 0;
    case TQ_CMP_LE: return c <= 0;
    case TQ_CMP_GT: return c > 0;
    case TQ_CMP_GE: return c >= 0;
    case TQ_CMP_EQ: return c == 0;
    default: return c != 0;
  }
}

struct FCompareInt {
  int op; bool ua, ub;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &, unsigned &, bool) const {
    o[0] = cmp_res_dev(op, cmp_int_dev(ua, ub, (int64_t)v[0], (int64_t)v[1]));
    onn[0] = nn[0] && nn[1];  // result.MergeNulls(buf0, buf1)
  }
};
struct FCompareReal {
  int op;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &, unsigned &, bool) const {
    onn[0] = nn[0] && nn[1];
    const double x = __longlong_as_double((long long)v[0]), y = __longlong_as_double((long long)v[1]);
    const int c = x < y ? -1 : (x == y ? 0 : 1);  // types.CompareFloat64
    o[0] = onn[0] ? cmp_res_dev(op, c) : 0;
  }
};

// signed overflow predicates written on unsigned words (no UB, no 64-bit division)
__device__ __forceinline__ bool add_overflows_ss(int64_t a, int64_t b) {
  // (lh > 0 && rh > MaxInt64-lh) || (lh < 0 && rh < MinInt64-lh)  builtin_arithmetic_vec.go:488
  const int64_t s = (int64_t)((uint64_t)a + (uint64_t)b);
  return ((a ^ s) & (b ^ s)) < 0;
}
__device__ __forceinline__ int64_t wneg(int64_t x) { return (int64_t)(0ull - (uint64_t)x); }  // Go's wrapping -x

struct FArithInt {
  int op; bool ua, ub;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &err, unsigned &, bool) const {
    onn[0] = nn[0] && nn[1];
    o[0] = 0;
    if (!onn[0]) return;  // `if result.IsNull(i) { continue }`
    const int64_t lh = (int64_t)v[0], rh = (int64_t)v[1];
    const uint64_t ul = v[0], ur = v[1];
    if (op == TQ_ARITH_PLUS) {
      if (ua && ub) { if (ul > ~0ull - ur) err |= ERR_UBIGINT; }                                        // plusUU :437
      else if (ua && !ub) {                                                                              // plusUS :448-459 (verbatim, lh twice)
        if (rh < 0 && (uint64_t)wneg(rh) > ul) err |= ERR_UBIGINT;
        if (rh > 0 && ul > ~0ull - ul) err |= ERR_UBIGINT;
      } else if (!ua && ub) {                                                                            // plusSU :464-476
        if (lh < 0 && (uint64_t)wneg(lh) > ur) err |= ERR_UBIGINT;
        if (lh > 0 && ur > ~0ull - ul) err |= ERR_UBIGINT;
      } else if (add_overflows_ss(lh, rh)) err |= ERR_BIGINT;                                            // plusSS :488
      o[0] = ul + ur;
    } else if (op == TQ_ARITH_MINUS) {
      if (ua && ub) { if (ul < ur) err |= ERR_UBIGINT; }                                                 // minusUU :208
      else if (ua && !ub) {                                                                              // minusUS :224-229
        if (rh >= 0 && ul < ur) err |= ERR_UBIGINT;
        if (rh < 0 && ul > ~0ull - (uint64_t)wneg(rh)) err |= ERR_UBIGINT;
      } else if (!ua && ub) {                                                                            // minusSU :245
        if ((ul - 0x8000000000000000ull) < ur) err |= ERR_UBIGINT;
      } else {                                                                                           // minusSS :260 (verbatim, with Go's wrapping -rh)
        const int64_t nr = wneg(rh);
        const int64_t max_minus = (int64_t)(0x7fffffffffffffffull - ul);
        const int64_t min_minus = (int64_t)(0x8000000000000000ull - ul);
        if ((lh > 0 && nr > max_minus) || (lh < 0 && nr < min_minus)) err |= ERR_BIGINT;
      }
      o[0] = ul - ur;
    } else {
      const uint64_t lo = ul * ur;
      if (ua || ub) {                                                                                    // MultiplyIntUnsigned :521-529 (either side unsigned: builtin_arithmetic.go:344-348)
        if (xp_umulhi(ul, ur) != 0) err |= ERR_UBIGINT;
      } else {                                                                                           // MultiplyInt :332-338
        // `x != 0 && tmp/x != y` with Go's wrapping quotient: a true overflow is missed exactly when
        // x == -1 and y == MinInt64 (tmp == MinInt64, MinInt64 / -1 wraps back to MinInt64 == y).
        const int64_t hi = xp_mulhi(lh, rh);
        const bool true_ovf = hi != ((int64_t)lo >> 63);
        if (true_ovf && !(lh == -1 && ur == 0x8000000000000000ull)) err |= ERR_BIGINT;
      }
      o[0] = lo;
    }
  }
};

struct FArithReal {
  int op;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &err, unsigned &cnt, bool) const {
    onn[0] = nn[0] && nn[1];
    o[0] = 0;
    if (!onn[0]) return;
    const double x = __longlong_as_double((long long)v[0]), y = __longlong_as_double((long long)v[1]);
    double r = 0;
    switch (op) {
      case TQ_ARITH_PLUS:                                                                 // builtin_arithmetic_vec.go:302-305
        if ((x > 0 && y > DBL_MAX - x) || (x < 0 && y < -DBL_MAX - x)) err |= ERR_DOUBLE;
        r = x + y; break;
      case TQ_ARITH_MINUS:                                                                // :80-83
        if ((x > 0 && -y > DBL_MAX - x) || (x < 0 && -y < -DBL_MAX - x)) err |= ERR_DOUBLE;
        r = x - y; break;
      case TQ_ARITH_MUL:                                                                  // :49-52
        r = x * y; if (xp_isinf(r)) err |= ERR_DOUBLE; break;
      default:                                                                            // :368-381
        if (y == 0) { cnt++; onn[0] = false; r = 0; }
        else { r = x / y; if (xp_isinf(r)) err |= ERR_DOUBLE; }
        break;
    }
    o[0] = (uint64_t)__double_as_longlong(r);
  }
};

struct FLogic {
  int op;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &, unsigned &, bool) const {
    const bool n0 = !nn[0], n1 = !nn[1];
    if (op == TQ_LOGIC_AND) {                                      // builtin_op_vec.go:192-211
      if ((!n0 && v[0] == 0) || (!n1 && v[1] == 0)) { o[0] = 0; onn[0] = true; }
      else if (n0 || n1) { o[0] = 0; onn[0] = false; }
      else { o[0] = 1; onn[0] = true; }
    } else {                                                       // builtin_op_vec.go:46-66
      if ((!n0 && v[0] != 0) || (!n1 && v[1] != 0)) { o[0] = 1; onn[0] = true; }
      else if (n0 || n1) { o[0] = 0; onn[0] = false; }
      else { o[0] = 0; onn[0] = true; }
    }
  }
};

struct FUnary {
  int op; bool ua;
  __device__ __forceinline__ void operator()(const uint64_t (&v)[1], const bool (&nn)[1], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &err, unsigned &, bool active) const {
    onn[0] = nn[0];
    o[0] = 0;
    switch (op) {
      case TQ_UNARY_NOT_INT: if (nn[0]) o[0] = (v[0] == 0); break;                                   // builtin_op_vec.go:255-265
      case TQ_UNARY_NOT_REAL: if (nn[0]) o[0] = (__longlong_as_double((long long)v[0]) == 0.0); break; // :152-165
      case TQ_UNARY_MINUS_INT:                                                                        // :221-243
        if (nn[0]) {
          if (ua) { if (v[0] > 0x8000000000000000ull) err |= ERR_BIGINT; }
          else if (v[0] == 0x8000000000000000ull) err |= ERR_BIGINT;
          o[0] = 0ull - v[0];
        }
        break;
      case TQ_UNARY_MINUS_REAL: if (nn[0]) o[0] = v[0] ^ 0x8000000000000000ull; break;               // :74-86 (-x flips the sign bit)
      default: o[0] = nn[0] ? 0 : 1; onn[0] = active; break;                                          // IsNull :98-106 — never NULL
    }
  }
};

struct FIf {
  __device__ __forceinline__ void operator()(const uint64_t (&v)[3], const bool (&nn)[3], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &, unsigned &, bool) const {
    const bool take_b = !nn[0] || v[0] == 0;                       // builtin_control_vec_generated.go:141-156
    onn[0] = take_b ? nn[2] : nn[1];
    o[0] = onn[0] ? (take_b ? v[2] : v[1]) : 0;
  }
};
struct FIfNull {
  __device__ __forceinline__ void operator()(const uint64_t (&v)[2], const bool (&nn)[2], uint64_t (&o)[1], bool (&onn)[1],
                                             unsigned &, unsigned &, bool) const {
    onn[0] = nn[0] || nn[1];                                       // builtin_control_vec_generated.go:38-45
    o[0] = nn[0] ? v[0] : (nn[1] ? v[1] : 0);
  }
};

// ------------------------------------------------------------------ the program over one row
// Runs ops[0, n_ops) over one row's register file: rv[k] / bit k of nn (NOT NULL) hold input k < n_in on entry, op i writes
// register n_in + i.  VecEvalBool's narrowing (expression.go:231-268):
//   alive — the row is still in the evaluation set (sel slice): errors and warnings of later ops count for it;
//   sel   — the row passes every FILTER item seen so far.
// Both start as `active`.  An ETInt NULL item leaves the row alive but not selected (the nulls[] quirk); TQ_X_COMPACT (the
// Selection -> Projection boundary) keeps only selected rows alive.  err collects ERR_* bits, cnt division-by-zero warnings.
template <int NREGS>
__device__ __forceinline__ void xp_run_row(const XOp *ops, int n_ops, int n_in, uint64_t (&rv)[NREGS], uint64_t &nn, bool active, bool &alive,
                                           bool &sel, unsigned &err, unsigned &cnt) {
  alive = active;
  sel = active;
  for (int i = 0; i < n_ops; i++) {
    const XOp x = ops[i];
    const uint64_t v2[2] = {rv[x.a], rv[x.b]};
    const bool n2[2] = {(bool)((nn >> x.a) & 1), (bool)((nn >> x.b) & 1)};
    uint64_t o1[1] = {0};
    bool on[1] = {true};
    unsigned e_ = 0, c_ = 0;
    switch (x.kind) {
      case TQ_X_CONST: o1[0] = x.imm; on[0] = !(x.flags & 4); break;
      case TQ_X_CMP_INT: FCompareInt{x.op, (bool)(x.flags & 1), (bool)(x.flags & 2)}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_CMP_REAL: FCompareReal{x.op}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_ARITH_INT: FArithInt{x.op, (bool)(x.flags & 1), (bool)(x.flags & 2)}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_ARITH_REAL: FArithReal{x.op}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_LOGIC: FLogic{x.op}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_UNARY: {
        const uint64_t v1[1] = {v2[0]};
        const bool n1[1] = {n2[0]};
        FUnary{x.op, (bool)(x.flags & 1)}(v1, n1, o1, on, e_, c_, active);
        break;
      }
      case TQ_X_IF: {
        const uint64_t v3[3] = {v2[0], v2[1], rv[x.c]};
        const bool n3[3] = {n2[0], n2[1], (bool)((nn >> x.c) & 1)};
        FIf{}(v3, n3, o1, on, e_, c_, active);
        break;
      }
      case TQ_X_IFNULL: FIfNull{}(v2, n2, o1, on, e_, c_, active); break;
      case TQ_X_FILTER: {                                          // VecEvalBool expression.go:231-268
        const bool isnull = !n2[0];
        const bool zero = x.op ? (fabs(__longlong_as_double((long long)v2[0])) < 0.5) : (v2[0] == 0);
        if (isnull) { sel = false; if (x.op) alive = false; }       // ETInt NULL stays in sel, flagged in nulls[]
        else if (zero) { sel = false; alive = false; }
        break;
      }
      default: alive = sel; break;                                 // TQ_X_COMPACT: Selection hands only selected rows on
    }
    if (alive) { err |= e_; cnt += c_; }
    rv[n_in + i] = o1[0];
    nn = (nn & ~(1ull << (n_in + i))) | ((uint64_t)on[0] << (n_in + i));
  }
}

// ------------------------------------------------------------------ OtherConditions of the joins
// A join's conditions as a program over the joined row: input register k is joined-row column in_col[k].  The comparison
// form (tq_join_cond) lowers to at most two inputs per condition, so a join program holds twice the inputs of tq_expr_eval.
static constexpr int JP_MAX_IN = 2 * TQ_EXPR_MAX_INPUTS;
static constexpr int JP_REGS = JP_MAX_IN + XP_MAX_OPS;
static_assert(JP_REGS <= 64, "the NOT-NULL bits of the register file are one 64-bit word");
static constexpr int JP_MAX_CONDS = 8;   // tq_join_cond entries per handle

struct JoinProg {
  int n_in = 0, n_ops = 0;
  bool want_counter = false;
  int in_col[JP_MAX_IN] = {};   // joined-row column (left ++ right) of each input register
  XOp ops[XP_MAX_OPS] = {};
};

// tq_*_set_other_program: checks the program and the types of its input columns (type_of(c) = TQ_TYPE_* of joined-row
// column c, n_cols of them).  FILTER at least once, no COMPACT, the limits of tq_expr_eval.
template <typename TypeOf>
static inline int32_t join_prog_from_ops(int32_t n_inputs, const int32_t *input_cols, int32_t n_ops, const tq_expr_op *ops, int n_cols, TypeOf type_of,
                                         JoinProg *P) {
  if (n_inputs < 0 || n_inputs > XP_MAX_IN || n_ops <= 0 || n_ops > XP_MAX_OPS || (n_inputs && !input_cols) || !ops) {
    set_error("OtherConditions program: 0..%d inputs and 1..%d ops", XP_MAX_IN, XP_MAX_OPS);
    return TQ_ERR_INVALID_ARG;
  }
  bool has_filter = false;
  for (int i = 0; i < n_ops; i++) {
    if (ops[i].kind == TQ_X_COMPACT) { set_error("OtherConditions program: op %d is TQ_X_COMPACT (there is no projection)", i); return TQ_ERR_INVALID_ARG; }
    has_filter |= ops[i].kind == TQ_X_FILTER;
  }
  if (!has_filter) { set_error("OtherConditions program: no TQ_X_FILTER item"); return TQ_ERR_INVALID_ARG; }
  for (int k = 0; k < n_inputs; k++)
    if (input_cols[k] < 0 || input_cols[k] >= n_cols) { set_error("OtherConditions program: input %d names column %d", k, input_cols[k]); return TQ_ERR_INVALID_ARG; }
  JoinProg p;
  TQ_TRY(xp_decode(n_inputs, n_ops, ops, p.ops, &p.want_counter));
  for (int k = 0; k < n_inputs; k++) {
    const int t = type_of(input_cols[k]);
    if (t != TQ_TYPE_INT64 && t != TQ_TYPE_UINT64 && t != TQ_TYPE_FLOAT64) {
      set_error("OtherConditions program: input %d (column %d) is not a BIGINT / BIGINT UNSIGNED / DOUBLE column", k, input_cols[k]);
      return TQ_ERR_UNSUPPORTED_TYPE;
    }
    p.in_col[k] = input_cols[k];
  }
  p.n_in = n_inputs;
  p.n_ops = n_ops;
  *P = p;
  return TQ_OK;
}

// The comparison form as a program: per condition CMP_INT (with the operands' unsigned flags) or CMP_REAL, CONST for the
// constant, then one ETInt FILTER.  A NULL operand makes the comparison NULL, which the FILTER does not select: the row fails,
// as VectorizedFilter has it.  Comparisons raise no errors.  The caller has checked the conditions and their types.
template <typename TypeOf>
static inline void join_prog_from_conds(int32_t n_conds, const tq_join_cond *conds, TypeOf type_of, JoinProg *P) {
  JoinProg p;
  auto input = [&](int col) {
    for (int k = 0; k < p.n_in; k++)
      if (p.in_col[k] == col) return k;
    p.in_col[p.n_in] = col;
    return p.n_in++;
  };
  int regs[JP_MAX_CONDS][2];
  for (int k = 0; k < n_conds; k++) {   // inputs first: registers n_in + i are the results of the ops
    regs[k][0] = input(conds[k].lhs_col);
    regs[k][1] = conds[k].rhs_col >= 0 ? input(conds[k].rhs_col) : -1;
  }
  auto emit = [&](int kind, int op, int a, int b, int flags, uint64_t imm) {
    XOp &x = p.ops[p.n_ops];
    x.kind = (int8_t)kind; x.op = (int8_t)op; x.a = (int8_t)a; x.b = (int8_t)b; x.c = 0; x.flags = (int8_t)flags; x.imm = imm;
    return p.n_in + p.n_ops++;
  };
  for (int k = 0; k < n_conds; k++) {
    const tq_join_cond &q = conds[k];
    const int ta = type_of(q.lhs_col), tb = q.rhs_col >= 0 ? type_of(q.rhs_col) : (q.const_type & 0xFF);
    const int b = regs[k][1] >= 0 ? regs[k][1] : emit(TQ_X_CONST, 0, 0, 0, 0, q.const_bits);
    const int flags = (ta == TQ_TYPE_UINT64 ? 1 : 0) | (tb == TQ_TYPE_UINT64 ? 2 : 0);
    const int c = emit(ta == TQ_TYPE_FLOAT64 ? TQ_X_CMP_REAL : TQ_X_CMP_INT, q.op, regs[k][0], b, flags, 0);
    emit(TQ_X_FILTER, 0, c, 0, 0, 0);
  }
  *P = p;
}

}  // namespace tq
