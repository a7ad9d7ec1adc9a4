// +build gpu

// Fused Selection + Projection on the device (SURVEY §8 f1): the expression trees of a SelectionExec's filters and of the
// ProjectionExec above it are lowered to ONE tq_expr_eval register program, so a chunk makes one trip through HBM instead of one
// per builtin (VectorizedFilter chunk_executor.go:196-245 → VecEvalBool expression.go:205-279; evalOneVec for projections).
//
// Only trees made of the fixed-width builtins the library implements lower (ETInt / ETReal compare, arithmetic, logic, NOT, unary
// minus, IS NULL, IF, IFNULL, IN, constants, columns); CompileProgram returns ok == false for anything else and the executor
// keeps the Go path for that operator — the same "capability check at plan time" the join and aggregate shims use.
package expression

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -ltinysql_b200
#include <stdlib.h>
#include "tinysql_b200.h"
*/
import "C"

import (
	"math"
	"unsafe"

	"github.com/pingcap/tidb/parser/ast"
	"github.com/pingcap/tidb/parser/mysql"
	"github.com/pingcap/tidb/types"
	"github.com/pingcap/tidb/util/chunk"
)

// GPUProgram is a compiled filter list + projection list.  The op array and the output-register array live in C memory
// (cgo pointer rules: nothing handed to C contains a Go pointer).
type GPUProgram struct {
	ops      *C.tq_expr_op
	nOps     int
	outRegs  *C.int32_t
	nOut     int
	inputs   []int // chunk column index of program input k
	hasSel   bool
	inViews  *chunk.CViewSet
	outViews *chunk.CViewSet
	selBuf   unsafe.Pointer // C bytes for `selected` (copied into the Go []bool after the call)
	selCap   int
}

type progBuilder struct {
	ops    []C.tq_expr_op
	inputs []int
	colReg map[int]int // chunk column index -> input register
	ok     bool
}

func evalKind(e Expression) (real, unsigned bool, ok bool) {
	tp := e.GetType()
	switch tp.EvalType() {
	case types.ETInt:
		return false, mysql.HasUnsignedFlag(tp.Flag), true
	case types.ETReal:
		return true, false, tp.Tp == mysql.TypeDouble // FLOAT columns are 4-byte slots: widen on the Go side first
	}
	return false, false, false
}

// emit appends op i and returns a TAGGED register (i + 2^20): the final number of an op result is nInputs + i, which is only
// known once every referenced column has been seen; CompileProgram patches the tags (inputs are plain small numbers).
func (b *progBuilder) emit(kind, op C.int32_t, a, bb, c int, ua, ub bool, isNull bool, imm uint64) int {
	var o C.tq_expr_op
	o.kind, o.op = kind, op
	o.a, o.b, o.c = C.int32_t(a), C.int32_t(bb), C.int32_t(c)
	o.a_unsigned, o.b_unsigned, o.is_null = cbool(ua), cbool(ub), cbool(isNull)
	o.imm = C.uint64_t(imm)
	b.ops = append(b.ops, o)
	return len(b.ops) - 1 + (1 << 20) // op results are tagged; inputs are plain small numbers
}

func (b *progBuilder) lower(e Expression) int {
	if !b.ok {
		return 0
	}
	switch x := e.(type) {
	case *Column:
		if _, _, ok := evalKind(x); !ok {
			b.ok = false
			return 0
		}
		if r, seen := b.colReg[x.Index]; seen {
			return r
		}
		r := len(b.inputs)
		b.inputs = append(b.inputs, x.Index)
		b.colReg[x.Index] = r
		return r
	case *Constant:
		real, _, ok := evalKind(x)
		if !ok {
			b.ok = false
			return 0
		}
		if x.Value.IsNull() {
			return b.emit(C.TQ_X_CONST, 0, 0, 0, 0, false, false, true, 0)
		}
		if real {
			return b.emit(C.TQ_X_CONST, 0, 0, 0, 0, false, false, false, math.Float64bits(x.Value.GetFloat64()))
		}
		return b.emit(C.TQ_X_CONST, 0, 0, 0, 0, false, false, false, uint64(x.Value.GetInt64())) // uint64 datums share the bits
	case *ScalarFunction:
		args := x.GetArgs()
		regs := make([]int, len(args))
		real, anyBad := false, false
		uns := make([]bool, len(args))
		for i, a := range args {
			r, u, ok := evalKind(a)
			anyBad = anyBad || !ok
			real = real || r
			uns[i] = u
		}
		if anyBad {
			b.ok = false
			return 0
		}
		name := x.FuncName.L
		if name == ast.In { // a IN (l0, l1, …) == (a = l0) OR (a = l1) OR … : the three-valued result of builtinIn{Int,Real}Sig
			a := b.lower(args[0])
			acc := -1
			for i := 1; i < len(args); i++ {
				kind := C.int32_t(C.TQ_X_CMP_INT)
				if real {
					kind = C.TQ_X_CMP_REAL
				}
				eq := b.emit(kind, C.TQ_CMP_EQ, a, b.lower(args[i]), 0, uns[0], uns[i], false, 0)
				if acc < 0 {
					acc = eq
				} else {
					acc = b.emit(C.TQ_X_LOGIC, C.TQ_LOGIC_OR, acc, eq, 0, false, false, false, 0)
				}
			}
			return acc
		}
		for i, a := range args {
			regs[i] = b.lower(a)
		}
		cmp := map[string]C.int32_t{ast.LT: C.TQ_CMP_LT, ast.LE: C.TQ_CMP_LE, ast.GT: C.TQ_CMP_GT, ast.GE: C.TQ_CMP_GE, ast.EQ: C.TQ_CMP_EQ, ast.NE: C.TQ_CMP_NE}
		arith := map[string]C.int32_t{ast.Plus: C.TQ_ARITH_PLUS, ast.Minus: C.TQ_ARITH_MINUS, ast.Mul: C.TQ_ARITH_MUL}
		cmpOp, isCmp := cmp[name]
		arithOp, isArith := arith[name]
		switch {
		case isCmp && len(args) == 2:
			kind := C.int32_t(C.TQ_X_CMP_INT)
			if real {
				kind = C.TQ_X_CMP_REAL
			}
			return b.emit(kind, cmpOp, regs[0], regs[1], 0, uns[0], uns[1], false, 0)
		case isArith && len(args) == 2:
			kind := C.int32_t(C.TQ_X_ARITH_INT)
			if real {
				kind = C.TQ_X_ARITH_REAL
			}
			return b.emit(kind, arithOp, regs[0], regs[1], 0, uns[0], uns[1], false, 0)
		case name == ast.Div && real: // builtinArithmeticDivideRealSig; integer '/' is decimal division: not lowered
			return b.emit(C.TQ_X_ARITH_REAL, C.TQ_ARITH_DIV, regs[0], regs[1], 0, false, false, false, 0)
		case name == ast.LogicAnd:
			return b.emit(C.TQ_X_LOGIC, C.TQ_LOGIC_AND, regs[0], regs[1], 0, false, false, false, 0)
		case name == ast.LogicOr:
			return b.emit(C.TQ_X_LOGIC, C.TQ_LOGIC_OR, regs[0], regs[1], 0, false, false, false, 0)
		case name == ast.UnaryNot:
			op := C.int32_t(C.TQ_UNARY_NOT_INT)
			if real {
				op = C.TQ_UNARY_NOT_REAL
			}
			return b.emit(C.TQ_X_UNARY, op, regs[0], 0, 0, false, false, false, 0)
		case name == ast.UnaryMinus:
			op := C.int32_t(C.TQ_UNARY_MINUS_INT)
			if real {
				op = C.TQ_UNARY_MINUS_REAL
			}
			return b.emit(C.TQ_X_UNARY, op, regs[0], 0, 0, uns[0], false, false, 0)
		case name == ast.IsNull:
			return b.emit(C.TQ_X_UNARY, C.TQ_UNARY_ISNULL, regs[0], 0, 0, false, false, false, 0)
		case name == ast.If:
			return b.emit(C.TQ_X_IF, 0, regs[0], regs[1], regs[2], false, false, false, 0)
		case name == ast.Ifnull:
			return b.emit(C.TQ_X_IFNULL, 0, regs[0], regs[1], 0, false, false, false, 0)
		}
	}
	b.ok = false
	return 0
}

// CompileProgram lowers `filters` (a CNF list) and `projections`; ok == false: keep the Go operators.
func CompileProgram(filters CNFExprs, projections []Expression) (p *GPUProgram, ok bool) {
	b := &progBuilder{colReg: map[int]int{}, ok: true}
	outTagged := make([]int, 0, len(projections))
	for _, f := range filters {
		r := b.lower(f)
		real, _, _ := evalKind(f)
		op := C.int32_t(0)
		if real {
			op = 1
		}
		b.emit(C.TQ_X_FILTER, op, r, 0, 0, false, false, false, 0)
	}
	if len(filters) > 0 && len(projections) > 0 {
		b.emit(C.TQ_X_COMPACT, 0, 0, 0, 0, false, false, false, 0)
	}
	for _, e := range projections {
		outTagged = append(outTagged, b.lower(e))
	}
	if !b.ok || len(b.inputs) > C.TQ_EXPR_MAX_INPUTS || len(b.ops) > C.TQ_EXPR_MAX_OPS || len(outTagged) > C.TQ_EXPR_MAX_OUTPUTS {
		return nil, false
	}
	// final register numbers: inputs 0..nIn-1, op i -> nIn + i
	nIn := len(b.inputs)
	fix := func(r int) C.int32_t {
		if r >= 1<<20 {
			return C.int32_t(r - (1 << 20) + nIn)
		}
		return C.int32_t(r)
	}
	p = &GPUProgram{nOps: len(b.ops), nOut: len(outTagged), inputs: b.inputs, hasSel: len(filters) > 0}
	p.ops = (*C.tq_expr_op)(C.calloc(C.size_t(len(b.ops)+1), C.size_t(unsafe.Sizeof(C.tq_expr_op{}))))
	dst := (*[1 << 16]C.tq_expr_op)(unsafe.Pointer(p.ops))
	for i, o := range b.ops {
		o.a, o.b, o.c = fix(int(o.a)), fix(int(o.b)), fix(int(o.c))
		dst[i] = o
	}
	p.outRegs = (*C.int32_t)(C.calloc(C.size_t(len(outTagged)+1), 4))
	regs := (*[1 << 16]C.int32_t)(unsafe.Pointer(p.outRegs))
	for i, r := range outTagged {
		regs[i] = fix(r)
	}
	p.inViews, p.outViews = chunk.NewCViewSet(nIn+1), chunk.NewCViewSet(len(outTagged)+1)
	return p, true
}

// Run evaluates the program over one chunk: results[i] receives projection i for ALL input rows (the caller compacts with
// `selected`, exactly as SelectionExec does with the []bool VectorizedFilter returns, executor.go:482-497).
func (p *GPUProgram) Run(input *chunk.Chunk, results []*chunk.Column, selected []bool) ([]bool, int64, error) {
	n := input.NumRows()
	for k, idx := range p.inputs {
		p.inViews.Fill(k, input.Column(idx))
	}
	for i, c := range results {
		c.PrepareFixedResult(n, 8)
		p.outViews.FillResult(i, c)
	}
	var sel unsafe.Pointer
	if p.hasSel {
		if n > p.selCap {
			if p.selBuf != nil {
				C.free(p.selBuf)
			}
			p.selBuf, p.selCap = C.malloc(C.size_t(n+n/2+64)), n+n/2+64
		}
		sel = p.selBuf
	}
	var warnings C.int64_t
	st := C.tq_expr_eval(C.int64_t(n), C.int32_t(len(p.inputs)), p.inViews.Ptr(), C.int32_t(p.nOps), p.ops, C.int32_t(p.nOut), p.outRegs,
		p.outViews.Ptr(), (*C.uint8_t)(sel), &warnings, C.TQ_MEM_HOST)
	p.inViews.Release()
	p.outViews.Release()
	if err := statusToError(st, "expression program"); err != nil {
		return nil, 0, err
	}
	for i, c := range results {
		p.outViews.CopyBack(i, c, n)
		c.SetResultRows(n)
	}
	if p.hasSel {
		selected = selected[:0]
		bytes := (*[1 << 30]byte)(sel)[:n:n]
		for _, v := range bytes {
			selected = append(selected, v != 0)
		}
	}
	return selected, int64(warnings), nil // warnings: one handleDivisionByZeroError call each (builtin_arithmetic_vec.go:369-375)
}

// JoinArgs hands a filter-only program to tq_join_set_other_program / tq_mjoin_set_other_program: the column each input
// register reads (an index into the joined row left ++ right when the filters are a join's OtherConditions) and the op
// array in C memory (a *C.tq_expr_op of the caller's package; cgo types do not cross packages).
func (p *GPUProgram) JoinArgs() (inputs []int, ops unsafe.Pointer, nOps int) {
	return p.inputs, unsafe.Pointer(p.ops), p.nOps
}

// Free releases the C memory of the program.
func (p *GPUProgram) Free() {
	C.free(unsafe.Pointer(p.ops))
	C.free(unsafe.Pointer(p.outRegs))
	if p.selBuf != nil {
		C.free(p.selBuf)
	}
	p.inViews.Free()
	p.outViews.Free()
}
