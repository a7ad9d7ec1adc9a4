// +build gpu

// GPUHashJoinExec: HashJoinExec (executor/join.go:31-146) with the hash table, the join workers and the joiners replaced
// by libtinysql_b200.  executorBuilder.buildHashJoin (builder.go:431-484) returns newGPUHashJoin(...) instead of
// &HashJoinExec{...} — for every key type the reference hashes (integers, FLOAT, DOUBLE, var-len; codec.go:216-236), for
// inner / left outer / right outer joins, with PhysicalHashJoin.DefaultValues passed through as defaultInner.  There is no
// fallback to the Go executor: a plan the library cannot run fails with the library's error (north_star: no CPU
// fallback on the named operators).
package executor

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -ltinysql_b200
#include <stdlib.h>
#include "tinysql_b200.h"
*/
import "C"

import (
	"context"
	"errors"
	"math"
	"unsafe"

	"github.com/pingcap/tidb/expression"
	"github.com/pingcap/tidb/parser/mysql"
	plannercore "github.com/pingcap/tidb/planner/core"
	"github.com/pingcap/tidb/sessionctx"
	"github.com/pingcap/tidb/types"
	"github.com/pingcap/tidb/util/chunk"
)

// tqType maps a FieldType onto the C-ABI's column types (util/chunk/codec.go:171-181 getFixedLen decides the layout).
func tqType(ft *types.FieldType) C.int32_t {
	switch ft.Tp {
	case mysql.TypeFloat:
		return C.TQ_TYPE_FLOAT32
	case mysql.TypeDouble:
		return C.TQ_TYPE_FLOAT64
	case mysql.TypeTiny, mysql.TypeShort, mysql.TypeInt24, mysql.TypeLong, mysql.TypeLonglong, mysql.TypeYear:
		if mysql.HasUnsignedFlag(ft.Flag) {
			return C.TQ_TYPE_UINT64
		}
		return C.TQ_TYPE_INT64
	default:
		return C.TQ_TYPE_BYTES
	}
}

type GPUHashJoinExec struct {
	baseExecutor

	outerSideExec, innerSideExec Executor
	outerSideFilter              expression.CNFExprs
	outerKeys, innerKeys         []*expression.Column
	otherConditions              expression.CNFExprs // run inside the library (setOtherConditions); what is left: see Next
	defaultValues                []types.Datum       // PhysicalHashJoin.DefaultValues (builder.go:449)
	joinType                     plannercore.JoinType
	outerIsRight                 bool

	h         *C.tq_join
	innerChk  *chunk.Chunk
	outerChk  *chunk.Chunk
	selected  []bool
	selBytes  []byte
	outTypes  []C.int32_t
	inViews   *chunk.CViewSet // argument blocks in C memory (cgo pointer rules: see util/chunk/gpu_bridge.go)
	outViews  *chunk.CViewSet
	desc      *C.tq_join_desc // C.malloc'ed together with the arrays it points to
	sizes     *C.int64_t
	prepared  bool
	outerDone bool
	warned    int64 // division-by-zero warnings of the OtherConditions program already in the statement context
}

// cInt32s builds an int32 array in C memory (a tq_join_desc in C memory may only point at C memory).
func cInt32s(n int, f func(i int) C.int32_t) *C.int32_t {
	p := (*C.int32_t)(C.malloc(C.size_t(4 * (n + 1))))
	a := (*[1 << 20]C.int32_t)(unsafe.Pointer(p))[:n:n]
	for i := range a {
		a[i] = f(i)
	}
	return p
}

// Open implements Executor (join.go:110-123).
func (e *GPUHashJoinExec) Open(ctx context.Context) error {
	if err := e.baseExecutor.Open(ctx); err != nil {
		return err
	}
	innerTypes, outerTypes := retTypes(e.innerSideExec), retTypes(e.outerSideExec)
	nb, np, nk := len(innerTypes), len(outerTypes), len(e.innerKeys)
	d := (*C.tq_join_desc)(C.calloc(1, C.size_t(unsafe.Sizeof(C.tq_join_desc{}))))
	e.desc = d
	d.join_type = C.int32_t(e.joinType) // InnerJoin=0, LeftOuterJoin=1, RightOuterJoin=2 (logical_plans.go:52-57)
	if e.outerIsRight {
		d.outer_is_right = 1
	}
	d.n_build_cols, d.build_types = C.int32_t(nb), cInt32s(nb, func(i int) C.int32_t { return tqType(innerTypes[i]) })
	d.n_probe_cols, d.probe_types = C.int32_t(np), cInt32s(np, func(i int) C.int32_t { return tqType(outerTypes[i]) })
	// nk == 0 (a cross join, or an ON without an equality: everything is in OtherConditions) is a key-less join, which
	// runs on the device too; cInt32s(0, …) still allocates one slot, and the library does not read it.
	d.n_keys = C.int32_t(nk)
	d.build_key_idx = cInt32s(nk, func(i int) C.int32_t { return C.int32_t(e.innerKeys[i].Index) })
	d.probe_key_idx = cInt32s(nk, func(i int) C.int32_t { return C.int32_t(e.outerKeys[i].Index) })
	if e.joinType != plannercore.InnerJoin && len(e.defaultValues) > 0 {
		// defaultInner (joiner.go:139-143): non-NULL defaults exist for integer / DOUBLE inner columns (COUNT -> 0 ...)
		bits := (*[1 << 16]C.uint64_t)(C.calloc(C.size_t(nb), 8))[:nb:nb]
		nn := (*[1 << 16]C.uint8_t)(C.calloc(C.size_t(nb), 1))[:nb:nb]
		for i := 0; i < nb && i < len(e.defaultValues); i++ {
			if !e.defaultValues[i].IsNull() {
				bits[i], nn[i] = C.uint64_t(datumBits(&e.defaultValues[i], innerTypes[i])), 1
			}
		}
		d.default_inner_bits, d.default_inner_not_null = &bits[0], &nn[0]
	}
	if st := C.tq_join_create(d, &e.h); st != C.TQ_OK {
		return chunk.StatusError(int32(st))
	}
	// OtherConditions (joiner.go:155-167) run inside the library, for outer joins too (a probe row whose joined rows all fail
	// becomes a miss row): see setOtherConditions.  Only trees that do not lower (string operands, ...) are left; for an
	// INNER join Next evaluates them with the tq_vec_* builtins on the returned chunk, an OUTER join fails here — there is no
	// Go-executor fallback.
	rest, err := setOtherConditions(e.otherConditions, e.outerIsRight, np, nb,
		func(n C.int32_t, cc *C.tq_join_cond) C.int32_t { return C.tq_join_set_other_conditions(e.h, n, cc) },
		func(nIn C.int32_t, in *C.int32_t, nOps C.int32_t, ops *C.tq_expr_op) C.int32_t {
			return C.tq_join_set_other_program(e.h, nIn, in, nOps, ops)
		})
	if err != nil {
		return err
	}
	e.otherConditions = rest
	if len(e.otherConditions) > 0 && e.joinType != plannercore.InnerJoin {
		return errors.New("tinysql_b200: this OtherCondition of an outer hash join is not supported on the device path")
	}
	// output = lhs ++ rhs (joiner.go:145-150)
	e.outTypes = e.outTypes[:0]
	lhs, rhs := outerTypes, innerTypes
	if e.outerIsRight {
		lhs, rhs = innerTypes, outerTypes
	}
	for _, ft := range append(append([]*types.FieldType{}, lhs...), rhs...) {
		e.outTypes = append(e.outTypes, tqType(ft))
	}
	e.inViews = chunk.NewCViewSet(maxInt(nb, np))
	e.outViews = chunk.NewCViewSet(len(e.outTypes))
	e.sizes = (*C.int64_t)(C.calloc(C.size_t(len(e.outTypes)), 8))
	e.innerChk, e.outerChk = newFirstChunk(e.innerSideExec), newFirstChunk(e.outerSideExec)
	e.prepared, e.outerDone, e.warned = false, false, 0
	return nil
}

// fetchAndBuildHashTable (join.go:148-158): drain the inner child into the device-side row container.
func (e *GPUHashJoinExec) build(ctx context.Context) error {
	for {
		if err := Next(ctx, e.innerSideExec, e.innerChk); err != nil {
			return err
		}
		if e.innerChk.NumRows() == 0 {
			break
		}
		e.inViews.FillChunk(e.innerChk)
		st := C.tq_join_put_build(e.h, e.inViews.Ptr(), C.TQ_MEM_HOST) // the library has copied the chunk when this returns
		e.inViews.Release()
		if st != C.TQ_OK {
			return chunk.StatusError(int32(st))
		}
	}
	if st := C.tq_join_finalize_build(e.h); st != C.TQ_OK {
		return chunk.StatusError(int32(st))
	}
	return nil
}

// Next implements Executor (join.go:125-146): fills req with <= req.RequiredRows() joined rows; 0 rows == EOF.
func (e *GPUHashJoinExec) Next(ctx context.Context, req *chunk.Chunk) error {
	req.Reset()
	if !e.prepared {
		if err := e.build(ctx); err != nil {
			return err
		}
		e.prepared = true
	}
	want := req.RequiredRows()
	sizes := (*[1 << 10]C.int64_t)(unsafe.Pointer(e.sizes))[:len(e.outTypes)]
	for {
		// size the result columns for this call (the *_next_size query of the ownership contract)
		if st := C.tq_join_next_bytes(e.h, C.int64_t(want), e.sizes); st != C.TQ_OK {
			return chunk.StatusError(int32(st))
		}
		for i := range e.outTypes {
			col := req.Column(i)
			switch e.outTypes[i] {
			case C.TQ_TYPE_BYTES:
				col.PrepareVarLenResult(want, int64(sizes[i]))
			case C.TQ_TYPE_FLOAT32:
				col.PrepareFixedResult(want, 4)
			default:
				col.PrepareFixedResult(want, 8)
			}
			e.outViews.FillResult(i, col)
		}
		var n C.int64_t
		var eof C.int32_t
		st := C.tq_join_next(e.h, C.int64_t(want), e.outViews.Ptr(), &n, &eof)
		e.outViews.Release()
		if st != C.TQ_OK {
			return chunk.StatusError(int32(st))
		}
		var warned C.int64_t
		C.tq_join_warnings(e.h, &warned)
		appendDivByZeroWarnings(e.ctx, int64(warned), &e.warned)
		if n > 0 || eof != 0 {
			for i := range e.outTypes {
				e.outViews.CopyBack(i, req.Column(i), int(n))
				req.Column(i).SetResultRows(int(n))
			}
			req.SetNumVirtualRows(int(n))
			if n > 0 && len(e.otherConditions) > 0 {
				// inner joins only (Open rejected the outer case): baseJoiner.filter (joiner.go:155-167) on the returned
				// chunk, the expressions themselves running through the tq_vec_* builtins (expression/gpu_builtin.go)
				var err error
				if e.selected, err = expression.VectorizedFilter(e.ctx, e.otherConditions, chunk.NewIterator4Chunk(req), e.selected); err != nil {
					return err
				}
				req.SetSel(selToIdx(e.selected))
				if req.NumRows() == 0 && eof == 0 {
					req.Reset()
					continue
				}
			}
			return nil
		}
		// fetchOuterSideChunks (join.go:194-221): feed one more outer chunk
		if e.outerDone {
			continue
		}
		if err := Next(ctx, e.outerSideExec, e.outerChk); err != nil {
			return err
		}
		if e.outerChk.NumRows() == 0 {
			e.outerDone = true
			C.tq_join_probe_eof(e.h)
			continue
		}
		var sel *C.uint8_t
		if len(e.outerSideFilter) > 0 { // join.go:328: rows the outer-side filter rejects are misses
			var err error
			if e.selected, err = expression.VectorizedFilter(e.ctx, e.outerSideFilter, chunk.NewIterator4Chunk(e.outerChk), e.selected); err != nil {
				return err
			}
			e.selBytes = e.selBytes[:0]
			for _, s := range e.selected {
				if s {
					e.selBytes = append(e.selBytes, 1)
				} else {
					e.selBytes = append(e.selBytes, 0)
				}
			}
			sel = (*C.uint8_t)(unsafe.Pointer(&e.selBytes[0])) // a []byte holds no Go pointers: legal as a direct argument
		}
		e.inViews.FillChunk(e.outerChk)
		st := C.tq_join_put_probe(e.h, e.inViews.Ptr(), sel, C.TQ_MEM_HOST)
		e.inViews.Release()
		if st != C.TQ_OK {
			return chunk.StatusError(int32(st))
		}
	}
}

func selToIdx(selected []bool) []int {
	idx := make([]int, 0, len(selected))
	for i, s := range selected {
		if s {
			idx = append(idx, i)
		}
	}
	return idx
}

// Close implements Executor (join.go:81-108); safe straight after Open and with rows still pending (`limit 1`).
func (e *GPUHashJoinExec) Close() error {
	if e.h != nil {
		C.tq_join_destroy(e.h)
		e.h = nil
	}
	if e.desc != nil {
		for _, p := range []unsafe.Pointer{unsafe.Pointer(e.desc.build_types), unsafe.Pointer(e.desc.probe_types), unsafe.Pointer(e.desc.build_key_idx),
			unsafe.Pointer(e.desc.probe_key_idx), unsafe.Pointer(e.desc.default_inner_bits), unsafe.Pointer(e.desc.default_inner_not_null), unsafe.Pointer(e.desc)} {
			C.free(p)
		}
		e.desc = nil
		e.inViews.Free()
		e.outViews.Free()
		C.free(unsafe.Pointer(e.sizes))
	}
	return e.baseExecutor.Close()
}

func maxInt(a, b int) int {
	if a > b {
		return a
	}
	return b
}

// datumBits: the 8-byte slot image of a default value (integers as they are, DOUBLE as its IEEE bits).
func datumBits(d *types.Datum, ft *types.FieldType) uint64 {
	if ft.Tp == mysql.TypeDouble {
		return math.Float64bits(d.GetFloat64())
	}
	return uint64(d.GetInt64())
}

// setOtherConditions hands a join's OtherConditions to the library and returns what it could not take.  A CNF made only of
// comparisons asJoinConds recognises goes to the comparison setter.  Otherwise, if CompileProgram lowers every item, the WHOLE
// CNF goes to the program setter (one form per handle).  Otherwise the comparisons go to the comparison setter and the rest is
// returned.  Column.Index of an OtherCondition is already an index into the joined row lhs ++ rhs, the program's input space.
func setOtherConditions(conds expression.CNFExprs, outerIsRight bool, nOuter, nInner int, setConds func(C.int32_t, *C.tq_join_cond) C.int32_t,
	setProgram func(C.int32_t, *C.int32_t, C.int32_t, *C.tq_expr_op) C.int32_t) (expression.CNFExprs, error) {
	if len(conds) == 0 {
		return nil, nil
	}
	cmps, rest, _ := asJoinConds(conds, outerIsRight, nOuter, nInner)
	if len(rest) > 0 {
		if prog, lowered := expression.CompileProgram(conds, nil); lowered {
			defer prog.Free()
			inputs, ops, nOps := prog.JoinArgs()
			in := cInt32s(len(inputs), func(i int) C.int32_t { return C.int32_t(inputs[i]) })
			defer C.free(unsafe.Pointer(in))
			if st := setProgram(C.int32_t(len(inputs)), in, C.int32_t(nOps), (*C.tq_expr_op)(ops)); st != C.TQ_OK {
				return nil, chunk.StatusError(int32(st))
			}
			return nil, nil
		}
	}
	if len(cmps) > 0 {
		cc := (*C.tq_join_cond)(C.malloc(C.size_t(len(cmps)) * C.size_t(unsafe.Sizeof(C.tq_join_cond{}))))
		defer C.free(unsafe.Pointer(cc))
		copy((*[1 << 10]C.tq_join_cond)(unsafe.Pointer(cc))[:len(cmps)], cmps)
		if st := setConds(C.int32_t(len(cmps)), cc); st != C.TQ_OK {
			return nil, chunk.StatusError(int32(st))
		}
	}
	return rest, nil
}

// appendDivByZeroWarnings adds the warnings a join's condition program raised since the last call to the statement context,
// one expression.ErrDivisionByZero each, as handleDivisionByZeroError does in a SELECT (expression/errors.go:65-77).
func appendDivByZeroWarnings(ctx sessionctx.Context, total int64, seen *int64) {
	sc := ctx.GetSessionVars().StmtCtx
	for ; *seen < total; *seen++ {
		sc.AppendWarning(expression.ErrDivisionByZero)
	}
}

// asJoinConds splits OtherConditions into the comparisons tq_join_set_other_conditions takes — `col op col` / `col op const`
// over the joined row lhs ++ rhs, BIGINT with BIGINT or DOUBLE with DOUBLE — and the rest.  ok is false when nothing qualifies.
func asJoinConds(conds expression.CNFExprs, outerIsRight bool, nOuter, nInner int) (out []C.tq_join_cond, rest expression.CNFExprs, ok bool) {
	ops := map[string]C.int32_t{"lt": C.TQ_CMP_LT, "le": C.TQ_CMP_LE, "gt": C.TQ_CMP_GT, "ge": C.TQ_CMP_GE, "eq": C.TQ_CMP_EQ, "ne": C.TQ_CMP_NE}
	for _, c := range conds {
		sf, isFn := c.(*expression.ScalarFunction)
		op, known := C.int32_t(0), false
		if isFn {
			op, known = ops[sf.FuncName.L]
		}
		if !known || len(sf.GetArgs()) != 2 {
			rest = append(rest, c)
			continue
		}
		l, lok := sf.GetArgs()[0].(*expression.Column)
		if !lok {
			rest = append(rest, c)
			continue
		}
		var jc C.tq_join_cond
		jc.op, jc.lhs_col, jc.rhs_col = op, C.int32_t(l.Index), -1 // Column.Index is already an index into lhs ++ rhs (joiner.go:157)
		switch r := sf.GetArgs()[1].(type) {
		case *expression.Column:
			jc.rhs_col = C.int32_t(r.Index)
		case *expression.Constant:
			if r.Value.IsNull() {
				rest = append(rest, c)
				continue
			}
			jc.const_type = tqType(r.RetType)
			jc.const_bits = C.uint64_t(datumBits(&r.Value, r.RetType))
		default:
			rest = append(rest, c)
			continue
		}
		out = append(out, jc)
	}
	return out, rest, len(out) > 0
}

