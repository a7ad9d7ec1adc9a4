// +build gpu

// GPUSortExec / GPUTopNExec / GPUMergeJoinExec: SortExec, TopNExec (executor/sort.go) and MergeJoinExec
// (executor/merge_join.go) replaced by libtinysql_b200 (csrc/sort.cu).  executorBuilder.buildSort / buildTopN / buildMergeJoin
// return them when every ByItem / join key is a column (the builder pre-projects other expressions, as it does for the
// hash operators).  Design reference like the rest of integration/go: not compiled in this image (no Go toolchain).
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
	"unsafe"

	"github.com/pingcap/tidb/expression"
	plannercore "github.com/pingcap/tidb/planner/core"
	"github.com/pingcap/tidb/types"
	"github.com/pingcap/tidb/util/chunk"
)

// resultPump hands a materialised device result to the parent in RequiredRows-sized chunks; shared by the three operators.
type resultPump struct {
	outTypes []C.int32_t
	outViews *chunk.CViewSet
	sizes    *C.int64_t // C memory, one entry per output column
}

func (p *resultPump) fill(req *chunk.Chunk, nextBytes func(C.int64_t, *C.int64_t) C.int32_t,
	next func(C.int64_t, *C.tq_column, *C.int64_t, *C.int32_t) C.int32_t) error {
	want := req.RequiredRows()
	if st := nextBytes(C.int64_t(want), p.sizes); st != C.TQ_OK { // sizes the var-len buffers of THIS call
		return chunk.StatusError(int32(st))
	}
	sizes := (*[1 << 10]C.int64_t)(unsafe.Pointer(p.sizes))[:len(p.outTypes)]
	for i, t := range p.outTypes {
		col := req.Column(i)
		switch t {
		case C.TQ_TYPE_BYTES:
			col.PrepareVarLenResult(want, int64(sizes[i]))
		case C.TQ_TYPE_FLOAT32:
			col.PrepareFixedResult(want, 4)
		default:
			col.PrepareFixedResult(want, 8)
		}
		p.outViews.FillResult(i, col)
	}
	var n C.int64_t
	var eof C.int32_t
	st := next(C.int64_t(want), p.outViews.Ptr(), &n, &eof)
	p.outViews.Release()
	if st != C.TQ_OK {
		return chunk.StatusError(int32(st))
	}
	for i := range p.outTypes {
		p.outViews.CopyBack(i, req.Column(i), int(n))
		req.Column(i).SetResultRows(int(n))
	}
	req.SetNumVirtualRows(int(n)) // 0 rows == end of stream (executor.go:146-162)
	return nil
}

// ---------------------------------------------------------------------------------------------- SortExec / TopNExec
type GPUSortExec struct {
	baseExecutor
	ByItems []*plannercore.ByItems
	limit   *plannercore.PhysicalLimit // nil: SortExec; else TopNExec (sort.go:159-166)

	h       *C.tq_sort
	fetched bool
	inViews *chunk.CViewSet
	childChk *chunk.Chunk
	pump    resultPump
}

// Open implements Executor (sort.go:50-55).
func (e *GPUSortExec) Open(ctx context.Context) error {
	if err := e.children[0].Open(ctx); err != nil {
		return err
	}
	fts := retTypes(e)
	types := cInt32s(len(fts), func(i int) C.int32_t { return tqType(fts[i]) })
	by := cInt32s(len(e.ByItems), func(i int) C.int32_t { return C.int32_t(e.ByItems[i].Expr.(*expression.Column).Index) }) // buildKeyColumns, sort.go:107-113
	desc := cInt32s(len(e.ByItems), func(i int) C.int32_t {
		if e.ByItems[i].Desc {
			return 1
		}
		return 0
	})
	defer C.free(unsafe.Pointer(types))
	defer C.free(unsafe.Pointer(by))
	defer C.free(unsafe.Pointer(desc))
	d := (*C.tq_sort_desc)(C.calloc(1, C.sizeof_tq_sort_desc)) // argument block in C memory (cgo pointer rules)
	defer C.free(unsafe.Pointer(d))
	d.n_cols, d.types = C.int32_t(len(fts)), types
	d.n_by, d.by_cols, d.by_desc = C.int32_t(len(e.ByItems)), by, desc
	d.limit_offset, d.limit_count = 0, -1
	if e.limit != nil { // totalLimit = Offset + Count, Idx starts at Offset (sort.go:210-214)
		d.limit_offset, d.limit_count = C.int64_t(e.limit.Offset), C.int64_t(e.limit.Count)
	}
	if st := C.tq_sort_create(d, &e.h); st != C.TQ_OK {
		return chunk.StatusError(int32(st))
	}
	e.fetched = false
	e.childChk = newFirstChunk(e.children[0])
	e.inViews = chunk.NewCViewSet(len(fts))
	e.pump = resultPump{outViews: chunk.NewCViewSet(len(fts)), sizes: (*C.int64_t)(C.calloc(C.size_t(len(fts)), 8))}
	for _, ft := range fts {
		e.pump.outTypes = append(e.pump.outTypes, tqType(ft))
	}
	return nil
}

// Next implements Executor (sort.go:58-76): a pipeline breaker — the first call drains the child (fetchRowChunks :77-86).
func (e *GPUSortExec) Next(ctx context.Context, req *chunk.Chunk) error {
	req.Reset()
	if !e.fetched {
		for {
			if err := Next(ctx, e.children[0], e.childChk); err != nil {
				return err
			}
			if e.childChk.NumRows() == 0 {
				break
			}
			e.inViews.FillChunk(e.childChk)
			st := C.tq_sort_put(e.h, e.inViews.Ptr(), C.TQ_MEM_HOST)
			e.inViews.Release()
			if st != C.TQ_OK {
				return chunk.StatusError(int32(st))
			}
		}
		if st := C.tq_sort_eof(e.h); st != C.TQ_OK { // the sort itself
			return chunk.StatusError(int32(st))
		}
		e.fetched = true
	}
	return e.pump.fill(req,
		func(want C.int64_t, sizes *C.int64_t) C.int32_t { return C.tq_sort_next_bytes(e.h, want, sizes) },
		func(want C.int64_t, out *C.tq_column, n *C.int64_t, eof *C.int32_t) C.int32_t { return C.tq_sort_next(e.h, want, out, n, eof) })
}

// Close implements Executor (sort.go:45-47).
func (e *GPUSortExec) Close() error {
	if e.h != nil {
		C.tq_sort_destroy(e.h)
		e.h = nil
		e.inViews.Free()
		e.pump.outViews.Free()
		C.free(unsafe.Pointer(e.pump.sizes))
	}
	return e.children[0].Close()
}

// ---------------------------------------------------------------------------------------------- MergeJoinExec
type GPUMergeJoinExec struct {
	baseExecutor
	joinType      plannercore.JoinType
	outerIdx      int // merge_join.go:41; the inner child is children[outerIdx^1]
	outerKeys     []*expression.Column
	innerKeys     []*expression.Column
	outerFilter   expression.CNFExprs
	otherConditions expression.CNFExprs // run inside the library (setOtherConditions, gpu_join.go); what is left: see Next
	defaultValues []types.Datum // PhysicalMergeJoin.DefaultValues -> defaultInner (joiner.go:139-143)

	h        *C.tq_mjoin
	prepared bool
	inViews  *chunk.CViewSet
	chk      [2]*chunk.Chunk
	selected []bool
	selBytes []byte
	filtered []bool
	pump     resultPump
}

// Open implements Executor (merge_join.go:185-198).  OtherConditions go to the library as the hash join hands them over
// (setOtherConditions, gpu_join.go): comparisons to tq_mjoin_set_other_conditions, any CNF CompileProgram lowers to
// tq_mjoin_set_other_program, for outer joins too.  Trees that do not lower stay with Next for an inner join; an outer join
// with such a condition fails here.
func (e *GPUMergeJoinExec) Open(ctx context.Context) error {
	if err := e.baseExecutor.Open(ctx); err != nil {
		return err
	}
	inner, outer := e.children[e.outerIdx^1], e.children[e.outerIdx]
	ift, oft := retTypes(inner), retTypes(outer)
	it := cInt32s(len(ift), func(i int) C.int32_t { return tqType(ift[i]) })
	ot := cInt32s(len(oft), func(i int) C.int32_t { return tqType(oft[i]) })
	ik := cInt32s(len(e.innerKeys), func(i int) C.int32_t { return C.int32_t(e.innerKeys[i].Index) })
	ok := cInt32s(len(e.outerKeys), func(i int) C.int32_t { return C.int32_t(e.outerKeys[i].Index) })
	d := (*C.tq_mjoin_desc)(C.calloc(1, C.sizeof_tq_mjoin_desc))
	defer func() {
		for _, p := range []unsafe.Pointer{unsafe.Pointer(it), unsafe.Pointer(ot), unsafe.Pointer(ik), unsafe.Pointer(ok), unsafe.Pointer(d)} {
			C.free(p)
		}
	}()
	d.join_type = C.int32_t(e.joinType) // InnerJoin 0, LeftOuterJoin 1, RightOuterJoin 2 = TQ_JOIN_*
	if e.outerIdx == 1 {
		d.outer_is_right = 1
	}
	d.n_inner_cols, d.inner_types, d.n_outer_cols, d.outer_types = C.int32_t(len(ift)), it, C.int32_t(len(oft)), ot
	d.n_keys, d.inner_keys, d.outer_keys = C.int32_t(len(e.innerKeys)), ik, ok
	if e.defaultValues != nil {
		bits := (*[1 << 10]C.uint64_t)(C.calloc(C.size_t(len(ift)), 8))
		nn := (*[1 << 10]C.uint8_t)(C.calloc(C.size_t(len(ift)), 1))
		defer C.free(unsafe.Pointer(bits))
		defer C.free(unsafe.Pointer(nn))
		for i := range ift {
			if !e.defaultValues[i].IsNull() {
				bits[i], nn[i] = C.uint64_t(datumBits(&e.defaultValues[i], ift[i])), 1
			}
		}
		d.default_inner_bits, d.default_inner_not_null = &bits[0], &nn[0]
	}
	if st := C.tq_mjoin_create(d, &e.h); st != C.TQ_OK {
		return chunk.StatusError(int32(st))
	}
	rest, err := setOtherConditions(e.otherConditions, e.outerIdx == 1, len(oft), len(ift),
		func(n C.int32_t, cc *C.tq_join_cond) C.int32_t { return C.tq_mjoin_set_other_conditions(e.h, n, cc) },
		func(nIn C.int32_t, in *C.int32_t, nOps C.int32_t, ops *C.tq_expr_op) C.int32_t {
			return C.tq_mjoin_set_other_program(e.h, nIn, in, nOps, ops)
		})
	if err != nil {
		return err
	}
	e.otherConditions = rest
	if len(e.otherConditions) > 0 && e.joinType != plannercore.InnerJoin {
		return errors.New("tinysql_b200: this OtherCondition of an outer merge join is not supported on the device path")
	}
	e.prepared = false
	e.chk = [2]*chunk.Chunk{newFirstChunk(inner), newFirstChunk(outer)}
	e.inViews = chunk.NewCViewSet(maxInt(len(ift), len(oft)))
	fts := retTypes(e)
	e.pump = resultPump{outViews: chunk.NewCViewSet(len(fts)), sizes: (*C.int64_t)(C.calloc(C.size_t(len(fts)), 8))}
	for _, ft := range fts {
		e.pump.outTypes = append(e.pump.outTypes, tqType(ft))
	}
	return nil
}

// Next implements Executor (merge_join.go:225-244).  The first call reads both children to the end — the inner child through
// mergeJoinInnerTable's reader loop (:127-152), the outer child chunk by chunk with its filter (fetchNextOuterRows :350-372).
func (e *GPUMergeJoinExec) Next(ctx context.Context, req *chunk.Chunk) error {
	req.Reset()
	if !e.prepared {
		inner, outer := e.children[e.outerIdx^1], e.children[e.outerIdx]
		for side, child := range []Executor{inner, outer} {
			for {
				chk := e.chk[side]
				if err := Next(ctx, child, chk); err != nil {
					return err
				}
				if chk.NumRows() == 0 {
					break
				}
				var sel *C.uint8_t
				if side == 1 && len(e.outerFilter) > 0 {
					var err error
					if e.selected, err = expression.VectorizedFilter(e.ctx, e.outerFilter, chunk.NewIterator4Chunk(chk), e.selected); err != nil {
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
					sel = (*C.uint8_t)(unsafe.Pointer(&e.selBytes[0]))
				}
				e.inViews.FillChunk(chk)
				var st C.int32_t
				if side == 0 {
					st = C.tq_mjoin_put_inner(e.h, e.inViews.Ptr(), C.TQ_MEM_HOST)
				} else {
					st = C.tq_mjoin_put_outer(e.h, e.inViews.Ptr(), sel, C.TQ_MEM_HOST)
				}
				e.inViews.Release()
				if st != C.TQ_OK {
					return chunk.StatusError(int32(st))
				}
			}
		}
		if st := C.tq_mjoin_finish(e.h); st != C.TQ_OK { // TQ_ERR_STATE: the inner child was not sorted by the keys
			return chunk.StatusError(int32(st))
		}
		e.prepared = true
		var warned C.int64_t
		C.tq_mjoin_warnings(e.h, &warned)
		var seen int64
		appendDivByZeroWarnings(e.ctx, int64(warned), &seen)
	}
	for {
		// an overflow of the OtherConditions program comes back from tq_mjoin_next_bytes / tq_mjoin_next
		if err := e.pump.fill(req,
			func(want C.int64_t, sizes *C.int64_t) C.int32_t { return C.tq_mjoin_next_bytes(e.h, want, sizes) },
			func(want C.int64_t, out *C.tq_column, n *C.int64_t, eof *C.int32_t) C.int32_t { return C.tq_mjoin_next(e.h, want, out, n, eof) }); err != nil {
			return err
		}
		if req.NumRows() == 0 || len(e.otherConditions) == 0 {
			return nil
		}
		// inner joins only (Open rejected the outer case): baseJoiner.filter (joiner.go:155-167) on the returned chunk
		var err error
		if e.filtered, err = expression.VectorizedFilter(e.ctx, e.otherConditions, chunk.NewIterator4Chunk(req), e.filtered); err != nil {
			return err
		}
		req.SetSel(selToIdx(e.filtered))
		if req.NumRows() > 0 {
			return nil
		}
		req.Reset()
	}
}

// Close implements Executor (merge_join.go:178-182).
func (e *GPUMergeJoinExec) Close() error {
	if e.h != nil {
		C.tq_mjoin_destroy(e.h)
		e.h = nil
		e.inViews.Free()
		e.pump.outViews.Free()
		C.free(unsafe.Pointer(e.pump.sizes))
	}
	return e.baseExecutor.Close()
}
