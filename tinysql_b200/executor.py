"""Host-side mirror of the reference's operator interface for the hot path:
executor.Executor{Open, Next, Close} (executor/executor.go:146-162) for HashJoinExec
(executor/join.go) and HashAggExec (executor/aggregate.go), driving the C-ABI exactly the way the
Go shim in INTEGRATION.md does: children hand up <=1024-row chunks, Next fills <=requiredRows rows,
0 rows == end of stream.  All operator logic (batching, hashing, matching, aggregation, re-slicing)
is inside libtinysql_b200.so; nothing here computes results.
"""
import ctypes as C

import numpy as np

from . import _lib as L
from .chunk import (BYTES, FLOAT64, INT64, MAX_CHUNK_SIZE, UINT64, Chunk, Column, DeviceColumn, VarColumn, device_to_host, tq_array)
from .expression import JoinProgram

INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN = 0, 1, 2  # planner/core/logical_plans.go:52-57
AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MAX, AGG_MIN, AGG_FIRSTROW = range(6)


class MockDataSource:
    """executor/benchmark_test.go:50-177 mockDataSource: replays prepared chunks of <= maxChunkSize rows."""

    def __init__(self, types, columns, chunk_size=MAX_CHUNK_SIZE):
        self.types = list(types)
        n = columns[0].length if columns else 0
        self.chunks = [Chunk([c.slice(lo, min(lo + chunk_size, n)) for c in columns]) for lo in range(0, n, chunk_size)]
        self.pos = 0

    def Open(self):
        self.pos = 0

    def Next(self):
        if self.pos >= len(self.chunks):
            return Chunk([Column(t, [] if t == BYTES else np.zeros(0)) for t in self.types])
        self.pos += 1
        return self.chunks[self.pos - 1]

    def Close(self):
        pass


def _i32arr(vals):
    return (C.c_int32 * max(len(vals), 1))(*vals)


class HashJoinExec:
    """executor/join.go:31-146.  inner = build side, outer = probe side; output = left ++ right."""

    def __init__(self, outer_exec, inner_exec, outer_keys, inner_keys, join_type=INNER_JOIN, outer_is_right=False,
                 outer_filter=None, probe_batch_rows=0, max_chunk_size=MAX_CHUNK_SIZE, stable_input=False, other_conditions=(), default_inner=None,
                 other_program=()):
        self.outer, self.inner = outer_exec, inner_exec
        self.outer_keys, self.inner_keys = list(outer_keys), list(inner_keys)
        self.join_type, self.outer_is_right = join_type, outer_is_right
        self.outer_filter = outer_filter  # callable(chunk) -> selected bytes (expression.VectorizedFilter result)
        self.probe_batch_rows = probe_batch_rows
        self.stable_input = stable_input  # TQ_JOIN_STABLE_INPUT: the children keep every chunk alive and unmodified until Close
        # OtherConditions (joiner.go:155-167) over the output row lhs ++ rhs, in one of two forms: other_conditions as
        # (op, lhs_col, rhs_col) or (op, lhs_col, None, const_type, const_value) comparisons (tq_join_set_other_conditions),
        # or other_program as a CNF list of expression.Expr filters, Col(i) = output column i (tq_join_set_other_program)
        self.other_conditions = list(other_conditions)
        self.other_program = list(other_program)
        self.warnings = 0   # division-by-zero warnings of other_program (tq_join_warnings), current after each Next
        # PhysicalHashJoin.DefaultValues (builder.go:449-465): per inner column the value a miss row of an outer join carries (None = NULL)
        self.default_inner = default_inner
        self.max_chunk_size = max_chunk_size
        self.handle = None
        self.prepared = False
        self.outer_done = False
        lhs, rhs = (inner_exec.types, outer_exec.types) if outer_is_right else (outer_exec.types, inner_exec.types)
        self.types = list(lhs) + list(rhs)

    def Open(self):
        self.outer.Open()
        self.inner.Open()
        lib = L.load()
        bt, pt = _i32arr(self.inner.types), _i32arr(self.outer.types)
        bk, pk = _i32arr(self.inner_keys), _i32arr(self.outer_keys)
        d = L.TQJoinDesc(self.join_type, 1 if self.outer_is_right else 0, len(self.inner.types), bt, len(self.outer.types), pt,
                         len(self.inner_keys), bk, pk, self.probe_batch_rows, L.TQ_JOIN_STABLE_INPUT if self.stable_input else 0)
        if self.default_inner is not None:
            np_t = {INT64: np.int64, UINT64: np.uint64, FLOAT64: np.float64}
            bits = [0 if v is None else int(np.array([v], dtype=np_t[t]).view(np.uint64)[0]) for v, t in zip(self.default_inner, self.inner.types)]
            self._dbits = (C.c_uint64 * len(bits))(*bits)
            self._dnn = (C.c_uint8 * len(bits))(*[0 if v is None else 1 for v in self.default_inner])
            d.default_inner_bits, d.default_inner_not_null = self._dbits, self._dnn
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
        self.handle = h
        if self.other_conditions:
            arr = (L.TQJoinCond * len(self.other_conditions))()
            for i, c in enumerate(self.other_conditions):
                if c[2] is None:
                    np_t = {INT64: np.int64, UINT64: np.uint64, FLOAT64: np.float64}[c[3]]
                    arr[i] = L.TQJoinCond(c[0], c[1], -1, c[3], int(np.array([c[4]], dtype=np_t).view(np.uint64)[0]))
                else:
                    arr[i] = L.TQJoinCond(c[0], c[1], c[2], 0, 0)
            L.check(lib.tq_join_set_other_conditions(h, len(self.other_conditions), arr))
        if self.other_program:
            JoinProgram(self.other_program).set_on(lib.tq_join_set_other_program, h)
        self.warnings = 0
        self.prepared = False
        self.outer_done = False

    def _build(self):
        """fetchAndBuildHashTable (join.go:148-158): drain the inner child into the row container."""
        lib = L.load()
        while True:
            chk = self.inner.Next()
            if chk.num_rows() == 0:
                break
            L.check(lib.tq_join_put_build(self.handle, tq_array(chk.cols), L.TQ_MEM_HOST))
        L.check(lib.tq_join_finalize_build(self.handle))

    def Next(self, required_rows=None):
        """Returns a Chunk with <= required_rows rows; 0 rows == EOF (join.go:125-146)."""
        lib = L.load()
        req = required_rows or self.max_chunk_size
        if not self.prepared:
            self._build()
            self.prepared = True
        has_var = BYTES in self.types
        out = [VarColumn.empty(BYTES, req) if t == BYTES else Column.empty(t, req) for t in self.types]
        arr = tq_array(out, req)
        n, eof = C.c_int64(0), C.c_int32(0)
        while True:
            if has_var:
                # size the var-len result buffers for this call (the *_next_size query of the ownership contract)
                need = (C.c_int64 * len(self.types))()
                L.check(lib.tq_join_next_bytes(self.handle, req, need))
                for i, t in enumerate(self.types):
                    if t == BYTES:
                        out[i] = VarColumn.empty(BYTES, req, int(need[i]))
                arr = tq_array(out, req)
            L.check(lib.tq_join_next(self.handle, req, arr, C.byref(n), C.byref(eof)))
            if n.value > 0 or eof.value:
                break
            # fetchOuterSideChunks (join.go:194-221): feed one more outer chunk
            chk = self.outer.Next()
            if chk.num_rows() == 0:
                L.check(lib.tq_join_probe_eof(self.handle))
                continue
            sel = None
            if self.outer_filter is not None:
                sel = np.ascontiguousarray(self.outer_filter(chk), dtype=np.uint8)
            L.check(lib.tq_join_put_probe(self.handle, tq_array(chk.cols), sel.ctypes.data if sel is not None else None, L.TQ_MEM_HOST))
        k = n.value
        w = C.c_int64(0)
        L.check(lib.tq_join_warnings(self.handle, C.byref(w)))
        self.warnings = w.value
        return Chunk([c.head(k) if t == BYTES else Column(t, c.values[:k], c.not_null()[:k]) for t, c in zip(self.types, out)])

    def Close(self):
        if self.handle is not None:
            L.load().tq_join_destroy(self.handle)
            self.handle = None
        self.outer.Close()
        self.inner.Close()

    def drain(self):
        chunks = []
        while True:
            c = self.Next()
            if c.num_rows() == 0:
                break
            chunks.append(c)
        return Chunk.concat(chunks, self.types)


class HashAggExec:
    """executor/aggregate.go:54-155.  funcs: list of (AGG_*, arg_col or -1); one GROUP BY column or none."""

    def __init__(self, child, group_by, funcs, est_groups=0, max_chunk_size=MAX_CHUNK_SIZE, not_null_cols=()):
        self.child, self.group_by, self.funcs = child, list(group_by), list(funcs)
        self.not_null_cols = set(not_null_cols)  # input columns whose FieldType carries mysql.NotNullFlag
        self.est_groups, self.max_chunk_size = est_groups, max_chunk_size
        self.handle = None
        self.prepared = False
        self.types = []

    def Open(self):
        self.child.Open()
        lib = L.load()
        it = _i32arr([t | (0x100 if i in self.not_null_cols else 0) for i, t in enumerate(self.child.types)])  # TQ_TYPE_NOT_NULL
        gb = _i32arr(self.group_by)
        fa = (L.TQAggFunc * max(len(self.funcs), 1))(*[L.TQAggFunc(f, a) for f, a in self.funcs])
        d = L.TQAggDesc(len(self.child.types), it, len(self.group_by), gb, len(self.funcs), fa, self.est_groups)
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
        self.handle = h
        self.types = []
        for i in range(len(self.funcs)):
            t = C.c_int32(0)
            L.check(lib.tq_agg_output_type(h, i, C.byref(t)))
            self.types.append(t.value)
        self.prepared = False

    def Next(self, required_rows=None):
        lib = L.load()
        req = required_rows or self.max_chunk_size
        if not self.prepared:  # fetchChildData + partial workers (aggregate.go:487-522,307-350)
            while True:
                chk = self.child.Next()
                if chk.num_rows() == 0:
                    break
                L.check(lib.tq_agg_put(self.handle, tq_array(chk.cols), L.TQ_MEM_HOST))
            L.check(lib.tq_agg_eof(self.handle))
            self.prepared = True
        out = [VarColumn.empty(BYTES, req) if t == BYTES else Column.empty(t, req) for t in self.types]
        if BYTES in self.types:
            # size the var-len result buffers for this call (the *_next_size query of the ownership contract)
            need = (C.c_int64 * len(self.types))()
            L.check(lib.tq_agg_next_bytes(self.handle, req, need))
            for i, t in enumerate(self.types):
                if t == BYTES:
                    out[i] = VarColumn.empty(BYTES, req, int(need[i]))
        arr = tq_array(out, req)
        n, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_agg_next(self.handle, req, arr, C.byref(n), C.byref(eof)))
        k = n.value
        return Chunk([c.head(k) if t == BYTES else Column(t, c.values[:k], c.not_null()[:k]) for t, c in zip(self.types, out)])

    def Close(self):
        if self.handle is not None:
            L.load().tq_agg_destroy(self.handle)
            self.handle = None
        self.child.Close()

    def drain(self):
        chunks = []
        while True:
            c = self.Next()
            if c.num_rows() == 0:
                break
            chunks.append(c)
        return Chunk.concat(chunks, self.types)


class HashAggFinalExec(HashAggExec):
    """FinalMode HashAggExec over pushed-down partial results (aggfuncs/builder.go:50-62,86-109; planner/core/task.go:564-625):
    the child returns PARTIAL rows — the layout store/mockstore/mocktikv/aggregate.go:81-124 produces (per function its
    GetPartialResult columns, then the GROUP BY columns).  funcs: list of (AGG_*, arg_col, arg_col2); arg_col2 is AVG's
    partial-sum column (arg_col its partial count), -1 otherwise."""

    def Open(self):
        self.child.Open()
        lib = L.load()
        it = _i32arr(list(self.child.types))
        gb = _i32arr(self.group_by)
        fa = (L.TQAggFinalFunc * max(len(self.funcs), 1))(*[L.TQAggFinalFunc(f, a, b) for f, a, b in self.funcs])
        d = L.TQAggFinalDesc(len(self.child.types), it, len(self.group_by), gb, len(self.funcs), fa, self.est_groups)
        h = C.c_void_p()
        L.check(lib.tq_agg_create_final(C.byref(d), C.byref(h)))
        self.handle = h
        self.types = []
        for i in range(len(self.funcs)):
            t = C.c_int32(0)
            L.check(lib.tq_agg_output_type(h, i, C.byref(t)))
            self.types.append(t.value)
        self.prepared = False


def _drain_result(lib, types, req, next_bytes, nxt, handle):
    """one Next() of an operator that hands out a materialised result in <= req-row chunks"""
    out = [VarColumn.empty(BYTES, req) if t == BYTES else Column.empty(t, req) for t in types]
    if BYTES in types:
        need = (C.c_int64 * len(types))()
        L.check(next_bytes(handle, req, need))
        for i, t in enumerate(types):
            if t == BYTES:
                out[i] = VarColumn.empty(BYTES, req, int(need[i]))
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(nxt(handle, req, tq_array(out, req), C.byref(n), C.byref(eof)))
    k = n.value
    return Chunk([c.head(k) if t == BYTES else Column(t, c.values[:k], c.not_null()[:k]) for t, c in zip(types, out)])


class SortExec:
    """executor/sort.go:28-157.  by_items: list of (column index, desc).  Ties keep child order (sort.Slice promises none)."""

    def __init__(self, child, by_items, max_chunk_size=MAX_CHUNK_SIZE):
        self.child, self.by_items, self.max_chunk_size = child, list(by_items), max_chunk_size
        self.limit_offset, self.limit_count = 0, -1
        self.handle, self.fetched = None, False
        self.types = list(child.types)

    def Open(self):
        self.child.Open()
        lib = L.load()
        d = L.TQSortDesc(len(self.types), _i32arr(self.types), len(self.by_items), _i32arr([c for c, _ in self.by_items]),
                         _i32arr([1 if x else 0 for _, x in self.by_items]), self.limit_offset, self.limit_count)
        h = C.c_void_p()
        L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
        self.handle, self.fetched = h, False

    def Next(self, required_rows=None):
        lib = L.load()
        if not self.fetched:  # fetchRowChunks (sort.go:77-86)
            while True:
                chk = self.child.Next()
                if chk.num_rows() == 0:
                    break
                L.check(lib.tq_sort_put(self.handle, tq_array(chk.cols), L.TQ_MEM_HOST))
            L.check(lib.tq_sort_eof(self.handle))
            self.fetched = True
        return _drain_result(lib, self.types, required_rows or self.max_chunk_size, lib.tq_sort_next_bytes, lib.tq_sort_next, self.handle)

    def Close(self):
        if self.handle is not None:
            L.load().tq_sort_destroy(self.handle)
            self.handle = None
        self.child.Close()

    def drain(self):
        chunks = []
        while True:
            c = self.Next()
            if c.num_rows() == 0:
                break
            chunks.append(c)
        return Chunk.concat(chunks, self.types)


class TopNExec(SortExec):
    """executor/sort.go:159-318: the rows [offset, offset + count) of the order (plannercore.PhysicalLimit)."""

    def __init__(self, child, by_items, offset, count, max_chunk_size=MAX_CHUNK_SIZE):
        super().__init__(child, by_items, max_chunk_size)
        self.limit_offset, self.limit_count = int(offset), int(count)


class MergeJoinExec:
    """executor/merge_join.go:31-373.  Both children sorted ascending by their keys; output = left ++ right in outer order."""

    def __init__(self, outer_exec, inner_exec, outer_keys, inner_keys, join_type=INNER_JOIN, outer_is_right=False, outer_filter=None,
                 max_chunk_size=MAX_CHUNK_SIZE, default_inner=None, other_conditions=(), other_program=()):
        # OtherConditions over the output row left ++ right, as in HashJoinExec: other_conditions = (op, lhs_col, rhs_col) or
        # (op, lhs_col, None, const_type, const_value) comparisons, other_program = a CNF list of expression.Expr filters
        self.other_conditions = list(other_conditions)
        self.other_program = list(other_program)
        self.warnings = 0   # division-by-zero warnings of other_program (tq_mjoin_warnings), current after each Next
        self.outer, self.inner = outer_exec, inner_exec
        self.outer_keys, self.inner_keys = list(outer_keys), list(inner_keys)
        self.join_type, self.outer_is_right, self.outer_filter = join_type, outer_is_right, outer_filter
        self.max_chunk_size, self.default_inner = max_chunk_size, default_inner
        self.handle, self.prepared = None, False
        self.types = (list(inner_exec.types) + list(outer_exec.types)) if outer_is_right else (list(outer_exec.types) + list(inner_exec.types))

    def Open(self):
        self.outer.Open()
        self.inner.Open()
        lib = L.load()
        dbits = dnn = None
        if self.default_inner is not None:
            from .chunk import _NP
            nb = len(self.inner.types)
            dbits = (C.c_uint64 * nb)(*[0 if v is None else int(np.array([v], dtype=_NP[t]).view(np.uint64)[0]) for v, t in zip(self.default_inner, self.inner.types)])
            dnn = (C.c_uint8 * nb)(*[0 if v is None else 1 for v in self.default_inner])
        self._keep = (dbits, dnn)
        d = L.TQMJoinDesc(self.join_type, 1 if self.outer_is_right else 0, len(self.inner.types), _i32arr(self.inner.types), len(self.outer.types),
                          _i32arr(self.outer.types), len(self.inner_keys), _i32arr(self.inner_keys), _i32arr(self.outer_keys), dbits, dnn)
        h = C.c_void_p()
        L.check(lib.tq_mjoin_create(C.byref(d), C.byref(h)))
        self.handle, self.prepared = h, False
        if self.other_conditions:
            from .chunk import _NP
            arr = (L.TQJoinCond * len(self.other_conditions))()
            for i, c in enumerate(self.other_conditions):
                if c[2] is None:
                    arr[i] = L.TQJoinCond(c[0], c[1], -1, c[3], int(np.array([c[4]], dtype=_NP[c[3]]).view(np.uint64)[0]))
                else:
                    arr[i] = L.TQJoinCond(c[0], c[1], c[2], 0, 0)
            L.check(lib.tq_mjoin_set_other_conditions(h, len(self.other_conditions), arr))
        if self.other_program:
            JoinProgram(self.other_program).set_on(lib.tq_mjoin_set_other_program, h)
        self.warnings = 0

    def Next(self, required_rows=None):
        lib = L.load()
        if not self.prepared:
            while True:  # mergeJoinInnerTable.nextRow's reader loop (merge_join.go:127-152)
                chk = self.inner.Next()
                if chk.num_rows() == 0:
                    break
                L.check(lib.tq_mjoin_put_inner(self.handle, tq_array(chk.cols), L.TQ_MEM_HOST))
            while True:  # fetchNextOuterRows (merge_join.go:350-372): one outer chunk + VectorizedFilter -> selected
                chk = self.outer.Next()
                if chk.num_rows() == 0:
                    break
                sel = None
                if self.outer_filter is not None:
                    sel = np.ascontiguousarray(self.outer_filter(chk), dtype=np.uint8)
                L.check(lib.tq_mjoin_put_outer(self.handle, tq_array(chk.cols), sel.ctypes.data if sel is not None else None, L.TQ_MEM_HOST))
            L.check(lib.tq_mjoin_finish(self.handle))
            self.prepared = True
            w = C.c_int64(0)
            L.check(lib.tq_mjoin_warnings(self.handle, C.byref(w)))
            self.warnings = w.value
        return _drain_result(lib, self.types, required_rows or self.max_chunk_size, lib.tq_mjoin_next_bytes, lib.tq_mjoin_next, self.handle)

    def Close(self):
        if self.handle is not None:
            L.load().tq_mjoin_destroy(self.handle)
            self.handle = None
        self.outer.Close()
        self.inner.Close()

    def drain(self):
        chunks = []
        while True:
            c = self.Next()
            if c.num_rows() == 0:
                break
            chunks.append(c)
        return Chunk.concat(chunks, self.types)
