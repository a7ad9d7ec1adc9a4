"""GPU suite: dist.BroadcastJoin — tq_partition_push_broadcast -> published slots -> tq_region_wait -> one device build chunk
per source -> the local probe shard — with W = 1, 2, 3 and 8 ranks emulated in one process (tests/broadcast_ref.py), against
the oracle on the concatenated inputs.  Keyed results are compared as multisets over all ranks; key-less results in order,
rank by rank (rank r = its probe shard against the rank-major concatenation of the build shards).  Also: the refusals of the
push (nothing written, nothing published) and a byte-area overflow the receiver reports instead of joining."""
import ctypes as C

import numpy as np
import pytest

import broadcast_ref as B
import exchange_ref as X
import oracle_py as O
from join_program_oracle import join_with_program
from keyless_oracle import keyless_hash_join, keyless_join_with_program
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, FLOAT64, INT64, UINT64, Chunk, Column, DeviceColumn
from tinysql_b200.dist import BroadcastJoin
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN
from tinysql_b200.expression import Col, Const, Func
from util import assert_same_multiset, assert_same_ordered

pytestmark = pytest.mark.gpu
WORLDS = [1, 2, 3, 8]
SHAPES = [(INNER_JOIN, True), (INNER_JOIN, False), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)]
LT = 0


def _col(rng, tp, n, lo, hi, null_frac):
    nn = rng.random(n) >= null_frac if null_frac else None
    if tp == BYTES:
        return Column(BYTES, [None if nn is not None and not nn[i] else b"s%d" % v for i, v in enumerate(rng.integers(lo, hi, n))], nn)
    if tp == UINT64:
        return Column(UINT64, rng.integers(lo, hi, n).astype(np.uint64) | np.uint64(1 << 63), nn)
    if tp == FLOAT64:
        return Column(FLOAT64, rng.integers(lo, hi, n).astype(np.float64) * 0.5, nn)
    return Column(INT64, rng.integers(lo, hi, n).astype(np.int64), nn)


# (build types, probe types, build keys, probe keys): key columns draw from a small domain so rows match several times
LAYOUTS = {
    "c1": ([INT64, BYTES], [INT64, BYTES, INT64], [0, 1], [0, 1]),                     # BIGINT + VARSTRING keys
    "two_keys_signed_unsigned": ([UINT64, FLOAT64, INT64], [INT64, UINT64], [2, 0], [0, 1]),
    "three_keys": ([INT64, UINT64, BYTES, INT64], [BYTES, INT64, UINT64, FLOAT64], [0, 1, 2], [1, 2, 0]),
    "string_payloads": ([INT64, BYTES], [BYTES, INT64, BYTES], [0], [1]),
}


def _side(rng, types, keys, n, null_frac):
    return [_col(rng, t, n, 0, 6 if c in keys else 1 << 40, null_frac) for c, t in enumerate(types)]


def _run(lib, W, bt, pt, bkeys, pkeys, bcols, pcols, jt, oir, sel=None, dflt=None, conds=(), program=(), bsizes=None, nullable=(False, False)):
    bsh = list(zip(*[B.shards(c, W, bsizes) for c in bcols]))
    psh = list(zip(*[B.shards(c, W) for c in pcols]))
    psel = None if sel is None else [np.asarray(s) for s in np.array_split(np.asarray(sel, bool), np.cumsum([p[0].length for p in psh])[:-1])]
    em = B.Emulated(lib, W, max(max(s[0].length for s in bsh), 1), bt, pt, build_keys=bkeys, probe_keys=pkeys, join_type=jt, outer_is_right=oir,
                    byte_caps=B.byte_caps(bt, bsh), build_nullable=nullable[0], probe_nullable=nullable[1], default_inner=dflt,
                    other_conditions=conds, other_program=program)
    try:
        return em.step(bsh, psh, psel), bsh, psh, psel
    finally:
        em.free()


@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("jt,oir", SHAPES)
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_keyed(lib, W, jt, oir, layout):
    """multi-column, signed / unsigned and string keys, string payloads, NULL keys and values, selected[] and defaultInner"""
    rng = np.random.default_rng(W * 100 + jt * 10 + oir + len(layout))
    bt, pt, bk, pk = LAYOUTS[layout]
    nb, npr = 300 * W + 7, 500 * W + 3
    bc, pc = _side(rng, bt, bk, nb, 0.1), _side(rng, pt, pk, npr, 0.1)
    outer = jt != INNER_JOIN
    sel = rng.random(npr) > 0.15 if outer else None
    dflt = [7 if t == INT64 else None for t in bt] if outer else None
    got, *_ = _run(lib, W, bt, pt, bk, pk, bc, pc, jt, oir, sel, dflt, nullable=(True, True))
    out_types = bt + pt if oir else pt + bt
    want = O.hash_join(jt, oir, bt, bc, pt, pc, bk, pk, sel, (), dflt)
    assert want.num_rows() > 0
    assert_same_multiset(Chunk.concat(got, out_types), want)


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("jt,oir", SHAPES)
@pytest.mark.parametrize("form", ["conds", "program"])
def test_keyed_conditions(lib, W, jt, oir, form):
    """OtherConditions as a comparison list and as a program; probe rows whose matches all fail the condition become miss
    rows of an outer join"""
    rng = np.random.default_rng(W + 10 * jt + oir + (form == "program") * 50)
    bt, pt = [INT64, INT64, BYTES], [INT64, INT64]
    nb, npr = 400 * W, 600 * W
    bc = [_col(rng, INT64, nb, 0, 50, 0.05), Column(INT64, rng.integers(0, 1000, nb)), _col(rng, BYTES, nb, 0, 99, 0.1)]
    pc = [_col(rng, INT64, npr, 0, 60, 0.05), Column(INT64, rng.integers(-200, 1200, npr))]
    n_left = len(bt) if oir else len(pt)
    bv, pv = (1, n_left + 1) if oir else (n_left + 1, 1)
    conds = [(LT, bv, pv)] if form == "conds" else ()
    program = [Func("ge", Func("plus", Col(pv), Const(0)), Col(bv))] if form == "program" else ()
    sel = rng.random(npr) > 0.1 if jt != INNER_JOIN else None
    got, *_ = _run(lib, W, bt, pt, [0], [0], bc, pc, jt, oir, sel, conds=conds, program=program, nullable=(True, True))
    out_types = bt + pt if oir else pt + bt
    if form == "conds":
        want = O.hash_join(jt, oir, bt, bc, pt, pc, [0], [0], sel, conds)
    else:
        want, _ = join_with_program("hash", jt, oir, bt, bc, pt, pc, [0], [0], program, sel)
    g = Chunk.concat(got, out_types)
    assert_same_multiset(g, want)
    if jt != INNER_JOIN:   # some outer row with matches had every pair fail: it is in the result once, as a miss row
        inner_c = 0 if oir else len(pt)
        assert (~g.cols[inner_c].not_null()).sum() > 0


@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("jt,oir", [(INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)])
@pytest.mark.parametrize("form", ["none", "conds", "program"])
def test_keyless_in_order(lib, W, jt, oir, form):
    """cross joins and ON a.x < b.y: rank r's output is exactly the single-GPU sequence of its probe shard against the
    build shards concatenated in rank order"""
    rng = np.random.default_rng(W * 7 + jt + (form == "conds") * 3 + (form == "program") * 5)
    bt, pt = [INT64, BYTES], [INT64, FLOAT64]
    nb, npr = 40 * W + 3, 90 * W + 1
    bc = [_col(rng, INT64, nb, 0, 100, 0.1), _col(rng, BYTES, nb, 0, 500, 0.1)]
    pc = [_col(rng, INT64, npr, 0, 100, 0.1), _col(rng, FLOAT64, npr, 0, 200, 0.0)]
    n_left = len(bt) if oir else len(pt)
    bx, px = (0, n_left) if oir else (n_left, 0)
    conds = [(LT, bx, px)] if form == "conds" else ()
    program = [Func("lt", Col(bx), Col(px))] if form == "program" else ()
    sel = rng.random(npr) > 0.2 if jt != INNER_JOIN else None
    dflt = [-1, None] if jt != INNER_JOIN else None
    got, bsh, psh, psel = _run(lib, W, bt, pt, [], [], bc, pc, jt, oir, sel, dflt, conds, program, nullable=(True, True))
    ball = B.concat(bsh, bt)
    for r in range(W):
        pr = list(psh[r])
        s = None if psel is None else psel[r]
        if form == "program":
            want, _ = keyless_join_with_program(jt, oir, bt, ball, pt, pr, program, s, dflt)
        else:
            want = keyless_hash_join(jt, oir, bt, ball, pt, pr, s, conds, dflt)
        assert_same_ordered(got[r], want)


@pytest.mark.parametrize("W", [3, 8])
@pytest.mark.parametrize("which", ["some", "all"])
@pytest.mark.parametrize("keyed", [True, False])
def test_empty_build_shards(lib, W, which, keyed):
    """build shards empty on some ranks or on every rank: an outer join still emits every probe row"""
    rng = np.random.default_rng(W + (which == "all") * 11 + keyed)
    bt, pt = [INT64, BYTES], [INT64, INT64]
    sizes = [0] * W if which == "all" else [0 if r % 2 else 37 + r for r in range(W)]
    nb = sum(sizes)
    bc = [_col(rng, INT64, nb, 0, 20, 0.0), _col(rng, BYTES, nb, 0, 50, 0.2)]
    pc = [_col(rng, INT64, 200 * W, 0, 25, 0.1), Column(INT64, np.arange(200 * W))]
    keys = [0] if keyed else []
    for jt, oir in ((INNER_JOIN, True), (LEFT_OUTER_JOIN, False)):
        got, bsh, psh, _ = _run(lib, W, bt, pt, keys, keys, bc, pc, jt, oir, bsizes=sizes, nullable=(True, True))
        out_types = bt + pt if oir else pt + bt
        if keyed:
            assert_same_multiset(Chunk.concat(got, out_types), O.hash_join(jt, oir, bt, bc, pt, pc, keys, keys))
        else:
            for r in range(W):
                assert_same_ordered(got[r], keyless_hash_join(jt, oir, bt, B.concat(bsh, bt), pt, list(psh[r])))


def test_two_epochs_reuse_one_exchange(lib):
    """a second step over the same regions (epoch 2) sees only its own rows"""
    W = 3
    rng = np.random.default_rng(5)
    bt, pt = [INT64, BYTES], [INT64, BYTES]
    em = B.Emulated(lib, W, 500, bt, pt, build_keys=[0, 1], probe_keys=[0, 1], byte_caps=[None, 8000])
    try:
        for step in range(2):
            nb, npr = 300 * W if step == 0 else 100 * W, 400 * W
            bc, pc = _side(rng, bt, [0, 1], nb, 0.0), _side(rng, pt, [0, 1], npr, 0.0)
            bsh = list(zip(*[B.shards(c, W) for c in bc]))
            psh = list(zip(*[B.shards(c, W) for c in pc]))
            got = em.step(bsh, psh)
            assert em.ex.epoch == step + 1
            assert_same_multiset(Chunk.concat(got, bt + pt), O.hash_join(0, True, bt, bc, pt, pc, [0, 1], [0, 1]))
    finally:
        em.free()


def _slots_and_regions_untouched(ex):
    for d in range(ex.world):
        assert not ex.read_slots(d).any(), "a refused push published a slot"
    raw = ex.buf.get(np.uint8)
    slot_block = ex.reg_off[0]
    for d in range(ex.world):
        assert np.all(raw[d * ex.bytes + slot_block:(d + 1) * ex.bytes] == X.SENTINEL_BYTE), "a refused push wrote a region"


def test_refusals_write_nothing(lib):
    """FLOAT32, offsets on the wrong columns, n > region_cap, bad destinations: refused before anything is enqueued"""
    W = 2
    bt = [INT64, BYTES]
    ex = B.EmuExchange(lib, W, BroadcastJoin.table_of(bt, 100, [None, 256], 1))
    cols = [DeviceColumn.from_host(Column(INT64, np.arange(50))), DeviceColumn.from_host(Column(BYTES, [b"ab"] * 50))]
    try:
        arr = (L.TQColumn * 2)(*[c.tq() for c in cols])
        dest, cnts = ex.push_tables(0, 0)
        caps = (C.c_int64 * 2)(0, 256)

        def push(types=(L.TQ_TYPE_INT64, L.TQ_TYPE_BYTES), a=arr, n=50, n_parts=W, d=dest, k=cnts, cap=ex.cap[0], slot=0):
            return lib.tq_partition_push_broadcast(len(types), a, (C.c_int32 * len(types))(*types), 1, n, n_parts, d, k, cap, caps, slot, 1)

        assert push(types=(L.TQ_TYPE_FLOAT32, L.TQ_TYPE_BYTES)) == L.TQ_ERR_UNSUPPORTED_TYPE
        assert push(types=(L.TQ_TYPE_INT64, L.TQ_TYPE_INT64)) == L.TQ_ERR_INVALID_ARG       # offsets on a non-BYTES column
        no_off = (L.TQColumn * 2)(arr[0], arr[1])
        no_off[1].offsets = None
        assert push(a=no_off) == L.TQ_ERR_INVALID_ARG                                      # a BYTES column without offsets
        assert push(n=ex.cap[0] + 1, cap=ex.cap[0]) == L.TQ_ERR_INVALID_ARG                  # n > region_cap
        assert push(n_parts=0) == L.TQ_ERR_INVALID_ARG
        assert push(n_parts=9) == L.TQ_ERR_INVALID_ARG
        holes = (C.c_void_p * len(dest))(*[None if i == 3 else dest[i] for i in range(len(dest))])
        assert push(d=holes) == L.TQ_ERR_INVALID_ARG
        assert push(k=(C.c_void_p * W)(cnts[0], None)) == L.TQ_ERR_INVALID_ARG
        assert push(slot=16) == L.TQ_ERR_INVALID_ARG
        X.compute_sync(lib)
        L.check(lib.tq_device_synchronize())
        _slots_and_regions_untouched(ex)
    finally:
        for c in cols:
            c.free()
        ex.free()


def test_byte_area_overflow_is_reported_not_joined(lib):
    """a shard whose cells exceed the byte cap: every slot it publishes reads ~0 and every rank's join raises"""
    W = 2
    bt, pt = [INT64, BYTES], [INT64]
    em = B.Emulated(lib, W, 100, bt, pt, build_keys=[0], probe_keys=[0], byte_caps=[None, 64])
    try:
        bsh = [[Column(INT64, np.arange(10)), Column(BYTES, [b"x" * 10] * 10)], [Column(INT64, np.arange(3)), Column(BYTES, [b"y"] * 3)]]
        psh = [[Column(INT64, np.arange(5))], [Column(INT64, np.arange(5))]]
        with pytest.raises(RuntimeError, match="region overflow"):
            em.step(bsh, psh)
        for d in range(W):
            assert int(em.ex.read_slots(d)[0, 0, 0]) == (1 << 64) - 1   # source 0 overflowed on every destination
            assert int(em.ex.read_slots(d)[0, 1, 0]) == 3
    finally:
        em.free()
