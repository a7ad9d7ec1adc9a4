"""util/chunk mirror: Column / Chunk laid out byte-for-byte like Go's chunk.Column
(util/chunk/column.go:28-34, Appendix A of SURVEY.md) on top of numpy buffers, plus the
pinned / device bridges the C-ABI works with.  Test-harness and benchmark plumbing only: the
operators themselves live in libtinysql_b200.so.
"""
import ctypes as C

import numpy as np

from . import _lib as L

MAX_CHUNK_SIZE = 1024  # DefMaxChunkSize sessionctx/variable/tidb_vars.go:241

INT64, UINT64, FLOAT64 = L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64, L.TQ_TYPE_FLOAT64
FLOAT32, BYTES = L.TQ_TYPE_FLOAT32, L.TQ_TYPE_BYTES  # FLOAT (4-byte slots) / var-len (offsets + data): join payload columns
_NP = {INT64: np.int64, UINT64: np.uint64, FLOAT64: np.float64, FLOAT32: np.float32}


def bitmap_bytes(n):
    return (n + 7) >> 3


def pack_not_null(not_null):
    """bool[n] -> nullBitmap bytes (bit i&7 of byte i>>3, 1 = NOT NULL; column.go:89-92)."""
    return np.packbits(np.asarray(not_null, dtype=bool), bitorder="little")


def unpack_not_null(bitmap, n):
    if bitmap is None:
        return np.ones(n, dtype=bool)
    return np.unpackbits(np.asarray(bitmap, dtype=np.uint8), count=n, bitorder="little").astype(bool)


class Column:
    """One fixed-width chunk.Column in host memory (8-byte slots; 4-byte for FLOAT).  Column(BYTES, [...]) and
    Column.empty(BYTES, ...) build the var-len flavour (VarColumn)."""

    def __new__(cls, tp=None, *args, **kw):
        if tp == L.TQ_TYPE_BYTES and cls is Column:
            return object.__new__(VarColumn)
        return object.__new__(cls)

    def __init__(self, tp, values, not_null=None):
        self.tp = tp
        v = np.ascontiguousarray(values)
        if v.dtype != _NP[tp]:
            v = v.astype(_NP[tp])
        self.values = v
        self.length = int(v.shape[0])
        self.bitmap = None if not_null is None else pack_not_null(not_null)

    @classmethod
    def empty(cls, tp, n):
        """Caller-allocated result column (data n*8 bytes + ceil(n/8) bitmap bytes)."""
        c = cls(tp, np.zeros(n, dtype=_NP[tp]))
        c.bitmap = np.zeros(bitmap_bytes(max(n, 1)), dtype=np.uint8)
        return c

    def not_null(self):
        return unpack_not_null(self.bitmap, self.length)

    def raw(self):
        if self.values.dtype.itemsize == 4:
            return self.values.view(np.uint32).astype(np.uint64)
        return self.values.view(np.uint64)

    def slice(self, lo, hi):
        nn = None if self.bitmap is None else self.not_null()[lo:hi]
        return Column(self.tp, self.values[lo:hi].copy(), nn)

    def tq(self, length=None):
        t = L.TQColumn()
        t.length = self.length if length is None else length
        t.data = self.values.ctypes.data if self.values.size else None
        t.null_bitmap = self.bitmap.ctypes.data if self.bitmap is not None else None
        t.offsets = None
        return t

    def tolist(self):
        nn = self.not_null()
        return [self.values[i].item() if nn[i] else None for i in range(self.length)]


class VarColumn(Column):
    """A var-len chunk.Column (util/chunk/column.go:28-34): int64 offsets[length+1] + the cells' bytes."""

    def __init__(self, tp, values, not_null=None):
        assert tp == BYTES
        self.tp = BYTES
        vals = [b"" if v is None else bytes(v) for v in values]
        if not_null is None and any(v is None for v in values):
            not_null = [v is not None for v in values]
        self.length = len(vals)
        self.offsets = np.zeros(self.length + 1, dtype=np.int64)
        if self.length:
            np.cumsum([len(v) for v in vals], out=self.offsets[1:])
        self.data = np.frombuffer(b"".join(vals), dtype=np.uint8).copy() if self.length else np.zeros(0, dtype=np.uint8)
        self.bitmap = None if not_null is None else pack_not_null(not_null)

    @classmethod
    def empty(cls, tp, n, nbytes=0):
        """Caller-allocated result column: offsets for n rows, `nbytes` of cell data, bitmap."""
        c = object.__new__(cls)
        c.tp, c.length = BYTES, n
        c.offsets = np.zeros(n + 1, dtype=np.int64)
        c.data = np.zeros(max(nbytes, 1), dtype=np.uint8)
        c.bitmap = np.zeros(bitmap_bytes(max(n, 1)), dtype=np.uint8)
        return c

    @property
    def values(self):
        """object array of the cells (bytes); NULL cells are b''"""
        return np.array([self.data[self.offsets[i]:self.offsets[i + 1]].tobytes() for i in range(self.length)], dtype=object)

    def raw(self):
        import hashlib
        return np.array([int.from_bytes(hashlib.blake2b(v, digest_size=8).digest(), "little") for v in self.values], dtype=np.uint64)

    def slice(self, lo, hi):
        nn = self.not_null()[lo:hi]
        return VarColumn(BYTES, [v if ok else None for v, ok in zip(self.values[lo:hi], nn)], None if self.bitmap is None else nn)

    def head(self, k):
        """first k rows of a filled result column"""
        nn = self.not_null()[:k]
        cells = [self.data[self.offsets[i]:self.offsets[i + 1]].tobytes() for i in range(k)]
        return VarColumn(BYTES, cells, nn)

    def tq(self, length=None):
        t = L.TQColumn()
        t.length = self.length if length is None else length
        t.data = self.data.ctypes.data if self.data.size else None
        t.null_bitmap = self.bitmap.ctypes.data if self.bitmap is not None else None
        t.offsets = self.offsets.ctypes.data
        return t

    def tolist(self):
        nn = self.not_null()
        v = self.values
        return [v[i] if nn[i] else None for i in range(self.length)]


def tq_array(cols, length=None):
    arr = (L.TQColumn * max(len(cols), 1))()
    for i, c in enumerate(cols):
        arr[i] = c.tq(length)
    return arr


class Chunk:
    """chunk.Chunk: a list of equally long columns (no sel vector on the operator boundary)."""

    def __init__(self, cols):
        self.cols = list(cols)

    def num_rows(self):
        return self.cols[0].length if self.cols else 0

    @classmethod
    def concat(cls, chunks, types):
        cols = []
        for ci, tp in enumerate(types):
            vals = [c.cols[ci].values for c in chunks if c.num_rows()]
            nns = [c.cols[ci].not_null() for c in chunks if c.num_rows()]
            if tp == BYTES:
                cells = [v if ok else None for va, na in zip(vals, nns) for v, ok in zip(va, na)]
                cols.append(VarColumn(BYTES, cells, np.concatenate(nns) if nns else None))
            elif vals:
                cols.append(Column(tp, np.concatenate(vals), np.concatenate(nns)))
            else:
                cols.append(Column(tp, np.zeros(0, dtype=_NP[tp]), np.zeros(0, dtype=bool)))
        return cls(cols)

    def rows(self):
        """list of tuples with None for NULL — the `testkit.Rows` view of a result."""
        lists = [c.tolist() for c in self.cols]
        return list(zip(*lists)) if lists else []


class DeviceColumn:
    """A column in HBM allocated through the C-ABI (tq_device_alloc)."""

    def __init__(self, tp, n, with_bitmap=True):
        lib = L.load()
        if tp in (FLOAT32, BYTES):
            raise ValueError("DeviceColumn holds 8-byte slots (INT64 / UINT64 / FLOAT64); DeviceColumn.from_host puts a var-len column "
                             "into a DeviceVarColumn; FLOAT32 columns enter through host chunks")
        self.tp, self.length = tp, int(n)
        self._data = C.c_void_p()
        L.check(lib.tq_device_alloc(max(self.length, 1) * 8, C.byref(self._data)))
        self._bm = C.c_void_p()
        self.bm_bytes = (((self.length + 63) >> 6) << 3) + 8  # 8-byte padded: kernels use 32-bit words
        if with_bitmap:
            L.check(lib.tq_device_alloc(self.bm_bytes, C.byref(self._bm)))
            L.check(lib.tq_memset_device(self._bm, 0, self.bm_bytes))

    @classmethod
    def from_host(cls, col):
        """the column in HBM: a DeviceColumn, or a DeviceVarColumn for a var-len (BYTES) column"""
        if col.tp == BYTES:
            return DeviceVarColumn.from_host(col)
        d = cls(col.tp, col.length, with_bitmap=col.bitmap is not None)
        lib = L.load()
        if col.length:
            L.check(lib.tq_memcpy_h2d(d._data, col.values.ctypes.data, col.values.nbytes))
            if col.bitmap is not None:
                L.check(lib.tq_memcpy_h2d(d._bm, col.bitmap.ctypes.data, bitmap_bytes(col.length)))
        return d

    def tq(self, length=None):
        t = L.TQColumn()
        t.length = self.length if length is None else length
        t.data = self._data.value
        t.null_bitmap = self._bm.value
        t.offsets = None
        return t

    def to_host(self, n=None):
        n = self.length if n is None else n
        return device_to_host(self.tp, self._data.value, self._bm.value, n)

    def free(self):
        lib = L.load()
        if self._data:
            lib.tq_device_free(self._data)
            self._data = C.c_void_p()
        if self._bm:
            lib.tq_device_free(self._bm)
            self._bm = C.c_void_p()


class DeviceVarColumn:
    """A var-len column in HBM (the TQ_MEM_DEVICE form of VarColumn): int64 offsets[length + 1] (8-byte aligned), the cells'
    bytes and the padded NOT-NULL bitmap of DeviceColumn.  `lead` puts that many filler bytes before the first cell, so
    offsets[0] == lead — the shape of a sliced column or of a cell range inside a larger buffer."""

    def __init__(self):
        self.tp, self.length, self.lead = BYTES, 0, 0
        self.off_bytes = self.data_bytes = 0
        self._off, self._data, self._bm = C.c_void_p(), C.c_void_p(), C.c_void_p()

    @classmethod
    def from_host(cls, col, lead=0):
        assert col.tp == BYTES
        lib = L.load()
        d = cls()
        d.length, d.lead = col.length, int(lead)
        offs = (np.asarray(col.offsets, dtype=np.int64) - int(col.offsets[0]) + d.lead) if col.length else np.full(1, d.lead, dtype=np.int64)
        nbytes = int(offs[-1])
        data = np.empty(max(nbytes, 1), dtype=np.uint8)
        data[: d.lead] = 0xEE
        data[d.lead: nbytes] = col.data[int(col.offsets[0]): int(col.offsets[0]) + nbytes - d.lead]
        d.off_bytes, d.data_bytes = offs.nbytes, data.nbytes
        L.check(lib.tq_device_alloc(offs.nbytes, C.byref(d._off)))
        L.check(lib.tq_memcpy_h2d(d._off, offs.ctypes.data, offs.nbytes))
        L.check(lib.tq_device_alloc(data.nbytes, C.byref(d._data)))
        L.check(lib.tq_memcpy_h2d(d._data, data.ctypes.data, data.nbytes))
        if col.bitmap is not None:
            bm_bytes = (((d.length + 63) >> 6) << 3) + 8
            L.check(lib.tq_device_alloc(bm_bytes, C.byref(d._bm)))
            L.check(lib.tq_memset_device(d._bm, 0, bm_bytes))
            if d.length:
                L.check(lib.tq_memcpy_h2d(d._bm, col.bitmap.ctypes.data, bitmap_bytes(d.length)))
        return d

    def tq(self, length=None):
        t = L.TQColumn()
        t.length = self.length if length is None else length
        t.data = self._data.value
        t.null_bitmap = self._bm.value
        t.offsets = self._off.value
        return t

    def to_host(self):
        return device_var_to_host(self._data.value, self._off.value, self._bm.value, self.length)

    def free(self):
        lib = L.load()
        for name in ("_off", "_data", "_bm"):
            p = getattr(self, name)
            if p:
                lib.tq_device_free(p)
                setattr(self, name, C.c_void_p())


def device_var_to_host(data_ptr, off_ptr, bm_ptr, n):
    """a var-len column in device memory (offsets[0] may be non-zero) copied into a VarColumn"""
    lib = L.load()
    offs = np.zeros(n + 1, dtype=np.int64)
    L.check(lib.tq_memcpy_d2h(offs.ctypes.data, off_ptr, offs.nbytes))
    nbytes = int(offs[n] - offs[0])
    data = np.zeros(max(nbytes, 1), dtype=np.uint8)
    if nbytes:
        L.check(lib.tq_memcpy_d2h(data.ctypes.data, data_ptr + int(offs[0]), nbytes))
    nn = None
    if bm_ptr and n:
        bm = np.zeros(bitmap_bytes(n), dtype=np.uint8)
        L.check(lib.tq_memcpy_d2h(bm.ctypes.data, bm_ptr, bm.nbytes))
        nn = unpack_not_null(bm, n)
    rel = offs - offs[0]
    cells = [data[rel[i]: rel[i + 1]].tobytes() for i in range(n)]
    return VarColumn(BYTES, [c if (nn is None or nn[i]) else None for i, c in enumerate(cells)], nn)


def device_to_host(tp, data_ptr, bm_ptr, n):
    lib = L.load()
    out = Column.empty(tp, n)
    if n:
        L.check(lib.tq_memcpy_d2h(out.values.ctypes.data, data_ptr, out.values.nbytes))
        if bm_ptr:
            L.check(lib.tq_memcpy_d2h(out.bitmap.ctypes.data, bm_ptr, bitmap_bytes(n)))
        else:
            out.bitmap = None
    return out


# ---------------------------------------------------------------------------------------------- chunk wire codec
def encode_chunk(types, cols):
    """chunk.Codec.Encode (util/chunk/codec.go:42-79) through the C-ABI: the wire bytes of the chunk."""
    lib = L.load()
    t = (C.c_int32 * max(len(types), 1))(*types)
    arr = tq_array(cols)
    need = C.c_int64(0)
    L.check(lib.tq_chunk_encoded_size(len(cols), t, arr, C.byref(need)))
    buf = np.zeros(max(need.value, 1), dtype=np.uint8)
    written = C.c_int64(0)
    L.check(lib.tq_chunk_encode(len(cols), t, arr, buf.ctypes.data, need.value, C.byref(written)))
    return buf[: written.value].tobytes()


def decode_chunk(buf, types):
    """chunk.Codec.DecodeToChunk (codec.go:92-143) through the C-ABI.  Returns (Chunk, bytes consumed); the columns are
    copied out of the views here (the views themselves are what a Go caller passes on to tq_join_put_probe)."""
    lib = L.load()
    raw = np.frombuffer(buf, dtype=np.uint8)
    t = (C.c_int32 * max(len(types), 1))(*types)
    out = (L.TQColumn * max(len(types), 1))()
    used = C.c_int64(0)
    L.check(lib.tq_chunk_decode(raw.ctypes.data if raw.size else None, raw.size, len(types), t, out, C.byref(used)))
    base = raw.ctypes.data
    cols = []
    for tp, v in zip(types, out):
        n = v.length
        nn = None
        if v.null_bitmap:
            o = v.null_bitmap - base
            nn = unpack_not_null(raw[o: o + bitmap_bytes(n)], n)
        if tp == BYTES:
            oo = v.offsets - base
            offs = raw[oo: oo + (n + 1) * 8].view(np.int64)
            d0 = (v.data - base) if v.data else 0
            cells = [raw[d0 + offs[i]: d0 + offs[i + 1]].tobytes() for i in range(n)]
            cols.append(VarColumn(BYTES, [c if (nn is None or nn[i]) else None for i, c in enumerate(cells)], nn))
        else:
            w = 4 if tp == FLOAT32 else 8
            d0 = (v.data - base) if v.data else 0
            cols.append(Column(tp, raw[d0: d0 + n * w].view(_NP[tp]).copy(), nn))
    return Chunk(cols), used.value


class DeviceChunk:
    """A chunk decoded straight into HBM (tq_chunk_decode_device): the wire bytes cross PCIe once and one kernel lays the
    columns out.  `tq_cols` are device tq_column views for the TQ_MEM_DEVICE entry points; reuse one DeviceChunk for a stream
    of wire chunks to decode without allocating."""

    def __init__(self):
        self.handle = C.c_void_p()
        self.types, self.tq_cols, self.consumed = [], None, 0

    def decode(self, buf, types):
        lib = L.load()
        raw = np.frombuffer(buf, dtype=np.uint8)
        t = (C.c_int32 * max(len(types), 1))(*types)
        out = (L.TQColumn * max(len(types), 1))()
        used = C.c_int64(0)
        L.check(lib.tq_chunk_decode_device(raw.ctypes.data if raw.size else None, raw.size, len(types), t, C.byref(self.handle), out, C.byref(used)))
        self.types, self.tq_cols, self.consumed = list(types), out, used.value
        return self

    def to_host(self):
        """copy the device columns back (tests / debugging)"""
        lib = L.load()
        cols = []
        for tp, v in zip(self.types, self.tq_cols):
            n = v.length
            nn = None
            if v.null_bitmap and n:
                bm = np.zeros(bitmap_bytes(n), dtype=np.uint8)
                L.check(lib.tq_memcpy_d2h(bm.ctypes.data, v.null_bitmap, bm.nbytes))
                nn = unpack_not_null(bm, n)
            if tp == BYTES:
                offs = np.zeros(n + 1, dtype=np.int64)
                L.check(lib.tq_memcpy_d2h(offs.ctypes.data, v.offsets, offs.nbytes))
                data = np.zeros(max(int(offs[n]), 1), dtype=np.uint8)
                if offs[n]:
                    L.check(lib.tq_memcpy_d2h(data.ctypes.data, v.data, int(offs[n])))
                cells = [data[offs[i]: offs[i + 1]].tobytes() for i in range(n)]
                cols.append(VarColumn(BYTES, [c if (nn is None or nn[i]) else None for i, c in enumerate(cells)], nn))
            else:
                vals = np.zeros(n, dtype=_NP[tp])
                if n:
                    L.check(lib.tq_memcpy_d2h(vals.ctypes.data, v.data, vals.nbytes))
                cols.append(Column(tp, vals, nn))
        return Chunk(cols)

    def free(self):
        if self.handle:
            L.load().tq_chunk_device_free(self.handle)
            self.handle = C.c_void_p()
