"""Key aiming for the hash tables (test infrastructure).

Both placement hashes of the library are bijections on 64-bit words (csrc/common.cuh):
  tqd::hash_key  xor-shift 32, multiply by an odd constant, xor-shift 32   (join tables: top bits = partition / sub-table,
                                                                            low 32 bits = home slot)
  tqd::mix64     murmur3 fmix64                                            (aggregation table: low bits = bucket;
                                                                            multi-GPU shard: bits 40.. = destination rank)
so a test can pick the hash value it wants and invert it into the key.  This module restates both hashes (numpy uint64,
vectorised), their inverses, the slot arithmetic of the join tables and the host-side table geometry of join.cu, so that an
edge test can compute — and assert — that its input really lies on the edge it is meant to exercise.
tests/test_hash_targets.py checks the restatement against the library's own functions."""
import numpy as np

U64 = np.uint64
EMPTY_KEY = 0xA5C3F00DDEADBEEF
MASK64 = (1 << 64) - 1

GOLDEN = 0x9E3779B97F4A7C15
FMIX_C1, FMIX_C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
GOLDEN_INV = pow(GOLDEN, -1, 1 << 64)
FMIX_C1_INV, FMIX_C2_INV = pow(FMIX_C1, -1, 1 << 64), pow(FMIX_C2, -1, 1 << 64)


def _u64(x):
    return np.asarray(x, dtype=np.int64).view(np.uint64) if np.asarray(x).dtype == np.int64 else np.asarray(x, dtype=np.uint64)


def _xs(k, s):
    return k ^ (k >> U64(s))


def hash_key(k):
    """tqd::hash_key over uint64 (or int64 bit patterns); returns uint64"""
    with np.errstate(over="ignore"):
        k = _xs(_u64(k), 32)
        k = k * U64(GOLDEN)
        return _xs(k, 32)


def hash_key_inv(h):
    with np.errstate(over="ignore"):
        h = _xs(_u64(h), 32)       # x ^ (x >> s) is its own inverse for s >= 32
        h = h * U64(GOLDEN_INV)
        return _xs(h, 32)


def mix64(k):
    """tqd::mix64 (murmur3 fmix64) over uint64 (or int64 bit patterns); returns uint64"""
    with np.errstate(over="ignore"):
        k = _xs(_u64(k), 33)
        k = k * U64(FMIX_C1)
        k = _xs(k, 33)
        k = k * U64(FMIX_C2)
        return _xs(k, 33)


def mix64_inv(h):
    with np.errstate(over="ignore"):
        h = _xs(_u64(h), 33)
        h = h * U64(FMIX_C2_INV)
        h = _xs(h, 33)
        h = h * U64(FMIX_C1_INV)
        return _xs(h, 33)


def as_int64(u):
    return np.asarray(u, dtype=np.uint64).view(np.int64)


# ---------------------------------------------------------------- join-table slot arithmetic (join.cu)
def home_slot(h, cap, shift):
    """join.cu home_slot: multiply-high of the low 32 hash bits by the capacity; 16-byte entries start on an even slot"""
    s = ((_u64(h) & U64(0xFFFFFFFF)) * U64(cap)) >> U64(32)
    return (s & ~U64(1)) if shift == 1 else s


def table_of(h, bits):
    """partition / sub-table index: the top `bits` hash bits (0 bits: the one table)"""
    return (_u64(h) >> U64(64 - bits)) if bits else np.zeros_like(_u64(h))


def slab_rows(n, parts, aos):
    """join.cu slab_rows: rows per slab of the optimistic scatter of n rows into `parts` bins"""
    slab = n // parts + n // parts // 4 + 4096
    return (slab + 31) & ~31 if aos else slab


PART_TARGET_ROWS = 150000
PART_MIN_BUILD_ROWS = 1 << 18
SA_MAX_PBITS, PART_MAX_BITS = 9, 12
BC_CLUSTER, BC_MAX_SLICE_BYTES = 8, 112 << 10
MAX_LOAD_PCT = 50


def stream_geometry(n, nb, part_rows=PART_TARGET_ROWS):
    """try_stream_build's host formulas for n unique NOT NULL build rows of nb columns; None when it does not try"""
    pbits = 0
    while (part_rows << pbits) < n:
        pbits += 1
    pbits = min(pbits, SA_MAX_PBITS)
    if pbits < 1:
        return None
    shift = 2 if nb > 2 else 1
    sbits = 0
    while True:
        if pbits + sbits > PART_MAX_BITS:
            return None
        mean = n / float((1 << pbits) << sbits)
        est_max = int(mean + 8.0 * np.sqrt(mean) + 64.0)
        cap = (est_max * 100 // MAX_LOAD_PCT + 15) & ~15
        if ((cap << shift) * 8) // BC_CLUSTER <= BC_MAX_SLICE_BYTES:
            break
        sbits += 1
    tbits = pbits + sbits
    bbits = min(tbits, SA_MAX_PBITS)
    return dict(pbits=pbits, sbits=sbits, tbits=tbits, bbits=bbits, lbits=tbits - bbits, shift=shift, cap=cap,
                slice=cap // BC_CLUSTER, max_rows=cap * MAX_LOAD_PCT // 100, n_bins=1 << bbits,
                bin_slab=slab_rows(n, 1 << bbits, True), n_slots=(1 << tbits) * cap)


def general_geometry(keys, nb, part_rows=PART_TARGET_ROWS, has_nulls=False):
    """join_build's general (non-streaming) table for these build keys (all valid, none equal to the empty marker counted)"""
    keys = _u64(keys)
    n = len(keys)
    row_words = nb + (1 if has_nulls else 0)
    shift = 2 if (row_words <= 4 and row_words > 2) else 1
    pbits, n_slots, cap = 0, 64, 0
    if n >= PART_MIN_BUILD_ROWS:
        P = 1
        while P * part_rows < n:
            P <<= 1
        pbits = min(int(P).bit_length() - 1, PART_MAX_BITS)
        regular = keys[keys != U64(EMPTY_KEY)]
        max_cnt = int(np.bincount(table_of(hash_key(regular), pbits).astype(np.int64), minlength=1 << pbits).max())
        cap = 64
        while cap * MAX_LOAD_PCT < max_cnt * 100:
            cap <<= 1
        if cap * (1 << pbits) > n * 12 + 4096:
            pbits, cap = 0, 0
        else:
            n_slots = (1 << pbits) * cap
    if pbits == 0:
        while n_slots < n * 2:
            n_slots <<= 1
        cap = n_slots
    return dict(pbits=pbits, shift=shift, cap=cap, n_slots=n_slots)


# ---------------------------------------------------------------- key generators
def _distinct(k):
    """sorted distinct values (a plain sort: numpy's hash-based unique is several times slower at 1e7 keys)"""
    k = np.sort(k)
    return k[np.concatenate([[True], k[1:] != k[:-1]])] if len(k) else k


def _finish(h, inv, rng, count, avoid_signbit, exclude):
    keys = inv(h)
    ok = keys != U64(EMPTY_KEY)
    if avoid_signbit:
        ok &= (keys >> U64(63)) == U64(0)
    keys = keys[ok]
    if exclude is not None:
        keys = keys[~np.isin(keys, _u64(exclude))]
    keys = _distinct(keys)
    rng.shuffle(keys)
    return keys[:count]


def join_keys(rng, count, top, top_bits, lo32_lo, lo32_hi, avoid_signbit=False, exclude=None):
    """`count` distinct int64 keys whose hash_key has its top `top_bits` bits equal to `top` and low 32 bits in
    [lo32_lo, lo32_hi); never the empty marker (nor a sign-bit key with avoid_signbit, nor a key in `exclude`)."""
    span = lo32_hi - lo32_lo
    assert 0 < span <= 1 << 32 and 0 <= top < (1 << top_bits) and top_bits <= 32
    m = count * 2 + 64
    mid_bits = 32 - top_bits
    mid = rng.integers(0, 1 << mid_bits, m, dtype=np.uint64) if mid_bits else np.zeros(m, np.uint64)
    lo = U64(lo32_lo) + rng.integers(0, span, m, dtype=np.uint64)
    h = (U64(top) << U64(64 - top_bits)) | (mid << U64(32)) | lo if top_bits else (mid << U64(32)) | lo
    keys = _finish(h, hash_key_inv, rng, count, avoid_signbit, exclude)
    assert len(keys) == count, "not enough distinct keys in the window"
    return as_int64(keys)


def join_keys_not_in_tables(rng, count, tables, bits, avoid_signbit=False, exclude=None):
    """random distinct int64 keys whose top `bits` hash bits are NOT one of `tables`"""
    out = np.zeros(0, np.uint64)
    bad = np.asarray(tables, np.uint64)
    while len(out) < count:
        h = rng.integers(0, 1 << 64, count - len(out) + 1024, dtype=np.uint64, endpoint=False)
        if len(bad):
            h = h[~np.isin(table_of(h, bits), bad)]
        k = hash_key_inv(h)   # distinct hashes are distinct keys
        ok = k != U64(EMPTY_KEY)
        if avoid_signbit:
            ok &= (k >> U64(63)) == U64(0)
        k = k[ok]
        if exclude is not None:
            k = k[~np.isin(k, _u64(exclude))]
        out = _distinct(np.concatenate([out, k]))
    rng.shuffle(out)
    return as_int64(out[:count])


def agg_keys(rng, count, low_bits, low_value, avoid_signbit=False, exclude=None):
    """`count` distinct int64 keys whose mix64 has its low `low_bits` bits equal to `low_value`"""
    m = count * 2 + 64
    h = (rng.integers(0, 1 << (64 - low_bits), m, dtype=np.uint64) << U64(low_bits)) | U64(low_value)
    keys = _finish(h, mix64_inv, rng, count, avoid_signbit, exclude)
    assert len(keys) == count
    return as_int64(keys)
