"""Key aiming for the two key dictionaries (test infrastructure), the companion of hash_targets.py.

  dict.cu     KeyDict: value -> dense id, slot = mix64(v) & (n_slots - 1), linear probing with wrap-around; MultiKeyEncoder
              folds the ids of N key columns into one word (pair = id_a << 32 | id_b, re-encoded by a pair dictionary between
              folds).
  strdict.cu  StringDict: byte string -> dense id, slot = sd_warp_hash(bytes) & (n_slots - 1); equality is decided on the
              bytes, the hash is only a filter.

This module restates sd_warp_hash, the slot and growth rules of both dictionaries and their id conventions, so that an edge test
can build inputs that provably share one probe chain (at the table's last slot, so the chain wraps to slot 0) and assert that
they still do at every table size the test reaches.  tests/test_emu_dicts.py checks the restatement against the library."""
import numpy as np

from hash_targets import EMPTY_KEY, FMIX_C1, GOLDEN, MASK64, U64, mix64, mix64_inv

# ---------------------------------------------------------------- id conventions (dict.cuh, strdict.cuh)
MK_ID_NULL, MK_ID_EMPTYVAL, MK_ID_MISS = 0, 1, 0xFFFFFFFF   # NULL under GROUP BY / the marker value / absent or NULL in a join
MK_PAIR_MISS = MASK64                                       # the folded word of a row without a valid encoding
DICT_MARKER = EMPTY_KEY                                     # KeyDict's empty-slot marker: the value 0xA5C3F00DDEADBEEF gets id 1
MK_FIRST_ID = 2                                             # regular ids are dense from here, in order of first claim
SD_ID_MISS = MASK64                                         # StringDict lookup of a string it does not hold

# ---------------------------------------------------------------- table geometry
KD_MIN_SLOTS, KD_SUB_BATCH = 1 << 12, 1 << 24
SD_MIN_SLOTS = 1 << 10
AGG_BATCH_ROWS = 1 << 22          # agg.cu batch_rows: host chunks are staged and encoded in device batches of this many rows


def _grow(n_slots, minimum, need):
    want = n_slots or minimum
    while want < 2 * need:
        want <<= 1
    return want


def kd_grow(n_slots, count, extra):
    """KeyDict::ensure: the table after making room for `extra` more values beside `count` (it never shrinks)"""
    return _grow(n_slots, KD_MIN_SLOTS, count + extra)


def kd_insert_slots(n_slots, count, rows, new_per_sub_batch):
    """KeyDict::insert of `rows` rows cut into KD_SUB_BATCH sub-batches; new_per_sub_batch[i] = distinct values that sub-batch
    adds.  Returns (n_slots, count) after the insert and the list of table sizes in force during each sub-batch."""
    sizes = []
    for i, off in enumerate(range(0, rows, KD_SUB_BATCH)):
        n_slots = kd_grow(n_slots, count, min(KD_SUB_BATCH, rows - off))
        sizes.append(n_slots)
        count += new_per_sub_batch[i]
    return n_slots, count, sizes


def sd_grow(n_slots, count, extra):
    """StringDict::ensure: an insert of a batch of `extra` rows makes room for all of them"""
    return _grow(n_slots, SD_MIN_SLOTS, count + extra)


def kd_slot(v, n_slots):
    return mix64(v) & U64(n_slots - 1)


def sd_slot(h, n_slots):
    return int(h) & (n_slots - 1)


# ---------------------------------------------------------------- sd_warp_hash restated
SD_SEED, SD_LANE = 0x9E3779B97F4A7C15, 0xD6E8FEB86659FD93


def _mix64_int(x):
    x ^= x >> 33
    x = (x * FMIX_C1) & MASK64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & MASK64
    return x ^ (x >> 33)


def _fold(h, w):
    h = ((h ^ w) * FMIX_C1) & MASK64
    return h ^ (h >> 32)


def _word(b, o):
    return int.from_bytes(b[o:o + 8], "little")   # a short last word is zero-extended


def _lane_state(b, lane):
    h = (SD_SEED + lane * SD_LANE) & MASK64
    for o in range(8 * lane, len(b), 256):
        h = _fold(h, _word(b, o))
    return h


def sd_hash(b):
    """sd_warp_hash: lane l folds the 8-byte words at 8l, 8l + 256, ...; the lanes' mixed states are summed"""
    b = bytes(b)
    s = 0
    for lane in range(32):
        s = (s + _mix64_int(_lane_state(b, lane))) & MASK64
    return _mix64_int(s ^ ((len(b) * GOLDEN) & MASK64))


def sd_hashes(cells):
    return np.array([sd_hash(c) for c in cells], dtype=np.uint64)


# ---------------------------------------------------------------- aimers
def chain_values(rng, count, low_bits=24, exclude=None):
    """`count` distinct uint64 values whose mix64 has its low `low_bits` bits all ones: one chain at the last slot of every KeyDict
    of up to 2^low_bits slots.  Never the marker value nor MK_PAIR_MISS."""
    h = (rng.integers(0, 1 << (64 - low_bits), count * 2 + 64, dtype=np.uint64) << U64(low_bits)) | U64((1 << low_bits) - 1)
    v = mix64_inv(h)                                   # distinct hashes are distinct values
    v = v[(v != U64(EMPTY_KEY)) & (v != U64(MK_PAIR_MISS))]
    if exclude is not None:
        v = v[~np.isin(v, np.asarray(exclude, dtype=np.uint64))]
    v = np.unique(v)
    rng.shuffle(v)
    assert len(v) >= count
    return v[:count]


def chain_strings(rng, count, length, low_bits=16, template=None, vary_at=0):
    """`count` distinct byte strings of `length` bytes whose sd_warp_hash has its low `low_bits` bits all ones: one chain at the
    last slot of every StringDict of up to 2^low_bits slots.  The strings equal `template` (random bytes by default) except in the
    8-byte word at offset `vary_at` (a multiple of 8), found by brute force over that word: the other lanes' contribution to the
    sum is computed once, the varied lane is folded for a whole vector of candidate words at a time."""
    assert vary_at % 8 == 0 and vary_at < length
    t = bytearray(rng.integers(0, 256, length, dtype=np.uint8).tobytes() if template is None else template)
    assert len(t) == length
    lane = (vary_at // 8) % 32
    others = 0
    for l in range(32):
        if l != lane:
            others = (others + _mix64_int(_lane_state(t, l))) & MASK64
    wbytes = min(8, length - vary_at)
    space = 1 << (8 * wbytes)
    want = U64((1 << low_bits) - 1)
    offs = list(range(8 * lane, length, 256))
    found = np.zeros(0, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for _ in range(256):
            w = rng.integers(0, space, 1 << 22, dtype=np.uint64) if space < (1 << 64) else rng.integers(0, 1 << 64, 1 << 22, dtype=np.uint64)
            h = np.full(len(w), U64((SD_SEED + lane * SD_LANE) & MASK64))
            for o in offs:
                x = w if o == vary_at else U64(_word(t, o))
                h = (h ^ x) * U64(FMIX_C1)
                h = h ^ (h >> U64(32))
            fin = mix64((U64(others) + mix64(h)) ^ U64((length * GOLDEN) & MASK64))
            found = np.unique(np.concatenate([found, w[(fin & want) == want]]))
            if len(found) >= count:
                break
    assert len(found) >= count, "not enough strings on the chain (the varied word is too short)"
    rng.shuffle(found)
    out = []
    for w in found[:count].tolist():
        s = bytearray(t)
        s[vary_at:vary_at + wbytes] = int(w).to_bytes(8, "little")[:wbytes]
        out.append(bytes(s))
    return out


def colliding_twin(s, at=256):
    """A different string of the same length with exactly the same sd_warp_hash: it differs from `s` in the 8-byte words at
    offsets `at` and `at + 256` (one lane folds both, and the second fold cancels the difference the first one made).  Byte
    at+1 is flipped; everything before `at` is shared, so only a byte-exact comparison past `at` tells the two apart."""
    s = bytes(s)
    assert at % 8 == 0 and len(s) >= at + 256 + 8
    lane = (at // 8) % 32
    h = (SD_SEED + lane * SD_LANE) & MASK64
    for o in range(8 * lane, at, 256):
        h = _fold(h, _word(s, o))
    w1 = _word(s, at)
    w1t = w1 ^ (0x01 << 8)
    st, stt = _fold(h, w1), _fold(h, w1t)
    w2t = _word(s, at + 256) ^ st ^ stt
    t = bytearray(s)
    t[at:at + 8] = w1t.to_bytes(8, "little")
    t[at + 256:at + 264] = w2t.to_bytes(8, "little")
    return bytes(t)


def differ_at(base, offset, count):
    """`count` strings equal to `base` except for the byte at `offset` (`base` itself first)"""
    base = bytes(base)
    out = [base]
    for k in range(1, count):
        t = bytearray(base)
        t[offset] = (t[offset] + k) & 0xFF
        out.append(bytes(t))
    return out


def trailing_nuls(base, count):
    """base, base + b"\\0", base + b"\\0\\0", ..."""
    return [bytes(base) + b"\0" * k for k in range(count)]


# ---------------------------------------------------------------- string columns from integer ids
def cells_from_table(v_off, v_data, ids, rows_per_step=1 << 20):
    """offsets (int64, len(ids) + 1) and bytes (uint8) of the cells whose ids are `ids`, cell i of the table being
    v_data[v_off[i]:v_off[i + 1]]; built with numpy, a bounded number of rows at a time"""
    ids = np.asarray(ids, dtype=np.int64)
    cl = v_off[1:][ids] - v_off[:-1][ids]
    off = np.zeros(len(ids) + 1, dtype=np.int64)
    np.cumsum(cl, out=off[1:])
    out = np.empty(off[-1], dtype=np.uint8)
    for lo in range(0, len(ids), rows_per_step):
        hi = min(len(ids), lo + rows_per_step)
        # byte j of cell i is v_data[v_off[ids[i]] + j]
        src = np.repeat(v_off[ids[lo:hi]] - off[lo:hi], cl[lo:hi]) + np.arange(off[lo], off[hi], dtype=np.int64)
        out[off[lo]:off[hi]] = v_data[src]
    return off, out


def cells_from_vocab(vocab, ids):
    """cells_from_table over a list of byte strings"""
    v_off = np.zeros(len(vocab) + 1, dtype=np.int64)
    np.cumsum([len(v) for v in vocab], out=v_off[1:])
    v_data = np.frombuffer(b"".join(vocab), dtype=np.uint8) if v_off[-1] else np.zeros(0, np.uint8)
    return cells_from_table(v_off, v_data, ids)
