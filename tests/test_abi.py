"""CPU suite, part 2: the C-ABI library loads, exports every symbol include/tinysql_b200.h declares, the ctypes
struct layouts match the header, and — with no GPU — every entry point fails loudly instead of falling back."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tinysql_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tinysql_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tq_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_bound_and_exported():
    lib = L.load()
    names = declared_symbols()
    assert len(names) >= 45
    for n in names:
        assert n in L.SYMBOLS, f"{n} declared in the header but not bound in tinysql_b200/_lib.py"
        assert getattr(lib, n) is not None
    for n in L.SYMBOLS:
        assert n in names, f"{n} bound but not declared in include/tinysql_b200.h"
    out = subprocess.run(["nm", "-D", "--defined-only", L.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r"\bT (tq_[a-z0-9_]+)", out))
    assert set(names) <= exported


def test_struct_layouts_match_header():
    assert C.sizeof(L.TQColumn) == 32  # int64 + 3 pointers
    assert L.TQColumn.length.offset == 0 and L.TQColumn.null_bitmap.offset == 8 and L.TQColumn.offsets.offset == 16 and L.TQColumn.data.offset == 24
    assert C.sizeof(L.TQAggFunc) == 8
    # ... int64 probe_batch_rows, int32 flags (+ pad), then the two defaultInner pointers
    assert C.sizeof(L.TQJoinDesc) == 96 and L.TQJoinDesc.flags.offset == 72 and L.TQJoinDesc.default_inner_bits.offset == 80 and L.TQJoinDesc.default_inner_not_null.offset == 88
    assert C.sizeof(L.TQAggDesc) == 56


def test_sass_carries_sm90a_tma():
    """the built library holds sm_90a SASS with TMA bulk copies (UBLKCP) — evidence, not a perf claim"""
    if not os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "UBLKCP" in out


def _has_gpu():
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU ") > 0
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="only meaningful without a GPU")
def test_no_gpu_means_loud_failure_not_cpu_fallback():
    lib = L.load()
    assert lib.tq_init(0) == L.TQ_ERR_NO_DEVICE
    assert "no CPU fallback" in L.last_error()
    from tinysql_b200 import expression as E
    from tinysql_b200.chunk import INT64, Column
    with pytest.raises(L.TQError) as ei:
        E.vec_compare_int(E.LT, Column(INT64, [1, 2]), Column(INT64, [2, 1]))
    assert ei.value.status == L.TQ_ERR_NO_DEVICE
    h = C.c_void_p()
    t = (C.c_int32 * 1)(1)
    k = (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(0, 0, 1, t, 1, t, 1, k, k, 0)
    assert lib.tq_join_create(C.byref(d), C.byref(h)) == L.TQ_ERR_NO_DEVICE and not h.value


def test_product_never_references_the_oracle():
    """oracle/ is test infrastructure: the product library must not link it and the package must not import it"""
    out = subprocess.run(["ldd", L.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in out
    pkg = os.path.join(ROOT, "tinysql_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle_py" not in src and "liboracle" not in src and "orc_" not in src, f
