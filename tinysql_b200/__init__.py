"""tinysql_b200 — H100-native vectorized execution path for TinySQL's HashJoin / HashAgg /
vectorized expressions.  The product is libtinysql_b200.so (hand-written sm_90a CUDA behind the
C-ABI in include/tinysql_b200.h); this package is the thin host-side mirror of the reference's
operator interface used by the tests, the benchmark and the multi-GPU driver.
"""
from . import _lib
from ._lib import TQError, load

__all__ = ["_lib", "TQError", "load"]
