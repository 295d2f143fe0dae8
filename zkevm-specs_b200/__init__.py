"""zkevm-specs_b200 — H100-native constraint checker behind the zkevm-specs Python API.

Host side mirrors the reference's interface for the hot path (FQ, Word, tables, witness
builders, verify_*); every check runs in hand-written sm_90a CUDA behind the C-ABI of
include/zkcheck.h (libzkcheck.so, loaded with ctypes by `native`).  There is no CPU path.
"""
from . import native, packing  # noqa: F401
from .util import FQ, RLC, Word, WordOrValue  # noqa: F401

__all__ = ["native", "packing", "FQ", "RLC", "Word", "WordOrValue"]
