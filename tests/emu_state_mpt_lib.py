"""TEST INFRASTRUCTURE: CPU emulation of zk_assign_state_circuit_mpt (tests/emu/zk_emu_state_mpt.cu) — the
__host__ __device__ bodies of csrc/assign.cu that k_state_mpt_* and k_assign_state_derive run, called serially.  The
product never uses this."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "zk_emu_state_mpt.cu")
OUT = os.path.join(ROOT, "tests", "emu", "_build", "libzkemu_state_mpt.so")
_LIB = None
# the rejections, by the return code of emu_assign_state_mpt, as the exception the mirror raises
ERRORS = {-1: "address", -2: "KeyError", -3: "AssertionError"}


def lib():
    global _LIB
    if _LIB is None:
        csrc = os.path.join(ROOT, "zkevm-specs_b200", "csrc")
        deps = [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)] + [
            os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            # host-only build with plain g++, as tests/emu_lib.py: the kernels sit under #ifdef __CUDACC__
            subprocess.run(["g++", "-x", "c++", "-std=c++17", "-O2", "-fPIC", "-shared", "-D__host__=", "-D__device__=",
                            "-D__forceinline__=inline", "-D__noinline__=__attribute__((noinline))", "-w",
                            "-o", OUT, SRC], check=True)
        _LIB = ctypes.CDLL(OUT)
        _LIB.emu_state_mpt_home_slot.restype = ctypes.c_uint64
    return _LIB


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def home_slot(key_cells, n_ops: int) -> int:
    """the slot zk_assign_state_circuit_mpt's hash table first tries for an MPT key (address, field_tag, storage_key
    lo, hi as ints) when it assigns n_ops operations"""
    k = np.array([[(int(v) >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in key_cells], dtype=np.uint64)
    return int(lib().emu_state_mpt_home_slot(_p(k), ctypes.c_uint64(n_ops)))


def assign_state_mpt(ops13, flags=None):
    """zk_assign_state_circuit_mpt's bodies run serially over canonical cells uint64[13][n][4]: (rows uint64[57][n][4],
    mpt uint64[12][U][4]), or (name of the rejection, failing op) where the device call rejects the input: "KeyError",
    "AssertionError" (the mirror's exceptions) or "address" (failing op None)"""
    ops = np.ascontiguousarray(ops13, dtype=np.uint64)
    assert ops.ndim == 3 and ops.shape[0] == 13 and ops.shape[2] == 4
    n = ops.shape[1]
    fl = None if flags is None else np.ascontiguousarray(flags, dtype=np.uint8)
    assert fl is None or fl.shape == (n,)
    rows = np.zeros((57, n, 4), dtype=np.uint64)
    mpt = np.zeros(12 * max(n, 1) * 4, dtype=np.uint64)  # [12][U][4], U <= n
    n_upd, fail = ctypes.c_uint64(0), ctypes.c_uint64(0)
    buf = ops if n else np.zeros((13, 1, 4), dtype=np.uint64)
    rc = lib().emu_assign_state_mpt(ctypes.c_uint64(n), _p(buf), None if fl is None or n == 0 else _p(fl), _p(rows),
                                    _p(mpt), ctypes.byref(n_upd), ctypes.byref(fail))
    if rc < 0:
        return ERRORS[rc], (None if rc == -1 else int(fail.value))
    u = int(n_upd.value)
    return rows, mpt[:12 * u * 4].reshape(12, u, 4)
