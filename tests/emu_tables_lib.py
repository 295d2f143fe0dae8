"""TEST INFRASTRUCTURE: CPU emulation of the tx-table and copy-table builders (tests/emu/zk_emu_tables.cu) — the
__host__ __device__ bodies of csrc/assign.cu that k_assign_tx_* and k_copy_table_* run, called serially.  The product
never uses this."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "zk_emu_tables.cu")
OUT = os.path.join(ROOT, "tests", "emu", "_build", "libzkemu_tables.so")
_LIB = None
COPY_TABLE_ERRORS = {-2: "Not enough rows in copy circuit", -3: "Invalid copy circuit"}


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
        _LIB.emu_tx_table_rows.restype = ctypes.c_int64
        _LIB.emu_assign_copy_table.restype = ctypes.c_int64
    return _LIB


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def tx_table_widths(records, offsets):
    """the column widths zk_assign_tx_table picks, or None where it rejects the input"""
    rec = np.ascontiguousarray(records, dtype=np.uint64).reshape(-1, 11, 4)
    offs = np.ascontiguousarray(offsets, dtype=np.uint64)
    w = np.zeros(5, dtype=np.uint8)
    n = lib().emu_tx_table_rows(ctypes.c_uint64(rec.shape[0]), _p(rec), _p(offs), _p(w))
    return None if n < 0 else w


def assign_tx_table(records, call_data, offsets):
    """zk_assign_tx_table's bodies run serially: (table uint64[5][rows][4], flags uint8[rows]), or None where the device
    call rejects the input"""
    rec = np.ascontiguousarray(records, dtype=np.uint64).reshape(-1, 11, 4)
    offs = np.ascontiguousarray(offsets, dtype=np.uint64)
    cd = np.ascontiguousarray(call_data, dtype=np.uint8)
    if len(cd) == 0:
        cd = np.zeros(1, dtype=np.uint8)
    n = lib().emu_tx_table_rows(ctypes.c_uint64(rec.shape[0]), _p(rec), _p(offs), None)
    if n < 0:
        return None
    out = np.zeros((5, n, 4), dtype=np.uint64)
    flags = np.zeros(max(n, 1), dtype=np.uint8)
    rc = lib().emu_assign_tx_table(ctypes.c_uint64(rec.shape[0]), _p(rec), _p(cd), _p(offs), ctypes.c_uint64(n),
                                   _p(out), _p(flags))
    assert rc == 0
    return out, flags[:n]


def assign_copy_table(circuit):
    """zk_assign_copy_table's bodies run serially over a canonical copy circuit uint64[20][n][4]: the table
    uint64[14][rows][4], or the reference's assert message (a str) where the device call returns it"""
    c = np.ascontiguousarray(circuit, dtype=np.uint64)
    n = c.shape[1]
    out = np.zeros(14 * max(n, 1) * 4, dtype=np.uint64)  # [14][table rows][4], table rows <= n
    rc = lib().emu_assign_copy_table(ctypes.c_uint64(n), _p(c) if n else None, ctypes.c_uint64(n), _p(out))
    if rc < 0:
        return COPY_TABLE_ERRORS[int(rc)]
    return out[:14 * rc * 4].reshape(14, rc, 4)
