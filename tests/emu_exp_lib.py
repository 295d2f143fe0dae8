"""TEST INFRASTRUCTURE: CPU emulation of the exp-circuit builder (tests/emu/zk_emu_exp.cu) — the __host__ __device__
bodies of csrc/assign.cu that k_assign_exp_chain / k_assign_exp_rows run, called serially.  The product never uses this."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "zk_emu_exp.cu")
OUT = os.path.join(ROOT, "tests", "emu", "_build", "libzkemu_exp.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        csrc = os.path.join(ROOT, "zkevm-specs_b200", "csrc")
        deps = [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)] + [
            os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            # host-only build with plain g++, as tests/emu_lib.py: the kernels sit under #ifdef __CUDACC__
            subprocess.run(["g++", "-x", "c++", "-std=c++17", "-O1", "-fPIC", "-shared", "-D__host__=", "-D__device__=",
                            "-D__forceinline__=inline", "-D__noinline__=__attribute__((noinline))", "-w",
                            "-o", OUT, SRC], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def exp_event_rows(exponent: int) -> int:
    """rows ExpCircuit.add_event emits for an exponent"""
    return 0 if exponent < 2 else (exponent.bit_length() - 1) + (bin(exponent).count("1") - 1)


def assign_exp(events, n_rows_min=0):
    """the exp bodies run serially on zk_assign_exp_circuit's events uint64[n][12]: (circuit uint64[21][rows][4], exp
    table uint64[11][table rows][4])"""
    ev = np.ascontiguousarray(events, dtype=np.uint64).reshape(-1, 12)
    used = sum(exp_event_rows(sum(int(x) << (64 * i) for i, x in enumerate(ev[k, 4:8]))) for k in range(ev.shape[0]))
    n = max(used, int(n_rows_min))
    n_table = used + (1 if n > used else 0)
    out = np.zeros((21, n, 4), dtype=np.uint64)
    tab = np.zeros((11, n_table, 4), dtype=np.uint64)
    c = ctypes.c_uint64
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))  # noqa: E731
    rc = lib().emu_assign_exp(c(ev.shape[0]), p(ev), c(int(n_rows_min)), c(n), c(n_table), p(out), p(tab))
    assert rc == 0
    return out, tab
