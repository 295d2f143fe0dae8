"""TEST INFRASTRUCTURE: CPU emulation of the public-inputs builder (tests/emu/zk_emu_pi.cu) — the __host__ __device__
bodies of csrc/assign.cu that the k_assign_pi_* kernels run, called serially.  The product never uses this."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "zk_emu_pi.cu")
OUT = os.path.join(ROOT, "tests", "emu", "_build", "libzkemu_pi.so")
_LIB = None
N_BLOCK_BYTES, SLOT_BYTES, WD_BYTES = 8454, 336, 56  # the stream's fixed part (block + empty tx row), a tx slot, a withdrawal


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
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))


def _limbs(v: int) -> np.ndarray:
    return np.array([(int(v) >> (64 * i)) & ((1 << 64) - 1) for i in range(4)], dtype=np.uint64)


def fr_inv(v: int) -> int:
    out = np.zeros(4, dtype=np.uint64)
    lib().emu_fr_inv(_p(_limbs(v)), _p(out))
    return sum(int(x) << (64 * i) for i, x in enumerate(out))


def assign_pi(raw: bytes, max_txs: int, max_cd: int, max_wd: int, keccak_rand: int, byte_pow_base: int):
    """zk_assign_pi_circuit's bodies run serially: (rows uint64[28][n][4], keccak table uint64[5][2][4], calldata gas
    table uint64[3][1 + used calldata bytes][4], digest Word as an int), or None where the device call rejects the input"""
    n = len(raw)
    buf = np.frombuffer(bytes(raw), dtype=np.uint8).copy() if n else np.zeros(1, dtype=np.uint8)
    rows = np.zeros((28, n, 4), dtype=np.uint64)
    kec = np.zeros((5, 2, 4), dtype=np.uint64)
    cdl = [int.from_bytes(bytes(raw[N_BLOCK_BYTES + SLOT_BYTES * k + 256:N_BLOCK_BYTES + SLOT_BYTES * k + 264]), "big")
           for k in range(max_txs)] if n >= N_BLOCK_BYTES + SLOT_BYTES * max_txs else []
    n_gas = 1 + min(sum(cdl), max_cd)  # the zero row + one row per used calldata byte
    gas = np.zeros((3, n_gas, 4), dtype=np.uint64)
    word = np.zeros(4, dtype=np.uint64)
    c = ctypes.c_uint64
    rc = lib().emu_assign_pi(c(max_txs), c(max_cd), c(max_wd), ctypes.c_void_p(buf.ctypes.data), c(n),
                             _p(_limbs(keccak_rand)), _p(_limbs(byte_pow_base)), _p(rows), _p(kec), c(n_gas), _p(gas), _p(word))
    if rc != 0:
        return None
    lo = int(word[0]) | int(word[1]) << 64
    hi = int(word[2]) | int(word[3]) << 64
    return rows, kec, gas, lo | hi << 128
