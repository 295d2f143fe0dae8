"""TEST INFRASTRUCTURE: CPU emulation of the product's gate programs (tests/emu/zk_emu.cu) —
the very __host__ __device__ functions the CUDA kernels call, run serially.  Lets the CPU
suite diff kernel logic against the oracle without a GPU.  The product never uses this."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "zk_emu.cu")
OUT = os.path.join(ROOT, "tests", "emu", "_build", "libzkemu.so")
_LIB = None
U64P = ctypes.POINTER(ctypes.c_uint64)
U32P = ctypes.POINTER(ctypes.c_uint32)
CHALLENGE = np.array([0x1234567, 0x89ABCDEF, 0x13579BDF, 0x02468ACE], dtype=np.uint64)


def lib():
    global _LIB
    if _LIB is None:
        csrc = os.path.join(ROOT, "zkevm-specs_b200", "csrc")
        deps = [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)] + [
            os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            # host-only build with plain g++: the gate programs are __host__ __device__ functions, the
            # kernels and other device-only declarations sit under #ifdef __CUDACC__ (20 s instead of the
            # 5 minutes nvcc needs to also generate sm_90a code nobody runs here)
            subprocess.run(["g++", "-x", "c++", "-std=c++17", "-O1", "-fPIC", "-shared", "-D__host__=", "-D__device__=",
                            "-D__forceinline__=inline", "-D__noinline__=__attribute__((noinline))", "-w",
                            "-o", OUT, SRC], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _p(a):
    return a.ctypes.data_as(U64P)


def check_evm(steps, bytecode, rw, fixed, row_begin=0, row_end=None, row_base=0, flags=0, n=None, challenge=None):
    steps, bytecode, rw, fixed = [np.ascontiguousarray(a) for a in (steps, bytecode, rw, fixed)]
    n = n or lib().emu_n_evm_constraints()
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    if row_end is None:
        row_end = steps.shape[1] - 1
    rc = lib().emu_check_evm(_p(steps), c(steps.shape[1]), _p(bytecode), c(bytecode.shape[1]), _p(rw),
                             c(rw.shape[1]), _p(fixed), c(fixed.shape[1]), c(row_begin), c(row_end), c(row_base),
                             ctypes.c_uint32(flags), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_bytecode(cols, push, keccak, r, row_begin=0, row_end=None, flags=1, n=22, challenge=None):
    cols, push, keccak = [np.ascontiguousarray(a) for a in (cols, push, keccak)]
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    if row_end is None:
        row_end = cols.shape[1]
    rc = lib().emu_check_bytecode(_p(cols), c(cols.shape[1]), _p(push), c(push.shape[1]), _p(keccak),
                                  c(keccak.shape[1]), _p(rr), c(row_begin), c(row_end), ctypes.c_uint32(flags),
                                  _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_copy(w, r, row_begin=0, row_end=None, flags=1, challenge=None):
    m = {k: np.ascontiguousarray(w[k]) for k in ("copy", "rw", "tx", "bytecode")}
    f = {k: np.ascontiguousarray(w[k], dtype=np.uint8) for k in ("copy_flags", "rw_flags", "tx_flags")}
    p8 = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if len(a) else None  # noqa: E731
    n = 64
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    n_rows = m["copy"].shape[1]
    if row_end is None:
        row_end = n_rows
    rc = lib().emu_check_copy(_p(m["copy"]), c(n_rows), p8(f["copy_flags"]), _p(m["rw"]), c(m["rw"].shape[1]),
                              p8(f["rw_flags"]), _p(m["bytecode"]), c(m["bytecode"].shape[1]), _p(m["tx"]),
                              c(m["tx"].shape[1]), p8(f["tx_flags"]), _p(rr), c(row_begin), c(row_end),
                              ctypes.c_uint32(flags), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_state(rows, flags, mpt, row_begin=0, row_end=None, cflags=1, challenge=None):
    rows, mpt = np.ascontiguousarray(rows), np.ascontiguousarray(mpt)
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    n = 128
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().emu_check_state(_p(rows), c(rows.shape[1]), flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                               _p(mpt), c(mpt.shape[1]), c(row_begin), c(row_end), ctypes.c_uint32(cflags), _p(ch),
                               ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def set_packed(on: bool) -> None:
    """store every witness / table matrix in the packed narrow-column format (fr.cuh:ld_col)"""
    ctypes.c_int.in_dll(lib(), "g_emu_packed").value = int(on)


def narrow_cols() -> int:
    return ctypes.c_longlong.in_dll(lib(), "g_emu_narrow_cols").value


def narrow_runs() -> int:
    """EVM checks that took the narrow form of the hot gate programs (StepCtx::narrow)"""
    return ctypes.c_longlong.in_dll(lib(), "g_emu_narrow_runs").value


def set_positional(on: bool) -> None:
    """toggle the positional (regular-table) lookup fast paths in the emulation; off = hash index only"""
    ctypes.c_int.in_dll(lib(), "g_emu_positional").value = int(on)


def positional_tables() -> int:
    """which tables of the last EVM / copy check took the positional lookup path: bit 0 bytecode, bit 1 rw; of the last
    bytecode-circuit check: bit 0 the push table"""
    return ctypes.c_int.in_dll(lib(), "g_emu_pos_ok").value


def heads_cap() -> int:
    """entries of the bytecode table's heads index (lookup.cuh ZK_HEADS_CAP)"""
    return int(lib().emu_heads_cap())


def check_evm_x(w, fixed, row_begin=0, row_end=None, row_base=0, flags=0, n=None, challenge=None):
    n = n or lib().emu_n_evm_constraints()
    m = {k: np.ascontiguousarray(w[k]) for k in ("steps", "bytecode", "rw", "copy", "keccak")}
    fixed = np.ascontiguousarray(fixed)
    rwf = np.ascontiguousarray(w["rw_flags"], dtype=np.uint8)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    if row_end is None:
        row_end = m["steps"].shape[1] - 1
    p8 = rwf.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if len(rwf) else None
    if w.get("tx") is not None or w.get("block") is not None:
        tx = np.ascontiguousarray(w["tx"] if w.get("tx") is not None else np.zeros((5, 0, 4)), dtype=np.uint64)
        blk = np.ascontiguousarray(w["block"] if w.get("block") is not None else np.zeros((4, 0, 4)), dtype=np.uint64)
        lib().emu_set_evm_context_tables(_p(tx), c(tx.shape[1]), _p(blk), c(blk.shape[1]))
    if w.get("wd") is not None or w.get("tx_flags") is not None or w.get("block_flags") is not None:  # BeginTx / EndTx / EndBlock
        p8_ = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if len(a) else None  # noqa: E731
        txf = np.ascontiguousarray(w.get("tx_flags") if w.get("tx_flags") is not None else np.zeros(0), dtype=np.uint8)
        blf = np.ascontiguousarray(w.get("block_flags") if w.get("block_flags") is not None else np.zeros(0), dtype=np.uint8)
        wd = np.ascontiguousarray(w["wd"] if w.get("wd") is not None else np.zeros((4, 0, 4)), dtype=np.uint64)
        check_evm_x._keep = [txf, blf, wd]
        lib().emu_set_evm_block_tables(p8_(txf), p8_(blf), _p(wd), c(wd.shape[1]))
    if w.get("exp") is not None:  # EXP: the exp table
        ex = np.ascontiguousarray(w["exp"], dtype=np.uint64)
        check_evm_x._keep_exp = ex
        lib().emu_set_evm_exp_table(_p(ex), c(ex.shape[1]))
    if w.get("aux") is not None:  # CREATE / CREATE2: StepState.aux_data as (step row, lo, hi) rows
        ax = np.ascontiguousarray(w["aux"], dtype=np.uint64)
        check_evm_x._keep_aux = ax
        lib().emu_set_evm_step_aux(_p(ax), c(ax.shape[1]))
    if w.get("flags") is not None:
        flags = int(w["flags"])
    rc = lib().emu_check_evm_x(_p(m["steps"]), c(m["steps"].shape[1]), _p(m["bytecode"]), c(m["bytecode"].shape[1]),
                               _p(m["rw"]), c(m["rw"].shape[1]), p8, _p(fixed), c(fixed.shape[1]), _p(m["copy"]),
                               c(m["copy"].shape[1]), _p(m["keccak"]), c(m["keccak"].shape[1]), c(row_begin), c(row_end),
                               c(row_base), ctypes.c_uint32(flags), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_exp(rows, row_begin=0, row_end=None, cflags=1):
    rows = np.ascontiguousarray(rows)
    ff = np.zeros(64, dtype=np.uint32)
    fc = np.zeros(64, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().emu_check_exp(_p(rows), c(rows.shape[1]), c(row_begin), c(row_end), ctypes.c_uint32(cflags),
                             ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_tx(rows, flags, keccak, r, row_begin=0, row_end=None, challenge=None):
    rows, keccak = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak)]
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    ff = np.zeros(16, dtype=np.uint32)
    fc = np.zeros(16, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().emu_check_tx(_p(rows), c(rows.shape[1]), flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _p(keccak),
                            c(keccak.shape[1]), _p(rr), c(row_begin), c(row_end), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_sig(rows, flags, keccak, r, row_begin=0, row_end=None, challenge=None):
    rows, keccak = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak)]
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    ff = np.zeros(16, dtype=np.uint32)
    fc = np.zeros(16, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().emu_check_sig(_p(rows), c(rows.shape[1]), flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _p(keccak),
                             c(keccak.shape[1]), _p(rr), c(row_begin), c(row_end), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


def check_pi(rows, keccak, gas, circuit_len, keccak_rand=255, byte_pow_base=255, row_begin=0, row_end=None, cflags=1, challenge=None):
    rows, keccak, gas = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak, gas)]
    ff = np.zeros(64, dtype=np.uint32)
    fc = np.zeros(64, dtype=np.uint64)
    c = ctypes.c_uint64
    ch = CHALLENGE if challenge is None else np.ascontiguousarray(challenge, dtype=np.uint64)
    if row_end is None:
        row_end = rows.shape[1]

    def lm(v):
        return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)

    rc = lib().emu_check_pi(_p(rows), c(rows.shape[1]), _p(keccak), c(keccak.shape[1]), _p(gas), c(gas.shape[1]),
                            _p(lm(keccak_rand)), _p(lm(byte_pow_base)), _p(lm(circuit_len)), c(row_begin), c(row_end),
                            ctypes.c_uint32(cflags), _p(ch), ff.ctypes.data_as(U32P), _p(fc))
    assert rc == 0
    return ff, fc


U8P = ctypes.POINTER(ctypes.c_uint8)


def _lm(v):
    return np.array([(int(v) >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def assign_bytecode(k, code, is_code_bits, code_offsets, hashes, r):
    """csrc/assign.cu bodies run serially: uint64[12][2^k][4]"""
    code, bits = np.ascontiguousarray(code, dtype=np.uint8), np.ascontiguousarray(is_code_bits, dtype=np.uint8)
    offs, hs = np.ascontiguousarray(code_offsets, dtype=np.uint64), np.ascontiguousarray(hashes, dtype=np.uint64)
    out = np.zeros((12, 1 << k, 4), dtype=np.uint64)
    rc = lib().emu_assign_bytecode(ctypes.c_uint32(k), ctypes.c_uint64(len(offs) - 1), code.ctypes.data_as(U8P), bits.ctypes.data_as(U8P),
                                   _p(offs), _p(hs), _p(_lm(r)), _p(out))
    assert rc == 0
    return out


def assign_state(ops):
    ops = np.ascontiguousarray(ops, dtype=np.uint64)
    assert ops.shape[0] == 15
    out = np.zeros((57, ops.shape[1], 4), dtype=np.uint64)
    assert lib().emu_assign_state(ctypes.c_uint64(ops.shape[1]), _p(ops), _p(out)) == 0
    return out


def assign_copy(events, data, bits, r):
    ev = np.ascontiguousarray(events, dtype=np.uint64).reshape(-1, 16)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    n = 2 * len(data)
    out = np.zeros((20, n, 4), dtype=np.uint64)
    fl = np.zeros(max(n, 1), dtype=np.uint8)
    b = None if bits is None else np.ascontiguousarray(bits, dtype=np.uint8)
    rc = lib().emu_assign_copy(ctypes.c_uint64(ev.shape[0]), _p(ev), data.ctypes.data_as(U8P),
                               None if b is None else b.ctypes.data_as(U8P), _p(_lm(r)), _p(out), fl.ctypes.data_as(U8P))
    assert rc == 0
    return out, fl[:n]
