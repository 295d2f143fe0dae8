"""ctypes loader for the CPU oracle (oracle/_build/libzkoracle.so) — TEST SIDE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may use the oracle."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
U64P = ctypes.POINTER(ctypes.c_uint64)
U32P = ctypes.POINTER(ctypes.c_uint32)

EXC_OF_CLASS = {
    0: "AssertionError",
    1: "LookupUnsatFailure",
    2: "LookupAmbiguousFailure",
    3: "ConstraintUnsatFailure",
    4: "ValueError",
    5: "NotImplementedError",
}


def build():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle")], check=True)


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(ROOT, "oracle", "_build", "libzkoracle.so")
        srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle"))
                if f.endswith((".c", ".h"))] + [os.path.join(ROOT, "include", "zk_constraints.h")]
        if not os.path.exists(path) or any(os.path.getmtime(s) > os.path.getmtime(path) for s in srcs):
            build()
        _LIB = ctypes.CDLL(path)
    return _LIB


def p64(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(U64P)


def limbs(v: int) -> np.ndarray:
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def from_limbs(a) -> int:
    return sum(int(a[i]) << (64 * i) for i in range(4))


def first_failure(first_fail: np.ndarray, classes):
    """(row, exception name) the reference would raise first: smallest (row, id)."""
    rows = first_fail.astype(np.int64)
    rows[first_fail == 0xFFFFFFFF] = 1 << 40
    r = int(rows.min())
    if r >= (1 << 40):
        return -1, ""
    cid = int(np.argmax(rows == r))
    return r, EXC_OF_CLASS[classes[cid]]


def check_bytecode(cols, push, keccak, r, row_begin=0, row_end=None, n=22):
    cols = np.ascontiguousarray(cols)
    push = np.ascontiguousarray(push)
    keccak = np.ascontiguousarray(keccak)
    n_rows = cols.shape[1]
    if row_end is None:
        row_end = n_rows
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    rc = lib().orc_check_bytecode(
        p64(cols), ctypes.c_uint64(n_rows), p64(push), ctypes.c_uint64(push.shape[1]),
        p64(keccak), ctypes.c_uint64(keccak.shape[1]), p64(rr), ctypes.c_uint64(row_begin),
        ctypes.c_uint64(row_end), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_evm(steps, bytecode, rw, fixed, row_begin=0, row_end=None, row_base=0, flags=0, n=None):
    steps, bytecode, rw, fixed = [np.ascontiguousarray(a) for a in (steps, bytecode, rw, fixed)]
    if n is None:
        n = lib().orc_n_constraints(3)
    n_steps = steps.shape[1]
    if row_end is None:
        row_end = n_steps - 1
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    rc = lib().orc_check_evm(p64(steps), c(n_steps), p64(bytecode), c(bytecode.shape[1]), p64(rw),
                             c(rw.shape[1]), p64(fixed), c(fixed.shape[1]), c(row_begin), c(row_end),
                             c(row_base), ctypes.c_uint32(flags), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def diff(ff, off):
    """the constraint ids where a first_fail array differs from the oracle's, with both values"""
    bad = np.nonzero(ff != off)[0]
    return f"ids {bad[:8].tolist()} cuda {ff[bad][:8].tolist()} oracle {off[bad][:8].tolist()}"


def same(got, want, what):
    """assert (first_fail, fail_count) == the oracle's, array for array"""
    ff, fc = got
    off, ofc = want
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc), \
        f"{what}: {diff(ff, off)}; counts differ at {np.nonzero(fc != ofc)[0][:8].tolist()}"


def constraint_classes(circuit_id):
    L = lib()
    n = L.orc_n_constraints(circuit_id)
    return [L.orc_constraint_class(circuit_id, i) for i in range(n)]


def _p8(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) if a is not None and len(a) else None


def check_copy(w, r, row_begin=0, row_end=None):
    """w: dict(copy, copy_flags, rw, rw_flags, tx, tx_flags, bytecode)"""
    m = {k: np.ascontiguousarray(w[k]) for k in ("copy", "rw", "tx", "bytecode")}
    f = {k: np.ascontiguousarray(w[k], dtype=np.uint8) for k in ("copy_flags", "rw_flags", "tx_flags")}
    n = lib().orc_n_constraints(2)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    n_rows = m["copy"].shape[1]
    if row_end is None:
        row_end = n_rows
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    rc = lib().orc_check_copy(p64(m["copy"]), c(n_rows), _p8(f["copy_flags"]), p64(m["rw"]), c(m["rw"].shape[1]),
                              _p8(f["rw_flags"]), p64(m["bytecode"]), c(m["bytecode"].shape[1]), p64(m["tx"]),
                              c(m["tx"].shape[1]), _p8(f["tx_flags"]), p64(rr), c(row_begin), c(row_end),
                              ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_state(rows, flags, mpt, row_begin=0, row_end=None):
    rows, mpt = np.ascontiguousarray(rows), np.ascontiguousarray(mpt)
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    n = lib().orc_n_constraints(1)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().orc_check_state(p64(rows), c(rows.shape[1]), _p8(flags), p64(mpt), c(mpt.shape[1]), c(row_begin),
                               c(row_end), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_evm_x(w, fixed, row_begin=0, row_end=None, row_base=0, flags=0):
    """w: dict(steps, bytecode, rw, rw_flags, copy, keccak) — EVM steps incl. SHA3 / CALLDATACOPY"""
    m = {k: np.ascontiguousarray(w[k]) for k in ("steps", "bytecode", "rw", "copy", "keccak")}
    fixed = np.ascontiguousarray(fixed)
    rwf = np.ascontiguousarray(w["rw_flags"], dtype=np.uint8)
    n = lib().orc_n_constraints(3)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = m["steps"].shape[1] - 1
    if w.get("tx") is not None or w.get("block") is not None:  # ORIGIN / GASPRICE / BlockCtx gadgets
        tx = np.ascontiguousarray(w["tx"] if w.get("tx") is not None else np.zeros((5, 0, 4)), dtype=np.uint64)
        blk = np.ascontiguousarray(w["block"] if w.get("block") is not None else np.zeros((4, 0, 4)), dtype=np.uint64)
        lib().orc_set_evm_context_tables(p64(tx), c(tx.shape[1]), p64(blk), c(blk.shape[1]))
    if w.get("wd") is not None or w.get("tx_flags") is not None or w.get("block_flags") is not None:  # BeginTx / EndTx / EndBlock: value type flags + withdrawals
        keep = getattr(check_evm_x, "_keep", None) or []
        txf = np.ascontiguousarray(w.get("tx_flags") if w.get("tx_flags") is not None else np.zeros(0), dtype=np.uint8)
        blf = np.ascontiguousarray(w.get("block_flags") if w.get("block_flags") is not None else np.zeros(0), dtype=np.uint8)
        wd = np.ascontiguousarray(w["wd"] if w.get("wd") is not None else np.zeros((4, 0, 4)), dtype=np.uint64)
        check_evm_x._keep = [txf, blf, wd]
        lib().orc_set_evm_block_tables(_p8(txf), _p8(blf), p64(wd), c(wd.shape[1]))
    if w.get("exp") is not None:  # EXP: the exp table
        ex = np.ascontiguousarray(w["exp"], dtype=np.uint64)
        check_evm_x._keep_exp = ex
        lib().orc_set_evm_exp_table(p64(ex), c(ex.shape[1]))
    if w.get("aux") is not None:  # CREATE / CREATE2: StepState.aux_data as (step row, lo, hi) rows
        ax = np.ascontiguousarray(w["aux"], dtype=np.uint64)
        check_evm_x._keep_aux = ax
        lib().orc_set_evm_step_aux(p64(ax), c(ax.shape[1]))
    if w.get("flags") is not None:
        flags = int(w["flags"])
    rc = lib().orc_check_evm_x(p64(m["steps"]), c(m["steps"].shape[1]), p64(m["bytecode"]), c(m["bytecode"].shape[1]),
                               p64(m["rw"]), c(m["rw"].shape[1]), _p8(rwf), p64(fixed), c(fixed.shape[1]),
                               p64(m["copy"]), c(m["copy"].shape[1]), p64(m["keccak"]), c(m["keccak"].shape[1]),
                               c(row_begin), c(row_end), c(row_base), ctypes.c_uint32(flags),
                               ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_exp(rows, row_begin=0, row_end=None):
    rows = np.ascontiguousarray(rows)
    n = lib().orc_n_constraints(4)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().orc_check_exp(p64(rows), c(rows.shape[1]), c(row_begin), c(row_end), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_tx(rows, flags, keccak, r, row_begin=0, row_end=None):
    """tx circuit Fr parts (oracle/tx.c): rows uint64[14][n][4], flags uint8[n], keccak uint64[5][k][4]"""
    rows, keccak = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak)]
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    n = lib().orc_n_constraints(5)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    rc = lib().orc_check_tx(p64(rows), c(rows.shape[1]), flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), p64(keccak),
                            c(keccak.shape[1]), p64(rr), c(row_begin), c(row_end), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


def check_sig(rows, flags, keccak, r, row_begin=0, row_end=None):
    """sig circuit Fr parts (oracle/tx.c): rows uint64[21][n][4], flags uint8[n] (bit 1 = ecdsa verdict)"""
    rows, keccak = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak)]
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    n = lib().orc_n_constraints(6)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rr = np.ascontiguousarray(r, dtype=np.uint64)
    rc = lib().orc_check_sig(p64(rows), c(rows.shape[1]), flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), p64(keccak),
                             c(keccak.shape[1]), p64(rr), c(row_begin), c(row_end), ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc


PI_KECCAK_RAND = 255  # module globals of the reference, pi_circuit.py:834-836
PI_BYTE_POW_BASE = 255


def check_pi(rows, keccak, gas, circuit_len, keccak_rand=PI_KECCAK_RAND, byte_pow_base=PI_BYTE_POW_BASE, row_begin=0, row_end=None):
    """public-inputs circuit (oracle/pi.c): rows uint64[28][n][4], keccak uint64[5][k][4], gas uint64[3][g][4]"""
    rows, keccak, gas = [np.ascontiguousarray(a, dtype=np.uint64) for a in (rows, keccak, gas)]
    n = lib().orc_n_constraints(7)
    ff = np.zeros(n, dtype=np.uint32)
    fc = np.zeros(n, dtype=np.uint64)
    c = ctypes.c_uint64
    if row_end is None:
        row_end = rows.shape[1]
    rc = lib().orc_check_pi(p64(rows), c(rows.shape[1]), p64(keccak), c(keccak.shape[1]), p64(gas), c(gas.shape[1]),
                            p64(limbs(keccak_rand)), p64(limbs(byte_pow_base)), p64(limbs(circuit_len)), c(row_begin), c(row_end),
                            ff.ctypes.data_as(U32P), p64(fc))
    assert rc == 0
    return ff, fc
