"""CPU-side diff of the product's gate programs (run through tests/emu, the same
__host__ __device__ code the CUDA kernels execute) against the oracle and the reference
goldens.  This is a pre-GPU safety net; the -m gpu tests repeat it through the real kernels."""
import numpy as np

import emu_lib
import golden_util
import oracle_lib
from zkevm_specs_b200 import synth
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix


def test_emu_bytecode_equals_oracle_on_goldens():
    """both push-table paths: positional (the regular table, verified on the fly) and hash index only"""
    for name, k, cols, push, kec, r, exp_row, exp_exc in golden_util.bytecode_vectors():
        off, ofc = oracle_lib.check_bytecode(cols, push, kec, r)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_bytecode(cols, push, kec, r)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{name}[{k}] positional={positional}"
    emu_lib.set_positional(True)


def test_emu_evm_equals_oracle_on_goldens():
    """both lookup paths: positional (regular rw / bytecode tables, verified on the fly; corrupted
    tables fall back by themselves) and hash index only"""
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    for name, k, s, b, r, flags, exp_row, exp_exc in golden_util.evm_vectors():
        off, ofc = oracle_lib.check_evm(s, b, r, fixed, flags=flags)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_evm(s, b, r, fixed, flags=flags, n=n)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{name}[{k}] positional={positional}"
    emu_lib.set_positional(True)


def test_emu_evm_synthetic_and_fuzz_equals_oracle():
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    w = synth.evm_trace(200, seed=2)
    S, B, R = w["steps"], w["bytecode"], w["rw"]
    ff, fc = emu_lib.check_evm(S, B, R, fixed, n=n)
    assert (ff == 0xFFFFFFFF).all(), [(int(i), int(ff[i])) for i in np.nonzero(ff != 0xFFFFFFFF)[0]]
    rng = np.random.default_rng(5)
    P = 21888242871839275222246405745257275088548364400416034343698204186575808495617
    for t in range(150):
        s, b, r = S, B, R
        kind = t % 5
        if kind == 0:
            r = R.copy(); r[8 + rng.integers(2), rng.integers(R.shape[1]), rng.integers(2)] ^= np.uint64(1 << int(rng.integers(64)))
        elif kind == 1:
            s = S.copy(); s[int(rng.integers(1, 13)), rng.integers(S.shape[1]), 0] += np.uint64(1 + rng.integers(3))
        elif kind == 2:
            b = B.copy(); b[int(rng.integers(2, 6)), 1 + rng.integers(B.shape[1] - 1), 0] ^= np.uint64(1 << int(rng.integers(8)))
        elif kind == 3:  # a random field element somewhere in the rw table
            r = R.copy()
            v = int(rng.integers(0, 1 << 62)) ** 4 % P
            r[int(rng.integers(0, 10)), rng.integers(R.shape[1]), :] = [(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]
        else:  # swap the execution state of a step for another hot state
            s = S.copy(); s[0, rng.integers(S.shape[1] - 1), 0] = np.uint64(rng.choice([5, 6, 40, 50]))
        ff, fc = emu_lib.check_evm(s, b, r, fixed, n=n)
        off, ofc = oracle_lib.check_evm(s, b, r, fixed)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (t, kind, ff[ff != off], off[ff != off], np.nonzero(ff != off))


def test_emu_copy_equals_oracle_on_goldens():
    n = oracle_lib.lib().orc_n_constraints(2)
    for name, k, w, r, exp_row, exp_exc in golden_util.copy_vectors():
        ff, fc = emu_lib.check_copy(w, r)
        off, ofc = oracle_lib.check_copy(w, r)
        assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k, ff[:n][ff[:n] != off], off[ff[:n] != off])


def test_emu_state_equals_oracle_on_goldens():
    n = oracle_lib.lib().orc_n_constraints(1)
    for name, k, s, f, m, exp_row, exp_exc in golden_util.state_vectors():
        ff, fc = emu_lib.check_state(s, f, m)
        off, ofc = oracle_lib.check_state(s, f, m)
        assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k, np.nonzero(ff[:n] != off), ff[:n][ff[:n] != off], off[ff[:n] != off])


def test_emu_evm_sha3_calldatacopy_equals_oracle_on_goldens():
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    for name, k, w, exp_row, exp_exc in golden_util.evm2_vectors():
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_evm_x(w, fixed, n=n)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k, positional, np.nonzero(ff != off), ff[ff != off], off[ff != off])
    emu_lib.set_positional(True)


def test_emu_evm_stop_equals_oracle_on_goldens():
    """STOP (root and internal call with the 12 restore-context lookups), both lookup paths"""
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    for name, k, w, exp_row, exp_exc in golden_util.evm3_vectors():
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_evm_x(w, fixed, n=n)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k, positional, np.nonzero(ff != off), ff[ff != off], off[ff != off])
    emu_lib.set_positional(True)


def test_emu_evm_memory_and_simple_gadgets_equal_oracle_on_goldens():
    """MLOAD / MSTORE / MSTORE8 and MSIZE / GAS / ISZERO / CMP / JUMP / JUMPI, both lookup paths"""
    import itertools

    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    for name, k, w, exp_row, exp_exc in itertools.chain(golden_util.evm4_vectors(), golden_util.evm5_vectors(), golden_util.evm6_vectors(), golden_util.evm7_vectors(), golden_util.evm8_vectors(), golden_util.evm9_vectors(), golden_util.evm10_vectors(), golden_util.evm12_vectors(), golden_util.evm13_vectors(), golden_util.evm14_vectors(), golden_util.evm15_vectors(), golden_util.evm16_vectors(), golden_util.evm17_vectors(), golden_util.evm18_vectors(), golden_util.evm19_vectors(), golden_util.evm20_vectors(), golden_util.evm21_vectors(), golden_util.evm22_vectors(), golden_util.evm23_vectors(), golden_util.evm24_vectors(), golden_util.evm25_vectors(), golden_util.evm26_vectors(), golden_util.evm27_vectors(), golden_util.evm28_vectors()):
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_evm_x(w, fixed, n=n)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k, positional, np.nonzero(ff != off), ff[ff != off], off[ff != off])
    emu_lib.set_positional(True)


def test_emu_evm_begin_end_tx_end_block_equal_oracle_on_goldens():
    """BeginTx / EndTx / EndBlock (evm11: 2,722 reference vectors), positional and hash lookup paths"""
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    for name, k, w, exp_row, exp_exc in golden_util.evm11_vectors():
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        for positional in (True, False):
            emu_lib.set_positional(positional)
            ff, fc = emu_lib.check_evm_x(w, fixed, n=n)
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k, positional, np.nonzero(ff != off), ff[ff != off], off[ff != off])
    emu_lib.set_positional(True)


def head_tail_order(w):
    """the rw rows as a block witness lays them out: every row but the `Start` padding ones by rw_counter, then the
    Start rows by rw_counter — the layout the dense-with-tail positional index serves (lookup.cuh)"""
    rw = w["rw"]
    is_start = (rw[2, :, 0] == 1) & (rw[2, :, 1:].sum(axis=1) == 0)
    key = np.lexsort((rw[0, :, 0], is_start))
    out = dict(w)
    out["rw"] = np.ascontiguousarray(rw[:, key, :])
    out["rw_flags"] = np.ascontiguousarray(w["rw_flags"][key])
    return out


def test_emu_dense_rw_table_with_start_tail_equals_oracle():
    """EndBlock / EndTx / BeginTx vectors with the rw table in head + tail order: the positional path (a dense head, a
    dense tail of Start rows) must give the oracle's arrays — the oracle does not care about row order"""
    fixed = fixed_table_matrix()
    n = oracle_lib.lib().orc_n_constraints(3)
    emu_lib.set_positional(True)
    m = 0
    for name, k, w, exp_row, exp_exc in golden_util.evm11_vectors():
        if k % 3 and not name.startswith("endblock"):
            continue
        w2 = head_tail_order(w)
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        ff, fc = emu_lib.check_evm_x(w2, fixed, n=n)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k, np.nonzero(ff != off), ff[ff != off], off[ff != off])
        m += 1
    assert m > 1200


def test_emu_exp_equals_oracle_on_goldens():
    n = oracle_lib.lib().orc_n_constraints(4)
    for name, k, r, exp_row, exp_exc in golden_util.exp_vectors():
        ff, fc = emu_lib.check_exp(r)
        off, ofc = oracle_lib.check_exp(r)
        assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k, np.nonzero(ff[:n] != off))


def test_emu_pi_equals_oracle_on_goldens():
    """public-inputs circuit (783 reference vectors): canonical and packed storage"""
    n = oracle_lib.lib().orc_n_constraints(7)
    for packed in (False, True):
        emu_lib.set_packed(packed)
        try:
            for name, k, R, K, G, clen, exp_row, exp_exc in golden_util.pi_vectors():
                if packed and k % 4:
                    continue
                ff, fc = emu_lib.check_pi(R, K, G, clen)
                off, ofc = oracle_lib.check_pi(R, K, G, clen)
                assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k, packed, np.nonzero(ff[:n] != off))
        finally:
            emu_lib.set_packed(False)


def test_emu_packed_columns_equal_oracle_on_every_golden_family():
    """the packed narrow-column storage (include/zkcheck.h "packed columns", fr.cuh:ld_col): every
    matrix stored at per-column minimal widths gives the oracle's arrays on every golden vector"""
    fixed = fixed_table_matrix()
    lib = oracle_lib.lib()
    emu_lib.set_packed(True)
    try:
        for name, k, cols, push, kec, r, exp_row, exp_exc in golden_util.bytecode_vectors():
            assert all(np.array_equal(a, b) for a, b in zip(emu_lib.check_bytecode(cols, push, kec, r),
                                                            oracle_lib.check_bytecode(cols, push, kec, r))), (name, k)
        n = lib.orc_n_constraints(3)
        for name, k, s, b, r, flags, exp_row, exp_exc in golden_util.evm_vectors():
            assert all(np.array_equal(a, b) for a, b in zip(emu_lib.check_evm(s, b, r, fixed, flags=flags, n=n),
                                                            oracle_lib.check_evm(s, b, r, fixed, flags=flags))), (name, k)
        for vectors in (golden_util.evm2_vectors, golden_util.evm3_vectors, golden_util.evm4_vectors, golden_util.evm5_vectors, golden_util.evm6_vectors, golden_util.evm7_vectors, golden_util.evm8_vectors, golden_util.evm9_vectors, golden_util.evm10_vectors, golden_util.evm11_vectors, golden_util.evm12_vectors, golden_util.evm13_vectors, golden_util.evm14_vectors, golden_util.evm15_vectors, golden_util.evm16_vectors, golden_util.evm17_vectors, golden_util.evm18_vectors, golden_util.evm19_vectors, golden_util.evm20_vectors, golden_util.evm21_vectors, golden_util.evm22_vectors, golden_util.evm23_vectors):
            for name, k, w, exp_row, exp_exc in vectors():
                assert all(np.array_equal(a, b) for a, b in zip(emu_lib.check_evm_x(w, fixed, n=n),
                                                                oracle_lib.check_evm_x(w, fixed))), (name, k)
        n = lib.orc_n_constraints(2)
        for name, k, w, r, exp_row, exp_exc in golden_util.copy_vectors():
            ff, fc = emu_lib.check_copy(w, r)
            off, ofc = oracle_lib.check_copy(w, r)
            assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k)
        n = lib.orc_n_constraints(1)
        for name, k, s, f, m, exp_row, exp_exc in golden_util.state_vectors():
            ff, fc = emu_lib.check_state(s, f, m)
            off, ofc = oracle_lib.check_state(s, f, m)
            assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k)
        n = lib.orc_n_constraints(4)
        for name, k, r, exp_row, exp_exc in golden_util.exp_vectors():
            ff, fc = emu_lib.check_exp(r)
            off, ofc = oracle_lib.check_exp(r)
            assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc), (name, k)
        assert emu_lib.narrow_cols() > 10000  # the packed path really ran
        assert emu_lib.narrow_runs() > 1000  # ... and so did the narrow form of the hot gate programs
    finally:
        emu_lib.set_packed(False)


def test_emu_div256_equals_python_integer_division():
    """evm.cu:div256 (Knuth D, 64-bit digits) against Python's // on random, boundary and
    nasty operands (tests/common.py:23-45 style values)"""
    import ctypes
    import random

    lib = emu_lib.lib()
    rnd = random.Random(256)
    nasty = [1, 2, 3, 0xFF, 1 << 64, (1 << 64) - 1, (1 << 64) + 1, (1 << 128) - 1, 1 << 128, (1 << 128) + 1,
             (1 << 192) - 1, 1 << 192, (1 << 255) - 1, 1 << 255, (1 << 256) - 1, (1 << 256) - 2, 0x8000000000000000,
             0xFFFFFFFF, 0x100000000, (1 << 63) - 1, ((1 << 64) - 1) << 192, (1 << 255) + (1 << 63)]
    cases = [(a, b) for a in nasty + [0] for b in nasty]
    for _ in range(20000):
        bits_n, bits_d = rnd.choice([256, 256, 200, 129, 128, 65, 64, 33]), rnd.choice([256, 255, 192, 129, 128, 65, 64, 63, 33, 32, 8, 1])
        n = rnd.getrandbits(bits_n)
        d = rnd.getrandbits(bits_d) | (1 << (bits_d - 1))
        if rnd.random() < 0.2:  # quotient digits of all ones / estimate corrections
            d = (d >> 64 << 64) | ((1 << 64) - 1) if bits_d > 64 else d
        cases.append((n, d))
    arr = ctypes.c_uint64 * 4
    for n, d in cases:
        q = arr()
        lib.emu_div256(arr(*[(n >> (64 * k)) & (2**64 - 1) for k in range(4)]),
                       arr(*[(d >> (64 * k)) & (2**64 - 1) for k in range(4)]), q)
        got = sum(int(q[k]) << (64 * k) for k in range(4))
        assert got == n // d, (hex(n), hex(d), hex(got), hex(n // d))


def test_device_keccak256_matches_host_reference():
    """csrc/keccak.cuh (run on the host through the emu build) against the Python sponge that the standard
    vectors pin (zkevm_specs_b200.util.hash), at every length around the 136-byte rate boundaries"""
    import ctypes

    import emu_lib
    from zkevm_specs_b200.util.hash import keccak256

    L = emu_lib.lib()
    rng = np.random.default_rng(7)
    out = (ctypes.c_uint8 * 32)()
    lo, hi = (ctypes.c_uint64 * 2)(), (ctypes.c_uint64 * 2)()
    for n in list(range(0, 140)) + [271, 272, 273, 407, 408, 1000, 24576]:
        msg = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        buf = (ctypes.c_uint8 * max(1, n)).from_buffer_copy(msg or b"\0")
        L.emu_keccak256(buf, ctypes.c_uint64(n), out)
        want = keccak256(msg)
        assert bytes(out) == want, n
        L.emu_keccak256_word(buf, ctypes.c_uint64(n), lo, hi)
        v = int.from_bytes(want, "big")
        assert lo[0] | (lo[1] << 64) == v & ((1 << 128) - 1) and hi[0] | (hi[1] << 64) == v >> 128
        # the table's input_rlc column, folded as the kernel folds it (128 chunks + tree)
        from zkevm_specs_b200.util import FQ
        r = 0x1234567ABCDEF0FEDCBA987654321
        rr = (ctypes.c_uint64 * 4)(*[(r >> (64 * k)) & (2**64 - 1) for k in range(4)])
        o4 = (ctypes.c_uint64 * 4)()
        L.emu_keccak_rlc(buf, ctypes.c_uint64(n), rr, o4)
        acc = FQ(0)
        for b in msg:
            acc = acc * FQ(r) + FQ(b)
        assert sum(int(o4[k]) << (64 * k) for k in range(4)) == acc.n, n
