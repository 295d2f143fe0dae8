"""GPU parity of the CUDA EVM-circuit checker (through the C-ABI) against the reference's
verdicts (tests/golden/evm.npz), the CPU oracle's full per-constraint result, and the
host API used the way the reference's tests use verify_steps."""
import numpy as np
import pytest

import golden_util
import oracle_lib
from zkevm_specs_b200 import native, synth
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

pytestmark = pytest.mark.gpu


def _device_check(ctx, steps, bytecode, rw, flags=0):
    ctx.upload_table(native.TABLE_BYTECODE, bytecode)
    ctx.upload_table(native.TABLE_RW, rw)
    evm_main.upload_fixed_table(ctx)
    ctx.upload_columns(native.CIRCUIT_EVM, steps)
    return ctx.check(native.CIRCUIT_EVM, 0, steps.shape[1] - 1, 0, flags)


def golden_parity_evm(ctx, transform=None):
    """evm.npz (ADD / MUL / POP / PUSH ... steps over bytecode + rw tables): CUDA == oracle array for array and ==
    the reference's verdicts.  `transform(w)` maps the witness dict (steps, bytecode, rw, rw_flags) to the one
    checked (tests/test_gpu_lookup.py: reordered tables).  Returns (vectors compared, declared-limit vectors)."""
    fixed = fixed_table_matrix()
    n = n_unsupported = 0
    for name, k, s, b, r, flags, exp_row, exp_exc in golden_util.evm_vectors():
        if transform is not None:
            w = transform({"steps": s, "bytecode": b, "rw": r, "rw_flags": None})
            s, b, r = w["steps"], w["bytecode"], w["rw"]
        ff, fc = _device_check(ctx, s, b, r, flags)
        off, ofc = oracle_lib.check_evm(s, b, r, fixed, flags=flags)
        assert np.array_equal(ff, off), f"{name}[{k}] first_fail differs from oracle: " + str((np.nonzero(ff != off)[0][:8].tolist(), ff[ff != off][:8].tolist(), off[ff != off][:8].tolist()))
        assert np.array_equal(fc, ofc), f"{name}[{k}] fail_count differs from oracle"
        hit = native.first_failure(ff, native.CIRCUIT_EVM)
        got = (-1, "") if hit is None else (hit[0], oracle_lib.EXC_OF_CLASS[hit[2]])
        if got[1] == "NotImplementedError" and exp_exc != got[1]:
            assert got[0] == exp_row  # declared limit, reported at the step the reference fails on
            n_unsupported += 1
            continue
        if got[1] == "ValueError" and exp_exc == "OverflowError":
            got = (got[0], exp_exc)
        assert got == (exp_row, exp_exc), f"{name}[{k}] cuda {got} reference {(exp_row, exp_exc)}"
        n += 1
    return n, n_unsupported


def test_evm_golden_and_oracle_parity():
    n, n_unsupported = golden_parity_evm(native.default_context())
    assert n > 250 and n_unsupported < 12


def test_evm_synthetic_trace_and_corruptions_match_oracle():
    """cfg2 generator at 2^12 steps: passes; 64 seeded corruptions (operand limb / gas_left /
    rw_counter / bytecode byte) give identical per-constraint results on GPU and oracle."""
    ctx = native.default_context()
    fixed = fixed_table_matrix()
    w = synth.evm_trace(1024, seed=2)
    S, B, R = w["steps"], w["bytecode"], w["rw"]
    ff, fc = _device_check(ctx, S, B, R)
    assert (ff == native.PASS).all() and fc.sum() == 0
    rng = np.random.default_rng(22)
    n_detected = 0
    for t in range(64):
        s, b, r = S, B, R
        kind = t % 4
        if kind == 0:  # flip one operand limb in the rw table
            r = R.copy()
            r[8 + rng.integers(2), rng.integers(R.shape[1]), rng.integers(2)] ^= np.uint64(1 << int(rng.integers(64)))
        elif kind == 1:  # gas_left
            s = S.copy()
            s[9, rng.integers(S.shape[1]), 0] += np.uint64(1)
        elif kind == 2:  # rw_counter of a step
            s = S.copy()
            s[1, rng.integers(S.shape[1]), 0] += np.uint64(1 + rng.integers(3))
        else:  # a bytecode byte
            b = B.copy()
            b[5, 1 + rng.integers(B.shape[1] - 1), 0] ^= np.uint64(1 << int(rng.integers(8)))
        ff, fc = _device_check(ctx, s, b, r)
        off, ofc = oracle_lib.check_evm(s, b, r, fixed)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"corruption {t} kind {kind}"
        n_detected += bool((ff != native.PASS).any())
    # a few corruptions are invisible to the EVM circuit by design (e.g. the value POP reads is
    # only constrained by the state circuit), most are caught
    assert n_detected >= 40


def test_evm_sharded_steps_match_whole():
    """steps split into two row shards (+1 halo step) and min-reduced == whole trace."""
    ctx = native.default_context()
    w = synth.evm_trace(64, seed=5)
    S = w["steps"].copy()
    S[9, 100, 0] += np.uint64(1)  # one gas corruption
    whole, _ = _device_check(ctx, S, w["bytecode"], w["rw"])
    n = S.shape[1] - 1
    half = n // 2
    ctx.upload_columns(native.CIRCUIT_EVM, np.ascontiguousarray(S[:, : half + 1]))
    a, _ = ctx.check(native.CIRCUIT_EVM, 0, half, 0, 0)
    ctx.upload_columns(native.CIRCUIT_EVM, np.ascontiguousarray(S[:, half:]))
    b, _ = ctx.check(native.CIRCUIT_EVM, 0, n - half, half, 0)
    assert np.array_equal(np.minimum(a, b), whole)


def test_verify_steps_host_api_like_reference_test_add_sub():
    """the reference's tests/evm/test_add_sub.py:27-76 written against our host API."""
    from zkevm_specs_b200.evm_circuit import (Block, Bytecode, ExecutionState, Opcode, RWDictionary, Tables)
    from zkevm_specs_b200.evm_circuit.main import verify_steps
    from zkevm_specs_b200.evm_circuit.step import StepState
    from zkevm_specs_b200.evm_circuit.table import LookupUnsatFailure
    from zkevm_specs_b200.util import Word

    for opcode, a, b in [(Opcode.ADD, 0x030201, 0x060504), (Opcode.SUB, 0x090705, 0x060504),
                         (Opcode.ADD, (1 << 256) - 1, (1 << 256) - 2), (Opcode.SUB, 0, (1 << 256) - 1)]:
        c = Word((a + b if opcode == Opcode.ADD else a - b) % 2**256)
        wa, wb = Word(a), Word(b)
        bytecode = Bytecode().add(wa, wb).stop() if opcode == Opcode.ADD else Bytecode().sub(wa, wb).stop()
        h = Word(bytecode.hash())

        def tables(rw_start=9, cc=c):
            return Tables(block_table=set(Block().table_assignments()), tx_table=set(), withdrawal_table=set(),
                          bytecode_table=set(bytecode.table_assignments()),
                          rw_table=set(RWDictionary(rw_start).stack_read(1, 1022, wa).stack_read(1, 1023, wb)
                                       .stack_write(1, 1023, cc).rws))

        def steps(gas=3):
            return [StepState(ExecutionState.ADD, rw_counter=9, call_id=1, is_root=True, code_hash=h,
                              program_counter=66, stack_pointer=1022, gas_left=gas),
                    StepState(ExecutionState.STOP, rw_counter=12, call_id=1, is_root=True, code_hash=h,
                              program_counter=67, stack_pointer=1023, gas_left=0)]

        verify_steps(tables(), steps())
        with pytest.raises(AssertionError):  # wrong result word
            verify_steps(tables(cc=Word((c.int_value() + 1) % 2**256)), steps())
        verify_steps(tables(cc=Word((c.int_value() + 1) % 2**256)), steps(), success=False)
        with pytest.raises(LookupUnsatFailure):  # rw rows missing: propagates even with success=False
            verify_steps(tables(rw_start=10), steps(), success=False)


def test_verify_steps_host_api_like_reference_test_exp():
    """the reference's tests/evm/test_exp.py:45-112 written against our host API: the exp table comes from the exp circuit's
    rows (Tables(exp_circuit=...)), the exp circuit itself is checked by verify_exp_circuit"""
    from zkevm_specs_b200.evm_circuit import (Block, Bytecode, ExecutionState, RWDictionary, Tables)
    from zkevm_specs_b200.evm_circuit.main import verify_steps
    from zkevm_specs_b200.evm_circuit.step import StepState
    from zkevm_specs_b200.exp_circuit import ExpCircuit, verify_exp_circuit
    from zkevm_specs_b200.util import Word

    for base, exponent in [(2, 5), (3, 101), (0xCAFE, 0), ((1 << 256) - 1, 1), ((1 << 256) - 1, 3), (7, 1023)]:
        result = pow(base, exponent, 1 << 256)
        bytecode = Bytecode().push(exponent, n_bytes=32).push(base, n_bytes=32).exp().stop()
        h = Word(bytecode.hash())
        rw = RWDictionary(3).stack_read(1, 1022, Word(base)).stack_read(1, 1023, Word(exponent)).stack_write(1, 1023, Word(result))
        exp_circuit = ExpCircuit().add_event(base, exponent, rw.rw_counter).fill_dummy_events()
        verify_exp_circuit(exp_circuit)
        gas = 50 * ((exponent.bit_length() + 7) // 8)  # Opcode.EXP.constant_gas_cost() is 0: the whole cost is dynamic

        def tables(res=result):
            rws = RWDictionary(3).stack_read(1, 1022, Word(base)).stack_read(1, 1023, Word(exponent)).stack_write(1, 1023, Word(res)).rws
            return Tables(block_table=set(Block().table_assignments()), tx_table=set(), withdrawal_table=set(),
                          bytecode_table=set(bytecode.table_assignments()), rw_table=set(rws), exp_circuit=exp_circuit.rows)

        steps = [StepState(ExecutionState.EXP, rw_counter=3, call_id=1, is_root=True, code_hash=h, program_counter=66,
                           stack_pointer=1022, gas_left=gas),
                 StepState(ExecutionState.STOP, rw_counter=6, call_id=1, is_root=True, code_hash=h, program_counter=67,
                           stack_pointer=1023, gas_left=0)]
        verify_steps(tables(), steps)
        with pytest.raises(AssertionError):  # wrong exponentiation on the stack
            verify_steps(tables(res=(result + 1) % (1 << 256)), steps)


_TABLES = {"bytecode": (native.TABLE_BYTECODE, 6), "rw": (native.TABLE_RW, 14), "copy": (native.TABLE_COPY, 14),
           "keccak": (native.TABLE_KECCAK, 5), "tx": (native.TABLE_TX, 5), "block": (native.TABLE_BLOCK, 4),
           "wd": (native.TABLE_WITHDRAWAL, 4), "exp": (native.TABLE_EXP, 11), "aux": (native.TABLE_STEP_AUX, 3)}


def _upload_tables(ctx, w, names):
    """uploads the named tables of a witness dict (an empty table where the dict has none), each with its
    `<name>_flags` row flags where the dict has them"""
    for name in names:
        tid, n_cols = _TABLES[name]
        m = w.get(name)
        if m is None:
            m = np.zeros((n_cols, 0, 4), dtype=np.uint64)
        flags = w.get(name + "_flags")
        if flags is None:
            ctx.upload_table(tid, m)
        else:
            ctx.upload_table(tid, m, flags=flags)


def golden_parity_x(ctx, vectors, tables, transform=None, value_errors=(), allow_unsupported=False):
    """vectors in the evm2 / evm11 layout (a witness dict per vector): upload `tables` of each witness, check the
    steps (with the witness's ZK_FLAG_EVM_* flags if it has them), CUDA == oracle array for array, first failure
    == the reference's verdict.  A CUDA ValueError stands for a reference exception named in `value_errors` (one
    "Python runtime error" class, ZK_ERR_VALUE); with `allow_unsupported`, a NotImplementedError (a declared limit)
    must be reported at the step the reference fails on.  `transform(w)` maps each witness dict to the one checked
    (tests/test_gpu_lookup.py: reordered tables).  Returns (vectors compared, declared-limit vectors)."""
    fixed = fixed_table_matrix()
    n = n_unsupported = 0
    for name, k, w, exp_row, exp_exc in vectors:
        if transform is not None:
            w = transform(w)
        _upload_tables(ctx, w, tables)
        evm_main.upload_fixed_table(ctx)
        ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
        ff, fc = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, w.get("flags", 0))
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{name}[{k}] differs from oracle: {_diff(ff, off)}"
        if w.get("order_dependent"):  # the reference's verdict was taken in generator order (table_perturb.has_flag_twins)
            n += 1
            continue
        hit = native.first_failure(ff, native.CIRCUIT_EVM)
        got = (-1, "") if hit is None else (hit[0], oracle_lib.EXC_OF_CLASS[hit[2]])
        if got[1] == "ValueError" and exp_exc in value_errors:
            got = (got[0], exp_exc)
        if allow_unsupported and got[1] == "NotImplementedError" and exp_exc != got[1]:
            # EV_AR_WITNESS_DOMAIN (ADDMOD / MULMOD / SDIV / SMOD with a stack word half >= 2^128): reported at the SAME
            # step the reference fails on
            assert got[0] == exp_row, f"{name}[{k}]"
            n_unsupported += 1
            continue
        assert got == (exp_row, exp_exc), f"{name}[{k}] cuda {got} reference {(exp_row, exp_exc)}"
        n += 1
    return n, n_unsupported


def clear_tables(ctx, names):
    """leave the context with empty side tables for the other tests"""
    _upload_tables(ctx, {}, names)


EVM2_TABLES = ("bytecode", "rw", "copy", "keccak")


def test_evm_sha3_calldatacopy_golden_and_oracle_parity():
    """SHA3 / CALLDATACOPY steps (copy-table + keccak-table + call-context lookups, memory
    expansion and copier gas): CUDA == oracle array for array, and == the reference's verdicts"""
    ctx = native.default_context()
    n, _ = golden_parity_x(ctx, golden_util.evm2_vectors(), EVM2_TABLES, value_errors=("OverflowError",))
    assert n > 380
    clear_tables(ctx, ("copy", "keccak"))


def test_evm_stop_golden_and_oracle_parity():
    """STOP steps (tests/evm/test_stop.py: root call -> EndTx, internal call -> restored caller
    context through 12 call-context lookups): CUDA == oracle array for array, == the reference"""
    ctx = native.default_context()
    n, _ = golden_parity_x(ctx, golden_util.evm3_vectors(), EVM2_TABLES)
    assert n > 550
    clear_tables(ctx, ("copy", "keccak"))


def test_evm_memory_golden_and_oracle_parity():
    """MLOAD / MSTORE / MSTORE8 steps (tests/evm/test_memory.py, 650 vectors) and MSIZE / GAS / ISZERO /
    CMP / JUMP / JUMPI (909), CALLER-family / CODESIZE (539), BITWISE / NOT / BYTE (639), SCMP / SIGNEXTEND
    (853), BlockCtx / ORIGIN / GASPRICE (526) steps: CUDA == oracle array for array, == the reference's verdicts"""
    ctx = native.default_context()
    clear_tables(ctx, ("copy", "keccak"))
    n, n_unsupported = golden_parity_x(ctx, memory_family_vectors(), MEMORY_TABLES, value_errors=MEMORY_VALUE_ERRORS,
                                       allow_unsupported=True)
    assert n > 9000 and n_unsupported <= 150
    clear_tables(ctx, ("aux", "copy", "tx", "block"))


# the evm4 .. evm28 families but evm11: CODECOPY / RETURNDATACOPY / EXTCODECOPY scenarios carry a copy table, EXP an exp
# table, CREATE / CREATE2 a step-aux table, CALLDATALOAD a tx table whose call-data rows are plain values (tx_flags),
# BLOCKHASH a block table whose current block number is a plain value (block_flags); the keccak table stays empty
MEMORY_TABLES = ("bytecode", "rw", "copy", "exp", "aux", "tx", "block")
MEMORY_VALUE_ERRORS = ("OverflowError", "UnboundLocalError", "AttributeError", "TypeError")


def memory_family_vectors():
    import itertools

    return itertools.chain(golden_util.evm4_vectors(), golden_util.evm5_vectors(), golden_util.evm6_vectors(), golden_util.evm7_vectors(), golden_util.evm8_vectors(), golden_util.evm9_vectors(), golden_util.evm10_vectors(), golden_util.evm12_vectors(), golden_util.evm13_vectors(), golden_util.evm14_vectors(), golden_util.evm15_vectors(), golden_util.evm16_vectors(), golden_util.evm17_vectors(), golden_util.evm18_vectors(), golden_util.evm19_vectors(), golden_util.evm20_vectors(), golden_util.evm21_vectors(), golden_util.evm22_vectors(), golden_util.evm23_vectors(), golden_util.evm24_vectors(), golden_util.evm25_vectors(), golden_util.evm26_vectors(), golden_util.evm27_vectors(), golden_util.evm28_vectors())


_diff = oracle_lib.diff


def test_evm_begin_end_tx_end_block_golden_and_oracle_parity():
    """BeginTx / EndTx / EndBlock steps (tests/evm/test_begin_tx.py, test_end_tx.py, test_end_block.py scenarios +
    seeded corruptions of every table, 2,722 reference vectors): rw lookups on other column subsets, the state_write
    reversion lookups, balance / gas word arithmetic, the RLP + Keccak contract address on the device, the
    table-derived constants of EndBlock: CUDA == oracle array for array, == the reference's verdicts"""
    ctx = native.default_context()
    n, _ = golden_parity_x(ctx, golden_util.evm11_vectors(), EVM11_TABLES, value_errors=("OverflowError",))
    assert n > 2700
    clear_tables(ctx, ("copy", "keccak", "tx", "block", "wd"))


EVM11_TABLES = ("bytecode", "rw", "copy", "keccak", "tx", "block", "wd")


def _upload_block(ctx, w, from_code=True, packed=False):
    from zkevm_specs_b200 import packing
    if from_code:
        ctx.upload_bytecode_table_from_code(**w["bytecode_src"])
    else:
        ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
    if packed:
        ctx.upload_table_packed(native.TABLE_RW, packing.pack_matrix(w["rw"]), flags=w["rw_flags"])
        ctx.upload_columns_packed(native.CIRCUIT_EVM, packing.pack_matrix(w["steps"]))
    else:
        ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
        ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
    ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
    ctx.upload_table(native.TABLE_BLOCK, w["block"], flags=w["block_flags"])
    ctx.upload_table(native.TABLE_WITHDRAWAL, w["wd"])
    ctx.upload_table(native.TABLE_COPY, w["copy"])
    ctx.upload_table(native.TABLE_KECCAK, w["keccak"])


def test_whole_block_trace_first_and_last_step_flags_match_oracle():
    """synth.block_trace: BeginTx .. STOP, EndTx per transaction over several contracts, EndBlock last, checked as ONE
    trace with ZK_FLAG_EVM_FIRST_STEP | ZK_FLAG_EVM_LAST_STEP (verify_steps(begin_with_first_step=True,
    end_with_last_step=True); the generator is accepted by the reference itself, tests/golden/gen_golden.py synth):
    passes on the device, corrupted copies equal the oracle array for array; packed storage and the
    bytecode-table-from-code upload give the same arrays; sharded == whole"""
    ctx = native.default_context()
    fixed = fixed_table_matrix()
    evm_main.upload_fixed_table(ctx)
    w = synth.block_trace(96, 24, 16, seed=9)
    n = w["n_steps"]
    _upload_block(ctx, w)
    ff, fc = ctx.check(native.CIRCUIT_EVM, 0, n, 0, w["flags"])
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_EVM)
    rng = np.random.default_rng(5)
    for trial in range(24):
        w2 = dict(w)
        which = trial % 4
        if which == 0:
            m = w["steps"].copy(); m[int(rng.integers(1, 13)), int(rng.integers(0, n)), 0] += np.uint64(1); w2["steps"] = m
        elif which == 1:
            m = w["rw"].copy(); m[int(rng.choice([3, 4, 5, 8, 10])), int(rng.integers(0, m.shape[1])), 0] ^= np.uint64(1); w2["rw"] = m
        elif which == 2:
            m = w["tx"].copy(); m[3, int(rng.integers(0, m.shape[1])), 0] += np.uint64(1); w2["tx"] = m
        else:
            m = w["block"].copy(); m[2, int(rng.integers(0, m.shape[1])), 0] += np.uint64(1); w2["block"] = m
        off, ofc = oracle_lib.check_evm_x(w2, fixed, row_end=n)
        for packed in (False, True):
            _upload_block(ctx, w2, from_code=packed, packed=packed)
            ff, fc = ctx.check(native.CIRCUIT_EVM, 0, n, 0, w["flags"])
            assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"trial {trial} packed={packed}: {_diff(ff, off)}"
        if trial < 4:  # row-sharded: every shard sees the whole tables, its steps + one halo step
            _upload_block(ctx, w2)
            acc_ff, acc_fc = np.full_like(off, native.PASS), np.zeros_like(ofc)
            for lo, hi in ((0, n // 3), (n // 3, 2 * n // 3), (2 * n // 3, n)):
                sff, sfc = ctx.check(native.CIRCUIT_EVM, lo, hi, 0, w["flags"])
                acc_ff, acc_fc = np.minimum(acc_ff, sff), acc_fc + sfc
            assert np.array_equal(acc_ff, off) and np.array_equal(acc_fc, ofc)
    for t, c in ((native.TABLE_TX, 5), (native.TABLE_BLOCK, 4)):
        ctx.upload_table(t, np.zeros((c, 0, 4), dtype=np.uint64))


def test_sha3_host_api_like_reference_test_sha3():
    """tests/evm/test_sha3.py:35-141 on our host API: copy circuit + keccak table + SHA3 step"""
    from zkevm_specs_b200.copy_circuit import verify_copy_table
    from zkevm_specs_b200.evm_circuit import (Block, Bytecode, CopyCircuit, CopyDataTypeTag, ExecutionState,
                                              KeccakCircuit, Opcode, RWDictionary, Tables)
    from zkevm_specs_b200.evm_circuit.main import verify_steps
    from zkevm_specs_b200.evm_circuit.step import StepState
    from zkevm_specs_b200.util import FQ, Word, keccak256

    r = FQ(0x5EED5EED5EED)
    offset, length = 0x20, 0x40
    mem = bytes((7 * i + 1) % 256 for i in range(offset + length))
    src = {i: mem[i] for i in range(offset, offset + length)}
    bc = Bytecode().push(offset, n_bytes=32).push(length, n_bytes=32).sha3().stop()
    h = Word(bc.hash())
    out = Word(int.from_bytes(keccak256(mem[offset:offset + length]), "big"))
    words = (offset + length + 31) // 32
    gas = Opcode.SHA3.constant_gas_cost() + ((length + 31) // 32) * 6
    rw = (RWDictionary(1).stack_write(1, 1023, Word(length)).stack_write(1, 1022, Word(offset))
          .stack_read(1, 1022, Word(offset)).stack_read(1, 1023, Word(length)).stack_write(1, 1023, out))
    cc = CopyCircuit().copy(r, rw, 1, CopyDataTypeTag.Memory, 1, CopyDataTypeTag.RlcAcc, offset, offset + length, 0, length, src)
    kc = KeccakCircuit().add(mem[offset:offset + length], r)

    def tables(keccak_rows):
        return Tables(block_table=set(Block().table_assignments()), tx_table=set(), withdrawal_table=set(),
                      bytecode_table=set(bc.table_assignments()), rw_table=set(rw.rws), copy_circuit=cc.rows,
                      keccak_table=keccak_rows)

    def steps(gas_left=gas):
        return [StepState(ExecutionState.SHA3, rw_counter=3, call_id=1, is_root=True, code_hash=h, program_counter=66,
                          stack_pointer=1022, memory_word_size=words, gas_left=gas_left),
                StepState(ExecutionState.STOP, rw_counter=rw.rw_counter, call_id=1, is_root=True, code_hash=h,
                          program_counter=67, stack_pointer=1023, memory_word_size=words, gas_left=0)]

    t = tables(kc.rows)
    verify_copy_table(cc, t, r)
    verify_steps(t, steps())
    with pytest.raises(AssertionError):
        verify_steps(t, steps(gas + 1))
    with pytest.raises(Exception) as ei:
        verify_steps(tables([]), steps())
    assert type(ei.value).__name__ == "LookupUnsatFailure"
    ctx = native.default_context()
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))


def test_step_aux_host_rows_reach_the_device():
    """StepState.aux_data -> evm_circuit.main.step_aux_rows -> ZK_TABLE_STEP_AUX: an ErrorOutOfGasSloadSstore (SSTORE) and a
    CREATE2 scenario of the goldens verify with the side table built by the HOST mirror from StepState objects, and fail
    with the aux-missing constraint when the table is left empty"""
    from zkevm_specs_b200.evm_circuit.step import StepState
    from zkevm_specs_b200.evm_circuit.spec import ExecutionState
    from zkevm_specs_b200.util.arithmetic import Word
    from zkevm_specs_b200 import packing

    ctx = native.default_context()
    evm_main.upload_fixed_table(ctx)
    ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_EXP, np.zeros((11, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_BLOCK, np.zeros((4, 0, 4), dtype=np.uint64))

    def to_int(cell):
        return sum(int(x) << (64 * k) for k, x in enumerate(cell))

    done = set()
    for vectors, want_missing, as_word in ((golden_util.evm25_vectors(), "EV_ESS_AUX_MISSING", False),
                                           (golden_util.evm24_vectors(), "EV_CR_AUX_MISSING", True)):
        for name, k, w, exp_row, exp_exc in vectors:
            if exp_row != -1 or "aux" not in w or name in done:
                continue
            if "sload" in name:
                continue  # SLOAD never reads aux_data
            done.add(name)
            steps = []
            for r in range(w["steps"].shape[1]):
                steps.append(StepState(execution_state=ExecutionState(to_int(w["steps"][0, r])), rw_counter=to_int(w["steps"][1, r])))
            for a in range(w["aux"].shape[1]):
                lo, hi = to_int(w["aux"][1, a]), to_int(w["aux"][2, a])
                steps[to_int(w["aux"][0, a])].aux_data = Word(lo + (hi << 128)) if as_word else lo + (hi << 128)
            rows = evm_main.step_aux_rows(steps)
            assert len(rows) == w["aux"].shape[1]
            ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
            ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
            ctx.upload_table(native.TABLE_COPY, w["copy"])
            if "tx_flags" in w:
                ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
            else:
                ctx.upload_table(native.TABLE_TX, w["tx"] if "tx" in w else np.zeros((5, 0, 4), dtype=np.uint64))
            ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
            ctx.upload_table(native.TABLE_STEP_AUX, packing.matrix_from_ints(rows, 3))
            ff, _ = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, 0)
            assert native.first_failure(ff, native.CIRCUIT_EVM) is None, name
            ctx.upload_table(native.TABLE_STEP_AUX, np.zeros((3, 0, 4), dtype=np.uint64))
            ff, _ = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, 0)
            hit = native.first_failure(ff, native.CIRCUIT_EVM)
            if as_word and hit is None:
                continue  # a CREATE without init code (or a failed pre-check) never reads aux_data
            assert hit is not None and hit[3].startswith(want_missing), (name, hit)
            if as_word and sum(1 for d in done if d.startswith("create_")) >= 20:
                break
    assert len(done) >= 40
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_TX, np.zeros((5, 0, 4), dtype=np.uint64))
