"""The tx-table and copy-table builders on the GPU (zk_assign_tx_table, zk_assign_copy_table, csrc/assign.cu): the
downloaded tables and flags equal the serial run of the same bodies (tests/emu/zk_emu_tables.cu), the mirror's
Transaction.table_assignments as a set, and the numpy restatements of the reference's conversions; the golden tx tables
rebuilt on the device reproduce the reference's EVM verdicts through verify_steps_resident; the copy table is built from
every storage form of the copy circuit; the copy and EVM checks give the host tables' verdicts against the device
tables; both builders run on a one-SM grid; rejected calls leave the previous table in place."""
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

import emu_tables_lib as et
import golden_util
import tables_assign_cases as tc
from zkevm_specs_b200 import assign, native, packing, synth
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.step import StepState
from zkevm_specs_b200.evm_circuit.typing import Transaction
from zkevm_specs_b200.util.arithmetic import FQ, FR_MODULUS

pytestmark = pytest.mark.gpu

CASES = list(tc.cases())


@pytest.fixture(scope="module")
def one_sm_ctx():
    """a context whose grids are sized for one SM (ZKCHECK_SM_COUNT=1): every thread walks several rows or bytes"""
    saved = os.environ.get("ZKCHECK_SM_COUNT")
    os.environ["ZKCHECK_SM_COUNT"] = "1"
    try:
        ctx = native.Context(0)
    finally:
        if saved is None:
            os.environ.pop("ZKCHECK_SM_COUNT", None)
        else:
            os.environ["ZKCHECK_SM_COUNT"] = saved
    yield ctx
    ctx.close()


def _device_tx(ctx, txs):
    rec, cd, offs = assign.tx_records(txs)
    ctx.assign_tx_table(rec, cd, offs)
    tab, fl = ctx.download_table(native.TABLE_TX), ctx.download_table_flags(native.TABLE_TX)
    want, want_fl = et.assign_tx_table(rec, cd, offs)
    assert np.array_equal(tab, want) and np.array_equal(fl, want_fl)
    return tab, fl


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("label,txs", CASES + [("one_tx_2_20_bytes", tc.big_tx())], ids=[c[0] for c in CASES] + ["one_tx_2_20_bytes"])
def test_device_tx_table_equals_emu_and_mirror(label, txs, strided, one_sm_ctx):
    ctx = one_sm_ctx if strided else native.default_context()
    tab, fl = _device_tx(ctx, txs)
    assert tc.table_set(tab, fl) == tc.mirror_set(txs)


def _steps_of(m):
    """the StepState objects of a packed step matrix (cells as they are, a corrupted one included)"""
    c = [[tc.cell(m[k, r]) for k in range(13)] for r in range(m.shape[1])]
    return [StepState(v[0], FQ(v[1]), FQ(v[2]), v[3], v[4], SimpleNamespace(lo=FQ(v[5]), hi=FQ(v[6])), FQ(v[7]), FQ(v[8]),
                      FQ(v[9]), FQ(v[10]), FQ(v[11]), FQ(v[12])) for v in c]


EXC = {"AssertionError", "LookupUnsatFailure", "LookupAmbiguousFailure", "ConstraintUnsatFailure", "ValueError",
       "NotImplementedError"}
VALUE_ERRORS = ("OverflowError", "UnboundLocalError", "AttributeError", "TypeError")


def test_golden_tx_tables_on_device_and_reference_verdicts():
    """every golden tx table that is exactly its transactions' table_assignments, rebuilt on the device, equals the golden
    table as a set; every vector of those scenarios that does not corrupt the tx table gets the reference's verdict
    through verify_steps_resident against the device-built table"""
    ctx = native.default_context()
    families = (("evm11", golden_util.evm11_vectors, (6, 8)), ("evm17", golden_util.evm17_vectors, (6, 12)),
                ("evm26", golden_util.evm26_vectors, (6, 12)), ("evm28", golden_util.evm28_vectors, (6, 12)))
    tables = {}
    for f, name, table, flags in tc.golden_tx_tables():
        txs = tc.txs_from_table(table, flags)
        assert txs is not None, (f, name)
        tab, fl = _device_tx(ctx, txs)
        assert tc.table_set(tab, fl) == tc.table_set(table, flags), (f, name)
        tables[(f, name)] = txs
    assert len(tables) == 150
    n = 0
    for f, vectors, tx_kinds in families:
        z = np.load(os.path.join(tc.GOLDEN, f + ".npz"))
        current = None
        for name, k, w, exp_row, exp_exc in vectors():
            if (f, name) not in tables or int(z[f"{name}/mut_kind"][k]) in tx_kinds:
                continue
            if current != name:
                assign.assign_tx_table(ctx, tables[(f, name)])
                current = name
            for t, tid, cols in (("bytecode", native.TABLE_BYTECODE, 6), ("copy", native.TABLE_COPY, 14),
                                 ("keccak", native.TABLE_KECCAK, 5), ("block", native.TABLE_BLOCK, 4),
                                 ("wd", native.TABLE_WITHDRAWAL, 4), ("exp", native.TABLE_EXP, 11)):
                m = w.get(t, np.zeros((cols, 0, 4), dtype=np.uint64))
                ctx.upload_table(tid, m, flags=w.get(t + "_flags"))
            ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
            flags = w.get("flags", 0)
            steps = _steps_of(w["steps"][:, :-1] if flags & 4 else w["steps"])
            try:
                evm_main.verify_steps_resident(steps, ctx, bool(flags & 2), bool(flags & 4))
                got = (-1, "")
            except Exception as e:  # noqa: BLE001
                name_ = type(e).__name__
                assert name_ in EXC, e
                got = (int(re.search(r"\bstep (\d+): ", str(e)).group(1)), name_)
            if got[1] == "ValueError" and exp_exc in VALUE_ERRORS:
                got = (got[0], exp_exc)
            assert got == (exp_row, exp_exc), f"{f} {name}[{k}] cuda {got} reference {(exp_row, exp_exc)}"
            n += 1
    assert n == 6067
    for tid, cols in ((native.TABLE_COPY, 14), (native.TABLE_KECCAK, 5), (native.TABLE_TX, 5), (native.TABLE_BLOCK, 4),
                      (native.TABLE_WITHDRAWAL, 4), (native.TABLE_EXP, 11)):
        ctx.upload_table(tid, np.zeros((cols, 0, 4), dtype=np.uint64))


def _torch_cells(m):
    torch = pytest.importorskip("torch")
    return torch.from_numpy(np.ascontiguousarray(m, dtype=np.uint64).view(np.int64)).to("cuda")


def _copy_table_or_assert(ctx):
    try:
        assign.assign_copy_table(ctx)
    except AssertionError as e:
        return str(e)
    return ctx.download_table(native.TABLE_COPY)


def test_copy_table_from_every_storage_form_of_the_copy_vectors():
    """every copy.npz vector (corruptions included), uploaded canonical, packed or bound: the device table equals the
    restatement, or both raise the same assert and the previous table stays in place"""
    import torch

    ctx = native.default_context()
    n = n_assert = 0
    for name, k, w, r, exp_row, exp_exc in golden_util.copy_vectors():
        c = w["copy"]
        want = tc.copy_table_restated(c)
        for form in ("canonical", "packed", "bound"):
            keep = None
            if form == "canonical":
                ctx.upload_columns(native.CIRCUIT_COPY, c, flags=w["copy_flags"])
            elif form == "packed":
                ctx.upload_columns_packed(native.CIRCUIT_COPY, packing.pack_matrix(c), flags=w["copy_flags"])
            else:
                keep = _torch_cells(c)
                torch.cuda.synchronize()
                ctx.bind_columns_device(native.CIRCUIT_COPY, c.shape[1], 20, keep.data_ptr())
            before = ctx.download_table(native.TABLE_COPY)
            got = _copy_table_or_assert(ctx)
            if isinstance(want, str):
                assert got == want, (name, k, form)
                assert np.array_equal(ctx.download_table(native.TABLE_COPY), before)
                n_assert += 1
            else:
                assert isinstance(got, np.ndarray) and np.array_equal(got, want), (name, k, form)
            del keep
        n += 1
    assert n == 257 and n_assert == 6
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))


@pytest.mark.parametrize("strided", [False, True])
def test_copy_table_from_assigned_copy_circuit_at_2_20_rows(strided, one_sm_ctx):
    ctx = one_sm_ctx if strided else native.default_context()
    w = synth.copy_events(512, 1024)
    ctx.set_challenge(native.CHALLENGE_KECCAK, w["r_int"])
    ctx.assign_copy_circuit(w["events"], w["data"])
    assert ctx.resident_rows(native.CIRCUIT_COPY) == 1 << 20
    assign.assign_copy_table(ctx)
    got = ctx.download_table(native.TABLE_COPY)
    circuit, _ = ctx.download_columns(native.CIRCUIT_COPY)
    want = tc.copy_table_restated(circuit)
    assert got.shape == (14, 512, 4) and np.array_equal(got, want) and np.array_equal(got, et.assign_copy_table(circuit))
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))


def test_sha3_scenario_with_device_tables_matches_verify_steps():
    """a CopyCircuit built with the mirror (the SHA3 scenario of tests/test_gpu_evm.py): verify_steps_resident after
    building the copy and tx tables on the device gives verify_steps(Tables(copy_circuit=...))'s verdict, clean and with
    a corrupted step"""
    from zkevm_specs_b200.evm_circuit import (Block, Bytecode, CopyCircuit, CopyDataTypeTag, ExecutionState, KeccakCircuit,
                                              Opcode, RWDictionary, Tables)
    from zkevm_specs_b200.util import Word, keccak256

    ctx = native.default_context()
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
    txs = [Transaction(1, callee_address=0xCAFE, call_data=b"\x01\x00\x02")]
    tables = Tables(block_table=set(Block().table_assignments()), tx_table=set(r_ for t in txs for r_ in t.table_assignments()),
                    withdrawal_table=set(), bytecode_table=set(bc.table_assignments()), rw_table=set(rw.rws),
                    copy_circuit=cc.rows, keccak_table=kc.rows)

    def steps(gas_left=gas):
        return [StepState(ExecutionState.SHA3, rw_counter=3, call_id=1, is_root=True, code_hash=h, program_counter=66,
                          stack_pointer=1022, memory_word_size=words, gas_left=gas_left),
                StepState(ExecutionState.STOP, rw_counter=rw.rw_counter, call_id=1, is_root=True, code_hash=h,
                          program_counter=67, stack_pointer=1023, memory_word_size=words, gas_left=0)]

    def verdict(run):
        try:
            run()
        except Exception as e:  # noqa: BLE001
            return type(e).__name__, str(e)
        return None

    for g in (gas, gas + 1):
        host = verdict(lambda: evm_main.verify_steps(tables, steps(g), ctx=ctx))
        rows = list(cc.table())  # the copy circuit, resident as the host mirror built it
        ctx.upload_columns(native.CIRCUIT_COPY, packing.pack(rows, packing.copy_circuit_row, 20))
        assign.assign_copy_table(ctx)
        assert tc.copy_table_set(ctx.download_table(native.TABLE_COPY)) == {
            tuple(packing.copy_table_row(x)) for x in tables.copy_table}
        assign.assign_tx_table(ctx, txs)
        dev = verdict(lambda: evm_main.verify_steps_resident(steps(g), ctx))
        assert dev == host, (g, dev, host)
    assert host is not None and host[0] == "AssertionError"
    for tid, cols in ((native.TABLE_COPY, 14), (native.TABLE_KECCAK, 5), (native.TABLE_TX, 5)):
        ctx.upload_table(tid, np.zeros((cols, 0, 4), dtype=np.uint64))


def _calldata_txs(tx):
    """transactions carrying the call-data rows of a partial tx table (synth.copy_events' TxCalldata rows)"""
    data = {}
    for r in range(tx.shape[1]):
        data.setdefault(int(tx[0, r, 0]), {})[int(tx[2, r, 0])] = int(tx[3, r, 0])
    return [Transaction(k, call_data=bytes(d.get(i, 0) for i in range(max(d) + 1))) for k, d in sorted(data.items())]


def test_copy_check_against_device_tx_table():
    ctx = native.default_context()
    w = synth.copy_events(64, 256)
    ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
    ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
    ctx.set_challenge(native.CHALLENGE_KECCAK, w["r_int"])
    txs = _calldata_txs(w["tx"])
    n = w["copy"].shape[1]

    def check():
        ctx.upload_columns(native.CIRCUIT_COPY, w["copy"], flags=w["copy_flags"])
        ff, fc = ctx.check(native.CIRCUIT_COPY, 0, n, 0, native.FLAG_WRAP)
        return ff, fc

    assign.assign_tx_table(ctx, txs)
    ff, _ = check()
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_COPY)
    rec, cd, offs = assign.tx_records(txs)
    j = int(offs[1]) + 7  # byte 7 of the second tx
    bad_cd = cd.copy()
    bad_cd[j] ^= 0x5A
    ctx.assign_tx_table(rec, bad_cd, offs)
    dev = check()
    bad = w["tx"].copy()
    hit = np.nonzero((bad[0, :, 0] == int(tc.cell(rec[1, 0]))) & (bad[2, :, 0] == 7))[0]
    assert len(hit) == 1
    bad[3, hit[0], 0] ^= np.uint64(0x5A)
    ctx.upload_table(native.TABLE_TX, bad, flags=w["tx_flags"])
    host = check()
    assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
    assert (host[0] != native.PASS).any()
    ctx.upload_table(native.TABLE_TX, np.zeros((5, 0, 4), dtype=np.uint64))


def test_block_trace_with_device_tx_table_equals_host_upload():
    ctx = native.default_context()
    w = synth.block_trace(64, 4, 8)
    txs = tc.txs_from_table(w["tx"], w["tx_flags"])
    assert txs is not None and len(txs) == 64
    from zkevm_specs_b200.evm_circuit.main import upload_fixed_table
    upload_fixed_table(ctx)
    ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
    ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
    for t, tid in (("block", native.TABLE_BLOCK), ("wd", native.TABLE_WITHDRAWAL), ("copy", native.TABLE_COPY),
                   ("keccak", native.TABLE_KECCAK)):
        ctx.upload_table(tid, w[t], flags=w.get(t + "_flags"))
    ctx.upload_table(native.TABLE_STEP_AUX, np.zeros((3, 0, 4), dtype=np.uint64))
    ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
    n = w["steps"].shape[1] - 1
    ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
    host = ctx.check(native.CIRCUIT_EVM, 0, n, 0, w["flags"])
    assign.assign_tx_table(ctx, txs)
    dev = ctx.check(native.CIRCUIT_EVM, 0, n, 0, w["flags"])
    assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1])
    assert (dev[0] == native.PASS).all(), native.first_failure(dev[0], native.CIRCUIT_EVM)
    for tid, cols in ((native.TABLE_TX, 5), (native.TABLE_BLOCK, 4)):
        ctx.upload_table(tid, np.zeros((cols, 0, 4), dtype=np.uint64))


def test_rejected_calls_leave_the_previous_table_in_place():
    ctx = native.default_context()
    txs = [Transaction(1, call_data=b"\x01\x00"), Transaction(2, callee_address=None, call_data=b"\x02")]
    tab, fl = _device_tx(ctx, txs)
    rec, cd, offs = assign.tx_records(txs)
    p = np.array([(FR_MODULUS >> (64 * i)) & ((1 << 64) - 1) for i in range(4)], dtype=np.uint64)
    bad = rec.copy()
    bad[0, 10] = p
    with pytest.raises(native.NativeError, match="canonical"):
        ctx.assign_tx_table(bad, cd, offs)
    # (2^31 - 1 rows needs gigabytes of call data here; the emulation runs the same host validation on it)
    for bad_offs, why in (([1, 2, 3], "offsets"), ([0, 3, 2], "non-decreasing")):
        with pytest.raises(native.NativeError, match=why):
            ctx.assign_tx_table(rec, np.zeros(3, dtype=np.uint8), np.array(bad_offs, dtype=np.uint64))
    assert np.array_equal(ctx.download_table(native.TABLE_TX), tab)
    assert np.array_equal(ctx.download_table_flags(native.TABLE_TX), fl)
    ctx.assign_tx_table(np.zeros((0, 11, 4), dtype=np.uint64), b"", np.zeros(1, dtype=np.uint64))
    assert ctx.table_rows(native.TABLE_TX) == 0
    # the copy table: the two asserts, then no resident copy circuit
    w = synth.copy_events(6, 40)
    ctx.upload_columns(native.CIRCUIT_COPY, w["copy"])
    assign.assign_copy_table(ctx)
    good = ctx.download_table(native.TABLE_COPY)
    for row, col, msg in ((-1, 1, "Not enough rows in copy circuit"), (1, 0, "Invalid copy circuit")):
        c = w["copy"].copy()
        c[col, row] = [1, 0, 0, 0]
        ctx.upload_columns(native.CIRCUIT_COPY, c)
        with pytest.raises(AssertionError, match=msg):
            assign.assign_copy_table(ctx)
        assert np.array_equal(ctx.download_table(native.TABLE_COPY), good)
    fresh = native.Context(0)
    with pytest.raises(native.NativeError, match="no resident copy circuit"):
        fresh.assign_copy_table()
    fresh.close()
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
