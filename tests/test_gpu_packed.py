"""Packed columns (include/zkcheck.h zk_upload_*_packed, csrc/fr.cuh:ld_col): every GPU parity
test of the other files is repeated with all witness matrices and tables stored at their minimal
per-column widths (constant columns collapsed to one cell) — the verdict arrays must still equal
the oracle's and the reference's golden verdicts bit for bit.  Plus: the type-width packing that
bench.py uses, and the packed ABI's argument checks."""
import numpy as np
import pytest

import oracle_lib
from zkevm_specs_b200 import native, packing, synth
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

pytestmark = pytest.mark.gpu


@pytest.fixture
def packed_ctx():
    ctx = native.default_context()
    ctx.packed_uploads = "min"
    yield ctx
    ctx.packed_uploads = None


def test_every_golden_family_with_packed_storage(packed_ctx):
    import test_gpu_bytecode
    import test_gpu_copy
    import test_gpu_evm
    import test_gpu_exp
    import test_gpu_pi
    import test_gpu_state

    before = packed_ctx.launch_count()
    test_gpu_bytecode.test_bytecode_golden_and_oracle_parity()
    test_gpu_bytecode.test_bytecode_row_sharding_with_halo()
    test_gpu_evm.test_evm_golden_and_oracle_parity()
    test_gpu_evm.test_evm_sha3_calldatacopy_golden_and_oracle_parity()
    test_gpu_evm.test_evm_stop_golden_and_oracle_parity()
    test_gpu_evm.test_evm_memory_golden_and_oracle_parity()
    test_gpu_evm.test_evm_sharded_steps_match_whole()
    test_gpu_copy.test_copy_golden_and_oracle_parity()
    test_gpu_state.test_state_golden_and_oracle_parity()
    test_gpu_state.test_state_sharded_rows_match_whole()
    test_gpu_exp.test_exp_golden_and_oracle_parity()
    test_gpu_pi.test_pi_golden_and_oracle_parity()
    assert packed_ctx.launch_count() > before


def test_synthetic_traces_and_corruptions_with_packed_storage(packed_ctx):
    import test_gpu_copy
    import test_gpu_evm
    import test_gpu_state

    test_gpu_evm.test_evm_synthetic_trace_and_corruptions_match_oracle()
    test_gpu_copy.test_copy_synthetic_2e14_rows_and_corruptions_match_oracle()
    test_gpu_state.test_state_synthetic_2e16_rows_and_corruptions_match_oracle()


def test_type_width_packing_equals_canonical_and_oracle():
    """bench.py's format: data-independent widths by column type (packing.TYPE_WIDTHS)"""
    ctx = native.default_context()
    fixed = fixed_table_matrix()
    from zkevm_specs_b200.evm_circuit import main as evm_main

    w = synth.evm_trace(512, seed=11)
    steps = w["steps"].copy()
    steps[9, 1000, 0] += np.uint64(1)  # gas_left of one step
    rw = w["rw"].copy()
    rw[8, 700, 0] ^= np.uint64(4)      # one stack value
    off, ofc = oracle_lib.check_evm(steps, w["bytecode"], rw, fixed)
    evm_main.upload_fixed_table(ctx)
    results = []
    for packed in (False, True):
        if packed:
            ps = packing.pack_matrix(steps, min_widths=packing.TYPE_WIDTHS["evm_steps"])
            pb = packing.pack_matrix(w["bytecode"], min_widths=packing.TYPE_WIDTHS["bytecode_table"])
            pr = packing.pack_matrix(rw, min_widths=packing.TYPE_WIDTHS["rw_table"])
            assert ps.nbytes * 4 < steps.nbytes and pb.nbytes * 4 < w["bytecode"].nbytes
            assert np.array_equal(ps.unpack(), steps) and np.array_equal(pr.unpack(), rw)
            ctx.upload_table_packed(native.TABLE_BYTECODE, pb)
            ctx.upload_table_packed(native.TABLE_RW, pr)
            ctx.upload_columns_packed(native.CIRCUIT_EVM, ps)
        else:
            ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
            ctx.upload_table(native.TABLE_RW, rw)
            ctx.upload_columns(native.CIRCUIT_EVM, steps)
        results.append(ctx.check(native.CIRCUIT_EVM, 0, steps.shape[1] - 1, 0, 0))
    for ff, fc in results:
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc)
    assert (results[0][0] != native.PASS).sum() >= 2


def test_packed_abi_rejects_bad_layouts():
    ctx = native.default_context()
    w = synth.evm_trace(8, seed=1)
    pm = packing.pack_matrix(w["rw"])
    bad = packing.PackedMatrix(pm.buf, pm.offsets.copy(), pm.widths.copy(), pm.n_rows)
    bad.widths[0] = 3
    with pytest.raises(native.NativeError, match="width"):
        ctx.upload_table_packed(native.TABLE_RW, bad)
    bad = packing.PackedMatrix(pm.buf, pm.offsets.copy(), pm.widths.copy(), pm.n_rows)
    bad.offsets[1] += np.uint64(8)
    with pytest.raises(native.NativeError, match="offset"):
        ctx.upload_table_packed(native.TABLE_RW, bad)
    bad = packing.PackedMatrix(pm.buf, pm.offsets.copy(), pm.widths.copy(), pm.n_rows)
    bad.offsets[-1] = np.uint64(pm.nbytes)
    with pytest.raises(native.NativeError, match="outside"):
        ctx.upload_table_packed(native.TABLE_RW, bad)
    ctx.upload_table_packed(native.TABLE_RW, pm)


def test_bytecode_table_from_code_equals_uploaded_table():
    """zk_upload_bytecode_table_from_code (Bytecode.table_assignments on the device) gives the same
    table as uploading the unrolled rows: same verdict arrays as the oracle on (a) a PUSH32-heavy
    trace with corruptions — every byte row of the table is looked up — and (b) the two-contract STOP
    goldens (restore-to-caller context reads the caller's code hash)."""
    import golden_util
    from zkevm_specs_b200.evm_circuit import main as evm_main

    ctx = native.default_context()
    fixed = fixed_table_matrix()
    evm_main.upload_fixed_table(ctx)
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
    w = synth.evm_trace(2048, seed=21)
    S, R = w["steps"].copy(), w["rw"].copy()
    rng = np.random.default_rng(77)
    for t in range(24):  # pushed values that no longer match the code, gas, pc
        if t % 3 == 0:
            R[8 + int(rng.integers(2)), int(rng.integers(R.shape[1])), int(rng.integers(2))] ^= np.uint64(1 << int(rng.integers(64)))
        else:
            S[9 if t % 3 == 1 else 7, int(rng.integers(1, S.shape[1] - 1)), 0] += np.uint64(1)
    off, ofc = oracle_lib.check_evm(S, w["bytecode"], R, fixed)
    assert (off != native.PASS).any()
    ctx.upload_table(native.TABLE_RW, R)
    ctx.upload_columns(native.CIRCUIT_EVM, S)
    ctx.upload_bytecode_table_from_code(**w["bytecode_src"])
    ff, fc = ctx.check(native.CIRCUIT_EVM, 0, S.shape[1] - 1, 0, 0)
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc)
    n = 0
    for name, k, v, exp_row, exp_exc in golden_util.evm3_vectors():
        src = packing.bytecode_src_from_table(v["bytecode"])
        if src is None or len(src["hashes"]) != 2:
            continue
        ctx.upload_bytecode_table_from_code(**src)
        ctx.upload_table(native.TABLE_RW, v["rw"], flags=v["rw_flags"])
        ctx.upload_columns(native.CIRCUIT_EVM, v["steps"])
        ff, fc = ctx.check(native.CIRCUIT_EVM, 0, v["steps"].shape[1] - 1, 0, 0)
        off, ofc = oracle_lib.check_evm_x(v, fixed)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (name, k)
        n += 1
    assert n > 400


def test_bytecode_table_from_code_with_duplicate_hashes_falls_back():
    """two contracts with the SAME code hash make every bytecode lookup ambiguous: the library-built
    table must then leave the positional path (k_heads_from_offsets clears the flag) and give the
    oracle's verdict (LookupAmbiguousFailure ids), like the explicitly uploaded table does"""
    from zkevm_specs_b200.evm_circuit import main as evm_main

    ctx = native.default_context()
    fixed = fixed_table_matrix()
    evm_main.upload_fixed_table(ctx)
    ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
    w = synth.evm_trace(32, seed=4)
    src = w["bytecode_src"]
    n = len(src["code"])
    # same hash, different bytes (rows identical in EVERY column would count once: the table is a set)
    other = src["code"] ^ np.uint8(1)
    dup = {"code": np.concatenate([src["code"], other]),
           "is_code_bits": np.packbits(np.concatenate([np.unpackbits(src["is_code_bits"], bitorder="little")[:n]] * 2), bitorder="little"),
           "code_offsets": np.array([0, n, 2 * n], dtype=np.uint64),
           "hashes": np.concatenate([src["hashes"], src["hashes"]])}
    second = w["bytecode"].copy()
    second[5, 1:, 0] = other.astype(np.uint64)
    table = np.ascontiguousarray(np.concatenate([w["bytecode"], second], axis=1))
    off, ofc = oracle_lib.check_evm(w["steps"], table, w["rw"], fixed)
    assert (off != native.PASS).any()
    ctx.upload_table(native.TABLE_RW, w["rw"])
    ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
    for from_code in (True, False):
        if from_code:
            ctx.upload_bytecode_table_from_code(**dup)
        else:
            ctx.upload_table(native.TABLE_BYTECODE, table)
        ff, fc = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, 0)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), from_code
