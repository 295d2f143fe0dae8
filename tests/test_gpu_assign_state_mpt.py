"""The state circuit's roots and MPT table from the operations alone on the GPU (zk_assign_state_circuit_mpt,
csrc/assign.cu): every state_mpt.npz list downloads as the reference's rows and MPT updates in order, or is rejected
with the mirror's exception; zk_check(STATE) after the call gives verify_state_circuit's verdicts on host-built rows and
tables (golden bases, synth 2^18 clean and corrupted); at scale the rows and table equal synth's (2^21 ops) and the
numpy restatement (2^20 unsorted ops over 2^16 keys, one key repeated 2^20 times, 64 keys sharing one home slot); the
builders run on a one-SM grid; rejected calls leave the previous matrix and table in place."""
import os

import numpy as np
import pytest

import emu_state_mpt_lib as em
import state_mpt_cases as smc
from zkevm_specs_b200 import assign, native, packing, synth
from zkevm_specs_b200 import state_circuit as sc

pytestmark = pytest.mark.gpu

GOLDEN = list(smc.golden_cases())


@pytest.fixture(scope="module")
def one_sm_ctx():
    """a context whose grids are sized for one SM (ZKCHECK_SM_COUNT=1): every thread walks several operations"""
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


def _assign(ctx, ops, flags):
    n_upd = assign.assign_state_circuit_mpt(ctx, ops, flags)
    rows, fl = ctx.download_columns(native.CIRCUIT_STATE)
    mpt = ctx.download_table(native.TABLE_MPT)
    assert mpt.shape[1] == n_upd
    return rows, fl, mpt


def _host_verdict(ctx, rows, flags, mpt):
    return sc.check_matrices(ctx, rows, flags, mpt)


def _device_verdict(ctx, ops, flags):
    assign.assign_state_circuit_mpt(ctx, ops, flags)
    return ctx.check(native.CIRCUIT_STATE, 0, ops.shape[1], 0, native.FLAG_WRAP)


def _same_verdict(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("case", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_device_golden_lists(case, strided, one_sm_ctx):
    ctx = one_sm_ctx if strided else native.default_context()
    name, ops, flags, rows, mpt, exc = case
    if exc:
        with pytest.raises({"KeyError": KeyError, "AssertionError": AssertionError}[exc]):
            assign.assign_state_circuit_mpt(ctx, ops, flags)
        return
    g_rows, g_fl, g_mpt = _assign(ctx, ops, flags)
    assert np.array_equal(g_rows, rows) and np.array_equal(g_fl, flags) and np.array_equal(g_mpt, mpt), name


def test_device_golden_verdicts():
    ctx = native.default_context()
    for name, ops, flags, rows, mpt, exc in GOLDEN:
        if not exc:
            _same_verdict(_device_verdict(ctx, ops, flags), _host_verdict(ctx, rows, flags, mpt))
    for name, rows, flags, mpt in smc.state_bases():
        ops = assign.state_op13_from_rows(rows)
        _same_verdict(_device_verdict(ctx, ops, flags), _host_verdict(ctx, rows, flags, mpt))
        assign.assign_state_circuit_mpt(ctx, ops, flags)
        sc.verify_state_circuit_resident(ctx)  # the reference passes these bases


def test_device_mirror_operations():
    """assign.state_op_cells packs mirror Operation objects: the device gives the mirror's rows and ordered table"""
    ctx = native.default_context()
    for seed in range(3):
        ops = smc.mirror_ops(seed, 300)
        rows, flags, mpt = smc.mirror_expected(ops)
        g_rows, g_fl, g_mpt = _assign(ctx, ops, None)
        assert np.array_equal(g_rows, rows) and np.array_equal(g_fl, flags) and np.array_equal(g_mpt, mpt)


@pytest.mark.parametrize("corrupt", [False, True])
def test_device_synth_2_18_verdicts(corrupt):
    ctx = native.default_context()
    w = synth.state_rows(1 << 18)
    rows = w["rows"]
    if corrupt:  # one Storage read value changed, on a row that repeats the previous row's key: not a first touch,
        rows = rows.copy()  # so the MPT table stays the same
        repeat = np.r_[False, (rows[2:8, 1:, :] == rows[2:8, :-1, :]).all(axis=(0, 2))]
        reads = np.nonzero((rows[1, :, 0] == 0) & (rows[2, :, 0] == 4) & repeat)[0]
        rows[50, reads[len(reads) // 2], 0] ^= 1
    host = _host_verdict(ctx, rows, w["flags"], w["mpt"])
    dev = _device_verdict(ctx, assign.state_op13_from_rows(rows), w["flags"])
    _same_verdict(dev, host)
    assert (host[0] != native.PASS).any() == corrupt


def test_device_synth_2_21():
    ctx = native.default_context()
    w = synth.state_rows(1 << 21)
    ops = packing.pack_matrix(assign.state_op13_from_rows(w["rows"]))  # narrow columns, as a caller would ship them
    roots = w["rows"][54:56].copy()
    del w["rows"]  # 3.8 GB of canonical cells: keep one such matrix in host memory at a time
    n_upd = assign.assign_state_circuit_mpt(ctx, ops, w["flags"])
    rows, _ = ctx.download_columns(native.CIRCUIT_STATE)
    assert np.array_equal(rows[54:56], roots)
    del rows
    mpt = ctx.download_table(native.TABLE_MPT)
    assert n_upd == w["mpt"].shape[1] and smc.row_set(mpt) == smc.row_set(w["mpt"])
    sc.verify_state_circuit_resident(ctx)


@pytest.mark.parametrize("strided", [False, True])
def test_device_restatements_at_scale(strided, one_sm_ctx):
    ctx = one_sm_ctx if strided else native.default_context()
    for ops, flags in (smc.spread_keys(1 << 20, 1 << 16, seed=9), smc.repeated_key(1 << 20),
                       smc.colliding_keys(64, em.home_slot, 256)):
        rows, _, mpt = _assign(ctx, ops, flags)
        roots, table = smc.restate(ops, flags)
        assert np.array_equal(rows[54, :, 0], roots) and not rows[54, :, 1:].any() and not rows[55].any()
        assert np.array_equal(mpt, table)
        assert np.array_equal(assign.state_op13_from_rows(rows), ops)


def test_rejected_calls_keep_the_previous_matrix_and_table():
    ctx = native.default_context()
    by_name = {c[0]: c for c in GOLDEN}
    _, rows, flags, _ = next(smc.state_bases())  # a witness the reference accepts
    ops = assign.state_op13_from_rows(rows)
    assign.assign_state_circuit_mpt(ctx, ops, flags)
    mpt = ctx.download_table(native.TABLE_MPT)
    for bad, bad_flags, exc in ((by_name["reject_word"][1], by_name["reject_word"][2], AssertionError),
                                (by_name["reject_field_tag"][1], by_name["reject_field_tag"][2], KeyError),
                                (smc.with_address_beyond_160_bits(ops, 3), flags, native.NativeError)):
        with pytest.raises(exc):
            assign.assign_state_circuit_mpt(ctx, bad, bad_flags)
        g_rows, g_fl = ctx.download_columns(native.CIRCUIT_STATE)
        assert np.array_equal(g_rows, rows) and np.array_equal(g_fl, flags)
        assert np.array_equal(ctx.download_table(native.TABLE_MPT), mpt)
    sc.verify_state_circuit_resident(ctx)
