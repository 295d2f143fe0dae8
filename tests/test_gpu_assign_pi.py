"""The public-inputs builder on the GPU (zk_assign_pi_circuit, csrc/assign.cu): the resident rows, downloaded, equal the
reference's rows (tests/golden/pi.npz), the host mirror's on edge cases and, at the bench shape and with 2^20 calldata
bytes, the serial run of the same bodies (tests/emu/zk_emu_pi.cu); the keccak and calldata gas tables equal theirs as
sets; the returned digest equals the host's; the checker accepts the rows where they stand on a full grid and on a
one-SM grid; corrupted streams get the oracle's verdicts; verify_public_data raises like verify_circuit; a rejected
call leaves the previous rows, tables and circuit length in place."""
import os

import numpy as np
import pytest

import emu_pi_lib
import oracle_lib
import pi_assign_cases as pcases
from test_pi_host import cases as golden_cases
from test_pi_host import load_public_data
from zkevm_specs_b200 import assign, native
from zkevm_specs_b200 import pi_circuit as pc
from zkevm_specs_b200.util.arithmetic import Word
from zkevm_specs_b200.util.hash import keccak256

pytestmark = pytest.mark.gpu

SYNTH = list(pcases.cases())


@pytest.fixture(autouse=True, scope="module")
def _empty_tables_after():
    """the calls replace the default context's keccak and calldata gas tables: leave them empty for later modules"""
    yield
    ctx = native.default_context()
    ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_CALLDATA_GAS, np.zeros((3, 0, 4), dtype=np.uint64))


def _assign(ctx, raw, mt, mc, mw):
    ctx.set_challenge(native.CHALLENGE_PI_KECCAK, pc.keccak_rand.n)
    ctx.set_challenge(native.CHALLENGE_PI_BYTE_BASE, pc.byte_pow_base.n)
    return ctx.assign_pi_circuit(mt, mc, mw, raw)


def _download(ctx):
    rows, _ = ctx.download_columns(native.CIRCUIT_PI)
    return rows, ctx.download_table(native.TABLE_KECCAK), ctx.download_table(native.TABLE_CALLDATA_GAS)


def _check(ctx, n):
    ff, fc = ctx.check(native.CIRCUIT_PI, 0, n, 0, native.FLAG_WRAP)
    return ff, fc


def test_device_rows_equal_reference_golden():
    ctx = native.default_context()
    for z, name, (mt, mc, mw) in golden_cases():
        pd = load_public_data(z, name)
        raw = pc.raw_public_inputs(pd, mt, mc, mw)
        digest = _assign(ctx, raw, mt, mc, mw)
        rows, kec, gas = _download(ctx)
        want = z[f"{name}/rows"]
        assert np.array_equal(rows, want), (name, np.argwhere((rows != want).any(axis=2))[:8])
        assert pcases.table_set(kec) == pcases.table_set(z[f"{name}/keccak"]), name
        assert pcases.table_set(gas) == pcases.table_set(z[f"{name}/gas"]), name
        # the digest: keccak256 of the bytes in processing order (rows n-1 .. 0), and the reference's row-0 cells
        seq = bytes(int(b) for b in want[pc.P_BYTES, ::-1, 0])
        assert digest == Word(keccak256(seq)).int_value()
        assert digest == int(want[pc.P_DIGEST_LO, 0, 0]) | int(want[pc.P_DIGEST_LO, 0, 1]) << 64 | (
            int(want[pc.P_DIGEST_HI, 0, 0]) | int(want[pc.P_DIGEST_HI, 0, 1]) << 64) << 128
        ff, _ = _check(ctx, len(raw))
        assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)


@pytest.mark.parametrize("label,pd,mt,mc,mw", SYNTH, ids=[c[0] for c in SYNTH])
def test_device_rows_equal_mirror(label, pd, mt, mc, mw):
    ctx = native.default_context()
    w = pc.public_data2witness(pd, mt, mc, mw)
    digest = _assign(ctx, pc.raw_public_inputs(pd, mt, mc, mw), mt, mc, mw)
    rows, kec, gas = _download(ctx)
    assert np.array_equal(rows, w.cells), np.argwhere((rows != w.cells).any(axis=2))[:8]
    assert pcases.table_set(kec) == w.keccak_table.table
    assert pcases.table_set(gas) == w.calldata_gas_cost_table
    assert digest == w.public_inputs.pi_keccak.int_value()
    ff, _ = _check(ctx, w.circuit_len)
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)


@pytest.fixture(scope="module")
def one_sm_ctx():
    """a context whose grids are sized for one SM (ZKCHECK_SM_COUNT=1): every thread of the row kernels and of the
    checker walks several rows"""
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


@pytest.mark.parametrize("max_cd", [1 << 18, 1 << 20], ids=["bench_shape", "calldata_2_20"])
def test_device_rows_at_scale_equal_emu_and_check(max_cd, one_sm_ctx):
    pd, mt, mc, mw = pcases.bench_shape(max_cd)
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    rows_e, kec_e, gas_e, digest_e = emu_pi_lib.assign_pi(raw, mt, mc, mw, pc.keccak_rand.n, pc.byte_pow_base.n)
    for ctx in (native.default_context(), one_sm_ctx):
        digest = _assign(ctx, raw, mt, mc, mw)
        assert digest == digest_e
        rows, kec, gas = _download(ctx)
        assert np.array_equal(rows, rows_e), np.argwhere((rows != rows_e).any(axis=2))[:8]
        del rows
        assert np.array_equal(kec, kec_e) and np.array_equal(gas, gas_e)
        ff, _ = _check(ctx, len(raw))
        assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)


def test_one_tx_owns_all_calldata():
    """one tx with 2^20 calldata bytes: the per-tx gas sum runs across every block of the scan"""
    mt, mc, mw = 2, 1 << 20, 1
    pd = pcases.public_data(1, mc, 1, 21, [mc])
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    rows_e, _, gas_e, _ = emu_pi_lib.assign_pi(raw, mt, mc, mw, pc.keccak_rand.n, pc.byte_pow_base.n)
    ctx = native.default_context()
    _assign(ctx, raw, mt, mc, mw)
    rows, _, gas = _download(ctx)
    assert np.array_equal(rows, rows_e) and np.array_equal(gas, gas_e)
    ff, _ = _check(ctx, len(raw))
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)


CORRUPT = list(pcases.corruptions())


@pytest.mark.parametrize("label,raw,mt,mc,mw,wd_row", CORRUPT, ids=[c[0] for c in CORRUPT])
def test_corrupted_streams_get_the_oracle_verdict(label, raw, mt, mc, mw, wd_row):
    ctx = native.default_context()
    _assign(ctx, raw, mt, mc, mw)
    rows, kec, gas = _download(ctx)
    rows_e, kec_e, gas_e, _ = emu_pi_lib.assign_pi(raw, mt, mc, mw, pc.keccak_rand.n, pc.byte_pow_base.n)
    assert np.array_equal(rows, rows_e) and np.array_equal(kec, kec_e) and np.array_equal(gas, gas_e)
    ff, fc = _check(ctx, len(raw))
    off, ofc = oracle_lib.check_pi(rows, kec, gas, len(raw))
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc), label
    assert (ff != native.PASS).any()
    if wd_row is not None:
        assert native.first_failure(ff, native.CIRCUIT_PI)[0] == wd_row


def test_verify_public_data():
    _, pd, mt, mc, mw = SYNTH[0]
    pi = pc.verify_public_data(pd, mt, mc, mw)
    assert pi.pi_keccak == pc.public_data2witness(pd, mt, mc, mw).public_inputs.pi_keccak
    pd.withdrawals[1].amount = 0
    with pytest.raises(Exception) as dev:
        pc.verify_public_data(pd, mt, mc, mw)
    with pytest.raises(Exception) as host:
        pc.verify_circuit(pc.public_data2witness(pd, mt, mc, mw), mt, mc, mw)
    assert type(dev.value) is type(host.value)
    assert str(dev.value) == str(host.value)
    n, _ = assign.assign_pi_circuit(native.default_context(), pd, mt, mc, mw)
    assert n == pc.public_data2witness(pd, mt, mc, mw).circuit_len


def test_rejected_calls_leave_rows_tables_and_length_in_place():
    ctx = native.default_context()
    _, pd, mt, mc, mw = SYNTH[1]
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    _assign(ctx, raw, mt, mc, mw)
    before = _download(ctx)
    ff, _ = _check(ctx, len(raw))
    assert (ff == native.PASS).all()
    _, pd2, mt2, mc2, mw2 = SYNTH[0]
    raw2 = pc.raw_public_inputs(pd2, mt2, mc2, mw2)
    used = sum(len(t.data) for t in pd2.txs)
    for bad in ((mt2, mc2, mw2, raw2[:-1]),                                                   # a wrong length
                (mt2, mc2, mw2, pcases.corrupt_cdl(raw2, mt2, 3, mc2 - used + 1)),             # calldata sum above the max
                (0, mc2, mw2, raw2)):                                                         # max_txs = 0
        with pytest.raises(native.NativeError):
            _assign(ctx, bad[3], *bad[:3])
    after = _download(ctx)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert ctx.resident_rows(native.CIRCUIT_PI) == len(raw)
    ff, _ = _check(ctx, len(raw))  # the keccak lookup reads the circuit length: still the first call's
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)
