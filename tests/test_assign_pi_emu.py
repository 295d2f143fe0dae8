"""The device public-inputs builder (zk_assign_pi_circuit, csrc/assign.cu), its per-thread bodies run serially on the CPU
(tests/emu/zk_emu_pi.cu): pi_circuit.raw_public_inputs builds the stream the host mirror joins; the rows built from it
equal the reference's rows (tests/golden/pi.npz) and the mirror's on edge cases cell for cell, the keccak and calldata
gas tables equal theirs as sets, and the oracle accepts the rows; corrupted streams are assigned as they are and the
oracle rejects them.  The GPU run of the same cases is tests/test_gpu_assign_pi.py."""
import numpy as np
import pytest

import emu_pi_lib
import oracle_lib
import pi_assign_cases as pcases
from test_pi_host import cases as golden_cases
from test_pi_host import load_public_data
from zkevm_specs_b200 import pi_circuit as pc
from zkevm_specs_b200.util.arithmetic import FR_MODULUS

PASS = 0xFFFFFFFF
SYNTH = list(pcases.cases())


def _emu(raw, mt, mc, mw):
    return emu_pi_lib.assign_pi(raw, mt, mc, mw, pc.keccak_rand.n, pc.byte_pow_base.n)


@pytest.mark.parametrize("label,pd,mt,mc,mw", SYNTH, ids=[c[0] for c in SYNTH])
def test_raw_stream_equals_mirror_copy_constrains(label, pd, mt, mc, mw):
    w = pc.public_data2witness(pd, mt, mc, mw)
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    assert raw == b"".join(w.copy_constrains)
    assert len(raw) == w.circuit_len


def test_emu_rows_and_tables_equal_reference_golden():
    n = 0
    for z, name, (mt, mc, mw) in golden_cases():
        pd = load_public_data(z, name)
        raw = pc.raw_public_inputs(pd, mt, mc, mw)
        w = pc.public_data2witness(pd, mt, mc, mw)
        assert raw == b"".join(w.copy_constrains), name
        rows, kec, gas, digest = _emu(raw, mt, mc, mw)
        want = z[f"{name}/rows"]
        assert np.array_equal(rows, want), (name, np.argwhere((rows != want).any(axis=2))[:8])
        assert pcases.table_set(kec) == pcases.table_set(z[f"{name}/keccak"]), name
        assert pcases.table_set(gas) == pcases.table_set(z[f"{name}/gas"]), name
        assert digest == w.public_inputs.pi_keccak.int_value()
        ff, _ = oracle_lib.check_pi(rows, kec, gas, len(raw))
        assert (ff == PASS).all(), name
        n += 1
    assert n == 3


@pytest.mark.parametrize("label,pd,mt,mc,mw", SYNTH, ids=[c[0] for c in SYNTH])
def test_emu_rows_and_tables_equal_mirror(label, pd, mt, mc, mw):
    w = pc.public_data2witness(pd, mt, mc, mw)
    assert w.cells.shape[1] < 1 << 16
    rows, kec, gas, digest = _emu(pc.raw_public_inputs(pd, mt, mc, mw), mt, mc, mw)
    assert np.array_equal(rows, w.cells), np.argwhere((rows != w.cells).any(axis=2))[:8]
    assert pcases.table_set(kec) == w.keccak_table.table
    assert pcases.table_set(gas) == w.calldata_gas_cost_table
    assert gas.shape[1] == 1 + sum(len(t.data) for t in pd.txs)  # the zero row, then one row per used calldata byte
    assert digest == w.public_inputs.pi_keccak.int_value()
    ff, _ = oracle_lib.check_pi(rows, kec, gas, w.circuit_len)
    assert (ff == PASS).all(), ff


def test_padded_withdrawal_slot_carries_the_stream_id():
    """with fewer withdrawals than slots the stream gives padded slot i the id i (withdrawal_raw_bytes(i)) while the
    mirror's table row keeps the default id 0; the reference's copy constraints reject that witness.  The builder takes
    the stream's id; every other cell equals the mirror's"""
    pd = pcases.public_data(2, 16, 1, 19, [3, 4])
    mt, mc, mw = 2, 16, 3
    w = pc.public_data2witness(pd, mt, mc, mw)
    rows, _, _, _ = _emu(pc.raw_public_inputs(pd, mt, mc, mw), mt, mc, mw)
    first = 10 * mt + 1 + mc
    diff = {tuple(x) for x in np.argwhere((rows != w.cells).any(axis=2))}
    assert diff == {(pc.P_WD_ID, first + 1), (pc.P_WD_ID, first + 2)}
    assert [int(rows[pc.P_WD_ID, first + k, 0]) for k in range(3)] == [0, 1, 2]
    with pytest.raises(AssertionError):
        pc._copy_constraints(w, mt, mc, mw)


def test_fr_inv():
    rng = np.random.default_rng(3)
    vals = [0, 1, 2, FR_MODULUS - 1, FR_MODULUS - 2] + list(range(3, 256)) + [
        int.from_bytes(rng.bytes(32), "little") % FR_MODULUS for _ in range(64)] + [(1 << 160) - 1, 1 << 128]
    for v in vals:
        assert emu_pi_lib.fr_inv(v) == (pow(v, -1, FR_MODULUS) if v else 0), v


CORRUPT = list(pcases.corruptions())


@pytest.mark.parametrize("label,raw,mt,mc,mw,wd_row", CORRUPT, ids=[c[0] for c in CORRUPT])
def test_corrupted_streams_are_assigned_and_rejected_by_the_oracle(label, raw, mt, mc, mw, wd_row):
    rows, kec, gas, _ = _emu(raw, mt, mc, mw)
    ff, fc = oracle_lib.check_pi(rows, kec, gas, len(raw))
    assert (ff != PASS).any(), label
    if wd_row is not None:  # only the amount gate fails, at the withdrawal's row
        assert int(ff.min()) == wd_row and (ff != PASS).sum() == 1, ff


def test_rejected_streams():
    _, pd, mt, mc, mw = SYNTH[0]
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    assert _emu(raw, mt, mc, mw) is not None
    assert _emu(raw[:-1], mt, mc, mw) is None  # a wrong length
    assert _emu(raw, mt + 1, mc, mw) is None
    assert _emu(pcases.corrupt_cdl(raw, mt, 3, mc - 49), mt, mc, mw) is None  # 50 bytes used: the sum becomes mc + 1
    assert _emu(pcases.corrupt_cdl(raw, mt, 3, mc - 50), mt, mc, mw) is not None  # exactly mc
    assert _emu(raw, 0, mc, mw) is None
    assert _emu(raw, mt, mc, 0) is None
