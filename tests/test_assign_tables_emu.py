"""The tx-table and copy-table builders (zk_assign_tx_table, zk_assign_copy_table, csrc/assign.cu), their per-thread bodies
run serially on the CPU (tests/emu/zk_emu_tables.cu): the tx table equals the mirror's Transaction.table_assignments as
a set of (cells, Word flag) and the numpy restatement row for row, on edge cases, on one tx of 2^20 call-data bytes and
on the transactions recovered from every golden tx table; the copy table equals the numpy restatement of
Tables._convert_copy_circuit_to_table on every copy.npz vector, or raises the same assert; rejected inputs are refused.
The GPU run is tests/test_gpu_assign_tables.py."""
import numpy as np
import pytest

import emu_tables_lib as et
import golden_util
import tables_assign_cases as tc
from zkevm_specs_b200 import assign, synth
from zkevm_specs_b200.evm_circuit.typing import Transaction
from zkevm_specs_b200.util.arithmetic import FR_MODULUS

CASES = list(tc.cases())


def _check_tx(txs):
    rec, cd, offs = assign.tx_records(txs)
    tab, fl = et.assign_tx_table(rec, cd, offs)
    want, want_fl = tc.tx_table_restated(rec, cd, offs)
    assert np.array_equal(tab, want) and np.array_equal(fl, want_fl)
    assert tc.table_set(tab, fl) == tc.mirror_set(txs)
    return rec, offs


@pytest.mark.parametrize("label,txs", CASES, ids=[c[0] for c in CASES])
def test_emu_tx_table_equals_mirror(label, txs):
    rec, offs = _check_tx(txs)
    if label == "many_small":  # small ids, bytes and counters: no 32-byte id or value column
        assert list(et.tx_table_widths(rec, offs)) == [2, 1, 1, 8, 1]


def test_emu_tx_table_one_tx_of_2_20_bytes():
    _check_tx(tc.big_tx())


def test_golden_tx_tables_rebuild_from_recovered_transactions():
    """every golden tx table of evm11 / evm17 / evm26 / evm28 is exactly the table_assignments of its transactions"""
    counts = {}
    for f, name, table, flags in tc.golden_tx_tables():
        txs = tc.txs_from_table(table, flags)
        assert txs is not None, (f, name)
        got, fl = et.assign_tx_table(*assign.tx_records(txs))
        assert got.shape == table.shape and tc.table_set(got, fl) == tc.table_set(table, flags), (f, name)
        counts[f] = counts.get(f, 0) + 1
    assert counts == {"evm11": 22, "evm17": 7, "evm26": 8, "evm28": 113}


def test_emu_tx_table_rejections():
    rec, cd, offs = assign.tx_records([Transaction(1, call_data=b"\x01\x00"), Transaction(2, call_data=b"\x02")])
    assert et.assign_tx_table(rec, cd, offs) is not None
    p = np.array([(FR_MODULUS >> (64 * i)) & ((1 << 64) - 1) for i in range(4)], dtype=np.uint64)
    for cell in (0, 1, 2, 6, 8, 9, 10):  # every value cell at p
        bad = rec.copy()
        bad[1, cell] = p
        assert et.assign_tx_table(bad, cd, offs) is None, cell
    big = rec.copy()
    big[1, 3] = np.uint64((1 << 64) - 1)  # a Word cell may use all 256 bits
    assert et.assign_tx_table(big, cd, offs) is not None
    for bad_offs in ([1, 2, 3], [0, 3, 2], [0, 2, (1 << 31) - 25]):  # not from 0, decreasing, 2^31 - 1 rows
        assert et.assign_tx_table(rec, cd, np.array(bad_offs, dtype=np.uint64)) is None, bad_offs
    with pytest.raises(AssertionError):  # a Word field outside [0, 2^256) is refused like Word()
        assign.tx_records([Transaction(1, value=1 << 256)])
    # value fields are reduced like FQ(); a creation has is_create 1 and callee 0
    rec2, _, _ = assign.tx_records([Transaction(FR_MODULUS + 5, nonce=FR_MODULUS, callee_address=None)])
    assert tc.cell(rec2[0, 0]) == 5 and tc.cell(rec2[0, 1]) == 0 and tc.cell(rec2[0, 5]) == 0 and tc.cell(rec2[0, 6]) == 1


def test_emu_copy_table_equals_restatement_on_copy_vectors():
    n = n_assert = 0
    for name, k, w, r, exp_row, exp_exc in golden_util.copy_vectors():
        want = tc.copy_table_restated(w["copy"])
        got = et.assign_copy_table(w["copy"])
        if isinstance(want, str):
            assert got == want, (name, k)
            n_assert += 1
        else:
            assert isinstance(got, np.ndarray) and np.array_equal(got, want), (name, k)
        n += 1
    assert n == 257 and n_assert == 2


def test_emu_copy_table_asserts_and_duplicates():
    w = synth.copy_events(6, 40)
    c = w["copy"]
    want = tc.copy_table_restated(c)
    assert want.shape == (14, 6, 4)
    dup = np.ascontiguousarray(np.concatenate([c, c], axis=1))  # duplicate events: duplicate rows
    got = et.assign_copy_table(dup)
    assert np.array_equal(got, np.concatenate([want, want], axis=1))
    last = c.copy()
    last[1, -1] = [1, 0, 0, 0]  # an is_first on the last row
    assert et.assign_copy_table(last) == tc.copy_table_restated(last) == "Not enough rows in copy circuit"
    both = last.copy()
    both[0, 1] = [1, 0, 0, 0]  # and, earlier, a next row with q_step != 0: the earlier assert wins
    assert et.assign_copy_table(both) == tc.copy_table_restated(both) == "Invalid copy circuit"
    near = c.copy()
    near[1, 0] = [1, 1, 0, 0]  # is_first must equal 1 exactly
    assert np.array_equal(et.assign_copy_table(near), tc.copy_table_restated(near))
    assert et.assign_copy_table(near).shape[1] == 5
    assert et.assign_copy_table(np.zeros((20, 0, 4), dtype=np.uint64)).shape == (14, 0, 4)
