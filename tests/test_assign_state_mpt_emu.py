"""The state circuit's roots and MPT table from the operations alone (zk_assign_state_circuit_mpt, csrc/assign.cu), its
per-thread bodies run serially on the CPU (tests/emu/zk_emu_state_mpt.cu): every state_mpt.npz list gives the
reference's rows and its MPT updates in order, or its rejection; the state.npz bases give their rows and MPT table;
synth.state_rows gives synth's roots and table; seeded unsorted lists give the mirror's.  The GPU run is
tests/test_gpu_assign_state_mpt.py."""
import numpy as np
import pytest

import emu_state_mpt_lib as em
import state_mpt_cases as smc
from zkevm_specs_b200 import assign, synth

GOLDEN = list(smc.golden_cases())


@pytest.mark.parametrize("case", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_emu_golden_lists(case):
    name, ops, flags, rows, mpt, exc = case
    got = em.assign_state_mpt(ops, flags)
    if exc:
        assert got[0] == exc, name
        return
    g_rows, g_mpt = got
    assert np.array_equal(assign.state_op13_from_rows(rows), ops)  # the fixture's cells are the rows' own
    assert np.array_equal(g_rows, rows), name
    assert np.array_equal(g_mpt, mpt), name


def test_emu_golden_rejections_name_the_first_failing_op():
    by_name = {c[0]: c for c in GOLDEN}
    assert em.assign_state_mpt(*by_name["reject_word"][1:3]) == ("AssertionError", 3)
    assert em.assign_state_mpt(*by_name["reject_field_tag"][1:3]) == ("KeyError", 2)


@pytest.mark.parametrize("base", list(smc.state_bases()), ids=lambda b: b[0])
def test_emu_state_bases(base):
    name, rows, flags, mpt = base
    g_rows, g_mpt = em.assign_state_mpt(assign.state_op13_from_rows(rows), flags)
    assert np.array_equal(g_rows, rows)
    assert smc.row_set(g_mpt) == smc.row_set(mpt)


def test_emu_synth_state_rows():
    w = synth.state_rows(1 << 14)
    g_rows, g_mpt = em.assign_state_mpt(assign.state_op13_from_rows(w["rows"]), w["flags"])
    assert np.array_equal(g_rows, w["rows"])
    assert smc.row_set(g_mpt) == smc.row_set(w["mpt"])


@pytest.mark.parametrize("seed", range(6))
def test_emu_seeded_lists_equal_mirror(seed):
    ops = smc.mirror_ops(seed, 40 + 60 * seed)
    want = smc.mirror_expected(ops)
    ops13, flags = assign.state_op_cells(ops)
    got = em.assign_state_mpt(ops13, flags)
    if isinstance(want, str):
        assert got[0] == want
        return
    rows, want_flags, mpt = want
    assert np.array_equal(flags, want_flags)
    assert np.array_equal(got[0], rows) and np.array_equal(got[1], mpt)


def test_emu_restatement_unsorted_spread_keys():
    ops, flags = smc.spread_keys(1 << 14, 1 << 10, seed=5)
    rows, mpt = em.assign_state_mpt(ops, flags)
    roots, table = smc.restate(ops, flags)
    assert np.array_equal(rows[54, :, 0], roots) and not rows[54, :, 1:].any() and not rows[55].any()
    assert np.array_equal(mpt, table)


def test_emu_colliding_keys_and_one_key():
    ops, flags = smc.colliding_keys(64, em.home_slot, 256)
    rows, mpt = em.assign_state_mpt(ops, flags)
    roots, table = smc.restate(ops, flags)
    assert mpt.shape[1] == 64 and np.array_equal(rows[54, :, 0], roots) and np.array_equal(mpt, table)
    ops, flags = smc.repeated_key(1 << 12)
    rows, mpt = em.assign_state_mpt(ops, flags)
    assert mpt.shape[1] == 1 and (rows[54, :-1, 0] == 3).all() and rows[54, -1, 0] == 8


def test_emu_edges_and_address_rejection():
    rows, mpt = em.assign_state_mpt(np.zeros((13, 0, 4), dtype=np.uint64))
    assert rows.shape == (57, 0, 4) and mpt.shape == (12, 0, 4)
    ops, flags = smc.repeated_key(8)
    assert em.assign_state_mpt(smc.with_address_beyond_160_bits(ops, 5), flags) == ("address", None)
