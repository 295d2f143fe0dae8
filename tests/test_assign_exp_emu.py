"""The device exp-circuit builder (zk_assign_exp_circuit, csrc/assign.cu), its per-thread bodies run serially on the CPU
(tests/emu/zk_emu_exp.cu): the rows equal, cell for cell, what the host mirror of ExpCircuit.add_event / fill_dummy_events produces,
the exp table equals the mirror's Tables(exp_circuit=...) rows as a set, and the mirror itself reproduces the
reference's rows (tests/golden/exp.npz).  The GPU run of the same cases is tests/test_gpu_assign_exp.py."""
import numpy as np
import pytest

import emu_exp_lib
import emu_lib
import exp_assign_cases as xc
import oracle_lib
import row_tables
from zkevm_specs_b200 import assign

XP = row_tables.constraint_ids("exp")


def test_host_mirror_reproduces_reference_exp_rows():
    """the events recovered from each golden scenario, padded to its length, give the reference's rows exactly"""
    n = 0
    for name, events, rows in xc.golden_events():
        assert events, name
        got, _, _ = xc.mirror(events, rows.shape[1])
        assert np.array_equal(got, rows), (name, np.argwhere((got != rows).any(axis=2))[:8])
        n += 1
    assert n == 3


@pytest.mark.parametrize("label,events,n_rows_min", list(xc.cases()), ids=[c[0] for c in xc.cases()])
def test_emu_exp_rows_and_table_equal_host_mirror(label, events, n_rows_min):
    want, want_table, used = xc.mirror(events, n_rows_min)
    got, tab = emu_exp_lib.assign_exp(assign.exp_events(events), n_rows_min)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(got, want), np.argwhere((got != want).any(axis=2))[:8]
    padded = want.shape[1] > used
    assert tab.shape == (11, used + padded, 4)
    rows = [tuple(xc.cell(tab[c, r]) for c in range(11)) for r in range(tab.shape[1])]
    assert set(rows) == want_table
    assert rows.count(xc.PAD_TABLE_ROW) == int(padded)


def test_emu_exp_rows_pass_the_checker_and_a_corruption_fails_at_its_row():
    events = xc.random_events(12, seed=9) + [(xc.MAX, xc.MAX, 1), (5, 2, 2)]
    rows, _ = emu_exp_lib.assign_exp(assign.exp_events(events), 3000)
    n = len(XP)
    ff, fc = emu_lib.check_exp(rows)
    assert (ff[:n] == 0xFFFFFFFF).all()
    off, _ = oracle_lib.check_exp(rows)
    assert (off == 0xFFFFFFFF).all()
    rng = np.random.default_rng(3)
    used = sum(xc.n_rows(x) for _, x, _ in events)
    for r in [0, used - 1, *rng.integers(1, used - 1, 6)]:
        bad = rows.copy()
        bad[8, r, 0] ^= np.uint64(1 << int(rng.integers(0, 64)))  # exponentiation.lo: only row r reads it
        ff, fc = emu_lib.check_exp(bad)
        assert int(ff[XP["XP_EXP_EQ_D"]]) == r and int(fc[XP["XP_EXP_EQ_D"]]) == 1
        assert int(ff[:n].min()) == r
        off, ofc = oracle_lib.check_exp(bad)
        assert np.array_equal(ff[:n], off) and np.array_equal(fc[:n], ofc)


def test_emu_evm_exp_steps_against_emu_built_table():
    """the events recovered from each reference exp table (tests/golden/evm19.npz) rebuild it as a set, and every vector
    that does not corrupt the exp table gets the reference's verdict from the EVM gate programs (emu) and the oracle
    against the rebuilt table"""
    import os

    import golden_util
    from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

    z = np.load(os.path.join(xc.GOLDEN, "evm19.npz"))
    tables = {}
    for name in (str(n) for n in z["names"]):
        if f"{name}/exp" in z.files:
            _, tables[name] = emu_exp_lib.assign_exp(assign.exp_events(xc.events_from_table(z[f"{name}/exp"])))
            assert xc.table_set(tables[name]) == xc.table_set(z[f"{name}/exp"]), name
    assert len(tables) == 12
    fixed = fixed_table_matrix()
    n = 0
    for name, k, w, exp_row, exp_exc in golden_util.evm19_vectors():
        if name not in tables or int(z[f"{name}/mut_kind"][k]) == 14:
            continue
        w = dict(w, exp=tables[name])
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        ff, fc = emu_lib.check_evm_x(w, fixed)
        assert np.array_equal(ff[:len(off)], off) and np.array_equal(fc[:len(off)], ofc), f"{name}[{k}]"
        bad = np.nonzero(off != 0xFFFFFFFF)[0]
        got = -1 if len(bad) == 0 else int(off[bad].min())
        assert got == exp_row, f"{name}[{k}] {got} reference {exp_row} {exp_exc}"
        n += 1
    assert n > 600
