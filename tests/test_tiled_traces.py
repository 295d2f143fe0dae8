"""Tiled golden traces on the CPU (tests/tile_trace.py): the oracle on every tiled trace satisfies the per-copy lower
bound, which guards the tiler itself (a re-keying mistake or a rule that depends on the row shows up here), and the
emulated gate programs equal the oracle on a sample of them, in canonical and packed storage."""
import time

import numpy as np
import pytest

import emu_lib
import oracle_lib
import tile_trace as tt
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

N_COPIES = 2048
EMU_EVERY = 16  # every k-th group of a family goes through the emu
EMU_COPIES = 256


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_tiled_traces.py wall time {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def fixed():
    return fixed_table_matrix()


def _multi(groups):
    return [g for g in groups if len(g[1]) >= 2]


@pytest.mark.parametrize("family", tt.EVM_FAMILIES)
def test_oracle_on_tiled_evm_traces_satisfies_the_per_copy_bound(family, fixed):
    """every group of >= 2 vectors (a scenario's base vector and its step mutations), N_COPIES copies (evm.npz's
    13-21-step vectors: a quarter of that)"""
    groups = _multi(tt.evm_groups(family))
    assert groups
    n_fail = 0
    for gi, (name, members) in enumerate(groups):
        t = tt.tile_evm(members, N_COPIES // 4 if family == "evm" else N_COPIES, gi, fixed)
        ff, fc = tt.oracle_evm(t.w, fixed)
        assert t.holds(ff, fc), f"{family} {name}: per-copy bound broken"
        n_fail += bool(t.lb_count.sum())
    assert n_fail >= len(groups) // 4  # many groups mix passing and failing copies


def test_tiled_traces_need_their_rekeyed_step_aux_rows(fixed):
    """CREATE / CREATE2 (evm24) read StepState.aux_data by the global step row: with every copy's aux rows keyed as if
    it were the first copy, the per-copy bound breaks; with the tiler's re-keying it holds"""
    n_broken = 0
    for gi, (name, members) in enumerate(_multi(tt.evm_groups("evm24"))):
        aux = members[0][1]["aux"]
        if not aux.shape[1]:
            continue
        t = tt.tile_evm(members, 64, gi, fixed)
        assert t.w["aux"].shape[1] == 64 * aux.shape[1]
        assert t.holds(*tt.oracle_evm(t.w, fixed))
        bad = dict(t.w)
        bad["aux"] = np.ascontiguousarray(np.tile(aux, (1, 64, 1)))
        n_broken += not t.holds(*tt.oracle_evm(bad, fixed))
    assert n_broken >= 3


def test_oracle_on_tiled_copy_traces_satisfies_the_per_row_bound():
    """copy.npz groups with identical tables, ~16k rows each, ZK_FLAG_WRAP"""
    groups = _multi(tt.copy_groups())
    assert len(groups) >= 3
    for gi, (name, members) in enumerate(groups):
        n_c = members[0][1]["copy"].shape[1]
        t = tt.tile_copy(members, -(-16384 // n_c), gi)
        ff, fc = oracle_lib.check_copy(t.w, t.r)
        assert t.holds(ff, fc), f"copy {name}: per-row bound broken"
        assert t.lb_count.sum() > 0


@pytest.mark.parametrize("packed", [False, True])
def test_emu_equals_oracle_on_tiled_traces(packed, fixed):
    """every EMU_EVERY-th group of every EVM family (EMU_COPIES copies) and every copy group: the emulated gate programs
    equal the oracle array for array"""
    emu_lib.set_packed(packed)
    try:
        n = 0
        for family in tt.EVM_FAMILIES:
            for gi, (name, members) in enumerate(_multi(tt.evm_groups(family))):
                if gi % EMU_EVERY:
                    continue
                t = tt.tile_evm(members, EMU_COPIES // 4 if family == "evm" else EMU_COPIES, gi, fixed)
                off, ofc = tt.oracle_evm(t.w, fixed)
                ff, fc = emu_lib.check_evm_x(t.w, fixed)
                assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{family} {name}"
                assert t.holds(ff, fc)
                n += 1
        for gi, (name, members) in enumerate(_multi(tt.copy_groups())):
            t = tt.tile_copy(members, 64, gi)
            off, ofc = oracle_lib.check_copy(t.w, t.r)
            ff, fc = emu_lib.check_copy(t.w, t.r)
            assert np.array_equal(ff[: len(off)], off) and np.array_equal(fc[: len(ofc)], ofc), f"copy {name}"
            n += 1
    finally:
        emu_lib.set_packed(False)
    assert n > 120
