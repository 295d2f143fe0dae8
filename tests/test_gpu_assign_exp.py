"""The exp-circuit builder on the GPU (zk_assign_exp_circuit, csrc/assign.cu): the resident rows, downloaded, equal the
host mirror of ExpCircuit.add_event / fill_dummy_events cell for cell and, at 2^20 rows, the serial run of the same
bodies (tests/emu/zk_emu_exp.cu); the resident exp table equals the emulation's table and the mirror's Tables(exp_circuit=...) rows;
the exp checker accepts the rows where they stand, on a full grid and on a one-SM grid; the EVM circuit's EXP steps give
the reference's verdicts (tests/golden/evm19.npz) against the table built on the device; a rejected call leaves the
previous rows and table in place."""
import os

import numpy as np
import pytest

import emu_exp_lib
import exp_assign_cases as xc
import golden_util
import oracle_lib
from zkevm_specs_b200 import assign, native
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix
from zkevm_specs_b200.util.arithmetic import FR_MODULUS

pytestmark = pytest.mark.gpu

CASES = list(xc.cases())


def _passes(ctx, n_rows):
    ff, _ = ctx.check(native.CIRCUIT_EXP, 0, n_rows, 0, native.FLAG_WRAP)
    return (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_EXP)


@pytest.mark.parametrize("label,events,n_rows_min", CASES, ids=[c[0] for c in CASES])
def test_device_exp_rows_and_table_equal_mirror_and_emu(label, events, n_rows_min):
    ctx = native.default_context()
    ev = assign.exp_events(events)
    ctx.assign_exp_circuit(ev, n_rows_min)
    want, want_table, used = xc.mirror(events, n_rows_min)
    got, _ = ctx.download_columns(native.CIRCUIT_EXP)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(got, want), np.argwhere((got != want).any(axis=2))[:8]
    tab = ctx.download_table(native.TABLE_EXP)
    _, emu_tab = emu_exp_lib.assign_exp(ev, n_rows_min)
    assert np.array_equal(tab, emu_tab)
    assert xc.table_set(tab) == want_table
    if want.shape[1]:
        ok, hit = _passes(ctx, want.shape[1])
        assert ok, hit


def _workload(n_rows, seed, exp_bits=256):
    """seeded events whose rows fill at most n_rows"""
    events, used, k = [], 0, 0
    while True:
        e = xc.random_events(1, seed=seed * 1000003 + k, exp_bits=exp_bits)[0]
        k += 1
        if used + xc.n_rows(e[1]) > n_rows:
            return events
        events.append(e)
        used += xc.n_rows(e[1])


def test_device_exp_rows_at_2_20_equal_emu_and_check():
    ctx = native.default_context()
    n = 1 << 20
    ev = assign.exp_events(_workload(n, seed=1))
    ctx.assign_exp_circuit(ev, n)
    want, want_tab = emu_exp_lib.assign_exp(ev, n)
    got, _ = ctx.download_columns(native.CIRCUIT_EXP)
    assert got.shape == want.shape and np.array_equal(got, want), np.argwhere((got != want).any(axis=2))[:8]
    del got, want
    assert np.array_equal(ctx.download_table(native.TABLE_EXP), want_tab)
    ok, hit = _passes(ctx, n)
    assert ok, hit


@pytest.fixture(scope="module")
def one_sm_ctx():
    """a context whose grids are sized for one SM (ZKCHECK_SM_COUNT=1): every thread of the row kernel and of the checker
    walks several rows"""
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


@pytest.mark.parametrize("strided", [False, True])
def test_checker_accepts_resident_rows_with_and_without_padding(strided, one_sm_ctx):
    ctx = one_sm_ctx if strided else native.default_context()
    events = _workload(6000, seed=2) + [(xc.MAX, xc.MAX, 1), (3, 2, FR_MODULUS - 1)]
    used = sum(xc.n_rows(x) for _, x, _ in events)
    assert used > 2 * 2048
    for n_min in (0, used + 1000):
        ctx.assign_exp_circuit(assign.exp_events(events), n_min)
        want, want_table, _ = xc.mirror(events, n_min)
        got, _ = ctx.download_columns(native.CIRCUIT_EXP)
        assert np.array_equal(got, want), np.argwhere((got != want).any(axis=2))[:8]
        assert xc.table_set(ctx.download_table(native.TABLE_EXP)) == want_table
        ok, hit = _passes(ctx, want.shape[1])
        assert ok, hit
        # the same rows with one exponentiation cell corrupted, uploaded in their place, fail at that row
        bad = got.copy()
        bad[8, used - 7, 1] ^= np.uint64(1)
        ctx.upload_columns(native.CIRCUIT_EXP, bad)
        ff, fc = ctx.check(native.CIRCUIT_EXP, 0, want.shape[1], 0, native.FLAG_WRAP)
        hit = native.first_failure(ff, native.CIRCUIT_EXP)
        assert hit is not None and hit[0] == used - 7 and hit[3].startswith("XP_EXP_EQ_D"), hit


def test_evm_exp_steps_against_device_built_table():
    """for every EXP scenario with an exp table: the events recovered from the reference's table, assigned on the device,
    rebuild that table as a set; every vector that does not corrupt the exp table gets the reference's verdict (and the
    oracle's arrays) against the device-built table"""
    ctx = native.default_context()
    fixed = fixed_table_matrix()
    for tid, cols in ((native.TABLE_TX, 5), (native.TABLE_BLOCK, 4), (native.TABLE_STEP_AUX, 3)):
        ctx.upload_table(tid, np.zeros((cols, 0, 4), dtype=np.uint64))
    z = np.load(os.path.join(xc.GOLDEN, "evm19.npz"))
    scenarios = [str(n) for n in z["names"] if f"{n}/exp" in z.files]
    assert len(scenarios) == 12 and {"exp_max_max", "exp_wide_exponent"} <= set(scenarios)
    tables = {}
    for name in scenarios:
        golden = z[f"{name}/exp"]
        events = xc.events_from_table(golden)
        ctx.assign_exp_circuit(assign.exp_events(events))
        tab = ctx.download_table(native.TABLE_EXP)
        assert xc.table_set(tab) == xc.table_set(golden), name
        assert tab.shape[1] == golden.shape[1], name  # no padding row, no duplicate
        tables[name] = events
    assert max(xc.n_rows(x) for _, x, _ in tables["exp_max_max"]) == 510
    n = 0
    current = None
    for name, k, w, exp_row, exp_exc in golden_util.evm19_vectors():
        if name not in tables or int(z[f"{name}/mut_kind"][k]) == 14:
            continue
        if current != name:
            ctx.assign_exp_circuit(assign.exp_events(tables[name]))
            current = name
        for t, tid in (("bytecode", native.TABLE_BYTECODE), ("copy", native.TABLE_COPY), ("keccak", native.TABLE_KECCAK)):
            ctx.upload_table(tid, w[t])
        ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
        evm_main.upload_fixed_table(ctx)
        ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
        ff, fc = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, w.get("flags", 0))
        off, ofc = oracle_lib.check_evm_x(w, fixed)
        assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{name}[{k}] differs from the oracle"
        hit = native.first_failure(ff, native.CIRCUIT_EVM)
        got = (-1, "") if hit is None else (hit[0], oracle_lib.EXC_OF_CLASS[hit[2]])
        if got[1] == "ValueError" and exp_exc in ("OverflowError", "UnboundLocalError", "AttributeError", "TypeError"):
            got = (got[0], exp_exc)
        assert got == (exp_row, exp_exc), f"{name}[{k}] cuda {got} reference {(exp_row, exp_exc)}"
        n += 1
    assert n > 500
    for tid, cols in ((native.TABLE_COPY, 14), (native.TABLE_KECCAK, 5), (native.TABLE_EXP, 11)):
        ctx.upload_table(tid, np.zeros((cols, 0, 4), dtype=np.uint64))


def test_rejected_calls_leave_rows_and_table_in_place():
    ctx = native.default_context()
    events = [(7, 1023, 12), (xc.MAX, 77, 13)]
    ctx.assign_exp_circuit(assign.exp_events(events), 100)
    rows, _ = ctx.download_columns(native.CIRCUIT_EXP)
    tab = ctx.download_table(native.TABLE_EXP)
    ok, _ = _passes(ctx, 100)
    assert ok
    bad_id = assign.exp_events([(2, 5, 1)])
    p = [(FR_MODULUS >> (64 * i)) & ((1 << 64) - 1) for i in range(4)]
    bad_id[0, 8:12] = p  # identifier == p: not canonical
    with pytest.raises(native.NativeError, match="canonical"):
        ctx.assign_exp_circuit(bad_id)
    with pytest.raises(native.NativeError, match="too many exp rows"):
        ctx.assign_exp_circuit(assign.exp_events(events), (1 << 31) - 1)
    assert ctx.resident_rows(native.CIRCUIT_EXP) == 100 and ctx.table_rows(native.TABLE_EXP) == tab.shape[1]
    assert np.array_equal(ctx.download_columns(native.CIRCUIT_EXP)[0], rows)
    assert np.array_equal(ctx.download_table(native.TABLE_EXP), tab)
    ok, hit = _passes(ctx, 100)
    assert ok, hit
    ctx.upload_table(native.TABLE_EXP, np.zeros((11, 0, 4), dtype=np.uint64))
