"""The row circuits' lookup tables reordered and duplicated on the device: the counterpart of test_gpu_lookup.py for
the bytecode (push, keccak), state (MPT), public-inputs (keccak, calldata gas), tx and sig (keccak) checkers.

The golden tables come in generator order, and the push table is the canonical 256-row one, so the golden runs take
the staged push path and barely probe the hash indexes.  Here every table is permuted, given identical copies of its
rows and near-copies differing in one column (each column in turn), and the push table is served by each of its
three paths with the same corruptions: staged in shared memory (canonical), dense by position (min-packed, or a
dense table that starts at 1), and the hash probe (permuted).  Every result == the oracle's, under several lookup
challenges."""
import time

import numpy as np
import pytest

import row_tables as rt
import table_perturb as tp
import test_gpu_row_tiled as T
from oracle_lib import same as _same
from zkevm_specs_b200 import native

pytestmark = pytest.mark.gpu
PASS = native.PASS
EVERY = {"bytecode": 3, "state": 3, "pi": 16, "tx": 3, "sig": 3}
DEFAULT_LOOKUP_CHALLENGE = 0x0FE3A95BD3A1C8E714057B7EF767814F5851F42D4C957F2D2545F4914F6CDD1D  # api.cu zk_ctx_create


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_row_lookup.py wall time {time.time() - t0:.1f} s")


def _every(fam, every):
    for j, (label, w) in enumerate(rt.vectors(fam)):
        if j % every == 0:
            yield j, label, w


@pytest.mark.parametrize("fam", rt.LOOKUP_FAMILIES)
def test_device_with_reordered_and_duplicated_tables(fam):
    """every 3rd (pi: 16th) golden vector, each table of the family permuted, with identical copies and with
    near-copies in every column: device == oracle(transformed), and the permuted / identical ones == oracle(original)"""
    ctx = native.default_context()
    never = [rt.constraint_ids(fam)[n] for n in rt.NEVER.get(fam, ())]
    n = 0
    for j, label, w in _every(fam, EVERY[fam]):
        base = rt.oracle(fam, w)
        for ti, table in enumerate(rt.TABLES[fam]):
            for kind, u in rt.transformed(w, table, 7 * j + ti):
                want = rt.oracle(fam, u)
                if kind in ("permuted", "identical"):
                    _same(want, base, f"oracle {fam} {label} {table} {kind}")
                assert not want[1][never].any()
                _same(T.device(ctx, fam, u), want, f"{fam} {label} {table} {kind}")
        n += 1
    assert n >= 40


def _push_corrupted():
    """the strided bytecode witness with push_data_size (column 11) wrong on Byte rows across the matrix, some
    in one warp: BC_PUSH_TABLE fails at each"""
    w, _, _ = T.witness("bytecode")
    m = w["m"].copy()
    byte_rows = np.nonzero(m[4, :, 0] == 2)[0]
    rows = np.unique(np.concatenate([byte_rows[::97], byte_rows[2048:2080:5], byte_rows[-3:]]))
    m[11, rows, 0] += np.uint64(1)
    return dict(w, m=m), rows


def test_push_table_paths_give_the_oracles_rows():
    """the same corruptions under the staged (canonical), dense positional (min-packed), hash (permuted, identical
    copy) push table, and a dense 256-row table starting at 1 (positional, not staged): == oracle, BC_PUSH_TABLE at
    the oracle's rows; the first four are the same set, so their verdicts are one"""
    ctx = native.default_context()
    w, rows = _push_corrupted()
    push = w["push"]
    bc_push = rt.constraint_ids("bytecode")["BC_PUSH_TABLE"]
    want = rt.oracle("bytecode", w)
    assert want[0][bc_push] == rows[0] and want[1][bc_push] >= len(rows)
    for name, t, packed in (("staged", push, None), ("dense", push, "min"), ("hash", tp.permute(push, None, 4)[0], None),
                            ("hash, a duplicate row", tp.with_identical_duplicates(push, None, k=2, seed=1)[0], None)):
        ctx.packed_uploads = packed
        try:
            _same(T.device(ctx, "bytecode", dict(w, push=t)), want, name)
        finally:
            ctx.packed_uploads = None
    shifted = push.copy()
    shifted[0, :, 0] += np.uint64(1)  # rows (v + 1, size(v)): dense by position, but not from 0
    u = dict(w, push=shifted)
    want1 = rt.oracle("bytecode", u)
    assert want1[1][bc_push] > want[1][bc_push]
    _same(T.device(ctx, "bytecode", u), want1, "dense from 1")


P = tp.P


def test_lookup_challenge_never_changes_a_row_verdict():
    """ZK_CHALLENGE_LOOKUP = 0, 1, p - 1 and a random value: every 10th golden vector of each family with each table
    permuted == oracle, and the push-path corruptions above; the default is restored"""
    ctx = native.default_context()
    rnd = int.from_bytes(np.random.default_rng(99).bytes(32), "little") % P
    pw, _ = _push_corrupted()
    pwant = rt.oracle("bytecode", pw)
    try:
        for c in (0, 1, P - 1, rnd):
            ctx.set_challenge(native.CHALLENGE_LOOKUP, c)
            for fam in rt.LOOKUP_FAMILIES:
                for j, label, w in _every(fam, 10 if fam != "pi" else 40):
                    for table in rt.TABLES[fam]:
                        u = dict(w, **{table: tp.permute(w[table], None, j)[0]})
                        _same(T.device(ctx, fam, u), rt.oracle(fam, u), f"challenge {c:#x} {fam} {label} {table}")
            _same(T.device(ctx, "bytecode", dict(pw, push=tp.permute(pw["push"], None, 6)[0])), pwant, f"push {c:#x}")
    finally:
        ctx.set_challenge(native.CHALLENGE_LOOKUP, DEFAULT_LOOKUP_CHALLENGE)
