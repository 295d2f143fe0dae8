"""Row order and duplicate rows of the row circuits' lookup tables, on the CPU: the counterpart of
test_lookup_order.py for the bytecode (push, keccak), state (MPT), public-inputs (keccak, calldata gas), tx and sig
(keccak) checkers.

The reference's tables are sets and these lookups name every column, so reordering a table or adding rows identical to
its own changes no verdict, and no lookup can be ambiguous.  The golden vectors come in generator order with a regular
push table, so the hash index is hardly ever probed on them.  Here every table is permuted, given identical copies of
its rows and near-copies that differ in one column (each column in turn): the oracle must not notice the first two,
and the product's checkers run through the emu must equal the oracle, with the positional paths on and off and under
several lookup challenges."""
import numpy as np
import pytest

import emu_lib
import row_tables as rt
import table_perturb as tp

PASS = 0xFFFFFFFF
EVERY = {"bytecode": 2, "state": 2, "pi": 8, "tx": 2, "sig": 2}


@pytest.fixture(autouse=True)
def _positional_restored():
    yield
    emu_lib.set_positional(True)


@pytest.mark.parametrize("family", rt.LOOKUP_FAMILIES)
def test_oracle_and_emu_ignore_row_order_and_duplicates(family):
    """every 2nd (pi: 8th) golden vector, every table of the family, every transform: oracle(permuted) and
    oracle(identical copies) == oracle(original); emu == oracle on each transformed vector with the positional paths
    on and off; the AMBIG ids of lookups that name every column never fire; on a valid witness no transform fails a row"""
    never = [rt.constraint_ids(family)[n] for n in rt.NEVER.get(family, ())]
    n = valid = 0
    for label, v in rt.vectors(family, EVERY[family]):
        base = rt.oracle(family, v)
        ok = bool((base[0] == PASS).all())
        valid += ok
        for ti, table in enumerate(rt.TABLES[family]):
            for kind, u in rt.transformed(v, table, 7 * n + ti):
                want = rt.oracle(family, u)
                what = f"{family} {label} {table} {kind}"
                if kind in ("permuted", "identical"):
                    rt.same(want, base, f"oracle {what}")
                if ok:
                    assert (want[0] == PASS).all(), what
                assert not want[1][never].any(), what
                for positional in (True, False):
                    emu_lib.set_positional(positional)
                    rt.same(rt.emu(family, u), want, f"emu positional={positional} {what}")
        n += 1
    assert n >= 90 and valid >= 1, (n, valid)


def test_ambiguity_ids_are_found_by_name():
    ids = {f: rt.constraint_ids(f) for f in rt.FAMILIES}
    assert ids["bytecode"]["BC_PUSH_TABLE"] == 10
    for f, names in rt.NEVER.items():
        for name in names:
            assert name in ids[f]
    assert len(ids["state"]) == len(rt.oracle("state", next(rt.vectors("state"))[1])[0])


def test_push_table_paths_in_the_emu():
    """a push table dense from row 0 is served by position (emu: positional flag set), the same table starting at 1,
    permuted, or with a duplicate row is not; the verdict is the oracle's on each"""
    label, v = next(rt.vectors("bytecode"))
    push = v["push"]
    shifted = push.copy()
    shifted[0, :, 0] += np.uint64(1)
    cases = [("canonical", push, 1), ("starts at 1", shifted, 1), ("permuted", tp.permute(push, None, 3)[0], 0),
             ("identical", tp.with_identical_duplicates(push, None, k=1, seed=2)[0], 0)]
    for name, t, pos in cases:
        u = dict(v, push=t)
        emu_lib.set_positional(True)
        got = rt.emu("bytecode", u)
        assert emu_lib.positional_tables() == pos, name
        rt.same(got, rt.oracle("bytecode", u), name)


P = tp.P


@pytest.mark.parametrize("family", rt.LOOKUP_FAMILIES)
def test_lookup_challenge_never_changes_a_row_verdict(family):
    """ZK_CHALLENGE_LOOKUP seeds the hash index only: 0, 1, p - 1 and a random value give the oracle's arrays on
    every 10th golden vector with each table permuted or with identical copies"""
    rnd = int.from_bytes(np.random.default_rng(99).bytes(32), "little") % P
    emu_lib.set_positional(False)
    n = 0
    for label, v in rt.vectors(family, 10):
        for ti, table in enumerate(rt.TABLES[family]):
            for kind, u in list(rt.transformed(v, table, n + ti))[:2]:
                want = rt.oracle(family, u)
                for c in (0, 1, P - 1, rnd):
                    ch = np.array([(c >> (64 * q)) & 0xFFFFFFFFFFFFFFFF for q in range(4)], dtype=np.uint64)
                    rt.same(rt.emu(family, u, challenge=ch), want, f"{family} {label} {table} {kind} challenge {c:#x}")
        n += 1
    assert n >= 30
