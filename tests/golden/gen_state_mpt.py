"""Generate tests/golden/state_mpt.npz by running the REFERENCE itself (zkevm-specs, pure Python).

    PYTHONPATH=oracle/pyshim:<zkevm-specs checkout>/src python tests/golden/gen_state_mpt.py

The fixture pins zk_assign_state_circuit_mpt: it holds operation lists with the 13 cells and type flags of each
operation, the rows the reference's assign_state_circuit gives, its _mock_mpt_updates in first-touch order and the
exception it raises.  It is not a verdict fixture, so it has a generator of its own beside gen_golden.py, whose cell
helpers it shares.  The tests only read the .npz file; they never need the reference.
"""
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import HERE, P, n_of, to_matrix  # noqa: E402


def state_mpt_cases():
    """The reference's assign_state_circuit and _mock_mpt_updates (state_circuit.py:861-933) on seeded operation
    lists: for each list its 13 operation cells (the 15 an operation brings without the root), the type flags, the
    reference's 57-cell rows, its MPT updates in first-touch order (the dict's order) and the exception class it
    raises.  The reference cannot build an Account op whose field tag has no proof type (its AccountOp takes an
    AccountFieldTag, and a plain int falls through to StorageMod): for that list the class recorded is the mirror's
    KeyError, and no rows."""
    import zkevm_specs.state_circuit as sc
    from zkevm_specs.evm_circuit import RW, AccountFieldTag, CallContextFieldTag
    from zkevm_specs.util import FQ, Word

    rng = random.Random(11)
    R_, W_ = RW.Read, RW.Write
    NONCE, BALANCE, CODEHASH, NONEX = (AccountFieldTag.Nonce, AccountFieldTag.Balance, AccountFieldTag.CodeHash,
                                       AccountFieldTag.NonExisting)

    def op_ints(o):
        return [int(o.rw_counter), 0 if o.rw == R_ else 1, int(o.tag), int(o.id), int(o.address), int(o.field_tag),
                int(o.storage_key) % (1 << 128), int(o.storage_key) >> 128, n_of(o.value.lo), n_of(o.value.hi),
                n_of(o.initial_value.lo), n_of(o.initial_value.hi), n_of(o.lexicographic_ordering_selector)]

    def row_ints(x):
        return ([n_of(x.rw_counter), n_of(x.is_write)] + [n_of(k) for k in x.keys[:4]] +
                [n_of(x.keys[4].lo), n_of(x.keys[4].hi)] + [n_of(l) for l in x.key2_limbs] +
                [n_of(b) for b in x.key45_bytes] + [n_of(x.value.lo), n_of(x.value.hi), n_of(x.initial_value.lo),
                                                    n_of(x.initial_value.hi), n_of(x.root.lo), n_of(x.root.hi),
                                                    n_of(x.lexicographic_ordering_selector)])

    def mpt_ints(x):
        return [n_of(x.address), n_of(x.proof_type), n_of(x.storage_key.lo), n_of(x.storage_key.hi), n_of(x.root.lo),
                n_of(x.root.hi), n_of(x.root_prev.lo), n_of(x.root_prev.hi), n_of(x.value.lo), n_of(x.value.hi),
                n_of(x.value_prev.lo), n_of(x.value_prev.hi)]

    def start(k):
        return [sc.StartOp(rw_counter=1, rw=R_, lexicographic_ordering_selector=0)] + [
            sc.StartOp(rw_counter=2 + j, rw=R_) for j in range(k - 1)]

    def all_tags():
        return start(2) + [
            sc.MemoryOp(rw_counter=1, rw=W_, call_id=1, mem_addr=0, value=FQ(42)),
            sc.StackOp(rw_counter=2, rw=W_, call_id=1, stack_ptr=1023, value=Word(533)),
            sc.StorageOp(rw_counter=3, rw=R_, tx_id=1, addr=0x12345678, key=0x1516, value=Word(789), committed_value=Word(789)),
            sc.StorageOp(rw_counter=4, rw=W_, tx_id=1, addr=0x12345678, key=(1 << 255) + 0x4959, value=Word(38491),
                         committed_value=Word(98765)),
            sc.CallContextOp(rw_counter=5, rw=R_, call_id=1, field_tag=CallContextFieldTag.IsStatic, value=FQ(0)),
            sc.AccountOp(rw_counter=6, rw=W_, addr=0x12345678, field_tag=NONCE, value=FQ(1), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=7, rw=R_, addr=0x12345678, field_tag=NONCE, value=FQ(1), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=8, rw=R_, addr=(1 << 160) - 1, field_tag=BALANCE, value=Word(3), committed_value=Word(0)),
            sc.TxRefundOp(rw_counter=9, rw=W_, tx_id=1, value=FQ(1)),
            sc.TxAccessListAccountOp(rw_counter=10, rw=W_, tx_id=1, addr=0x12345678, value=FQ(1)),
            sc.TxAccessListAccountStorageOp(rw_counter=11, rw=W_, tx_id=1, addr=0x12345678, key=0x1516, value=FQ(1)),
        ]

    def unsorted():
        ops = all_tags() + [sc.StorageOp(rw_counter=20 + j, rw=W_, tx_id=1 + j % 3, addr=0xAB, key=j % 4, value=Word(j),
                                         committed_value=Word(0)) for j in range(12)]
        rng.shuffle(ops)
        return ops

    def storage_multi_tx():
        ops = start(1)
        for tx in (1, 2, 3):
            ops.append(sc.StorageOp(rw_counter=10 * tx, rw=W_, tx_id=tx, addr=0xBEEF, key=7, value=Word(tx), committed_value=Word(0)))
            ops.append(sc.MemoryOp(rw_counter=10 * tx + 1, rw=W_, call_id=tx, mem_addr=5, value=FQ(tx)))
            ops.append(sc.StorageOp(rw_counter=10 * tx + 2, rw=R_, tx_id=tx, addr=0xBEEF, key=8 + tx, value=Word(1), committed_value=Word(1)))
        # a repeated touch whose Word value is >= 2^256: only first touches become MPT rows, so no assert
        ops.append(sc.StorageOp(rw_counter=40, rw=W_, tx_id=4, addr=0xBEEF, key=7,
                                value=Word((FQ(5), FQ(1 << 128)), check=False), committed_value=Word(0)))
        return ops

    def account_interleaved():
        ops = start(1)
        tags = [NONCE, BALANCE, CODEHASH, NONEX]
        for j in range(16):
            t = tags[(3 * j) % 4]
            v = FQ(j) if t == NONCE else Word(rng.randrange(1 << 256)) if t in (BALANCE, CODEHASH) else FQ(0)
            p = FQ(0) if t in (NONCE, NONEX) else Word(rng.randrange(1 << 256))
            ops.append(sc.AccountOp(rw_counter=2 + j, rw=W_ if j % 2 else R_, addr=0xC0FFEE, field_tag=t, value=v, committed_value=p))
        return ops

    def nonce_big():
        return start(1) + [
            sc.AccountOp(rw_counter=2, rw=W_, addr=0x1, field_tag=NONCE, value=FQ((1 << 200) + 5), committed_value=FQ(1 << 130)),
            sc.AccountOp(rw_counter=3, rw=W_, addr=0x1, field_tag=NONCE, value=FQ(P - 1), committed_value=FQ((1 << 200) + 5)),
            sc.AccountOp(rw_counter=4, rw=W_, addr=0x2, field_tag=NONCE, value=FQ(P - 1), committed_value=FQ(1 << 128))]

    def words():
        return start(1) + [
            sc.AccountOp(rw_counter=2, rw=W_, addr=0x7, field_tag=BALANCE, value=Word((1 << 255) + 7), committed_value=Word((1 << 256) - 1)),
            sc.AccountOp(rw_counter=3, rw=W_, addr=0x7, field_tag=CODEHASH, value=Word(rng.randrange(1 << 256)),
                         committed_value=Word(rng.randrange(1 << 256))),
            sc.StorageOp(rw_counter=4, rw=W_, tx_id=1, addr=0x7, key=(1 << 256) - 1, value=Word((1 << 256) - 1),
                         committed_value=Word(1 << 128))]

    def nonexisting():
        return start(1) + [
            sc.AccountOp(rw_counter=2, rw=R_, addr=0x99, field_tag=NONEX, value=FQ(0), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=3, rw=R_, addr=0x99, field_tag=NONEX, value=FQ(1), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=4, rw=R_, addr=0x98, field_tag=NONEX, value=FQ(0), committed_value=FQ(0))]

    def no_mpt():
        return start(2) + [sc.MemoryOp(rw_counter=1 + j, rw=W_, call_id=1, mem_addr=j, value=FQ(j)) for j in range(5)] + [
            sc.StackOp(rw_counter=10, rw=W_, call_id=1, stack_ptr=1023, value=Word(9))]

    def one_key():
        return [sc.StorageOp(rw_counter=1 + j, rw=W_ if j % 3 == 0 else R_, tx_id=1, addr=0x5, key=0x77, value=Word(j),
                             committed_value=Word(0)) for j in range(24)]

    def seeded(seed, n):
        r = random.Random(seed)
        ops = start(2)
        for j in range(n):
            k = r.randrange(6)
            a = r.choice([0x10, 0x11, (1 << 160) - 1])
            if k == 0:
                ops.append(sc.MemoryOp(rw_counter=j, rw=W_, call_id=1, mem_addr=r.randrange(8), value=FQ(r.randrange(256))))
            elif k == 1:
                ops.append(sc.StackOp(rw_counter=j, rw=W_, call_id=1, stack_ptr=r.randrange(1024), value=Word(r.randrange(1 << 256))))
            elif k in (2, 3):
                ops.append(sc.StorageOp(rw_counter=j, rw=r.choice([R_, W_]), tx_id=r.randrange(1, 4), addr=a,
                                        key=r.choice([0, 1, 2, (1 << 256) - 1]), value=Word(r.randrange(1 << 256)),
                                        committed_value=Word(r.randrange(1 << 256))))
            else:
                t = r.choice([NONCE, BALANCE, CODEHASH, NONEX])
                v = Word(r.randrange(1 << 256)) if t in (BALANCE, CODEHASH) else FQ(r.randrange(P))
                ops.append(sc.AccountOp(rw_counter=j, rw=r.choice([R_, W_]), addr=a, field_tag=t, value=v, committed_value=v))
        r.shuffle(ops)
        return ops

    def reject_word():  # a Word value >= 2^256 at op 3 decides, before the field-tag error at op 5
        return start(1) + [
            sc.StorageOp(rw_counter=2, rw=W_, tx_id=1, addr=0x1, key=1, value=Word(1), committed_value=Word(0)),
            sc.MemoryOp(rw_counter=3, rw=W_, call_id=1, mem_addr=0, value=FQ(1)),
            sc.StorageOp(rw_counter=4, rw=W_, tx_id=1, addr=0x1, key=2, value=Word(1),
                         committed_value=Word((FQ(0), FQ(1 << 128)), check=False)),
            sc.AccountOp(rw_counter=5, rw=W_, addr=0x1, field_tag=NONCE, value=FQ(1), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=6, rw=W_, addr=0x1, field_tag=9, value=FQ(1), committed_value=FQ(0))]

    def reject_field_tag():  # an Account field tag without a proof type at op 2 decides, before the Word error at op 4
        return start(1) + [
            sc.AccountOp(rw_counter=2, rw=W_, addr=0x1, field_tag=NONCE, value=FQ(1), committed_value=FQ(0)),
            sc.AccountOp(rw_counter=3, rw=W_, addr=0x1, field_tag=5, value=FQ(1), committed_value=FQ(0)),
            sc.MemoryOp(rw_counter=4, rw=W_, call_id=1, mem_addr=0, value=FQ(1)),
            sc.StorageOp(rw_counter=5, rw=W_, tx_id=1, addr=0x1, key=2, value=Word((FQ(1), FQ((1 << 128) + 1)), check=False),
                         committed_value=Word(0))]

    cases = [("all_tags", all_tags()), ("unsorted", unsorted()), ("storage_multi_tx", storage_multi_tx()),
             ("account_interleaved", account_interleaved()), ("nonce_big", nonce_big()), ("words", words()),
             ("nonexisting", nonexisting()), ("no_mpt", no_mpt()), ("only_start", start(5)), ("one_key", one_key()),
             ("seeded_a", seeded(101, 120)), ("seeded_b", seeded(202, 300)), ("reject_word", reject_word()),
             ("reject_field_tag", reject_field_tag())]
    out = {"names": np.array([nm for nm, _ in cases])}
    for name, ops in cases:
        exc, rows, mpt = "", [], []
        if name == "reject_field_tag":
            exc = "KeyError"  # the mirror's; the reference has no such op (see above)
        else:
            try:
                rows = sc.assign_state_circuit(ops)
                mpt = list(sc._mock_mpt_updates(ops).values())
            except Exception as e:  # noqa: BLE001
                exc = type(e).__name__
        out[f"{name}/ops"] = to_matrix([op_ints(o) for o in ops])
        out[f"{name}/flags"] = np.array([int(o.value.is_word) | (int(o.initial_value.is_word) << 1) for o in ops], dtype=np.uint8)
        out[f"{name}/rows"] = to_matrix([row_ints(x) for x in rows]) if rows else np.zeros((57, 0, 4), dtype=np.uint64)
        out[f"{name}/mpt"] = to_matrix([mpt_ints(x) for x in mpt]) if mpt else np.zeros((12, 0, 4), dtype=np.uint64)
        out[f"{name}/exc"] = np.array(exc)
        print(name, len(ops), "ops", len(rows), "rows", len(mpt), "mpt rows", exc or "accepted")
    np.savez_compressed(os.path.join(HERE, "state_mpt.npz"), **out)


if __name__ == "__main__":
    state_mpt_cases()
