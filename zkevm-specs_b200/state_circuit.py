"""State circuit, host side — API of /root/reference/src/zkevm_specs/state_circuit.py.

`Row`, the `*Op` constructors, `op2row`, `assign_state_circuit` and the mock MPT updates build
the witness like the reference (:63-152, :617-933); the checks of `check_state_row` (:492-613)
run on the device.  `verify_state_circuit(rows, tables)` packs all rows (57 cells + the
WordOrValue type flags) and makes ONE zk_check(ZK_CIRCUIT_STATE) with wrap-around rotations —
the loop the reference's test driver runs row by row (tests/test_state_circuit.py:17-38);
`check_state_row` keeps the per-row signature."""
from __future__ import annotations

from typing import Dict, Iterable, List, NamedTuple, Optional, Set, Tuple

import numpy as np

from . import native, packing
from .evm_circuit.main import raise_first_failure
from .evm_circuit.spec import RW, AccountFieldTag, MPTProofType, StateTag as Tag
from .evm_circuit.table import MPTTableRow
from .util.arithmetic import FQ, Word, WordOrValue


class Row(NamedTuple):
    rw_counter: FQ
    is_write: FQ
    keys: Tuple[FQ, FQ, FQ, FQ, Word]  # tag, id, address, field_tag, storage_key
    key2_limbs: Tuple[FQ, ...]  # address as 10 little-endian 16-bit limbs
    key45_bytes: Tuple[FQ, ...]  # storage key as 32 little-endian bytes
    value: WordOrValue
    initial_value: WordOrValue
    root: Word
    lexicographic_ordering_selector: FQ

    def tag(self): return self.keys[0]  # noqa: E704
    def id(self): return self.keys[1]  # noqa: E704
    def address(self): return self.keys[2]  # noqa: E704
    def field_tag(self): return self.keys[3]  # noqa: E704
    def storage_key(self): return self.keys[4]  # noqa: E704


class Operation(NamedTuple):
    rw_counter: int
    rw: RW
    tag: int
    id: int
    address: int
    field_tag: int
    storage_key: int
    value: WordOrValue
    initial_value: WordOrValue
    lexicographic_ordering_selector: FQ


def _op(rw_counter, rw, tag, id=0, address=0, field_tag=0, storage_key=0, value=FQ(0), initial=FQ(0), selector=1):
    return Operation(rw_counter, rw, int(tag), int(id), int(address), int(field_tag), int(storage_key),
                     WordOrValue(value), WordOrValue(initial), FQ(selector))


# constructors with the reference's names and argument order (state_circuit.py:634-824)
def StartOp(rw_counter, rw, lexicographic_ordering_selector=1):
    return _op(rw_counter, rw, Tag.Start, selector=lexicographic_ordering_selector)


def MemoryOp(rw_counter, rw, call_id, mem_addr, value):
    return _op(rw_counter, rw, Tag.Memory, call_id, mem_addr, value=FQ(value))


def StackOp(rw_counter, rw, call_id, stack_ptr, value: Word):
    return _op(rw_counter, rw, Tag.Stack, call_id, stack_ptr, value=value)


def StorageOp(rw_counter, rw, tx_id, addr, key, value: Word, committed_value: Word):
    return _op(rw_counter, rw, Tag.Storage, tx_id, addr, 0, key, value, committed_value)


def CallContextOp(rw_counter, rw, call_id, field_tag, value):
    return _op(rw_counter, rw, Tag.CallContext, call_id, 0, field_tag, value=value)


def AccountOp(rw_counter, rw, addr, field_tag, value, committed_value):
    return _op(rw_counter, rw, Tag.Account, 0, addr, field_tag, 0, value, committed_value)


def TxRefundOp(rw_counter, rw, tx_id, value):
    return _op(rw_counter, rw, Tag.TxRefund, tx_id, value=value)


def TxAccessListAccountOp(rw_counter, rw, tx_id, addr, value):
    return _op(rw_counter, rw, Tag.TxAccessListAccount, tx_id, addr, value=value)


def TxAccessListAccountStorageOp(rw_counter, rw, tx_id, addr, key, value):
    return _op(rw_counter, rw, Tag.TxAccessListAccountStorage, tx_id, addr, 0, key, value)


def TxLogOp(rw_counter, rw, tx_id, log_id, field_tag, index, value):
    return _op(rw_counter, rw, Tag.TxLog, tx_id, log_id, field_tag, index, value)


def TxReceiptOp(rw_counter, rw, tx_id, field_tag, value):
    return _op(rw_counter, rw, Tag.TxReceipt, tx_id, 0, field_tag, value=value)


def op2row(op: Operation, root: Word) -> Row:
    """operation -> circuit row: address limbs and key bytes decomposed (reference :827-857)"""
    addr_bytes = op.address.to_bytes(20, "little")
    limbs = tuple(FQ(int.from_bytes(addr_bytes[k:k + 2], "little")) for k in range(0, 20, 2))
    key_bytes = tuple(FQ(b) for b in op.storage_key.to_bytes(32, "little"))
    keys = (FQ(op.tag), FQ(op.id), FQ(op.address), FQ(op.field_tag), Word(op.storage_key))
    return Row(FQ(op.rw_counter), FQ(0 if op.rw == RW.Read else 1), keys, limbs, key_bytes, op.value,
               op.initial_value, root, FQ(op.lexicographic_ordering_selector))


def _mpt_key(op: Operation):
    if op.tag not in (int(Tag.Account), int(Tag.Storage)):
        return None
    return (op.address, op.field_tag, op.storage_key)


def _mock_mpt_updates(ops: Iterable[Operation]) -> Dict[tuple, MPTTableRow]:
    """fake MPT updates: the root starts at 3 and grows by 5 per first touch of an Account /
    Storage key (reference :903-933)"""
    out: Dict[tuple, MPTTableRow] = {}
    root = 3
    for op in ops:
        key = _mpt_key(op)
        if key is None or key in out:
            continue
        proof = int(MPTProofType.StorageMod) if op.tag == int(Tag.Storage) else int(
            {int(AccountFieldTag.Nonce): MPTProofType.NonceMod, int(AccountFieldTag.Balance): MPTProofType.BalanceMod,
             int(AccountFieldTag.CodeHash): MPTProofType.CodeHashMod,
             int(AccountFieldTag.NonExisting): MPTProofType.NonExistingAccountProof}[op.field_tag])
        out[key] = MPTTableRow(FQ(op.address), FQ(proof), Word(op.storage_key), Word(root + 5), Word(root),
                               Word(op.value.int_value()), Word(op.initial_value.int_value()))
        root += 5
    return out


def mpt_table_from_ops(ops: List[Operation]) -> Set[MPTTableRow]:
    return set(_mock_mpt_updates(ops).values())


def assign_state_circuit(ops: List[Operation]) -> List[Row]:
    """rows with the state root each operation sees (reference :861-889): an Account/Storage
    row carries the root BEFORE its own update applies... every other row the next one's."""
    updates = _mock_mpt_updates(ops)
    roots: List[Optional[Word]] = []
    for op in ops:
        key = _mpt_key(op)
        roots.append(None if key is None else updates[key].root_prev)
    final = Word(3 + 5 * len(updates))
    roots.append(final)
    nxt = final
    for k in range(len(roots) - 1, -1, -1):
        if roots[k] is None:
            roots[k] = nxt
        else:
            nxt = roots[k]
    return [op2row(op, roots[k + 1]) for k, op in enumerate(ops)]


class Tables:
    def __init__(self, mpt_table: Set[MPTTableRow]):
        self.mpt_table = set(mpt_table)


# ---- packing + device check ----------------------------------------------------------------
def state_row(r: Row) -> List[int]:
    c = packing.cell_int
    return ([c(r.rw_counter), c(r.is_write)] + [c(k) for k in r.keys[:4]] + [c(r.keys[4].lo), c(r.keys[4].hi)] +
            [c(x) for x in r.key2_limbs] + [c(x) for x in r.key45_bytes] +
            [c(r.value.lo), c(r.value.hi), c(r.initial_value.lo), c(r.initial_value.hi), c(r.root.lo), c(r.root.hi),
             c(r.lexicographic_ordering_selector)])


def mpt_row(r: MPTTableRow) -> List[int]:
    c = packing.cell_int
    return [c(r.address), c(r.proof_type), c(r.storage_key.lo), c(r.storage_key.hi), c(r.root.lo), c(r.root.hi),
            c(r.root_prev.lo), c(r.root_prev.hi), c(r.value.lo), c(r.value.hi), c(r.value_prev.lo), c(r.value_prev.hi)]


def pack_rows(rows: List[Row]):
    cols = packing.matrix_from_ints([state_row(r) for r in rows], 57)
    flags = np.array([packing.word_flag(r.value) | (packing.word_flag(r.initial_value) << 1) for r in rows], dtype=np.uint8)
    return cols, flags


def check_matrices(ctx: native.Context, cols, flags, mpt, row_begin=0, row_end=None, row_base=0, cflags=native.FLAG_WRAP):
    ctx.upload_table(native.TABLE_MPT, mpt)
    ctx.upload_columns(native.CIRCUIT_STATE, cols, flags=flags)
    return ctx.check(native.CIRCUIT_STATE, row_begin, cols.shape[1] if row_end is None else row_end, row_base, cflags)


def verify_state_circuit(rows: List[Row], tables: Tables, ctx: Optional[native.Context] = None) -> None:
    ctx = ctx or native.default_context()
    cols, flags = pack_rows(rows)
    mpt = packing.matrix_from_ints([mpt_row(r) for r in tables.mpt_table], 12)
    ff, _ = check_matrices(ctx, cols, flags, mpt)
    raise_first_failure(ff, native.CIRCUIT_STATE, "state row")


def verify_state_circuit_resident(ctx: native.Context) -> None:
    """verify_state_circuit over the resident rows and MPT table (assign.assign_state_circuit_mpt leaves both): ONE
    zk_check(ZK_CIRCUIT_STATE) with wrap-around rotations, raising like verify_state_circuit"""
    ff, _ = ctx.check(native.CIRCUIT_STATE, 0, ctx.resident_rows(native.CIRCUIT_STATE), 0, native.FLAG_WRAP)
    raise_first_failure(ff, native.CIRCUIT_STATE, "state row")


def check_state_row(row: Row, row_prev: Row, row_next: Row, tables: Tables, ctx: Optional[native.Context] = None) -> None:
    """Reference signature (state_circuit.py:492): checks `row` with its neighbours on the device."""
    ctx = ctx or native.default_context()
    cols, flags = pack_rows([row_prev, row, row_next])
    mpt = packing.matrix_from_ints([mpt_row(r) for r in tables.mpt_table], 12)
    ff, _ = check_matrices(ctx, cols, flags, mpt, 1, 2, 0, 0)
    raise_first_failure(ff, native.CIRCUIT_STATE, "state row")
