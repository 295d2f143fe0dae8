"""Witness assignment on the device — host side of include/zkcheck.h "witness assignment" (csrc/assign.cu).

The reference builds circuit rows with Python object loops (assign_bytecode_circuit, bytecode_circuit.py:104-167;
op2row / assign_state_circuit and its mock MPT updates, state_circuit.py:827-933; CopyCircuit.copy,
evm_circuit/typing.py:1010-1147; ExpCircuit.add_event, evm_circuit/typing.py:880-994; public_data2witness,
pi_circuit.py:839-1073; Transaction.table_assignments, evm_circuit/typing.py:209-281;
Tables._convert_copy_circuit_to_table, evm_circuit/table.py:627-652).  The functions here hand the device the compact
data those loops start from — raw code bytes, 15 operation cells (or 13, the roots and the MPT table then built on the
device), copy events + the copied bytes, (base, exponent, identifier) per exponentiation, the raw public-input stream,
11 cells + the call data per transaction, the resident copy circuit — and leave the expanded witness or table resident
for zk_check."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from . import native, packing
from .evm_circuit.spec import RW, CopyDataTypeTag
from .util.arithmetic import FQ, Word
from .util.hash import keccak256


def is_code_bits(code: bytes) -> np.ndarray:
    """one bit per byte, LSB first: the byte is an opcode, not PUSH data (Bytecode.table_assignments, typing.py:390-427)"""
    n = len(code)
    flags = np.zeros(n, dtype=np.uint8)
    i = 0
    while i < n:
        flags[i] = 1
        b = code[i]
        i += 1 + (b - 0x5F if 0x60 <= b <= 0x7F else 0)
    return flags


def bytecode_src(codes: Sequence[bytes]) -> Dict[str, np.ndarray]:
    """arguments of Context.upload_bytecode_table_from_code / Context.assign_bytecode_circuit for these contracts"""
    flags = [is_code_bits(bytes(c)) for c in codes]
    offs = np.zeros(len(codes) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in codes])
    code = np.frombuffer(b"".join(bytes(c) for c in codes), dtype=np.uint8).copy()
    bits = np.packbits(np.concatenate(flags), bitorder="little") if len(code) else np.zeros(1, dtype=np.uint8)
    hashes = np.zeros((len(codes), 4), dtype=np.uint64)
    for k, c in enumerate(codes):
        h = Word(int.from_bytes(keccak256(bytes(c)), "big"))
        hashes[k] = [h.lo.n & 0xFFFFFFFFFFFFFFFF, h.lo.n >> 64, h.hi.n & 0xFFFFFFFFFFFFFFFF, h.hi.n >> 64]
    return {"code": code, "is_code_bits": bits, "code_offsets": offs, "hashes": hashes}


def assign_bytecode_circuit(ctx: native.Context, k: int, codes: Sequence[bytes], keccak_randomness, stream: int = 0) -> None:
    """the reference's assign_bytecode_circuit(k, [UnrolledBytecode(code, Bytecode(code).table_assignments()) ...], r)
    as one device call; the rows stay resident as ZK_CIRCUIT_BYTECODE"""
    ctx.set_challenge(native.CHALLENGE_KECCAK, packing.cell_int(keccak_randomness))
    ctx.assign_bytecode_circuit(k, stream=stream, **bytecode_src(codes))


STATE_OP_COLS = list(range(8)) + list(range(50, 57))  # the 15 cells of a 57-cell state row an operation brings


def state_ops_from_rows(rows57: np.ndarray) -> np.ndarray:
    """the operation cells of packed state rows: uint64[57][n][4] -> uint64[15][n][4]"""
    return np.ascontiguousarray(rows57[STATE_OP_COLS])


def assign_state_circuit(ctx: native.Context, ops, flags=None, stream: int = 0) -> None:
    """op2row for every operation on the device.  `ops`: a list of state_circuit.Operation (roots from the mock MPT
    updates like state_circuit.assign_state_circuit) or an operation-cell matrix uint64[15][n][4]"""
    if isinstance(ops, np.ndarray):
        m = ops
    else:
        from . import state_circuit as sc
        rows = sc.assign_state_circuit(list(ops))
        cols, flags = sc.pack_rows(rows)  # host op2row only to read the 15 operation cells and the roots
        m = state_ops_from_rows(cols)
    ctx.assign_state_circuit(packing.pack_matrix(m), flags=flags, stream=stream)


STATE_OP13_COLS = list(range(8)) + [50, 51, 52, 53, 56]  # the 13 cells of a state row an operation brings: no root


def state_op13_from_rows(rows57: np.ndarray) -> np.ndarray:
    """the operation cells of packed state rows without the root: uint64[57][n][4] -> uint64[13][n][4]"""
    return np.ascontiguousarray(rows57[STATE_OP13_COLS])


def state_op_cells(ops):
    """state_circuit.Operation objects -> (uint64[13][n][4], flags uint8[n]): the 13 cells and the WordOrValue type bits
    the operations bring, without op2row or the MPT walk"""
    c = packing.cell_int
    rows = [[int(op.rw_counter), 0 if op.rw == RW.Read else 1, int(op.tag), int(op.id), int(op.address), int(op.field_tag),
             int(op.storage_key) & ((1 << 128) - 1), int(op.storage_key) >> 128, c(op.value.lo), c(op.value.hi),
             c(op.initial_value.lo), c(op.initial_value.hi), c(op.lexicographic_ordering_selector)] for op in ops]
    flags = np.array([packing.word_flag(op.value) | (packing.word_flag(op.initial_value) << 1) for op in ops], dtype=np.uint8)
    return packing.matrix_from_ints(rows, 13), flags


# the two data rejections of zk_assign_state_circuit_mpt and the exception the mirror's _mock_mpt_updates raises there
STATE_MPT_ERRORS = (("the Account field tag is not Nonce, Balance, CodeHash or NonExisting", KeyError),
                    ("a Word value or initial value is >= 2^256", AssertionError))


def assign_state_circuit_mpt(ctx: native.Context, ops, flags=None, stream: int = 0) -> int:
    """state_circuit.assign_state_circuit(ops) and mpt_table_from_ops(ops) as one device call: the rows stay resident as
    ZK_CIRCUIT_STATE, the MPT updates (first-touch order) as ZK_TABLE_MPT; returns their number.  `ops`: a list of
    state_circuit.Operation, or the 13 operation cells uint64[13][n][4] (or a PackedMatrix of them) with `flags`.  An
    Account field tag without a proof type raises KeyError, a Word value >= 2^256 AssertionError, as the mirror does;
    the previous matrix and table stay in place"""
    if not isinstance(ops, (np.ndarray, packing.PackedMatrix)):
        ops, flags = state_op_cells(list(ops))
    try:
        return ctx.assign_state_circuit_mpt(ops, flags=flags, stream=stream)
    except native.NativeError as e:
        for msg, exc in STATE_MPT_ERRORS:
            if msg in str(e):
                raise exc(str(e)) from None
        raise


def copy_event(src_id, src_tag, dst_id, dst_tag, src_addr: int, src_addr_end: int, dst_addr: int, copy_length: int,
               rw_counter: int, log_id: int = 0) -> List[int]:
    """one row of the events array of zk_assign_copy_circuit — the arguments of CopyCircuit.copy plus the rw_counter the
    event starts at"""
    def cell(x):
        if isinstance(x, Word) and not hasattr(x, "is_word"):
            return x.lo.n, x.hi.n, 1
        if hasattr(x, "is_word"):
            return packing.cell_int(x.lo), packing.cell_int(x.hi), int(x.is_word)
        return packing.cell_int(x), 0, 0

    s_lo, s_hi, s_w = cell(src_id)
    d_lo, d_hi, d_w = cell(dst_id)
    M = 0xFFFFFFFFFFFFFFFF
    return [int(src_tag) | (s_w << 8), int(dst_tag) | (d_w << 8), int(src_addr), int(src_addr_end), int(dst_addr), int(copy_length),
            int(log_id), int(rw_counter), s_lo & M, s_lo >> 64, s_hi & M, s_hi >> 64, d_lo & M, d_lo >> 64, d_hi & M, d_hi >> 64]


def assign_copy_circuit(ctx: native.Context, r, events: Sequence[Sequence[int]], data: bytes,
                        is_code: Optional[Sequence[int]] = None, stream: int = 0) -> None:
    """CopyCircuit.copy of every event as one device call: `events` from copy_event(), `data` the copied bytes of all
    events back to back (0 where the source is out of bounds), `is_code` one flag per data byte (events that touch
    bytecode)"""
    ctx.set_challenge(native.CHALLENGE_KECCAK, packing.cell_int(r))
    ev = np.array(events, dtype=np.uint64).reshape(-1, 16)
    bits = None
    if is_code is not None:
        bits = np.packbits(np.asarray(is_code, dtype=np.uint8), bitorder="little") if len(data) else np.zeros(1, dtype=np.uint8)
    ctx.assign_copy_circuit(ev, np.frombuffer(bytes(data), dtype=np.uint8), bits, stream=stream)


def exp_events(triples) -> np.ndarray:
    """(base, exponent, identifier) per ExpCircuit.add_event -> the uint64[n][12] events of zk_assign_exp_circuit.  Base
    and exponent become Words as in the reference (an int outside [0, 2^256) raises there, and here); the identifier is
    reduced mod p like FQ()"""
    M = (1 << 64) - 1
    out = np.zeros((len(triples), 12), dtype=np.uint64)
    for k, (base, exponent, identifier) in enumerate(triples):
        ident = FQ(packing.cell_int(identifier)).n
        for j, v in enumerate((Word(int(base)).int_value(), Word(int(exponent)).int_value(), ident)):
            out[k, 4 * j:4 * j + 4] = [(v >> (64 * i)) & M for i in range(4)]
    return out


def assign_exp_circuit(ctx: native.Context, triples, max_exp_steps: Optional[int] = None, stream: int = 0) -> None:
    """ExpCircuit(max_exp_steps).add_event(...) for every (base, exponent, identifier), then fill_dummy_events() when
    max_exp_steps is given, as one device call: the rows stay resident as ZK_CIRCUIT_EXP, the exp table the EVM circuit's
    EXP lookups read (Tables(exp_circuit=...)) as ZK_TABLE_EXP"""
    from .exp_circuit import ExpCircuit

    n_min = 0 if max_exp_steps is None else int(max_exp_steps) * ExpCircuit.OFFSET_INCREMENT
    ctx.assign_exp_circuit(exp_events(list(triples)), n_rows_min=n_min, stream=stream)


def assign_pi_circuit(ctx: native.Context, public_data, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int,
                      stream: int = 0):
    """public_data2witness(public_data, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS) as one device call from the raw
    public-input stream, under the module's challenges (pi_circuit.keccak_rand, byte_pow_base, as check_matrices sets
    them): the rows stay resident as ZK_CIRCUIT_PI, the keccak and calldata gas tables as TABLE_KECCAK /
    TABLE_CALLDATA_GAS.  Returns (circuit_len, PublicInputs)"""
    from . import pi_circuit as pc

    ctx.set_challenge(native.CHALLENGE_PI_KECCAK, pc.keccak_rand.n)
    ctx.set_challenge(native.CHALLENGE_PI_BYTE_BASE, pc.byte_pow_base.n)
    raw = pc.raw_public_inputs(public_data, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS)
    digest = ctx.assign_pi_circuit(MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS, raw, stream=stream)
    b = public_data.block
    return len(raw), pc.PublicInputs(Word(digest), Word(b.hash), Word(b.state_root), Word(public_data.state_root_prev))


TX_SIGN_HASH = 1234  # the mirror's (and the reference's) mock sign hash, Transaction.table_fixed


def tx_records(txs):
    """evm_circuit.typing.Transaction objects -> the arguments of Context.assign_tx_table: (records uint64[n][11][4], call
    data uint8, offsets uint64[n + 1]).  A record is id, nonce, gas, gas_price, caller_address, callee_address,
    is_create, value, tx_invalid, access_list_gas_cost, tx_sign_hash.  Value fields are reduced mod p like FQ(); Word
    fields (gas_price, caller, callee, value) are checked like Word() (outside [0, 2^256) raises); a creation (callee
    None) has is_create 1 and callee 0; the access-list gas cost is computed here"""
    M = (1 << 64) - 1
    txs = list(txs)
    rec = np.zeros((len(txs), 11, 4), dtype=np.uint64)
    fq = lambda x: FQ(packing.cell_int(x)).n  # noqa: E731
    word = lambda x: Word(int(x)).int_value()  # noqa: E731
    for k, t in enumerate(txs):
        callee = t.callee_address
        cells = (fq(t.id), fq(t.nonce), fq(t.gas), word(t.gas_price), word(t.caller_address),
                 word(0 if callee is None else callee), int(callee is None), word(t.value), fq(t.invalid_tx),
                 fq(t.access_list_gas_cost()), TX_SIGN_HASH)
        for c, v in enumerate(cells):
            rec[k, c] = [(v >> (64 * i)) & M for i in range(4)]
    offs = np.zeros(len(txs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(t.call_data) for t in txs], dtype=np.uint64)
    data = np.frombuffer(b"".join(bytes(t.call_data) for t in txs), dtype=np.uint8)
    return rec, data, offs


def assign_tx_table(ctx: native.Context, txs, stream: int = 0) -> None:
    """Tables(tx_table=set(row for tx in txs for row in tx.table_assignments()), ...) as one device call: the tx table
    (with its Word type flags) stays resident as ZK_TABLE_TX"""
    rec, data, offs = tx_records(txs)
    ctx.assign_tx_table(rec, data, offs, stream=stream)


COPY_TABLE_ASSERTS = ("Not enough rows in copy circuit", "Invalid copy circuit")


def assign_copy_table(ctx: native.Context, stream: int = 0) -> None:
    """Tables(copy_circuit=...)'s copy table from the resident copy circuit (uploaded or assigned by
    assign_copy_circuit) as one device call, left resident as ZK_TABLE_COPY.  The reference's two asserts raise
    AssertionError with its message, and leave the previous table in place"""
    try:
        ctx.assign_copy_table(stream=stream)
    except native.NativeError as e:
        for msg in COPY_TABLE_ASSERTS:
            if f"zk_assign_copy_table: {msg} (rc=-1)" == str(e):
                raise AssertionError(msg) from None
        raise
