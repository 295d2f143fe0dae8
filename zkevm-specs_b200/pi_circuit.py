"""Public-inputs circuit, host side — API of /root/reference/src/zkevm_specs/pi_circuit.py.

`Block`, `Transaction`, `Withdrawal`, `PublicData` hold the public data like the reference's dataclasses
(:461-631); `public_data2witness` lays the raw public-input bytes out exactly as the reference does (:839-1073: one
circuit row per byte, accumulated from the last byte backwards, the tx-table / calldata / withdrawal rows riding
on the first rows) and `verify_circuit` keeps the reference signature (:337-459): the copy constraints between
the tables and the raw bytes are compared on the host like the reference's loops (:364-444), every row's gates
and lookups (`check_row`, :150-321) run in one zk_check(ZK_CIRCUIT_PI) on the device.

The witness keeps its rows as the cell matrix of include/zkcheck.h (uint64[28][n][4]); `Witness.rows` gives
`Row` objects for a range of rows when a test wants to look at or override them (`Witness.set_row`)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import native, packing
from .evm_circuit.main import raise_first_failure
from .util.arithmetic import FQ, FR_MODULUS, Word, WordOrValue, bytes_to_fq
from .util.hash import keccak256

BLOCK_LEN = (8 + 256) * 2  # util/param.py:126 PUBLIC_INPUTS_BLOCK_LEN
TX_LEN = 10  # util/param.py:128 PUBLIC_INPUTS_TX_LEN
GAS_COST_TX_CALL_DATA_PER_NON_ZERO_BYTE = 16  # util/param.py:64
GAS_COST_TX_CALL_DATA_PER_ZERO_BYTE = 4  # util/param.py:66
TAG_CALLDATA_LENGTH, TAG_CALLDATA = 8, 13  # TxContextFieldTag (evm_circuit/table.py:147-167)
N_BYTES_ONE, N_BYTES_U64, N_BYTES_TX, N_BYTES_WITHDRAWAL = 1, 8, 176, 56  # pi_circuit.py:813-819
N_BYTES_BLOCK = 20 + 8 + 8 + 8 + 32 + 32 + 8 + 32 + 32 * 256  # :820-830
N_BYTES_EXTRA_VALUE = 32 * 3
byte_pow_base = FQ(255)  # module globals of the reference (:834-836)
evm_rand = FQ(255)
keccak_rand = FQ(255)
N_CELLS = 28

(P_Q_BYTES_LAST, P_Q_TX_TABLE, P_Q_TX_CALLDATA, P_Q_TX_CALLDATA_START, P_Q_KECCAK, P_Q_VALUE_START, P_TXID_INV,
 P_VALUE_LO_INV, P_TXID_DIFF_INV, P_CD_GAS, P_IS_FINAL, P_Q_WD, P_BYTES, P_KRLC, P_VALUE_LC, P_DIGEST_LO, P_DIGEST_HI,
 P_Q_BYTE_EN, P_TX_ID, P_TX_TAG, P_TX_INDEX, P_TX_VAL_LO, P_TX_VAL_HI, P_WD_ID, P_WD_VALIDATOR, P_WD_ADDR_LO,
 P_WD_ADDR_HI, P_WD_AMOUNT) = range(N_CELLS)


def _inv(v: int) -> int:
    v %= FR_MODULUS
    return pow(v, -1, FR_MODULUS) if v else 0


def _word(v: int) -> WordOrValue:
    return WordOrValue(Word(v))


def _value(v: int) -> WordOrValue:
    return WordOrValue(FQ(v))


def _lo_hi(v: int) -> Tuple[int, int]:
    return v & ((1 << 128) - 1), v >> 128


# ------------------------------------------------------------------------------------------ public data
@dataclass
class Block:
    """Block header (pi_circuit.py:461-482)"""
    hash: int
    parent_hash: int
    uncle_hash: int
    coinbase: int
    state_root: int
    tx_hash: int
    receipt_hash: int
    bloom: bytes
    prev_randao: int
    number: int
    gas_limit: int
    gas_used: int
    time: int
    extra: bytes
    mix_digest: int
    nonce: int
    base_fee: int
    withdrawals_root: int


@dataclass
class Transaction:
    """pi_circuit.py:485-604"""
    nonce: int
    gas_price: int
    gas: int
    from_addr: int
    to_addr: Optional[int]
    value: int
    data: bytes
    tx_sign_hash: int

    @classmethod
    def default(cls):
        return Transaction(0, 0, 0, 0, 0, 0, bytes([]), 0)

    def call_data_gas_cost(self) -> int:
        return sum(GAS_COST_TX_CALL_DATA_PER_ZERO_BYTE if b == 0 else GAS_COST_TX_CALL_DATA_PER_NON_ZERO_BYTE for b in self.data)

    def tx_table_value_column(self) -> List[WordOrValue]:
        """the ten tx-table values of this tx, no calldata (:499-522)"""
        return [_value(self.nonce), _value(self.gas), _word(self.gas_price), _value(self.from_addr), _value(self.to_addr or 0),
                _value(1 if self.to_addr is None else 0), _word(self.value), _value(len(self.data)),
                _value(self.call_data_gas_cost()), _word(self.tx_sign_hash)]

    def tx_raw_bytes(self, tx_id: int, call_data_gas_cost: Optional[int] = None) -> List[bytes]:
        """(tx_id, index = 0, value lo, [value hi]) big-endian per field (:524-583); `call_data_gas_cost` saves the
        per-byte sum when the caller has it"""
        out: List[bytes] = []

        def put(lo: bytes, hi: bytes = b""):
            out.append(int(tx_id).to_bytes(8, "big"))
            out.append((0).to_bytes(8, "big"))
            out.append(lo)
            if hi != b"":
                out.append(hi)

        def put_word(v: int):
            lo, hi = _lo_hi(v)
            put(lo.to_bytes(16, "big"), hi.to_bytes(16, "big"))

        put(int(self.nonce).to_bytes(8, "big"))
        put(int(self.gas).to_bytes(8, "big"))
        put_word(self.gas_price)
        put(int(self.from_addr).to_bytes(20, "big"))
        put(int(self.to_addr or 0).to_bytes(20, "big"))
        put((1 if self.to_addr is None else 0).to_bytes(8, "big"))
        put_word(self.value)
        put(len(self.data).to_bytes(8, "big"))
        gas = self.call_data_gas_cost() if call_data_gas_cost is None else call_data_gas_cost
        put(int(gas).to_bytes(8, "big"))
        put_word(self.tx_sign_hash)
        return out


@dataclass
class Withdrawal:
    """pi_circuit.py:606-627"""
    id: int
    validator_id: int
    address: int
    amount: int

    @classmethod
    def default(cls):
        return Withdrawal(0, 0, 0, 0)

    def withdrawal_raw_bytes(self, id: int) -> List[bytes]:
        lo, hi = _lo_hi(self.address)
        return [int(id).to_bytes(8, "big"), int(self.validator_id).to_bytes(8, "big"), lo.to_bytes(16, "big"),
                hi.to_bytes(16, "big"), int(self.amount).to_bytes(8, "big")]


@dataclass
class PublicData:
    """pi_circuit.py:630-810"""
    chain_id: int
    block: Block
    state_root_prev: int
    block_hashes: List[int]
    txs: List[Transaction]
    withdrawals: List[Withdrawal]

    def block_table_value_column(self) -> List[WordOrValue]:
        b = self.block
        assert len(self.block_hashes) == 256
        return [_value(0), _value(b.coinbase), _value(b.gas_limit), _value(b.number), _value(b.time), _word(b.prev_randao),
                _word(b.base_fee), _value(self.chain_id), _word(b.withdrawals_root)] + [_word(h) for h in self.block_hashes]

    def block_table_raw_byte_values(self) -> List[bytes]:
        b = self.block
        out = [(0).to_bytes(1, "big"), int(b.coinbase).to_bytes(20, "big"), int(b.gas_limit).to_bytes(8, "big"),
               int(b.number).to_bytes(8, "big"), int(b.time).to_bytes(8, "big")]

        def put_word(v: int):
            lo, hi = _lo_hi(v)
            out.append(lo.to_bytes(16, "big"))
            out.append(hi.to_bytes(16, "big"))

        put_word(b.prev_randao)
        put_word(b.base_fee)
        out.append(int(self.chain_id).to_bytes(8, "big"))
        put_word(b.withdrawals_root)
        assert len(self.block_hashes) == 256
        for h in self.block_hashes:
            put_word(h)
        return out

    def _txs_padded(self, MAX_TXS: int) -> List[Transaction]:
        assert len(self.txs) <= MAX_TXS
        return list(self.txs) + [Transaction.default() for _ in range(MAX_TXS - len(self.txs))]

    def _withdrawals_padded(self, MAX_WITHDRAWALS: int) -> List[Withdrawal]:
        assert len(self.withdrawals) <= MAX_WITHDRAWALS
        return list(self.withdrawals) + [Withdrawal.default() for _ in range(MAX_WITHDRAWALS - len(self.withdrawals))]

    def withdrawal_table_raw_bytes(self, MAX_WITHDRAWALS: int) -> List[bytes]:
        assert len(self.withdrawals) > 0
        out: List[bytes] = []
        for i, wd in enumerate(self._withdrawals_padded(MAX_WITHDRAWALS)):
            out.extend(wd.withdrawal_raw_bytes(i))
        return out

    def tx_table_raw_bytes(self, MAX_TXS: int) -> List[bytes]:
        assert len(self.txs) > 0
        out = [(0).to_bytes(8, "big"), (0).to_bytes(8, "big"), (0).to_bytes(1, "big")]  # the empty first row
        for i, tx in enumerate(self._txs_padded(MAX_TXS)):
            out.extend(tx.tx_raw_bytes(i + 1))
        return out

    def tx_table_calldata_raw_bytes(self, MAX_CALLDATA_BYTES: int) -> List[bytes]:
        data = b"".join(bytes(tx.data) for tx in self.txs)
        assert len(data) <= MAX_CALLDATA_BYTES
        data += bytes(MAX_CALLDATA_BYTES - len(data))
        return [bytes([b]) for b in data]


# ------------------------------------------------------------------------------------------ witness
@dataclass
class TxTableRow:
    tx_id: FQ
    tag: FQ
    index: FQ
    value: WordOrValue


@dataclass
class TxTable:
    table: List[TxTableRow] = field(default_factory=list)


@dataclass
class BlockTable:
    table: List[WordOrValue] = field(default_factory=list)


@dataclass
class WithdrawalTableRow:
    id: FQ
    validator_id: FQ
    address: Word
    amount: FQ


@dataclass
class WithdrawalTable:
    table: List[WithdrawalTableRow] = field(default_factory=list)


class KeccakTable:
    """rows (is_enabled, input_rlc, input_len, output); always holds the all-zero row (pi_circuit.py:78-102)"""

    def __init__(self):
        self.table = {(0, 0, 0, 0, 0)}

    def add(self, input: bytes, keccak_randomness: FQ):
        acc = 0
        r = packing.cell_int(keccak_randomness)
        for b in input:  # RLC(reversed(input), r) little-endian = Horner over the bytes in order
            acc = (acc * r + b) % FR_MODULUS
        out = Word(keccak256(input))
        self.table.add((1, acc, len(input), out.lo.n, out.hi.n))

    def matrix(self) -> np.ndarray:
        return packing.matrix_from_ints(sorted(self.table), 5)


@dataclass
class Row:
    """PublicInputs circuit row (pi_circuit.py:104-133)"""
    q_bytes_last: FQ
    q_tx_table: FQ
    q_tx_calldata: FQ
    q_tx_calldata_start: FQ
    q_rpi_keccak_lookup: FQ
    q_rpi_value_start: FQ
    tx_id_inv: FQ
    tx_value_lo_inv: FQ
    tx_id_diff_inv: FQ
    calldata_gas_cost: FQ
    is_final: FQ
    q_withdrawal_table: FQ
    rpi_bytes: FQ
    rpi_bytes_keccakrlc: FQ
    rpi_value_lc: FQ
    rpi_digest_word: Word
    q_rpi_byte_enable: FQ
    tx_table: TxTableRow
    withdrawal_table: WithdrawalTableRow

    def cells(self) -> List[int]:
        c = packing.cell_int
        t, w = self.tx_table, self.withdrawal_table
        return [c(self.q_bytes_last), c(self.q_tx_table), c(self.q_tx_calldata), c(self.q_tx_calldata_start),
                c(self.q_rpi_keccak_lookup), c(self.q_rpi_value_start), c(self.tx_id_inv), c(self.tx_value_lo_inv),
                c(self.tx_id_diff_inv), c(self.calldata_gas_cost), c(self.is_final), c(self.q_withdrawal_table),
                c(self.rpi_bytes), c(self.rpi_bytes_keccakrlc), c(self.rpi_value_lc), c(self.rpi_digest_word.lo),
                c(self.rpi_digest_word.hi), c(self.q_rpi_byte_enable), c(t.tx_id), c(t.tag), c(t.index), c(t.value.lo),
                c(t.value.hi), c(w.id), c(w.validator_id), c(w.address.lo), c(w.address.hi), c(w.amount)]


@dataclass
class PublicInputs:
    pi_keccak: Word
    block_hash: Word
    state_root: Word
    state_root_prev: Word


@dataclass
class Witness:
    cells: np.ndarray  # uint64[28][n][4]: the circuit rows in the layout of include/zkcheck.h ZK_CIRCUIT_PI
    public_inputs: PublicInputs
    calldata_gas_cost_table: set  # {(tx_id, is_final, gas_cost_acc)} as ints
    keccak_table: KeccakTable
    block_table: BlockTable
    tx_table: TxTable
    withdrawal_table: WithdrawalTable
    circuit_len: int
    copy_constrains: List[bytes]

    def row(self, i: int) -> Row:
        v = [packing.cell_to_int(self.cells[c, i]) for c in range(N_CELLS)]
        f = [FQ(x) for x in v]
        val = WordOrValue(FQ(v[P_TX_VAL_LO]))
        val.hi = FQ(v[P_TX_VAL_HI])
        return Row(*f[:15], Word((f[15], f[16]), check=False), f[17], TxTableRow(f[18], f[19], f[20], val),
                   WithdrawalTableRow(f[23], f[24], Word((f[25], f[26]), check=False), f[27]))

    @property
    def rows(self) -> List[Row]:
        return [self.row(i) for i in range(self.cells.shape[1])]

    def set_row(self, i: int, row: Row) -> None:
        for c, v in enumerate(row.cells()):
            self.cells[c, i] = packing.int_to_cell(v)

    def gas_matrix(self) -> np.ndarray:
        return packing.matrix_from_ints(sorted(self.calldata_gas_cost_table), 3)


def flatten_len(a: Sequence[bytes]) -> int:
    return sum(len(b) for b in a)


def public_data2witness(public_data: PublicData, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int) -> Witness:
    """pi_circuit.py:839-1073.  Raw public-input values: block table (value lo, [hi]) ..., block hash / state root /
    previous state root (lo, hi), tx table (id, index, value lo, [hi]) per field incl. the empty first row, one calldata
    byte per row, withdrawals (id, validator_id, address lo, hi, amount); one circuit row per BYTE, row i holding the
    i-th byte from the end."""
    pd = public_data
    values: List[bytes] = list(pd.block_table_raw_byte_values())
    for v in (pd.block.hash, pd.block.state_root, pd.state_root_prev):
        lo, hi = _lo_hi(v)
        values += [lo.to_bytes(16, "big"), hi.to_bytes(16, "big")]
    assert flatten_len(values) == N_BYTES_ONE + N_BYTES_BLOCK + N_BYTES_EXTRA_VALUE
    values += pd.tx_table_raw_bytes(MAX_TXS)
    circuit_len = (N_BYTES_ONE + N_BYTES_BLOCK + N_BYTES_EXTRA_VALUE + 2 * (N_BYTES_U64 * TX_LEN * MAX_TXS + N_BYTES_U64)
                   + N_BYTES_TX * MAX_TXS + N_BYTES_ONE)
    assert flatten_len(values) == circuit_len
    values += pd.tx_table_calldata_raw_bytes(MAX_CALLDATA_BYTES)
    circuit_len += MAX_CALLDATA_BYTES
    values += pd.withdrawal_table_raw_bytes(MAX_WITHDRAWALS)
    circuit_len += N_BYTES_WITHDRAWAL * MAX_WITHDRAWALS
    assert flatten_len(values) == circuit_len
    n = circuit_len

    # processing order of the reference: values from the last to the first, each value's bytes first to last; the
    # t-th processed byte sits on row n - 1 - t
    seq = b"".join(reversed(values))
    starts = np.zeros(n, dtype=np.uint64)  # q_rpi_value_start by processing step
    t = 0
    for v in reversed(values):
        starts[t] = 1
        t += len(v)
    rand, base = keccak_rand.n, byte_pow_base.n
    krlc, vlc = [0] * n, [0] * n
    acc = lc = 0
    for t, b in enumerate(seq):
        acc = (acc * rand + b) % FR_MODULUS if t else b
        lc = b if starts[t] else (lc * base + b) % FR_MODULUS
        krlc[t], vlc[t] = acc, lc
    cells = np.zeros((N_CELLS, n, 4), dtype=np.uint64)

    def put(col: int, by_row: Sequence[int]):
        cells[col] = packing.matrix_from_ints([[int(x)] for x in by_row], 1)[0]

    put(P_BYTES, seq[::-1])
    put(P_KRLC, krlc[::-1])
    put(P_VALUE_LC, vlc[::-1])
    cells[P_Q_VALUE_START, :, 0] = starts[::-1]
    cells[P_Q_BYTE_EN, :, 0] = 1
    cells[P_Q_BYTES_LAST, n - 1, 0] = 1
    cells[P_Q_KECCAK, 0, 0] = 1
    digest = Word(keccak256(seq))
    cells[P_DIGEST_LO, 0] = packing.int_to_cell(digest.lo.n)
    cells[P_DIGEST_HI, 0] = packing.int_to_cell(digest.hi.n)

    # tx table: the empty row, TX_LEN rows per tx slot, one row per calldata byte (:727-810)
    txs = pd._txs_padded(MAX_TXS)
    tx_id_col, index_col, value_col = [0], [0], [_value(0)]
    for i, tx in enumerate(txs):
        tx_id_col += [i + 1] * TX_LEN
        index_col += [0] * TX_LEN
        value_col += tx.tx_table_value_column()
    cd_tx, cd_idx, cd_val, cd_gas, cd_final = [], [], [], [], []
    for i, tx in enumerate(pd.txs):
        g = 0
        for k, b in enumerate(tx.data):
            g += GAS_COST_TX_CALL_DATA_PER_ZERO_BYTE if b == 0 else GAS_COST_TX_CALL_DATA_PER_NON_ZERO_BYTE
            cd_tx.append(i + 1)
            cd_idx.append(k)
            cd_val.append(b)
            cd_gas.append(g)
            cd_final.append(int(k == len(tx.data) - 1))
    assert len(cd_val) <= MAX_CALLDATA_BYTES
    pad = MAX_CALLDATA_BYTES - len(cd_val)
    for lst in (cd_tx, cd_idx, cd_val, cd_gas, cd_final):
        lst += [0] * pad
    tx_table_len = TX_LEN * MAX_TXS + 1
    tx_and_calldata_len = tx_table_len + MAX_CALLDATA_BYTES
    tx_id_col += cd_tx
    index_col += cd_idx
    value_col += [_value(b) for b in cd_val]
    gas_table = {(0, 0, 0)}
    tx_table = TxTable()
    rows_ints = {c: [0] * tx_and_calldata_len for c in (P_TX_ID, P_TX_TAG, P_TX_INDEX, P_TX_VAL_LO, P_TX_VAL_HI, P_TXID_INV,
                                                         P_VALUE_LO_INV, P_TXID_DIFF_INV, P_CD_GAS, P_IS_FINAL)}
    for i in range(tx_and_calldata_len):
        tx_id, index, value = tx_id_col[i], index_col[i], value_col[i]
        lo, hi = packing.cell_int(value.lo), packing.cell_int(value.hi)
        if i == 0:
            tag = 0
        elif i < tx_table_len:
            tag = i % TX_LEN or TX_LEN
        else:
            tag = TAG_CALLDATA
        rows_ints[P_TX_ID][i], rows_ints[P_TX_TAG][i], rows_ints[P_TX_INDEX][i] = tx_id, tag, index
        rows_ints[P_TX_VAL_LO][i], rows_ints[P_TX_VAL_HI][i] = lo, hi
        rows_ints[P_VALUE_LO_INV][i] = _inv(lo)
        if i < tx_table_len:
            rows_ints[P_TXID_INV][i] = _inv(tag - TAG_CALLDATA_LENGTH)
        else:
            k = i - tx_table_len
            nxt = tx_id_col[i + 1] if i < tx_and_calldata_len - 1 else 0
            rows_ints[P_TXID_INV][i] = _inv(tx_id)
            rows_ints[P_TXID_DIFF_INV][i] = _inv(nxt - tx_id)
            rows_ints[P_CD_GAS][i], rows_ints[P_IS_FINAL][i] = cd_gas[k], cd_final[k]
            gas_table.add((tx_id, cd_final[k], cd_gas[k]))
        tx_table.table.append(TxTableRow(FQ(tx_id), FQ(tag), FQ(index), value))
    for c, lst in rows_ints.items():
        cells[c, :tx_and_calldata_len] = packing.matrix_from_ints([[x] for x in lst], 1)[0]
    cells[P_Q_TX_TABLE, :tx_table_len, 0] = 1
    cells[P_Q_TX_CALLDATA, tx_table_len:tx_and_calldata_len, 0] = 1
    if MAX_CALLDATA_BYTES:
        cells[P_Q_TX_CALLDATA_START, tx_table_len, 0] = 1

    withdrawal_table = WithdrawalTable()
    for k, wd in enumerate(pd._withdrawals_padded(MAX_WITHDRAWALS)):
        i = tx_and_calldata_len + k
        lo, hi = _lo_hi(wd.address)
        for c, v in ((P_WD_ID, wd.id), (P_WD_VALIDATOR, wd.validator_id), (P_WD_ADDR_LO, lo), (P_WD_ADDR_HI, hi),
                     (P_WD_AMOUNT, wd.amount)):
            cells[c, i] = packing.int_to_cell(int(v) % FR_MODULUS)
        cells[P_Q_WD, i, 0] = 1
        withdrawal_table.table.append(WithdrawalTableRow(FQ(wd.id), FQ(wd.validator_id), Word(wd.address), FQ(wd.amount)))

    block_table = BlockTable(list(pd.block_table_value_column()[: BLOCK_LEN // 2 + 1])
                             + [_word(pd.block.hash), _word(pd.block.state_root), _word(pd.state_root_prev)])
    keccak_table = KeccakTable()
    keccak_table.add(seq, keccak_rand)
    public_inputs = PublicInputs(Word(digest.int_value()), Word(pd.block.hash), Word(pd.block.state_root),
                                 Word(pd.state_root_prev))
    return Witness(cells, public_inputs, gas_table, keccak_table, block_table, tx_table, withdrawal_table, circuit_len,
                   copy_constrains=values)


def raw_public_inputs(public_data: PublicData, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int) -> bytes:
    """the raw public-input stream b"".join(public_data2witness(...).copy_constrains) (pi_circuit.py:845-856), built
    without a Python object per calldata byte: what zk_assign_pi_circuit expands on the device"""
    pd = public_data
    values: List[bytes] = list(pd.block_table_raw_byte_values())
    for v in (pd.block.hash, pd.block.state_root, pd.state_root_prev):
        lo, hi = _lo_hi(v)
        values += [lo.to_bytes(16, "big"), hi.to_bytes(16, "big")]
    assert len(pd.txs) > 0
    values += [(0).to_bytes(8, "big"), (0).to_bytes(8, "big"), (0).to_bytes(1, "big")]  # the empty first tx row
    data = [np.frombuffer(bytes(tx.data), dtype=np.uint8) for tx in pd.txs]
    for i, tx in enumerate(pd._txs_padded(MAX_TXS)):
        d = data[i] if i < len(data) else data[0][:0]
        gas = GAS_COST_TX_CALL_DATA_PER_ZERO_BYTE * len(d) + (GAS_COST_TX_CALL_DATA_PER_NON_ZERO_BYTE
                                                               - GAS_COST_TX_CALL_DATA_PER_ZERO_BYTE) * int(np.count_nonzero(d))
        values += tx.tx_raw_bytes(i + 1, gas)
    calldata = np.concatenate(data).tobytes()
    assert len(calldata) <= MAX_CALLDATA_BYTES
    values += [calldata, bytes(MAX_CALLDATA_BYTES - len(calldata))]
    values += pd.withdrawal_table_raw_bytes(MAX_WITHDRAWALS)
    return b"".join(values)


# ------------------------------------------------------------------------------------------ verification
def check_matrices(ctx: native.Context, cells: np.ndarray, keccak: np.ndarray, gas: np.ndarray, circuit_len: int,
                   row_begin: int = 0, row_end: Optional[int] = None, row_base: int = 0, flags: int = native.FLAG_WRAP):
    """check_row over rows [row_begin, row_end) of an already packed witness: (first_fail, fail_count)"""
    ctx.set_challenge(native.CHALLENGE_PI_KECCAK, keccak_rand.n)
    ctx.set_challenge(native.CHALLENGE_PI_BYTE_BASE, byte_pow_base.n)
    ctx.set_challenge(native.PARAM_PI_CIRCUIT_LEN, int(circuit_len) % FR_MODULUS)
    ctx.upload_table(native.TABLE_KECCAK, keccak)
    ctx.upload_table(native.TABLE_CALLDATA_GAS, gas)
    ctx.upload_columns(native.CIRCUIT_PI, cells)
    return ctx.check(native.CIRCUIT_PI, row_begin, cells.shape[1] if row_end is None else row_end, row_base, flags)


def _copy_constraints(witness: Witness, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int) -> None:
    """the table cells equal the raw public-input bytes in vertical order (pi_circuit.py:364-444); consumes
    witness.copy_constrains like the reference"""
    cc = witness.copy_constrains
    pi = witness.public_inputs
    digest = Word((FQ(packing.cell_to_int(witness.cells[P_DIGEST_LO, 0])), FQ(packing.cell_to_int(witness.cells[P_DIGEST_HI, 0]))),
                  check=False)
    assert digest == pi.pi_keccak

    def lo_hi(value: WordOrValue):
        lo = cc.pop(0)[::-1]
        hi = cc.pop(0)[::-1] if value.is_word else bytes(0)
        return bytes_to_fq(lo), bytes_to_fq(hi)

    for i in range(BLOCK_LEN // 2 + 1):
        row = witness.block_table.table[i]
        lo, hi = lo_hi(row)
        assert row.lo.expr() == lo
        assert row.hi.expr() == hi
    for w in (pi.block_hash, pi.state_root, pi.state_root_prev):
        lo, hi = bytes_to_fq(cc.pop(0)[::-1]), bytes_to_fq(cc.pop(0)[::-1])
        assert w.lo.expr() == lo
        assert w.hi.expr() == hi
    tx_len = TX_LEN * MAX_TXS + 1
    for i in range(tx_len):
        r = witness.tx_table.table[i]
        assert r.tx_id == bytes_to_fq(cc.pop(0)[::-1])
        assert r.index == bytes_to_fq(cc.pop(0)[::-1])
        lo, hi = lo_hi(r.value)
        assert r.value.lo.expr() == lo
        assert r.value.hi.expr() == hi
    for i in range(MAX_CALLDATA_BYTES):
        v = witness.tx_table.table[tx_len + i].value
        lo, hi = lo_hi(v)
        assert v.lo.expr() == lo
        assert v.hi.expr() == hi
    for i in range(MAX_WITHDRAWALS):
        wd = witness.withdrawal_table.table[i]
        assert wd.id == bytes_to_fq(cc.pop(0)[::-1])
        assert wd.validator_id == bytes_to_fq(cc.pop(0)[::-1])
        lo, hi = bytes_to_fq(cc.pop(0)[::-1]), bytes_to_fq(cc.pop(0)[::-1])
        assert wd.address.lo.expr() == lo
        assert wd.address.hi.expr() == hi
        assert wd.amount == bytes_to_fq(cc.pop(0)[::-1])


def verify_public_data(public_data: PublicData, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int,
                       ctx: Optional[native.Context] = None) -> PublicInputs:
    """verify_circuit(public_data2witness(public_data, ...), ...) with the witness built on the device
    (assign.assign_pi_circuit) and checked where it stands: every row's gates and lookups in one zk_check, failures
    raised like verify_circuit.  The copy-constraint half of verify_circuit holds by construction here: the tables'
    cells and the raw bytes it compares are both read from the one raw public-input stream.  Returns the public inputs
    (the digest computed on the device)."""
    from . import assign

    ctx = ctx or native.default_context()
    n, public_inputs = assign.assign_pi_circuit(ctx, public_data, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS)
    ff, _ = ctx.check(native.CIRCUIT_PI, 0, n, 0, native.FLAG_WRAP)
    raise_first_failure(ff, native.CIRCUIT_PI, "pi row")
    return public_inputs


def verify_circuit(witness: Witness, MAX_TXS: int, MAX_CALLDATA_BYTES: int, MAX_WITHDRAWALS: int,
                   ctx: Optional[native.Context] = None) -> None:
    """pi_circuit.py:337-459: copy constraints (host), then check_row of every row (device)"""
    _copy_constraints(witness, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS)
    ctx = ctx or native.default_context()
    ff, _ = check_matrices(ctx, witness.cells, witness.keccak_table.matrix(), witness.gas_matrix(), witness.circuit_len)
    raise_first_failure(ff, native.CIRCUIT_PI, "pi row")
