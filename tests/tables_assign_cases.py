"""Cases and references for the tx-table and copy-table builders (zk_assign_tx_table, zk_assign_copy_table): edge-case
transactions, the host mirror's tx table (Transaction.table_assignments) as a set of (cells, Word flag), numpy
restatements of the two reference conversions over matrices (records -> tx table; copy circuit -> copy table,
Tables._convert_copy_circuit_to_table with its two asserts), and the transactions recovered from a golden tx table."""
import os

import numpy as np

from zkevm_specs_b200 import packing
from zkevm_specs_b200.evm_circuit.typing import AccessTuple, Transaction
from zkevm_specs_b200.util.arithmetic import FR_MODULUS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX_WORD = (1 << 256) - 1
P1 = FR_MODULUS - 1
WORD_TAGS = (3, 4, 5, 7)


def cell(c) -> int:
    return sum(int(x) << (64 * i) for i, x in enumerate(c))


def _bytes(n, seed, zero_share=0.3):
    rng = np.random.default_rng(seed)
    b = rng.integers(1, 256, n, dtype=np.uint8)
    b[rng.random(n) < zero_share] = 0
    return b.tobytes()


def small_txs(n_txs, max_len, seed):
    rng = np.random.default_rng(seed)
    return [Transaction(k + 1, nonce=int(rng.integers(0, 1 << 20)), gas=int(rng.integers(21000, 1 << 24)),
                        caller_address=int(rng.integers(1, 1 << 62)), callee_address=int(rng.integers(1, 1 << 62)),
                        value=int(rng.integers(0, 1 << 62)), call_data=_bytes(int(rng.integers(0, max_len + 1)), seed + k))
            for k in range(n_txs)]


def cases():
    """(label, [Transaction]) edge cases of the tx table"""
    yield "no_txs", []
    yield "empty_call_data", [Transaction(1), Transaction(2, callee_address=0xBEEF)]
    yield "all_zero_and_all_ff", [Transaction(1, call_data=bytes(100)), Transaction(2, callee_address=5, call_data=b"\xff" * 77)]
    yield "creation", [Transaction(1, callee_address=None, call_data=_bytes(300, 1)),
                       Transaction(2, callee_address=0xCAFE, access_list=[AccessTuple(0xAA, [1, 2]), AccessTuple(0xBB, [])])]
    yield "extremes", [Transaction(P1, nonce=P1, gas=P1, gas_price=MAX_WORD, caller_address=MAX_WORD, callee_address=MAX_WORD,
                                   value=MAX_WORD, call_data=b"\x00\xff\x01", invalid_tx=P1),
                       Transaction(FR_MODULUS + 3, gas_price=1 << 128, value=(1 << 128) - 1, callee_address=None)]
    yield "duplicated_ids", [Transaction(7, call_data=_bytes(40, 2)), Transaction(7, call_data=_bytes(41, 3)),
                             Transaction(7, call_data=_bytes(40, 2))]
    yield "many_small", small_txs(4096, 64, 4)


def big_tx():
    """one tx owning 2^20 call-data bytes"""
    return [Transaction(1, callee_address=0x1234, call_data=_bytes(1 << 20, 5))]


def mirror_set(txs):
    """the mirror's tx table as a set of (tx_id, tag, index, value lo, value hi, is_word)"""
    c = packing.cell_int
    return {(c(r.tx_id), c(r.field_tag), c(r.call_data_index_or_zero), c(r.value.lo), c(r.value.hi), int(r.value.is_word))
            for t in txs for r in t.table_assignments()}


def column_ints(col):
    """a column uint64[n][4] as a list of python ints"""
    l0, l1, l2, l3 = (col[:, i].tolist() for i in range(4))
    return [a | b << 64 | c << 128 | d << 192 for a, b, c, d in zip(l0, l1, l2, l3)]


def table_set(table, flags):
    """a downloaded tx table uint64[5][n][4] + its flags as the same set"""
    return set(zip(*(column_ints(table[c]) for c in range(5)), (np.asarray(flags) & 1).tolist()))


def tx_table_restated(rec, cd, offs):
    """Transaction.table_assignments over the records of assign.tx_records, in tx order: (table uint64[5][n][4], flags)"""
    rec = np.asarray(rec, dtype=np.uint64).reshape(-1, 11, 4)
    cd = np.asarray(cd, dtype=np.uint8)
    parts, flags = [], []
    for k in range(rec.shape[0]):
        lo, hi = int(offs[k]), int(offs[k + 1])
        data = cd[lo:hi]
        zeros = int((data == 0).sum())
        fixed = np.zeros((5, 12, 4), dtype=np.uint64)
        fixed[0] = rec[k, 0]
        fixed[1, :, 0] = np.arange(1, 13)
        for tag in range(1, 13):
            v = rec[k, tag if tag <= 7 else tag - 2]  # the record cell of the tag (CallDataLength / GasCost: unused)
            if tag == 8:
                fixed[3, tag - 1, 0] = hi - lo
            elif tag == 9:
                fixed[3, tag - 1, 0] = 16 * (hi - lo) - 12 * zeros
            elif tag in WORD_TAGS:
                fixed[3, tag - 1, :2], fixed[4, tag - 1, :2] = v[:2], v[2:]
            else:
                fixed[3, tag - 1] = v
        body = np.zeros((5, hi - lo, 4), dtype=np.uint64)
        body[0] = rec[k, 0]
        body[1, :, 0] = 13
        body[2, :, 0] = np.arange(hi - lo)
        body[3, :, 0] = data
        parts += [fixed, body]
        flags += [np.array([int(t in WORD_TAGS) for t in range(1, 13)], dtype=np.uint8), np.zeros(hi - lo, dtype=np.uint8)]
    if not parts:
        return np.zeros((5, 0, 4), dtype=np.uint64), np.zeros(0, dtype=np.uint8)
    return np.concatenate(parts, axis=1), np.concatenate(flags)


def _access_list(gas):
    """access tuples whose gas cost is `gas` (2,400 per address, 1,900 per storage key), or None"""
    for a in range(gas // 2400 + 1):
        rest = gas - 2400 * a
        if rest % 1900 == 0 and (a or not rest):
            s = rest // 1900
            return [AccessTuple(i, list(range(s)) if i == 0 else []) for i in range(a)]
    return None


def txs_from_table(table, flags):
    """the transactions whose table_assignments are exactly this tx table (with its flags), or None if there are none"""
    rows = {}
    n = table.shape[1]
    for r in range(n):
        tx_id, tag, idx, lo, hi = (cell(table[c, r]) for c in range(5))
        rows.setdefault(tx_id, {})[(tag, idx)] = (lo, hi, int(flags[r]) & 1)
    txs = []
    for tx_id, f in rows.items():
        if any((t, 0) not in f for t in range(1, 13)):
            return None
        v = {t: f[(t, 0)] for t in range(1, 13)}
        if any(v[t][2] != (t in WORD_TAGS) or (t not in WORD_TAGS and v[t][1]) for t in v):
            return None
        w = {t: v[t][0] | v[t][1] << 128 for t in v}
        n_cd = sum(1 for (t, _) in f if t == 13)
        data = []
        for i in range(n_cd):
            b = f.get((13, i))
            if b is None or b[0] > 255 or b[1] or b[2]:
                return None
            data.append(b[0])
        al = _access_list(w[11])
        if w[6] not in (0, 1) or (w[6] and w[5]) or w[12] != 1234 or al is None:
            return None
        txs.append(Transaction(tx_id, nonce=w[1], gas=w[2], gas_price=w[3], caller_address=w[4],
                               callee_address=None if w[6] else w[5], value=w[7], call_data=bytes(data),
                               invalid_tx=w[10], access_list=al))
    if len(set(table_set(table, flags))) != n or mirror_set(txs) != table_set(table, flags):
        return None
    return txs


def golden_tx_tables():
    """(file, scenario, tx table, flags) of every golden scenario of evm11 / evm17 / evm26 / evm28 that has a tx table"""
    for f in ("evm11", "evm17", "evm26", "evm28"):
        z = np.load(os.path.join(GOLDEN, f + ".npz"))
        for name in z["names"]:
            name = str(name)
            if f"{name}/tx" in z.files:
                yield f, name, z[f"{name}/tx"], z[f"{name}/tx_flags"]


COPY_SRC = (1, 3, 4, 5, 3, 4, 5, 6, 7, 6, 8, 10, 13, 14)
COPY_NEXT = (0, 0, 0, 0, 1, 1, 1, 0, 0, 1, 0, 0, 0, 0)


def copy_table_restated(circuit):
    """Tables._convert_copy_circuit_to_table over a copy circuit uint64[20][n][4]: the table uint64[14][rows][4] in
    circuit order, or the message of the first assert it raises"""
    c = np.asarray(circuit, dtype=np.uint64)
    n = c.shape[1]
    first = np.nonzero((c[1, :, 0] == 1) & ~c[1, :, 1:].any(axis=1))[0]
    for i in first:
        if i + 1 == n:
            return "Not enough rows in copy circuit"
        if c[0, i + 1].any():
            return "Invalid copy circuit"
    return np.ascontiguousarray(np.stack([c[s, first + d] for s, d in zip(COPY_SRC, COPY_NEXT)]))


def copy_table_set(table):
    return set(zip(*(column_ints(table[c]) for c in range(14))))
