"""Cases for the public-inputs builder (zk_assign_pi_circuit): seeded PublicData at the edges of the stream's layout, and
corruptions of a raw public-input stream.  Shared by tests/test_assign_pi_emu.py (CPU) and tests/test_gpu_assign_pi.py."""
import numpy as np

from zkevm_specs_b200 import packing, synth
from zkevm_specs_b200 import pi_circuit as pc

TX0, SLOT, WD = 8454, 336, 56  # the first tx slot's offset in the stream, a tx slot's bytes, a withdrawal's bytes
CDL = 256                       # the CallDataLength value inside a slot


def public_data(n_txs, max_cd, n_wd, seed, datas=None):
    pd = synth.pi_public_data(n_txs, max_cd, n_wd, seed=seed)
    if datas is not None:
        rng = np.random.default_rng(seed + 1)
        for tx, d in zip(pd.txs, datas):
            tx.data = bytes(rng.integers(0, 256, d, dtype=np.uint8)) if isinstance(d, int) else bytes(d)
    return pd


def cases():
    """(label, PublicData, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS).  Every withdrawal slot is used: the stream
    gives a padded slot i the id i, its table row the default id 0, and the reference's copy constraints reject that"""
    yield "empty_between", public_data(3, 64, 2, 11, [20, b"", 30]), 4, 64, 2
    yield "exact_fill", public_data(3, 96, 2, 12, [40, bytes(16), 40]), 3, 96, 2
    yield "single_tx", public_data(1, 50, 1, 13, [17]), 5, 50, 1
    yield "all_withdrawals", public_data(2, 32, 6, 14, [5, 9]), 2, 32, 6
    yield "leading_empties", public_data(3, 40, 3, 15, [b"", b"", 33]), 3, 40, 3
    yield "no_calldata", public_data(1, 0, 1, 16, [b""]), 2, 0, 1
    yield "zero_bytes_only", public_data(2, 70, 2, 17, [bytes(31), bytes(1)]), 2, 70, 2
    yield "wide", public_data(12, 1 << 15, 4, 18), 16, 1 << 15, 4


def bench_shape(max_cd=1 << 18):
    """bench.py --workload pi: 48 txs in 64 slots, 16 withdrawals"""
    return synth.pi_public_data(48, max_cd, 16, seed=7), 64, max_cd, 16


def table_set(m):
    return {tuple(packing.cell_to_int(m[c, r]) for c in range(m.shape[0])) for r in range(m.shape[1])}


def calldata_offset(max_txs):
    return TX0 + SLOT * max_txs


def corrupt_cdl(raw, max_txs, slot, delta):
    """the CallDataLength field of a tx slot off by `delta`"""
    b = bytearray(raw)
    o = TX0 + SLOT * slot + CDL
    b[o:o + 8] = (int.from_bytes(b[o:o + 8], "big") + delta).to_bytes(8, "big")
    return bytes(b)


def corrupt_calldata_byte(raw, max_txs, k):
    """calldata byte k turned from zero to non-zero or back: the CallDataGasCost field no longer matches"""
    b = bytearray(raw)
    o = calldata_offset(max_txs) + k
    b[o] = 0 if b[o] else 7
    return bytes(b)


def corrupt_withdrawal_amount(raw, max_txs, max_cd, k):
    """withdrawal k's amount set to 0"""
    b = bytearray(raw)
    o = calldata_offset(max_txs) + max_cd + WD * k + 48
    b[o:o + 8] = bytes(8)
    return bytes(b)


def corruptions():
    """(label, raw stream, MAX_TXS, MAX_CALLDATA_BYTES, MAX_WITHDRAWALS, withdrawal row or None) on the empty_between case"""
    _, pd, mt, mc, mw = next(cases())
    raw = pc.raw_public_inputs(pd, mt, mc, mw)
    n_tx = 10 * mt + 1
    yield "cdl_plus_one", corrupt_cdl(raw, mt, 0, 1), mt, mc, mw, None
    yield "cdl_minus_one", corrupt_cdl(raw, mt, 2, -1), mt, mc, mw, None
    yield "calldata_byte", corrupt_calldata_byte(raw, mt, 25), mt, mc, mw, None
    yield "zero_amount", corrupt_withdrawal_amount(raw, mt, mc, 1), mt, mc, mw, n_tx + mc + 1
