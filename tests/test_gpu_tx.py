"""GPU parity of the tx circuit's Fr parts (ZK_CIRCUIT_TX, csrc/tx.cu) against the reference's
verdicts (tests/golden/tx.npz), the oracle's per-constraint arrays, and the host API
(zkevm_specs_b200.tx_circuit.verify_circuit keeps the reference signature, tx_circuit.py:253)."""
import numpy as np
import pytest

import golden_util
import oracle_lib
from zkevm_specs_b200 import native
from zkevm_specs_b200 import tx_circuit as tc
from zkevm_specs_b200.util import FQ, Word, keccak256

pytestmark = pytest.mark.gpu


def test_tx_golden_and_oracle_parity():
    ctx = native.default_context()
    n = 0
    for packed in (None, "min"):
        ctx.packed_uploads = packed
        try:
            for k, rows, flags, kec, r, exp_row, exp_exc in golden_util.tx_vectors():
                ff, fc = tc.check_matrices(ctx, rows, flags, kec, sum(int(r[j]) << (64 * j) for j in range(4)))
                off, ofc = oracle_lib.check_tx(rows, flags, kec, r)
                assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"[{k}] differs from oracle"
                hit = native.first_failure(ff, native.CIRCUIT_TX)
                got = (-1, "") if hit is None else (hit[0], oracle_lib.EXC_OF_CLASS[hit[2]])
                assert got == (exp_row, exp_exc), f"[{k}] cuda {got} reference {(exp_row, exp_exc)}"
                n += 1
        finally:
            ctx.packed_uploads = None
    assert n > 700


class _Ecdsa:
    """stands in for ECDSAVerifyChip (tx_circuit.py:107-158): eth_keys is third-party"""

    def __init__(self, pk: bytes, msg: bytes, ok=True):
        self.pub_key_x_bytes, self.pub_key_y_bytes = bytes(reversed(pk[:32])), bytes(reversed(pk[32:]))
        self.msg_hash_bytes, self.ok = bytes(reversed(msg)), ok

    def verify(self, assert_msg):
        assert self.ok, f"{assert_msg}: ecdsa_verify failed"


def _witness(r, n_txs, max_txs, bad=None):
    rng = np.random.default_rng(7)
    kt, rows, chips = tc.KeccakTable(), [], []
    for i in range(max_txs):
        if i < n_txs:
            pk, msg = bytes(rng.integers(0, 256, 64, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
            kt.add(pk, r)
            h = keccak256(pk)
            addr, mw = FQ(int.from_bytes(h[-20:], "big")), Word(int.from_bytes(msg, "big"))
            chip = tc.SignVerifyChip(h, addr, mw, _Ecdsa(pk, msg, ok=not (bad == "ecdsa" and i == 2)))
        else:  # padding tx: all zero (tx_circuit.py:273-275)
            addr, mw = FQ(0), Word(0)
            chip = tc.SignVerifyChip(bytes(32), addr, mw, _Ecdsa(bytes(64), bytes(32)))
        chips.append(chip)
        for tag in range(1, 13):
            v = addr if tag == 4 else mw if tag == 12 else FQ(0)
            if bad == "caller" and i == 1 and tag == 4:
                v = FQ(addr.n + 1)
            rows.append(tc.Row(FQ(i + 1), FQ(tag), FQ(0), v))
    return tc.Witness(rows, kt, chips)


def test_verify_circuit_host_api_like_reference_test_tx_circuit():
    r = FQ(0xA5A5A5A5A5A5A5A5A5A5)
    tc.verify_circuit(_witness(r, 5, 8), 8, 0, r)
    with pytest.raises(AssertionError, match="tx_index = 1"):
        tc.verify_circuit(_witness(r, 5, 8, bad="caller"), 8, 0, r)
    with pytest.raises(AssertionError, match="tx_index = 2.*ecdsa"):
        tc.verify_circuit(_witness(r, 5, 8, bad="ecdsa"), 8, 0, r)
    with pytest.raises(AssertionError, match="tx_index = 0.*keccak"):  # another randomness: the RLC no longer matches
        tc.verify_circuit(_witness(r, 5, 8), 8, 0, FQ(r.n + 1))


def test_sig_golden_and_oracle_parity():
    from zkevm_specs_b200 import sig_circuit as sc

    ctx = native.default_context()
    n = 0
    for packed in (None, "min"):
        ctx.packed_uploads = packed
        try:
            for k, rows, flags, kec, r, exp_row, exp_exc in golden_util.sig_vectors():
                ff, fc = sc.check_matrices(ctx, rows, flags, kec, sum(int(r[j]) << (64 * j) for j in range(4)))
                off, ofc = oracle_lib.check_sig(rows, flags, kec, r)
                assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"[{k}] differs from oracle"
                hit = native.first_failure(ff, native.CIRCUIT_SIG)
                got = (-1, "") if hit is None else (hit[0], oracle_lib.EXC_OF_CLASS[hit[2]])
                assert got == (exp_row, exp_exc), f"[{k}] cuda {got} reference {(exp_row, exp_exc)}"
                n += 1
        finally:
            ctx.packed_uploads = None
    assert n > 700


class _LE:
    def __init__(self, v):
        self.le_bytes = int(v).to_bytes(32, "little")


class _SigChip:
    """stands in for the ECDSA chip of the sig circuit (sig_circuit.py): its verdict is given"""

    def __init__(self, pk, msg, ok=True):
        self.pub_key_x_bytes, self.pub_key_y_bytes = bytes(reversed(pk[:32])), bytes(reversed(pk[32:]))
        self.msg_hash_bytes, self.sig_v, self.sig_r, self.sig_s, self.ok = msg, _LE(1), _LE(12345), _LE(67890), ok

    def verify(self):
        return self.ok


def _sig_rows(r):
    """six signatures, the one at row 4 invalid (and marked so): (rows, keccak table) of a valid sig witness"""
    from zkevm_specs_b200 import sig_circuit as sc

    rng = np.random.default_rng(9)
    kt, rows = tc.KeccakTable(), []
    for i in range(6):
        pk, msg = bytes(rng.integers(0, 256, 64, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        kt.add(pk, r)
        h = keccak256(pk)
        rows.append(sc.Row(h, FQ(int.from_bytes(h[-20:], "big")), Word(msg), _SigChip(pk, msg, ok=i != 4), is_valid=i != 4))
    return rows, kt


def test_sig_verify_circuit_host_api_and_scale():
    """host API like tests/test_sig_circuit.py; then 2^14 rows in one check (64 Fr products per row)"""
    from zkevm_specs_b200 import sig_circuit as sc

    r = FQ(0x77777777777777777)
    rows, kt = _sig_rows(r)
    sc.verify_circuit(sc.Witness(rows, kt), r)
    rows[2].recovered_addr = FQ(rows[2].recovered_addr.n ^ 1)
    with pytest.raises(AssertionError, match="row = 2"):
        sc.verify_circuit(sc.Witness(rows, kt), r)
    rows[2].recovered_addr = FQ(rows[2].recovered_addr.n ^ 1)
    rows[4].is_valid = True  # the chip says the signature is invalid
    with pytest.raises(AssertionError, match="row = 4.*is_valid"):
        sc.verify_circuit(sc.Witness(rows, kt), r)
    rows[4].is_valid = False
    # scale: tile the 6 valid rows to 2^14 and plant one corruption; GPU == oracle
    cells, flags, kec = sc.pack_witness(sc.Witness(rows, kt))
    reps = (1 << 14) // 6 + 1
    big = np.ascontiguousarray(np.tile(cells, (1, reps, 1))[:, : 1 << 14, :])
    bflags = np.tile(flags, reps)[: 1 << 14]
    big[8, 9999, 0] ^= np.uint64(1)
    ctx = native.default_context()
    ff, fc = sc.check_matrices(ctx, big, bflags, kec, r)
    rl = np.array([(r.n >> (64 * j)) & (2**64 - 1) for j in range(4)], dtype=np.uint64)
    off, ofc = oracle_lib.check_sig(big, bflags, kec, rl)
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc) and fc.sum() == 1
