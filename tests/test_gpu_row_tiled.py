"""The six row checkers (bytecode, state, exp, public inputs, tx, sig) against the oracle with their grids forced to
stride.

Golden witnesses are far smaller than one grid, so in a golden check no thread of k_check_bytecode / k_state_fold /
k_check_state / k_check_exp / k_check_pi / k_check_tx / k_check_sig reaches a second row, and no rotation reads a row
that another round of the grid-stride loop owns.  Here a context created with ZKCHECK_SM_COUNT=1 (DESIGN.md §3) sizes
every grid for one SM, and each witness has more than 2 x 2048 checked rows (2048 = the most resident threads of one
SM), so every thread walks at least two rows.  Corruptions sit at the ends of the possible rounds and warps, at rows
whose +1 / -1 neighbour another round owns, and in one warp whose lanes fail at different constraints.  Each witness
runs canonical and min-packed, whole with FLAG_WRAP, as row shards with halos, and once with row_begin > 0; the golden
families run once on the strided context, and valid witnesses cut to 1 .. 257 rows run with FLAG_WRAP."""
import time

import numpy as np
import pytest

import oracle_lib
import row_tables as rt
import test_gpu_tiled as tiled
import test_gpu_tx
from oracle_lib import same as _same
from row_tables import oracle
from zkevm_specs_b200 import exp_circuit as xc
from zkevm_specs_b200 import native, packing, synth
from zkevm_specs_b200 import pi_circuit as pc
from zkevm_specs_b200 import sig_circuit as sgc
from zkevm_specs_b200 import tx_circuit as tc
from zkevm_specs_b200.util import FQ

pytestmark = pytest.mark.gpu
PASS = native.PASS
RESIDENT = 2048  # most resident threads of one SM
WRAP = native.FLAG_WRAP
FAMILIES = rt.FAMILIES
CIRCUIT = {"bytecode": native.CIRCUIT_BYTECODE, "state": native.CIRCUIT_STATE, "exp": native.CIRCUIT_EXP,
           "pi": native.CIRCUIT_PI, "tx": native.CIRCUIT_TX, "sig": native.CIRCUIT_SIG}
ROT = {"bytecode": (0, 1), "state": (1, 1), "exp": (0, 1), "pi": (0, 1), "tx": (0, 0), "sig": (0, 0)}  # rows before / after
# columns whose corruption breaks a row (or its neighbour's check), cycled over the planted rows
COLS = {"bytecode": (6, 9, 5, 8, 10, 7, 4), "state": (50, 0, 4, 54, 2, 8),
        "exp": (16, 10, 6, 20, 2, 18, 12), "pi": (pc.P_KRLC, pc.P_IS_FINAL, pc.P_TX_INDEX, pc.P_VALUE_LC, pc.P_TXID_DIFF_INV),
        "tx": (0, 5, 7, 11, 1, 12), "sig": (1, 6, 0, 11, 2, 15)}


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_row_tiled.py wall time {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def strided():
    ctx, = tiled._contexts(1, (None,))
    yield ctx
    ctx.close()


# ---- witnesses: dict(m = the circuit's matrix, flags = its row flags or None, tables, r) ------------------------------
def _bytecode_witness():
    w = synth.bytecode_circuit_rows(13, n_contracts=5, seed=21)
    return {"m": w["rows"], "flags": None, "push": w["push"], "keccak": w["keccak"], "r": w["r"]}


def _state_witness():
    w = synth.state_rows(3 * RESIDENT + 517, seed=12, n_start=64)
    return {"m": w["rows"].copy(), "flags": w["flags"], "mpt": w["mpt"]}


def _exp_witness():
    c = xc.ExpCircuit()
    rng = np.random.default_rng(31)
    ident = 1
    while len(c.rows) < 2 * RESIDENT + 300:
        c.add_event(int.from_bytes(rng.bytes(32), "little"), int(rng.integers(2, 1 << 40)), ident)
        ident += 7
    c.max_exp_steps = (len(c.rows) + 6) // 7 + 3
    c.fill_dummy_events()
    return {"m": packing.matrix_from_ints([xc.exp_row(r) for r in c.rows], 21), "flags": None}


def _pi_witness():
    max_txs, max_cd, max_wd = 16, 2 * RESIDENT + 700, 8
    w = pc.public_data2witness(synth.pi_public_data(11, max_cd, max_wd, seed=13), max_txs, max_cd, max_wd)
    return {"m": w.cells.copy(), "flags": None, "keccak": w.keccak_table.matrix(), "gas": w.gas_matrix(),
            "clen": w.circuit_len}


def _tiled_rows(cells, flags, n):
    reps = n // cells.shape[1] + 1
    return np.ascontiguousarray(np.tile(cells, (1, reps, 1))[:, :n, :]), np.ascontiguousarray(np.tile(flags, reps)[:n])


def _tx_witness():
    r = FQ(0xA5A5A5A5A5A5A5A5A5A5)
    cells, flags, kec = tc.pack_witness(test_gpu_tx._witness(r, 5, 8), 8)
    m, f = _tiled_rows(cells, flags, 2 * RESIDENT + 333)
    return {"m": m, "flags": f, "keccak": kec, "r": oracle_lib.limbs(r.n)}


def _sig_witness():
    r = FQ(0x77777777777777777)
    rows, kt = test_gpu_tx._sig_rows(r)
    cells, flags, kec = sgc.pack_witness(sgc.Witness(rows, kt))
    m, f = _tiled_rows(cells, flags, 2 * RESIDENT + 211)
    return {"m": m, "flags": f, "keccak": kec, "r": oracle_lib.limbs(r.n)}


BUILD = {"bytecode": _bytecode_witness, "state": _state_witness, "exp": _exp_witness, "pi": _pi_witness,
         "tx": _tx_witness, "sig": _sig_witness}


def upload_tables(ctx, fam, w):
    if fam == "bytecode":
        ctx.set_challenge(native.CHALLENGE_KECCAK, packing.cell_to_int(w["r"]))
        ctx.upload_table(native.TABLE_PUSH, w["push"])
        ctx.upload_table(native.TABLE_KECCAK, w["keccak"])
    elif fam == "state":
        ctx.upload_table(native.TABLE_MPT, w["mpt"])
    elif fam == "pi":
        ctx.set_challenge(native.CHALLENGE_PI_KECCAK, pc.keccak_rand.n)
        ctx.set_challenge(native.CHALLENGE_PI_BYTE_BASE, pc.byte_pow_base.n)
        ctx.set_challenge(native.PARAM_PI_CIRCUIT_LEN, int(w["clen"]))
        ctx.upload_table(native.TABLE_KECCAK, w["keccak"])
        ctx.upload_table(native.TABLE_CALLDATA_GAS, w["gas"])
    elif fam in ("tx", "sig"):
        ctx.set_challenge(native.CHALLENGE_KECCAK, packing.cell_to_int(w["r"]))
        ctx.upload_table(native.TABLE_KECCAK, w["keccak"])


def device(ctx, fam, w, row_begin=0, row_end=None, row_base=0, flags=WRAP, m=None, f=None):
    """upload the tables and the matrix (`m`, `f`: a shard of it), then check [row_begin, row_end)"""
    upload_tables(ctx, fam, w)
    m = w["m"] if m is None else m
    f = w["flags"] if f is None else f
    ctx.upload_columns(CIRCUIT[fam], m, flags=f)
    if fam in ("tx", "sig"):
        flags = 0  # no rotation: tx / sig rows never wrap
    return ctx.check(CIRCUIT[fam], row_begin, m.shape[1] if row_end is None else row_end, row_base, flags)


def sharded(ctx, fam, w, cuts):
    """rows [lo, hi) of each shard uploaded with the halo rows its rotations read (taken cyclically, as the whole
    matrix wraps) and checked without FLAG_WRAP at row base lo: min / sum over the shards"""
    n = w["m"].shape[1]
    back, fwd = ROT[fam]
    bounds = [0, *cuts, n]
    acc_ff = acc_fc = None
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        idx = np.arange(lo - back, hi + fwd) % n
        m = np.ascontiguousarray(w["m"][:, idx])
        f = None if w["flags"] is None else np.ascontiguousarray(w["flags"][idx])
        ff, fc = device(ctx, fam, w, back, back + hi - lo, (lo - back) % (1 << 64), 0, m=m, f=f)
        acc_ff = ff if acc_ff is None else np.minimum(acc_ff, ff)
        acc_fc = fc if acc_fc is None else acc_fc + fc
    return acc_ff, acc_fc


def plant(fam, w, seed):
    """corruptions at the last and first rows of every possible round of one SM's grid (a round is a whole number of
    128- or 256-thread blocks, at most 2048 threads: rows t - 1 and t for every multiple t of 128 up to 4096), at both
    ends of the witness (the wrap-around rotations), and in six lanes of one warp of the second round at different
    columns: the planted rows"""
    m = w["m"]
    n = m.shape[1]
    rows = {0, 1, n - 1, n - 2}
    for t in range(128, 2 * RESIDENT + 1, 128):
        rows |= {t - 1, t}
    rows |= {RESIDENT + 96 + d for d in (0, 3, 7, 12, 20, 31)}
    rows = sorted(r for r in rows if r < n)
    cols = COLS[fam]
    rng = np.random.default_rng(seed)
    for j, i in enumerate(rows):
        m[cols[j % len(cols)], i, 0] ^= np.uint64(1 << int(rng.integers(0, 3)))
    return rows


CACHE = {}


def witness(fam):
    """(valid witness, corrupted copy, planted rows), built once per module"""
    if fam not in CACHE:
        w = BUILD[fam]()
        bad = dict(w, m=w["m"].copy())
        rows = plant(fam, bad, 5)
        CACHE[fam] = (w, bad, rows)
    return CACHE[fam]


@pytest.mark.parametrize("fam", FAMILIES)
def test_row_checker_forced_to_stride(fam, strided):
    """> 2 x 2048 checked rows with corruptions at round and warp boundaries on a grid for one SM: canonical and
    min-packed, whole with FLAG_WRAP, 3 shards with halos (cuts not multiples of 32), and rows [b, e) inside the matrix
    with b > 0: first_fail and fail_count == the oracle's"""
    w, bad, rows = witness(fam)
    n = w["m"].shape[1]
    assert n > 2 * RESIDENT
    good = oracle(fam, w)
    assert (good[0] == PASS).all(), f"{fam}: the generated witness is not valid"
    _same(device(strided, fam, w), good, f"{fam} valid")
    want = oracle(fam, bad)
    hit = {int(r) for r in want[0] if r != PASS}
    assert want[1].sum() >= len(rows) // 2 and len(hit) >= 3, f"{fam}: the planted rows break too little"
    _same(device(strided, fam, bad), want, f"{fam} whole")
    strided.packed_uploads = "min"
    try:
        _same(device(strided, fam, bad), want, f"{fam} min-packed")
    finally:
        strided.packed_uploads = None
    cuts = [RESIDENT - 5, RESIDENT + 1501]
    _same(sharded(strided, fam, bad, cuts), want, f"{fam} shards at {cuts}")
    b, e = 37, n - 45
    _same(device(strided, fam, bad, b, e), oracle(fam, bad, b, e), f"{fam} rows [{b}, {e})")


@pytest.mark.parametrize("fam", FAMILIES)
def test_golden_families_on_the_strided_context(fam, strided):
    """every golden vector of the six families on the context sized for one SM: == oracle"""
    n = 0
    for label, w in rt.vectors(fam):
        _same(device(strided, fam, w), oracle(fam, w), f"{fam} {label}")
        n += 1
    assert n > 300


@pytest.mark.parametrize("fam", FAMILIES)
def test_tiny_witnesses_wrap_onto_themselves(fam, strided):
    """the valid strided witness cut to 1, 2, 3, 31, 33 and 257 rows and checked with FLAG_WRAP: the +1 / -1
    rotations land on the row itself or its neighbour across the wrap; == oracle"""
    w, bad, rows = witness(fam)
    for n in (1, 2, 3, 31, 33, 257):
        for src in (w, bad):
            v = dict(src, m=np.ascontiguousarray(src["m"][:, :n]))
            if src["flags"] is not None:
                v["flags"] = np.ascontiguousarray(src["flags"][:n])
            _same(device(strided, fam, v), oracle(fam, v), f"{fam} {n} rows")
