"""Every EVM gate program on long tiled traces (tests/tile_trace.py) against the oracle, with the persistent grids
forced to stride.

A golden vector holds 2 to 21 steps, so in a golden check no thread of a persistent grid takes a second step and a
warp almost never holds two failing lanes.  Here a context created with ZKCHECK_SM_COUNT=1 (DESIGN.md §3) sizes
every grid for one SM, and each tiled trace gives every bucket more than 2 x 2048 steps (2048 = the most resident
threads of one SM), so every thread walks at least two steps: the grid-stride loops, the per-thread code-hash caches
of the PUSH kernels, warps whose lanes fail at different constraints, the TX group on its auxiliary stream and in
line, and the copy circuit's deferred-warp list.  The real grid is covered by traces of 2^19 checked steps."""
import os
import time

import numpy as np
import pytest

import oracle_lib
import table_perturb as tp
import test_gpu_evm as ge
import tile_trace as tt
from zkevm_specs_b200 import native, packing, synth
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

pytestmark = pytest.mark.gpu
PASS = native.PASS
RESIDENT = 2048  # most resident threads of one SM
LAST_STEP = 4  # ZK_FLAG_EVM_LAST_STEP
ALL_TABLES = tuple(tt.EMPTY)
ENV = ("ZKCHECK_SM_COUNT", "ZKCHECK_TX_OVERLAP")
AXES = ("plain", "packed", "permuted", "inline", "shards")


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_tiled.py wall time {time.time() - t0:.1f} s")


def _contexts(sm_count, tx_overlap_flags):
    """one context per ZKCHECK_TX_OVERLAP value, all created with ZKCHECK_SM_COUNT = sm_count (None: unset); the
    environment is restored afterwards"""
    saved = {k: os.environ.get(k) for k in ENV}
    out = []
    try:
        for k in ENV:
            os.environ.pop(k, None)
        if sm_count is not None:
            os.environ["ZKCHECK_SM_COUNT"] = str(sm_count)
        for ov in tx_overlap_flags:
            if ov is not None:
                os.environ["ZKCHECK_TX_OVERLAP"] = ov
            out.append(native.Context(0))
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    for c in out:
        evm_main.upload_fixed_table(c)
    return out


@pytest.fixture(scope="module")
def strided():
    """(context, context with the TX group in line), both sized for one SM"""
    ctxs = _contexts(1, (None, "0"))
    yield tuple(ctxs)
    for c in ctxs:
        c.close()


@pytest.fixture(scope="module")
def fixed():
    return fixed_table_matrix()


def _upload(ctx, w):
    for name in ALL_TABLES:
        tid, _ = ge._TABLES[name]
        fl = w.get(tp.FLAGS_OF.get(name, "-"))
        if fl is not None and len(fl) and len(fl) == w[name].shape[1]:
            ctx.upload_table(tid, w[name], flags=fl)
        else:
            ctx.upload_table(tid, w[name])


def _device(ctx, w):
    _upload(ctx, w)
    ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
    return ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, w["flags"])


def _sharded(ctx, w, seed):
    """3 to 7 row shards at seeded cut points, each uploaded with one halo step and checked with its global row base;
    the LAST flag goes to the last shard only (it names the resident matrix's last checked step)"""
    n = w["steps"].shape[1] - 1
    rng = np.random.default_rng(seed)
    cuts = np.unique(rng.integers(1, n, 2 + seed % 5))
    bounds = [0, *cuts.tolist(), n]
    _upload(ctx, w)
    acc_ff, acc_fc = None, None
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ctx.upload_columns(native.CIRCUIT_EVM, np.ascontiguousarray(w["steps"][:, lo:hi + 1]))
        ff, fc = ctx.check(native.CIRCUIT_EVM, 0, hi - lo, lo, w["flags"] if hi == n else w["flags"] & ~LAST_STEP)
        acc_ff = ff if acc_ff is None else np.minimum(acc_ff, ff)
        acc_fc = fc if acc_fc is None else acc_fc + fc
    return acc_ff, acc_fc


def _same(got, want, what):
    ff, fc = got
    off, ofc = want
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc), \
        f"{what}: {ge._diff(ff, off)}; counts differ at {np.nonzero(fc != ofc)[0][:8].tolist()}"


def _check_axis(strided, t, axis, seed, fixed, want):
    ctx, ctx_inline = strided
    w = t.w
    if axis == "plain":
        got = _device(ctx, w)
    elif axis == "packed":
        ctx.packed_uploads = "min"
        try:
            got = _device(ctx, w)
        finally:
            ctx.packed_uploads = None
    elif axis == "permuted":  # the hash path: k_evm_push_hash, the POS = 0 gadgets, the other indexes
        v = tp.permute_witness(w, seed)
        want = tt.oracle_evm(v, fixed)
        if not v.get("order_dependent"):
            assert t.holds(*want)
        got = _device(ctx, v)
    elif axis == "inline":
        got = _device(ctx_inline, w)
    else:
        got = _sharded(ctx, w, seed)
    return got, want


def _multi(groups):
    return [g for g in groups if len(g[1]) >= 2]


@pytest.mark.parametrize("family", tt.EVM_FAMILIES)
def test_every_scenario_forced_to_stride(family, strided, fixed):
    """every group of >= 2 vectors, tiled until each execution state of its base vector fills more than 2 x 2048
    steps, on grids for one SM: arrays == oracle and the per-copy bound holds; the groups take turns at plain, packed
    storage, permuted tables, the TX group in line, and 3 to 7 row shards (a family with fewer groups than axes
    runs every axis on every group)"""
    groups = _multi(tt.evm_groups(family))
    for gi, (name, members) in enumerate(groups):
        t = tt.tile_evm(members, tt.copies_for(members[0][1], 2 * RESIDENT), gi, fixed)
        want = tt.oracle_evm(t.w, fixed)
        assert t.holds(*want), f"{family} {name}"
        for axis in AXES if len(groups) < len(AXES) else (AXES[gi % len(AXES)],):
            got, ref = _check_axis(strided, t, axis, gi, fixed, want)
            _same(got, ref, f"{family} {name} {axis}")
    _upload(strided[0], tt.full_witness({"steps": None}))


@pytest.mark.parametrize("family", tt.EVM_FAMILIES)
def test_table_mutated_vectors_tiled_alone(family, strided, fixed):
    """a vector whose tables differ from every other vector's (a table mutation) tiled alone, 128 copies, so whole
    warps fail the same way: arrays == oracle (every 6th such vector of a family, at least one)"""
    ctx = strided[0]
    singles = [g for g in tt.evm_groups(family) if len(g[1]) == 1]
    assert singles
    for gi, (name, members) in enumerate(singles):
        if gi % 6:
            continue
        t = tt.tile_evm(members, 32 if family == "evm" else 128, gi, fixed)
        want = tt.oracle_evm(t.w, fixed)
        assert t.holds(*want)
        _same(_device(ctx, t.w), want, f"{family} {name}")
    _upload(ctx, tt.full_witness({"steps": None}))


def _planted(n_groups, seed, n_bad):
    """synth.evm_trace with n_bad operand / gas / rw_counter corruptions at seeded steps"""
    w = synth.evm_trace(n_groups, seed=seed)
    S, R = w["steps"].copy(), w["rw"].copy()
    n = S.shape[1] - 1
    rng = np.random.default_rng(seed + 100)
    for t in range(n_bad):
        i = int(rng.integers(1, n))
        if t % 3 == 0:
            R[8 + t % 2, int(rng.integers(R.shape[1])), 0] ^= np.uint64(1 << int(rng.integers(64)))
        elif t % 3 == 1:
            S[9, i, 0] += np.uint64(1)
        else:
            S[1, i, 0] += np.uint64(1 + t % 3)
    return S, w["bytecode"], R


def _narrow_upload(ctx, S, B, R, from_code):
    """the bench's storage: steps and rw table packed to their type widths, the bytecode table either unrolled on the
    device from the raw code or packed to its type widths (the narrow instances of the hot kernels)"""
    if from_code:
        src = packing.bytecode_src_from_table(B)
        assert src is not None
        ctx.upload_bytecode_table_from_code(**src)
    else:
        ctx.upload_table_packed(native.TABLE_BYTECODE, packing.pack_matrix(B, min_widths=packing.TYPE_WIDTHS["bytecode_table"]))
    ctx.upload_table_packed(native.TABLE_RW, packing.pack_matrix(R, min_widths=packing.TYPE_WIDTHS["rw_table"]))
    ctx.upload_columns_packed(native.CIRCUIT_EVM, packing.pack_matrix(S, min_widths=packing.TYPE_WIDTHS["evm_steps"]))


def test_hot_kernels_on_the_real_grid_2e19_steps(fixed):
    """2^19 steps (PUSH32, PUSH32, ADD / SUB / MUL / DIV / MOD, POP) with 384 planted corruptions on the default grid:
    positional canonical tables (k_evm_push_pos<0>, k_evm_gadget<*, 1>), type-width packing with the bytecode table
    from the code and packed (the narrow instances), every table permuted (k_evm_push_hash, k_evm_gadget<*, 0>):
    each == oracle"""
    ctx = native.default_context()
    evm_main.upload_fixed_table(ctx)
    ge.clear_tables(ctx, ("copy", "keccak", "tx", "block", "wd", "exp", "aux"))
    S, B, R = _planted(1 << 17, 2, 384)
    n = S.shape[1] - 1
    want = oracle_lib.check_evm(S, B, R, fixed)
    assert want[1].sum() >= 300
    _same(ge._device_check(ctx, S, B, R), want, "positional")
    for from_code in (True, False):
        _narrow_upload(ctx, S, B, R, from_code)
        _same(ctx.check(native.CIRCUIT_EVM, 0, n, 0, 0), want, f"narrow from_code={from_code}")
    Bp, _ = tp.permute(B, None, 3, kind="bytecode")
    Rp, _ = tp.permute(R, None, 4, kind="rw")
    _same(ge._device_check(ctx, S, Bp, Rp), want, "permuted")


@pytest.mark.parametrize("family", ["evm5", "evm7", "evm2", "evm10", "evm11", "evm16"])
def test_group_kernel_on_the_real_grid_2e19_steps(family, fixed):
    """one scenario per k_evm_group instance (SIMPLE evm5, BYTES32 evm7, COPY evm2, WIDE evm10, TX evm11, ARITH evm16)
    tiled to 2^19 checked steps on the default grid: == oracle"""
    ctx = native.default_context()
    evm_main.upload_fixed_table(ctx)
    name, members = max(_multi(tt.evm_groups(family)), key=lambda g: len(g[1]))
    n_c = members[0][1]["steps"].shape[1]
    t = tt.tile_evm(members, (1 << 19) // n_c + 1, 5, fixed)
    want = tt.oracle_evm(t.w, fixed)
    assert t.holds(*want) and want[1].sum() > 0
    _same(_device(ctx, t.w), want, f"{family} {name}")
    _upload(ctx, tt.full_witness({"steps": None}))


def _two_contracts(n_groups, seed):
    """synth.evm_trace plus a second contract in the bytecode table: the first one's code with every byte changed
    and another code hash (a run of its own, so the table stays positional)"""
    w = synth.evm_trace(n_groups, seed=seed)
    B = w["bytecode"]
    B2 = B.copy()
    B2[0, :, 0] ^= np.uint64(0x5A5A5A5A)
    B2[5, 1:, 0] ^= np.uint64(1)
    return w["steps"].copy(), np.ascontiguousarray(np.concatenate([B, B2], axis=1)), w["rw"], B2[:, 0]


def _plant_code_hashes(S, other_hash, seed, frac=0.01):
    """about frac of the PUSH steps run under the other contract's code hash, as many under a hash no run has"""
    push = np.nonzero(S[0, :-1, 0] == S[0, 0, 0])[0]
    rng = np.random.default_rng(seed)
    k = max(8, int(len(push) * frac))
    rows = rng.choice(push[1:], size=2 * k, replace=False)
    for i in rows[:k]:
        S[5, i], S[6, i] = other_hash[0], other_hash[1]  # code hash lo / hi
    for i in rows[k:]:
        S[5, i, 0] ^= np.uint64(0xDEADBEEF)
    return S


@pytest.mark.parametrize("grid", ["one_sm", "default"])
def test_push_code_hash_caches(grid, strided, fixed):
    """PUSH steps that switch to another contract's code hash and to a hash no run has, among steps of the usual
    contract: the head cache of k_evm_push_pos (positional, canonical and type-width packed) and the per-lane code-hash
    cache of k_evm_push_hash (permuted tables) must not carry a verdict over.  Arrays == oracle, and every planted
    step is caught at its own row or the one before it (its predecessor's same-context check)"""
    ctx = strided[0] if grid == "one_sm" else native.default_context()
    evm_main.upload_fixed_table(ctx)
    ge.clear_tables(ctx, ("copy", "keccak", "tx", "block", "wd", "exp", "aux"))
    S, B, R, other = _two_contracts(1 << 14 if grid == "one_sm" else 1 << 16, 7)
    S = _plant_code_hashes(S, other, 8)
    n = S.shape[1] - 1
    assert tp.is_runs(B)
    want = oracle_lib.check_evm(S, B, R, fixed)
    assert want[1].sum() >= 16
    _same(ge._device_check(ctx, S, B, R), want, "positional")
    _narrow_upload(ctx, S, B, R, from_code=False)
    _same(ctx.check(native.CIRCUIT_EVM, 0, n, 0, 0), want, "type-width packed")
    Bp, _ = tp.permute(B, None, 9, kind="bytecode")
    Rp, _ = tp.permute(R, None, 10, kind="rw")
    _same(ge._device_check(ctx, S, Bp, Rp), want, "permuted")


def _copy_ctx_check(ctx, w, r, packed):
    ctx.packed_uploads = "min" if packed else None
    try:
        ctx.set_challenge(native.CHALLENGE_KECCAK, packing.cell_to_int(r))
        ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
        ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
        ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
        ctx.upload_columns(native.CIRCUIT_COPY, w["copy"], flags=w["copy_flags"])
        return ctx.check(native.CIRCUIT_COPY, 0, w["copy"].shape[1], 0, native.FLAG_WRAP)
    finally:
        ctx.packed_uploads = None


@pytest.mark.parametrize("packed", [False, True])
def test_copy_groups_tiled_on_one_sm(packed, strided):
    """copy.npz groups tiled to ~16k rows: the small kernel strides and the general kernel walks a long deferred-warp
    list on grids for one SM; arrays == oracle and the per-row bound holds"""
    ctx = strided[0]
    n = 0
    for gi, (name, members) in enumerate(_multi(tt.copy_groups())):
        t = tt.tile_copy(members, -(-16384 // members[0][1]["copy"].shape[1]), gi)
        want = oracle_lib.check_copy(t.w, t.r)
        assert t.holds(*want)
        _same(_copy_ctx_check(ctx, t.w, t.r, packed), want, f"copy {name}")
        n += 1
    assert n >= 3
    ctx.upload_table(native.TABLE_TX, np.zeros((5, 0, 4), dtype=np.uint64))


def test_copy_general_kernel_2e20_rows_with_non_small_cells():
    """cfg4 (2^20 rows) with a non-small cell in about 1 % of the warps (a value p - 1, an address 2^64 + k, an
    is_pad flag 2) and 40 small corruptions: k_check_copy_general walks thousands of deferred warps on the real grid;
    == oracle, packed == canonical"""
    ctx = native.default_context()
    w = synth.copy_events(512, 1024, seed=4)
    v = dict(w)
    v["copy"] = w["copy"].copy()
    n = v["copy"].shape[1]
    rng = np.random.default_rng(44)
    warps = rng.choice(n // 32, size=n // 32 // 100, replace=False)
    p1 = oracle_lib.limbs(tp.P - 1)
    for j, wi in enumerate(warps):
        i = 32 * int(wi) + int(rng.integers(32))
        if j % 3 == 0:
            v["copy"][9, i] = p1
        elif j % 3 == 1:
            v["copy"][6, i, 1] = 1
            v["copy"][6, i, 0] = np.uint64(j)
        else:
            v["copy"][12, i] = [2, 0, 0, 0]
    for t in range(40):
        v["copy"][9 if t % 2 else 13, int(rng.integers(n)), 0] ^= np.uint64(1)
    want = oracle_lib.check_copy(v, w["r"])
    assert want[1].sum() >= len(warps)
    for packed in (False, True):
        _same(_copy_ctx_check(ctx, v, w["r"], packed), want, f"packed={packed}")
    ctx.upload_table(native.TABLE_TX, np.zeros((5, 0, 4), dtype=np.uint64))


@pytest.mark.parametrize("grid", ["one_sm", "default"])
def test_block_trace_tx_group_overlapped_and_in_line(grid, strided, fixed):
    """synth.block_trace with 1024 transactions (about 9,000 steps in the TX group) and its corruption loop:
    the TX group on its auxiliary stream and in line give the same arrays, both == oracle"""
    ctxs = strided if grid == "one_sm" else _contexts(None, (None, "0"))
    try:
        w = synth.block_trace(1024, 4, 16, seed=9)
        n = w["n_steps"]
        rng = np.random.default_rng(12)
        for trial in range(9):
            w2 = dict(w)
            which = trial % 4
            if trial == 0:
                pass
            elif which == 0:
                m = w["steps"].copy(); m[int(rng.integers(1, 13)), int(rng.integers(0, n)), 0] += np.uint64(1); w2["steps"] = m
            elif which == 1:
                m = w["rw"].copy(); m[int(rng.choice([3, 4, 5, 8, 10])), int(rng.integers(0, m.shape[1])), 0] ^= np.uint64(1); w2["rw"] = m
            elif which == 2:
                m = w["tx"].copy(); m[3, int(rng.integers(0, m.shape[1])), 0] += np.uint64(1); w2["tx"] = m
            else:
                m = w["block"].copy(); m[2, int(rng.integers(0, m.shape[1])), 0] += np.uint64(1); w2["block"] = m
            want = oracle_lib.check_evm_x(w2, fixed, row_end=n)
            if trial == 0:
                assert (want[0] == PASS).all()
            for c in ctxs:
                ge._upload_block(c, w2)
                _same(c.check(native.CIRCUIT_EVM, 0, n, 0, w["flags"]), want, f"{grid} trial {trial}")
        for c in ctxs:
            ge.clear_tables(c, ("copy", "keccak", "tx", "block", "wd"))
    finally:
        if grid == "default":
            for c in ctxs:
                c.close()
