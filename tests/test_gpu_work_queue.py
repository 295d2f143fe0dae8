"""The hot EVM kernels' work queue (k_evm_push_pos, k_evm_push_hash, k_evm_gadget<MUL|ADD|POP>) and their side-by-side
launch on four streams, against the oracle.

A warp of a hot kernel takes chunks of 32 consecutive sorted entries of its group (MUL: its MUL, DIV and MOD
sub-buckets in one chunk space) until the group's chunks run out.  The sorted order inside a bucket is not known to
the host, so the traces here corrupt the rw_counter of every checked step (or of every third one): each such step
then fails in its own hot kernel (the prologue does not read rw_counter), and a chunk that is skipped, run twice or
mapped to another bucket changes the fail counts.  Bucket sizes are exact: synth.evm_trace assigns its five ops in
turn, and the traces here replace that cycle."""
import numpy as np
import pytest
import torch

import oracle_lib
import table_perturb as tp
import test_gpu_evm as ge
import test_gpu_tiled as tiled
from zkevm_specs_b200 import native, synth
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

pytestmark = pytest.mark.gpu
EVM = native.CIRCUIT_EVM
MIXED = ("MUL", "DIV", "MOD", "ADD", "SUB")
# (op cycle, groups): a group is PUSH32, PUSH32, op, POP; ADD and SUB share a bucket, and with positional tables MUL,
# DIV and MOD are three sub-buckets of the MUL kernel
EDGES = [
    (("ADD",) * 5, 1),      # ADD 1, POP 1, PUSH 2; no MUL kernel
    (("ADD",) * 5, 31),     # one partial chunk; PUSH 62
    (("SUB",) * 5, 32),     # exactly one chunk; PUSH 64 = two
    (("ADD",) * 5, 33),     # one chunk and one step; PUSH 66
    (("DIV",) * 5, 33),     # a MUL kernel with DIV steps only: MUL 0, DIV 33, MOD 0
    (("MOD",) * 5, 1),      # MUL 0, DIV 0, MOD 1
    (MIXED, 4),             # MUL 1, DIV 1, MOD 0, ADD 1
    (MIXED, 165),           # MUL, DIV, MOD 33 each, ADD 66
    (synth.OPS, (1 << 17) + 1),  # POP 2^17 + 1, PUSH 2^18 + 2, ADD 52,430, MUL 26,215, DIV and MOD 26,214
]
TABLES = ("narrow", "canonical", "permuted")


@pytest.fixture(scope="module")
def fixed():
    return fixed_table_matrix()


@pytest.fixture(scope="module")
def grids():
    """{"default": a context on the device's grids, "one_sm": one whose grids are sized for one SM, so that each warp
    takes many chunks}"""
    out = {"default": tiled._contexts(None, (None,))[0], "one_sm": tiled._contexts(1, (None,))[0]}
    yield out
    for c in out.values():
        c.close()


def _trace(ops, g, seed=5):
    saved = synth.OPS
    synth.OPS = ops
    try:
        w = synth.evm_trace(g, seed=seed)
    finally:
        synth.OPS = saved
    return w["steps"].copy(), w["bytecode"], w["rw"]


def _corrupt(S, every):
    """rw_counter + 1 on every `every`-th checked step"""
    S = S.copy()
    S[1, :-1:every, 0] += np.uint64(1)
    return S


def _check(ctx, S, B, R, tables, seed):
    n = S.shape[1] - 1
    if tables == "narrow":
        tiled._narrow_upload(ctx, S, B, R, from_code=True)
        return ctx.check(EVM, 0, n, 0, 0)
    if tables == "permuted":
        B, _ = tp.permute(B, None, seed, kind="bytecode")
        R, _ = tp.permute(R, None, seed + 1, kind="rw")
    return ge._device_check(ctx, S, B, R)


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("ops,g", EDGES, ids=[f"{o[0] if len(set(o)) == 1 else 'mixed'}-{g}" for o, g in EDGES])
def test_bucket_edges(ops, g, every, grids, fixed):
    """hot buckets of 0, 1, 31, 32, 33 and about 2^17 + 1 steps, MUL sub-buckets of 0 and 1 step and a MUL kernel
    with DIV steps only; every (or every third) step corrupted: on both grids, with positional narrow, positional
    canonical and permuted tables (every instance of the four kernels), arrays == oracle"""
    S, B, R = _trace(ops, g)
    S = _corrupt(S, every)
    want = oracle_lib.check_evm(S, B, R, fixed)
    assert want[1].sum() >= (S.shape[1] - 1) // every
    for grid, ctx in grids.items():
        for tables in TABLES:
            tiled._same(_check(ctx, S, B, R, tables, g), want, f"{grid} {tables}")


@pytest.mark.parametrize("tables", ["narrow", "permuted"])
def test_queue_counters_reset_between_checks(tables, grids, fixed):
    """the same trace checked twice without invalidating the indexes, then a trace of another step count, then that
    one again, on grids for one SM (each warp takes many chunks after its first): every check == oracle.  A counter
    left over from the previous check would make the next one skip chunks"""
    ctx = grids["one_sm"]
    runs = []
    for g in (4096, 4096, 5003, 5003):
        S, B, R = _trace(synth.OPS, g, seed=g)
        runs.append((g, _corrupt(S, 1), B, R))
    wants = {g: oracle_lib.check_evm(S, B, R, fixed) for g, S, B, R in runs}
    for j, (g, S, B, R) in enumerate(runs):
        tiled._same(_check(ctx, S, B, R, tables, 7), wants[g], f"check {j}: {g} groups")


def _two_lanes(ctxs):
    return [(c, torch.cuda.Stream()) for c in ctxs]


def test_two_contexts_on_two_streams_full_workload(fixed):
    """the bench's 2^20-step workload with 384 planted corruptions on two contexts whose checks are enqueued on two
    streams before either result is read, four times, alternating: every result == oracle"""
    S, B, R = tiled._planted(1 << 18, 2, 384)
    n = S.shape[1] - 1
    want = oracle_lib.check_evm(S, B, R, fixed)
    assert want[1].sum() >= 300
    lanes = _two_lanes(tiled._contexts(None, (None, None)))
    try:
        for c, _ in lanes:
            tiled._narrow_upload(c, S, B, R, from_code=True)
        torch.cuda.synchronize()
        for rnd in range(4):
            order = lanes if rnd % 2 == 0 else lanes[::-1]
            for c, s in order:
                c.check_async(EVM, 0, n, 0, 0, s.cuda_stream)
            for c, s in order:
                tiled._same(c.fetch_result(EVM, s.cuda_stream), want, f"round {rnd}")
    finally:
        for c, _ in lanes:
            c.close()


def test_two_contexts_block_trace_tx_group_overlapped_and_in_line(fixed):
    """synth.block_trace (1024 transactions) with one corrupted step, on a context that forks the TX group to its own
    stream and one that runs it in line, their checks enqueued on two streams before either result is read: both ==
    oracle"""
    w = dict(synth.block_trace(1024, 4, 16, seed=9))
    n = w["n_steps"]
    w["steps"] = w["steps"].copy()
    w["steps"][1, n // 2, 0] += np.uint64(1)
    want = oracle_lib.check_evm_x(w, fixed, row_end=n)
    assert want[1].sum() > 0
    lanes = _two_lanes(tiled._contexts(None, (None, "0")))
    try:
        for c, _ in lanes:
            ge._upload_block(c, w)
        torch.cuda.synchronize()
        for rnd in range(2):
            for c, s in lanes:
                c.check_async(EVM, 0, n, 0, w["flags"], s.cuda_stream)
            for j, (c, s) in enumerate(lanes):
                tiled._same(c.fetch_result(EVM, s.cuda_stream), want, f"round {rnd} context {j}")
    finally:
        for c, _ in lanes:
            c.close()
