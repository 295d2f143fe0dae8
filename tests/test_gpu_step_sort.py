"""The EVM step sort (k_evm_sort: classify, grid-wide barrier, scatter in one cooperative launch) and the histogram it
hands to the host, against the oracle.

The host launches a gate-program group only when the histogram names steps of it, and sizes its grid from the
counts, so a histogram read from an earlier check would skip or mis-size a group.  The sort walks tiles of 256
threads x 4 steps (narrow storage) or x 2 steps (canonical storage), a thread's steps 256 apart, and every block
walks its tiles once per phase; the traces here put bucket ends, steps that fail in the prologue and steps whose
opcode peek picks another bucket at those edges.  Every step of a trace is also checked by its gate program with a
corrupted rw_counter on every second step, so a step that the scatter drops, writes twice or files in another
bucket changes the fail counts."""
import numpy as np
import pytest
import torch

import oracle_lib
import table_perturb as tp
import test_gpu_evm as ge
import test_gpu_tiled as tiled
from zkevm_specs_b200 import native, synth
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix
from zkevm_specs_b200.evm_circuit.spec import ExecutionState

pytestmark = pytest.mark.gpu
EVM = native.CIRCUIT_EVM
SIDE = ("copy", "keccak", "tx", "block", "wd", "exp", "aux")
# checked steps: ends of a thread's step range (256 apart), of a canonical tile (512), of a narrow tile (1024), and
# past one round of a one-SM grid
SIZES = [1, 2, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2047, 4097, 3 * 8192 + 1]
EDGES = (0, 255, 256, 511, 512, 1023, 1024, 1025, 2047, 2048, 4096)
BAD_STATE = 250  # not an execution state: the step fails in the prologue (ZK_BK_NONE)


@pytest.fixture(scope="module")
def fixed():
    return fixed_table_matrix()


@pytest.fixture(scope="module")
def grids():
    out = {"default": tiled._contexts(None, (None,))[0], "one_sm": tiled._contexts(1, (None,))[0]}
    for c in out.values():
        ge.clear_tables(c, SIDE)
    yield out
    for c in out.values():
        c.close()


def _edge_trace(n):
    """a cfg2 trace of n checked steps: BAD_STATE at the edges, MUL-state steps near the edges pointed at a DIV opcode
    (the peek files them as DIV, the gate program fails them) or past the code (the peek gives up), and rw_counter + 1
    on every second step"""
    g = (n + 4) // 4 + 1
    w = synth.evm_trace(g, seed=n)
    S = np.ascontiguousarray(w["steps"][:, : n + 1]).copy()
    mul = np.nonzero(S[0, :n, 0] == int(ExecutionState.MUL))[0]
    div_pc = 68 * 3 + 66  # group 3's op: synth.OPS[3] == "DIV"
    for j, e in enumerate(EDGES):
        if e >= n:
            break
        if len(mul):
            k = mul[np.argmin(np.abs(mul - e))]
            S[7, k, 0] = div_pc if j % 2 == 0 else 1 << 40
        S[0, e, 0] = BAD_STATE
    S[1, :n:2, 0] += np.uint64(1)
    return S, w["bytecode"], w["rw"]


def _upload_check(ctx, S, B, R, tables, rb, re, base):
    if tables == "narrow":
        tiled._narrow_upload(ctx, S, B, R, from_code=True)
    else:
        if tables == "permuted":  # the hash path: no opcode peek
            B, _ = tp.permute(B, None, 3, kind="bytecode")
            R, _ = tp.permute(R, None, 4, kind="rw")
        ctx.upload_table(native.TABLE_BYTECODE, B)
        ctx.upload_table(native.TABLE_RW, R)
        ctx.upload_columns(EVM, S)
    return ctx.check(EVM, rb, re, base, 0)


@pytest.mark.parametrize("n", SIZES)
def test_sort_edges(n, grids, fixed):
    """n checked steps with prologue failures and wrong opcode peeks at the ends of a thread's, a tile's and a grid
    round's step ranges: on a one-SM grid and the full grid, positional narrow (peek on, NARROW = 1), positional
    canonical (peek on, NARROW = 0) and permuted tables (peek off), arrays == oracle"""
    S, B, R = _edge_trace(n)
    want = oracle_lib.check_evm(S, B, R, fixed)
    assert want[1].sum() >= n // 2
    for grid, ctx in grids.items():
        for tables in ("narrow", "canonical", "permuted"):
            tiled._same(_upload_check(ctx, S, B, R, tables, 0, n, 0), want, f"{grid} {tables}")


@pytest.mark.parametrize("rb,re,base", [(1, 1026, 0), (255, 4352, 1000), (1023, 3 * 8192, 37)])
def test_sort_shards(rb, re, base, grids, fixed):
    """steps [rb, re) of a resident trace, reported from row `base`: the sort's local step indices start at 0 while
    its cells come from row rb on; arrays == oracle on every grid and storage form"""
    S, B, R = _edge_trace(3 * 8192 + 1)
    want = oracle_lib.check_evm(S, B, R, fixed, row_begin=rb, row_end=re, row_base=base)
    assert want[1].sum() > 0
    for grid, ctx in grids.items():
        for tables in ("narrow", "canonical", "permuted"):
            tiled._same(_upload_check(ctx, S, B, R, tables, rb, re, base), want, f"{grid} {tables}")


def _cfg2(seed):
    S, B, R = tiled._planted(4096, seed, 48)
    return {"kind": "cfg2", "S": S, "B": B, "R": R}


def _block(seed):
    """synth.block_trace with rw_counter + 1 on its first BeginTx / EndTx steps (TX group) and on a few others"""
    w = dict(synth.block_trace(256, 4, 16, seed=seed))
    n = w["n_steps"]
    S = w["steps"] = w["steps"].copy()
    tx = np.nonzero(np.isin(S[0, :n, 0], [int(ExecutionState.BeginTx), int(ExecutionState.EndTx)]))[0]
    rng = np.random.default_rng(seed)
    for i in [*tx[:6].tolist(), *rng.integers(1, n, 6).tolist()]:
        S[1, i, 0] += np.uint64(1)
    return {"kind": "block", "w": w}


def _want(run, fixed):
    if run["kind"] == "cfg2":
        return oracle_lib.check_evm(run["S"], run["B"], run["R"], fixed)
    w = run["w"]
    return oracle_lib.check_evm_x(w, fixed, row_end=w["n_steps"])


def _upload(ctx, run):
    if run["kind"] == "cfg2":
        ge.clear_tables(ctx, SIDE)
        tiled._narrow_upload(ctx, run["S"], run["B"], run["R"], from_code=True)
        return run["S"].shape[1] - 1, 0
    ge._upload_block(ctx, run["w"])
    return run["w"]["n_steps"], run["w"]["flags"]


def test_stale_histogram_one_context(fixed):
    """cfg2, then a block trace with failures in TX-group steps, then cfg2 again (another trace) on one context,
    without invalidating anything: each == oracle.  The group sets differ from check to check, so a histogram read
    from the previous check would skip the TX group or run a group sized for another trace"""
    runs = [_cfg2(1), _block(9), _cfg2(2), _block(10)]
    wants = [_want(r, fixed) for r in runs]
    assert all(w[1].sum() > 0 for w in wants)
    ctx = tiled._contexts(None, (None,))[0]
    try:
        for j, (run, want) in enumerate(zip(runs, wants)):
            n, flags = _upload(ctx, run)
            tiled._same(ctx.check(EVM, 0, n, 0, flags), want, f"check {j}: {run['kind']}")
    finally:
        ctx.close()


def test_stale_histogram_two_contexts_two_streams(fixed):
    """two contexts on two streams, each alternating cfg2 and block traces in opposite phase, both checks of a round
    enqueued before either result is read: every result == oracle"""
    runs = [_cfg2(3), _block(11)]
    wants = [_want(r, fixed) for r in runs]
    ctxs = tiled._contexts(None, (None, None))
    lanes = [(c, torch.cuda.Stream()) for c in ctxs]
    try:
        for rnd in range(4):
            picks = [(rnd + j) % 2 for j in range(2)]
            args = []
            for (c, s), p in zip(lanes, picks):
                args.append(_upload(c, runs[p]))
            torch.cuda.synchronize()
            for (c, s), (n, flags) in zip(lanes, args):
                c.check_async(EVM, 0, n, 0, flags, s.cuda_stream)
            for j, ((c, s), p) in enumerate(zip(lanes, picks)):
                tiled._same(c.fetch_result(EVM, s.cuda_stream), wants[p], f"round {rnd} context {j}: {runs[p]['kind']}")
    finally:
        for c, _ in lanes:
            c.close()
