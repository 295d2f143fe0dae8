"""The index phase's positional flags are rebuilt from scratch by every build: a context that checks positional tables,
then reordered (non-positional) ones, then positional ones again, with every index invalidated in between, must equal
the oracle at every check.  So must two contexts on two streams that alternate between the two kinds, as the
double-buffered end-to-end pipeline of bench.py does.  A flag or per-block verify result left over from an earlier
build would send lookups down the wrong path and change the arrays."""
import numpy as np
import pytest
import torch

import oracle_lib
import table_perturb as tp
import test_gpu_evm as ge
from zkevm_specs_b200 import native, packing, synth
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

pytestmark = pytest.mark.gpu


def _witness(n_groups=1 << 12, seed=2):
    """cfg2 trace with 48 planted corruptions of steps and rw values"""
    w = synth.evm_trace(n_groups, seed=seed)
    S, R = w["steps"].copy(), w["rw"].copy()
    n = S.shape[1] - 1
    rng = np.random.default_rng(303 + seed)
    for t in range(48):
        i = int(rng.integers(1, n))
        if t % 3 == 0:
            R[8 + int(rng.integers(2)), int(rng.integers(R.shape[1])), int(rng.integers(2))] ^= np.uint64(1 << int(rng.integers(64)))
        elif t % 3 == 1:
            S[9, i, 0] += np.uint64(1)
        else:
            S[1, i, 0] += np.uint64(1 + int(rng.integers(3)))
    return w, S, R


def _arrangements(w, R):
    """(label, upload function, bytecode matrix, rw matrix): the bench's data path in generator order, then
    both tables reordered so that neither is positional"""
    B = w["bytecode"]
    Bp, _ = tp.permute(B, None, 41, kind="bytecode")
    Rp, _ = tp.permute(R, None, 42, kind="rw")
    assert not tp.is_regular(Bp, "bytecode") and not tp.is_regular(Rp, "rw")

    def positional(ctx, stream=0):
        ctx.upload_bytecode_table_from_code(**w["bytecode_src"], stream=stream)
        ctx.upload_table_packed(native.TABLE_RW, packing.pack_matrix(R), stream=stream)

    def permuted(ctx, stream=0):
        ctx.upload_table_packed(native.TABLE_BYTECODE, packing.pack_matrix(Bp), stream=stream)
        ctx.upload_table_packed(native.TABLE_RW, packing.pack_matrix(Rp), stream=stream)

    return [("positional", positional, B, R), ("permuted", permuted, Bp, Rp)]


def _setup(ctx, S, stream=0):
    evm_main.upload_fixed_table(ctx)
    ge.clear_tables(ctx, ("copy", "keccak"))
    ctx.upload_columns_packed(native.CIRCUIT_EVM, packing.pack_matrix(S), stream=stream)


def test_positional_then_permuted_then_positional_one_context():
    w, S, R = _witness()
    n = S.shape[1] - 1
    fixed = fixed_table_matrix()
    arr = _arrangements(w, R)
    expect = {label: oracle_lib.check_evm(S, B, RR, fixed) for label, _, B, RR in arr}
    assert np.array_equal(expect["positional"][0], expect["permuted"][0])
    ctx = native.Context(0)
    try:
        _setup(ctx, S)
        for k, (label, upload, _, _) in enumerate(arr + arr + arr[:1]):
            upload(ctx)
            ctx.invalidate_indexes()
            for rep in range(2):  # the second check rebuilds over unchanged tables, as every bench pass does
                ff, fc = ctx.check(native.CIRCUIT_EVM, 0, n, 0, 0)
                off, ofc = expect[label]
                assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (k, label, rep, ge._diff(ff, off))
                ctx.invalidate_indexes()
        assert fc.sum() >= 48
    finally:
        ctx.close()


def test_two_contexts_on_two_streams_alternate_kinds():
    w, S, R = _witness(seed=3)
    n = S.shape[1] - 1
    fixed = fixed_table_matrix()
    arr = _arrangements(w, R)
    expect = {label: oracle_lib.check_evm(S, B, RR, fixed) for label, _, B, RR in arr}
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ctxs = [native.Context(0), native.Context(0)]
    try:
        for c, s in zip(ctxs, streams):
            _setup(c, S, s.cuda_stream)
        for rnd in range(4):
            # round r: context i holds arrangement (r + i) % 2; both checks are in flight before either result is read
            labels = []
            for i, (c, s) in enumerate(zip(ctxs, streams)):
                label, upload, _, _ = arr[(rnd + i) % 2]
                upload(c, s.cuda_stream)
                c.invalidate_indexes()
                c.check_async(native.CIRCUIT_EVM, 0, n, 0, 0, s.cuda_stream)
                labels.append(label)
            for i, (c, s) in enumerate(zip(ctxs, streams)):
                ff, fc = c.fetch_result(native.CIRCUIT_EVM, s.cuda_stream)
                off, ofc = expect[labels[i]]
                assert np.array_equal(ff, off) and np.array_equal(fc, ofc), (rnd, i, labels[i], ge._diff(ff, off))
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            c.close()
