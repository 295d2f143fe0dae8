"""Borrowed device storage (include/zkcheck.h zk_bind_columns_device / zk_bind_table_device): torch CUDA tensors
bound as the witness matrix and the lookup tables give the upload path's arrays, a tensor edited in place and bound
again is read as new contents (its index rebuilt), and a pointer the kernels could not read in place — not 16-byte
aligned, host memory, null — is refused before anything is stored."""
import time

import numpy as np
import pytest

import golden_util
import oracle_lib
import row_tables as rt
import test_gpu_evm as ge
import test_gpu_row_tiled as T
from oracle_lib import same as _same
from zkevm_specs_b200 import native
from zkevm_specs_b200.evm_circuit import main as evm_main
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
TABLE_ID = {"push": native.TABLE_PUSH, "keccak": native.TABLE_KECCAK, "mpt": native.TABLE_MPT,
            "gas": native.TABLE_CALLDATA_GAS}


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_borrowed.py wall time {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def own():
    """a context of this module's own, so that no other test sees what it borrows; every test hands its bound
    storage back (uploads host copies over it) before its tensors go"""
    ctx = native.Context(0)
    evm_main.upload_fixed_table(ctx)
    ge.clear_tables(ctx, ("copy", "keccak", "tx", "block", "wd", "exp", "aux"))
    yield ctx
    ctx.close()


def _tensor(m):
    """a CUDA tensor holding the canonical matrix uint64[n_cols][n_rows][4] (as int64: same bits)"""
    return torch.from_numpy(np.ascontiguousarray(m, dtype=np.uint64).view(np.int64)).to("cuda")


def _row_flags(ctx, circuit_id, flags):
    f = np.ascontiguousarray(flags, dtype=np.uint8)
    ctx._ck(ctx._L.zk_upload_row_flags(ctx._h, circuit_id, f.shape[0], f.ctypes.data, None), "zk_upload_row_flags")


def _bind(ctx, fam, w, keep, names):
    """bind the named tables ("m": the witness matrix) from the CUDA tensors in `keep` (made from `w` when missing),
    uploading nothing"""
    for name in names:
        t = keep.setdefault(name, _tensor(w[name]))
        if name == "m":
            ctx.bind_columns_device(T.CIRCUIT[fam], w["m"].shape[1], w["m"].shape[0], t.data_ptr())
            if w["flags"] is not None:
                _row_flags(ctx, T.CIRCUIT[fam], w["flags"])
        else:
            ctx.bind_table_device(TABLE_ID[name], w[name].shape[1], w[name].shape[0], t.data_ptr())
    torch.cuda.synchronize()


def _check(ctx, fam, w):
    return ctx.check(T.CIRCUIT[fam], 0, w["m"].shape[1], 0, 0 if fam in ("tx", "sig") else native.FLAG_WRAP)


def _bound(ctx, fam, w, keep):
    """T.device with every table and the matrix bound from CUDA tensors (kept alive in `keep`)"""
    T.upload_tables(ctx, fam, w)  # the challenges (the tables are bound over right after)
    _bind(ctx, fam, w, keep, (*rt.TABLES[fam], "m"))
    return _check(ctx, fam, w)


@pytest.mark.parametrize("fam", rt.FAMILIES)
def test_bound_tensors_equal_the_upload_path(fam, own):
    """every 25th golden vector of a row family: bound tensors == uploaded matrices == oracle"""
    ctx = own
    n = 0
    for j, (label, w) in enumerate(rt.vectors(fam)):
        if j % 25:
            continue
        want = rt.oracle(fam, w)
        keep = {}
        _same(_bound(ctx, fam, w, keep), want, f"{fam} {label} bound")
        _same(T.device(ctx, fam, w), want, f"{fam} {label} uploaded")  # also hands the bound storage back
        n += 1
    assert n >= 10


def test_bound_evm_tensors_equal_the_upload_path(own):
    """every 20th evm.npz vector with the steps, bytecode and rw tables bound: == upload path == oracle"""
    ctx = own
    fixed = fixed_table_matrix()
    n = 0
    for name, k, s, b, r, flags, _, _ in golden_util.evm_vectors():
        if k % 20:
            continue
        want = oracle_lib.check_evm(s, b, r, fixed, flags=flags)
        keep = [_tensor(b), _tensor(r), _tensor(s)]
        ctx.bind_table_device(native.TABLE_BYTECODE, b.shape[1], b.shape[0], keep[0].data_ptr())
        ctx.bind_table_device(native.TABLE_RW, r.shape[1], r.shape[0], keep[1].data_ptr())
        ctx.bind_columns_device(native.CIRCUIT_EVM, s.shape[1], s.shape[0], keep[2].data_ptr())
        torch.cuda.synchronize()
        _same(ctx.check(native.CIRCUIT_EVM, 0, s.shape[1] - 1, 0, flags), want, f"evm {name}[{k}] bound")
        ctx.upload_table(native.TABLE_BYTECODE, b)  # also hands the bound storage back
        ctx.upload_table(native.TABLE_RW, r)
        ctx.upload_columns(native.CIRCUIT_EVM, s)
        _same(ctx.check(native.CIRCUIT_EVM, 0, s.shape[1] - 1, 0, flags), want, f"evm {name}[{k}] uploaded")
        n += 1
    assert n >= 5


def _swap_rows(t, a, b):
    t[:, [a, b]] = t[:, [b, a]]


def _equal(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_rebinding_an_edited_tensor_rebuilds_the_index(own):
    """the strided bytecode witness bound from tensors, then edited in place step by step, each step rebinding only
    the edited tensor at the same pointer (nothing uploaded).  Each step changes the oracle's arrays and the device
    must follow them, which a stale index could not:
      1. keccak: the corrupted RLC of row 2 restored, row 0's corrupted instead.  The hash index of the first bind
         holds row 2 under its corrupted key, so a stale probe of contract 3's true key would miss.
      2. push: rows 0x61 / 0x62, bound swapped (an irregular table, served by the hash index), swapped back (a regular
         table, staged) and row 0x63's push size made wrong.  A stale hash index would send the (0x61, 2) probe to
         row 0x62, and a stale positional flag would keep the table off the staged path.
      3. witness: one RLC cell of a Byte row."""
    ctx = own
    w, _, _ = T.witness("bytecode")
    w = dict(w, m=w["m"].copy(), keccak=w["keccak"].copy(), push=w["push"].copy())
    assert w["keccak"].shape[1] >= 3 and ((w["m"][4, :, 0] == 2) & (w["m"][6, :, 0] == 0x61)).any()
    w["keccak"][1, 2, 0] ^= np.uint64(1)
    _swap_rows(w["push"], 0x61, 0x62)
    keep = {}

    def keccak_edit(k):
        k[1, 2, 0] ^= np.uint64(1)
        k[1, 0, 0] ^= np.uint64(1)

    def push_edit(p):
        _swap_rows(p, 0x61, 0x62)
        p[1, 0x63, 0] += np.uint64(1)

    def witness_edit(m):
        m[9, 3001, 0] ^= np.uint64(1)

    try:
        prev = rt.oracle("bytecode", w)
        assert (prev[0] != native.PASS).any()
        _same(_bound(ctx, "bytecode", w, keep), prev, "first bind")
        ptrs = {name: t.data_ptr() for name, t in keep.items()}
        for name, edit, what in (("keccak", keccak_edit, "keccak rows edited in place"),
                                 ("push", push_edit, "push rows swapped back and one push size changed in place"),
                                 ("m", witness_edit, "a witness cell edited in place")):
            edit(w[name])
            keep[name].copy_(_tensor(w[name]))  # the same storage, new contents
            want = rt.oracle("bytecode", w)
            assert not _equal(want, prev), f"{what}: the edit must change the verdict"
            _bind(ctx, "bytecode", w, keep, (name,))
            _same(_check(ctx, "bytecode", w), want, what)
            prev = want
        assert {name: t.data_ptr() for name, t in keep.items()} == ptrs
    finally:
        T.device(ctx, "bytecode", w)  # hand the bound storage back before the tensors go


def _aligned_host(a):
    """a host copy of `a` at a 64-byte-aligned address, so that only its memory type can refuse it"""
    raw = np.zeros(a.nbytes + 64, dtype=np.uint8)
    off = -raw.ctypes.data % 64
    out = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
    out[...] = a
    assert out.ctypes.data % 16 == 0
    return out


def test_bind_refuses_misaligned_host_and_null_pointers():
    """a view 8 bytes into a tensor, an aligned host numpy array and a null pointer with rows, as the witness matrix
    and as a table: each raises NativeError for its own reason.  On a context of its own that never runs a check, so
    a refused pointer is never read"""
    ctx = native.Context(0)
    try:
        w = next(rt.vectors("tx"))[1]
        m = _tensor(w["m"])
        k = _tensor(w["keccak"])
        host_m, host_k = _aligned_host(w["m"]), _aligned_host(w["keccak"])
        n, nc = w["m"].shape[1], w["m"].shape[0]
        kn, kc = w["keccak"].shape[1], w["keccak"].shape[0]
        for ptr, why in ((m.data_ptr() + 8, "not 16-byte aligned"), (host_m.ctypes.data, "not device"), (0, "null")):
            with pytest.raises(native.NativeError, match=why):
                ctx.bind_columns_device(native.CIRCUIT_TX, n, nc, ptr)
        for ptr, why in ((k.data_ptr() + 8, "not 16-byte aligned"), (host_k.ctypes.data, "not device"), (0, "null")):
            with pytest.raises(native.NativeError, match=why):
                ctx.bind_table_device(native.TABLE_KECCAK, kn, kc, ptr)
        ctx.bind_columns_device(native.CIRCUIT_TX, n, nc, m.data_ptr())  # the aligned tensor itself is taken
        ctx.bind_table_device(native.TABLE_KECCAK, kn, kc, k.data_ptr())
        ctx.bind_columns_device(native.CIRCUIT_TX, 0, nc, 0)  # no rows: nothing to read
    finally:
        ctx.close()
