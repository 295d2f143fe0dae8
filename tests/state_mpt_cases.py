"""Cases of zk_assign_state_circuit_mpt shared by the CPU emulation test and the GPU test: the golden operation lists of
state_mpt.npz (the reference's rows, MPT updates and exceptions), the state.npz bases, seeded operation lists run
through the mirror, and numpy restatements of the roots and the MPT table for lists too long for the mirror."""
import os
import random

import numpy as np

import golden_util
from zkevm_specs_b200 import packing
from zkevm_specs_b200 import state_circuit as sc
from zkevm_specs_b200.evm_circuit.spec import RW, AccountFieldTag
from zkevm_specs_b200.util.arithmetic import FQ, FR_MODULUS, Word


def golden_cases():
    """yield (name, ops13, flags, rows57, mpt12 in first-touch order, exception class name or "")"""
    z = np.load(os.path.join(golden_util.GOLDEN, "state_mpt.npz"))
    for name in z["names"]:
        name = str(name)
        yield (name, z[f"{name}/ops"], z[f"{name}/flags"], z[f"{name}/rows"], z[f"{name}/mpt"], str(z[f"{name}/exc"]))


def state_bases():
    """the unmutated bases of state.npz: yield (name, rows57, flags, mpt12 as the reference's set)"""
    z = np.load(os.path.join(golden_util.GOLDEN, "state.npz"))
    for name in z["names"]:
        name = str(name)
        yield name, z[f"{name}/rows"], z[f"{name}/flags"], z[f"{name}/mpt"]


def row_set(m):
    """the rows of a matrix uint64[c][n][4] as a sorted list (set comparison that keeps duplicates visible)"""
    return sorted(tuple(int(x) for x in m[:, r, :].reshape(-1)) for r in range(m.shape[1]))


def mirror_ops(seed: int, n: int):
    """a seeded, unsorted operation list of the mirror: Start, Memory, Stack, Storage (one small key pool touched under
    several tx ids) and Account ops of every field tag, Words and field values >= 2^128 among them"""
    r = random.Random(seed)
    ops = [sc.StartOp(1, RW.Read, 0)]
    addrs = [0x10, 0x11, (1 << 160) - 1, r.randrange(1 << 160)]
    for j in range(n):
        k = r.randrange(7)
        rw = r.choice([RW.Read, RW.Write])
        if k == 0:
            ops.append(sc.MemoryOp(j, rw, 1, r.randrange(8), r.randrange(256)))
        elif k == 1:
            ops.append(sc.StackOp(j, rw, 1, r.randrange(1024), Word(r.randrange(1 << 256))))
        elif k in (2, 3):
            ops.append(sc.StorageOp(j, rw, r.randrange(1, 5), r.choice(addrs), r.choice([0, 1, 5, (1 << 256) - 1]),
                                    Word(r.randrange(1 << 256)), Word(r.randrange(1 << 256))))
        elif k == 4:
            ops.append(sc.StartOp(j, RW.Read))
        else:
            t = r.choice(list(AccountFieldTag))
            word = t in (AccountFieldTag.Balance, AccountFieldTag.CodeHash)
            v = Word(r.randrange(1 << 256)) if word else FQ(r.randrange(FR_MODULUS))
            p = Word(r.randrange(1 << 256)) if word else FQ(r.randrange(1 << 130))
            ops.append(sc.AccountOp(j, rw, r.choice(addrs), int(t), v, p))
    r.shuffle(ops)
    return ops


def mirror_expected(ops):
    """the mirror's (rows57, flags, mpt12 in first-touch order), or the exception class name it raises"""
    try:
        rows = sc.assign_state_circuit(ops)
        upd = list(sc._mock_mpt_updates(ops).values())
    except (KeyError, AssertionError) as e:
        return type(e).__name__
    cols, flags = sc.pack_rows(rows)
    return cols, flags, packing.matrix_from_ints([sc.mpt_row(u) for u in upd], 12)


def ops_matrix(tag, addr, field, klo, khi, vlo, vhi, ilo, ihi):
    """13 operation cells from per-op uint64 arrays (each cell below 2^64; rw_counter = index, selector 1)"""
    n = len(tag)
    m = np.zeros((13, n, 4), dtype=np.uint64)
    m[0, :, 0] = np.arange(n, dtype=np.uint64)
    for c, v in ((2, tag), (4, addr), (5, field), (6, klo), (7, khi), (8, vlo), (9, vhi), (10, ilo), (11, ihi)):
        m[c, :, 0] = v
    m[12, :, 0] = 1
    return m


def spread_keys(n: int, n_keys: int, seed: int):
    """n unsorted ops, about a quarter Memory, the rest Storage / Account over n_keys keys (Storage keys touched under
    several tx ids): (ops13, flags), value Words where flag bit 0 is set"""
    rng = np.random.default_rng(seed)
    key = rng.integers(0, n_keys, n)
    is_acc = key % 5 == 0
    tag = np.where(is_acc, 6, 4).astype(np.uint64)
    mem = rng.random(n) < 0.25
    tag[mem] = 2
    addr = (0x1000 + key // 8).astype(np.uint64)
    field = np.where(is_acc, 1 + key % 4, 0).astype(np.uint64)
    klo = np.where(is_acc, 0, key * 0x9E3779B9).astype(np.uint64)
    khi = np.where(is_acc, 0, key % 3).astype(np.uint64)
    ops = ops_matrix(tag, addr, field, klo, khi, rng.integers(0, 1 << 63, n, dtype=np.uint64),
                     rng.integers(0, 1 << 63, n, dtype=np.uint64), rng.integers(0, 1 << 63, n, dtype=np.uint64), 0 * key)
    ops[3, :, 0] = rng.integers(1, 9, n)  # tx ids: one Storage key shares its MPT key across them
    flags = np.where(field == 2, 1, 0).astype(np.uint8) | np.where((~is_acc) & (tag == 4), 1, 0).astype(np.uint8)
    ops[9, flags == 0, 0] = 0  # a field value has no hi half
    ops[11, :, 0] = 0
    return ops, flags


def restate(ops, flags):
    """the roots (uint64[n]) and MPT table (uint64[12][U][4]) of 13 operation cells whose cells are below 2^64 and whose
    values are below 2^128: first touches from np.unique(return_index), the next MPT op of each row by searchsorted"""
    n = ops.shape[1]
    tag = ops[2, :, 0]
    is_mpt = (tag == 4) | (tag == 6)
    pos = np.nonzero(is_mpt)[0]
    keys = np.stack([ops[4, pos, 0], ops[5, pos, 0], ops[6, pos, 0], ops[7, pos, 0]], axis=1)
    uniq, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)  # first-touch order of the distinct keys
    rank = np.empty(len(order), dtype=np.int64)
    rank[order] = np.arange(len(order))
    U = len(order)
    op_rank = rank[inv.reshape(-1)]  # the update rank of each MPT op's key
    j = np.searchsorted(pos, np.arange(n), side="right")  # the first MPT op after each row
    roots = np.full(n, 3 + 5 * U, dtype=np.uint64)
    has = j < len(pos)
    roots[has] = (3 + 5 * op_rank[j[has]]).astype(np.uint64)
    src = pos[first[order]]  # the op of update u
    t = np.zeros((12, U, 4), dtype=np.uint64)
    t[0, :, 0] = ops[4, src, 0]
    t[1, :, 0] = np.where(tag[src] == 4, 6, ops[5, src, 0])
    t[2, :, 0], t[3, :, 0] = ops[6, src, 0], ops[7, src, 0]
    t[4, :, 0] = 3 + 5 * (np.arange(U, dtype=np.uint64) + 1)
    t[6, :, 0] = 3 + 5 * np.arange(U, dtype=np.uint64)
    for c, lo in ((8, 8), (10, 10)):  # Word(lo + hi 2^128) of a value below 2^128 in each half: lo, hi as they are
        bit = 1 if lo == 8 else 2
        t[c, :, 0] = ops[lo, src, 0]
        t[c + 1, :, 0] = np.where(flags[src] & bit, ops[lo + 1, src, 0], 0)
    return roots, t


def repeated_key(n: int):
    """one Storage key touched by all n ops"""
    z = np.zeros(n, dtype=np.uint64)
    ops = ops_matrix(z + 4, z + 0xAB, z, z + 0x77, z, np.arange(n, dtype=np.uint64), z, z + 5, z)
    return ops, np.zeros(n, dtype=np.uint8)


def colliding_keys(n_keys: int, home_slot, n_ops: int):
    """n_keys distinct Storage keys (address 0x42, key lo searched) that share one home slot of the hash table of n_ops
    ops, each touched twice; home_slot(key_cells, n_ops) is the emulation's slot function"""
    want = home_slot((0x42, 0, 0, 0), n_ops)
    found = [0]
    k = 1
    while len(found) < n_keys:
        if home_slot((0x42, 0, k, 0), n_ops) == want:
            found.append(k)
        k += 1
    klo = np.array(found * 2 + [0] * (n_ops - 2 * n_keys), dtype=np.uint64)
    tag = np.array([4] * (2 * n_keys) + [2] * (n_ops - 2 * n_keys), dtype=np.uint64)
    z = np.zeros(n_ops, dtype=np.uint64)
    return ops_matrix(tag, z + 0x42, z, klo, z, np.arange(n_ops, dtype=np.uint64), z, z, z), np.zeros(n_ops, dtype=np.uint8)


def with_address_beyond_160_bits(ops, i):
    out = ops.copy()
    out[4, i, :] = [0, 0, 1 << 32, 0]
    return out

