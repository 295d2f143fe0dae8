"""Long traces tiled from the golden vectors (pure numpy), with a verdict bound that needs no device.

Every golden EVM vector holds 2 to 21 steps, so on the device no thread of a persistent grid ever takes a
second step, and a warp almost never holds two failing lanes.  A tiled trace concatenates C copies of the step
matrices of one group of vectors (one scenario, identical tables) in a seeded order and keeps the group's tables,
so the same gate programs see thousands of steps in one launch.

The bound: a copy that is neither the first nor the last has the same steps, the same successor and the same
tables as its small vector, so it fails exactly where that vector fails when checked without the FIRST / LAST
step flags (those bind only the first and last step of the whole trace).  Hence, for every constraint id,
fail_count[id] >= the sum of the interior copies' small counts, and first_fail[id] <= the first such row.  The
successor row of each copy is checked against the next copy's first step; those verdicts are left to the oracle.

The copy circuit is tiled the same way (ZK_FLAG_WRAP): a row whose +1 and +2 rotations stay inside its copy keeps
its small verdict."""
import hashlib

import numpy as np

import golden_util
import oracle_lib

PASS = 0xFFFFFFFF
EVM_FAMILIES = ("evm",) + tuple(f"evm{i}" for i in range(2, 29))
# every side table an EVM witness may carry, and its empty form: a missing table is uploaded (and handed to the
# oracle) empty, so no table of an earlier witness is ever left behind
EMPTY = {"bytecode": (6,), "rw": (14,), "copy": (14,), "keccak": (5,), "tx": (5,), "block": (4,), "wd": (4,),
         "exp": (11,), "aux": (3,)}
ROW_FLAGS = ("rw_flags", "tx_flags", "block_flags")
EVM_TABLES = tuple(EMPTY)
COPY_TABLES = ("rw", "rw_flags", "tx", "tx_flags", "bytecode")


def full_witness(w):
    """the witness dict with every side table present (empty where the vector has none) and `flags` set"""
    out = dict(w)
    for name, (n_cols,) in EMPTY.items():
        if out.get(name) is None:
            out[name] = np.zeros((n_cols, 0, 4), dtype=np.uint64)
    for fl in ROW_FLAGS:
        if out.get(fl) is None:
            out[fl] = np.zeros(0, dtype=np.uint8)
    out["flags"] = int(out.get("flags") or 0)
    return out


def family_vectors(family):
    """(scenario, k, witness dict) of an EVM golden family; evm.npz's (steps, bytecode, rw, flags) tuples become
    witness dicts too"""
    if family == "evm":
        for name, k, s, b, r, flags, _row, _exc in golden_util.evm_vectors():
            yield name, k, full_witness({"steps": s, "bytecode": b, "rw": r, "flags": flags})
    else:
        vecs = golden_util.evm11_vectors() if family == "evm11" else golden_util.evm2_vectors(family)
        for name, k, w, _row, _exc in vecs:
            yield name, k, full_witness(w)


def _digest(w, keys):
    h = hashlib.sha1()
    for key in keys:
        a = w.get(key)
        if isinstance(a, np.ndarray):
            h.update(key.encode() + str(a.shape).encode() + np.ascontiguousarray(a).tobytes())
        else:
            h.update(key.encode() + repr(a).encode())
    return h.hexdigest()


def groups(vectors, table_keys):
    """[(scenario, [(k, witness), ...])]: vectors of one scenario whose tables (`table_keys`, row flags and `flags`
    included) are identical byte for byte, in file order"""
    out = {}
    for name, k, w in vectors:
        out.setdefault((name, _digest(w, table_keys)), (name, []))[1].append((k, w))
    return list(out.values())


def evm_groups(family):
    return groups(family_vectors(family), EVM_TABLES + ROW_FLAGS + ("flags",))


def oracle_evm(w, fixed, row_end=None, flags=None):
    """the oracle on a full witness dict (full_witness): every checked row, the dict's flags unless `flags`"""
    v = dict(w)
    v["flags"] = w["flags"] if flags is None else flags
    return oracle_lib.check_evm_x(v, fixed, row_end=row_end)


def copies_for(w, min_bucket):
    """copies of `w`'s step matrix after which every execution state in it fills more than min_bucket steps"""
    st = w["steps"][0, :, 0]
    _, counts = np.unique(st, return_counts=True)
    return int(-(-(min_bucket + 1) // int(counts.min())))


class Tiled:
    """a tiled witness (`w`, a full witness dict), the vector index of every copy (`pick`), their first rows
    (`offsets`) and the per-copy lower bound (`lb_first`, `lb_count`)"""

    def __init__(self, w, pick, offsets, lb_first, lb_count):
        self.w, self.pick, self.offsets, self.lb_first, self.lb_count = w, pick, offsets, lb_first, lb_count

    @property
    def n_rows(self):
        return self.w["steps"].shape[1] if "steps" in self.w else self.w["copy"].shape[1]

    def holds(self, ff, fc):
        """the per-copy lower bound holds for the arrays (first_fail, fail_count) of the whole trace"""
        return bool((ff.astype(np.int64) <= self.lb_first).all() and (fc >= self.lb_count).all())


def _lower_bound(small, pick, offsets, interior):
    """small[j] = (first_fail, fail_count) of vector j; the bound over the copies c where interior[c]"""
    n = len(small[0][0])
    lb_first = np.full(n, PASS, dtype=np.int64)
    lb_count = np.zeros(n, dtype=np.uint64)
    for c in np.nonzero(interior)[0]:
        ff, fc = small[pick[c]]
        hit = ff != PASS
        lb_first[hit] = np.minimum(lb_first[hit], offsets[c] + ff[hit].astype(np.int64))
        lb_count += fc
    return lb_first, lb_count


def tile_evm(members, n_copies, seed, fixed, small=None):
    """a tiled EVM trace of n_copies copies of the members' step matrices (members: [(k, full witness)] of one
    group); `small`: their flag-free oracle verdicts, if already known"""
    ws = [w for _, w in members]
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, len(ws), n_copies)
    lens = np.array([ws[j]["steps"].shape[1] for j in pick], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)[:-1]])
    out = dict(ws[0])
    out["steps"] = np.ascontiguousarray(np.concatenate([ws[j]["steps"] for j in pick], axis=1))
    aux = ws[0]["aux"]
    if aux.shape[1]:  # the step-aux key is the global step row
        tiles = np.repeat(aux[None], n_copies, axis=0)  # [C][3][m][4]
        tiles[:, 0, :, 0] += offsets.astype(np.uint64)[:, None]
        out["aux"] = np.ascontiguousarray(tiles.transpose(1, 0, 2, 3).reshape(3, -1, 4))
    if small is None:
        small = [oracle_evm(w, fixed, flags=0) for w in ws]
    interior = np.ones(n_copies, dtype=bool)
    interior[[0, -1]] = False
    return Tiled(out, pick, offsets, *_lower_bound(small, pick, offsets, interior))


def copy_groups():
    """[(scenario, [(k, witness, r)])] of copy.npz, grouped like the EVM families"""
    vecs = [(name, k, (w, r)) for name, k, w, r, _row, _exc in golden_util.copy_vectors()]
    out = {}
    for name, k, (w, r) in vecs:
        out.setdefault((name, _digest(w, COPY_TABLES)), (name, []))[1].append((k, w, r))
    return list(out.values())


def tile_copy(members, n_copies, seed, small=None):
    """a tiled copy-circuit witness (checked with ZK_FLAG_WRAP over every row); `small`: the members' oracle verdicts
    over rows [0, n - 2), if already known"""
    ws = [w for _, w, _ in members]
    r = members[0][2]
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, len(ws), n_copies)
    lens = np.array([ws[j]["copy"].shape[1] for j in pick], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)[:-1]])
    out = dict(ws[0])
    out["copy"] = np.ascontiguousarray(np.concatenate([ws[j]["copy"] for j in pick], axis=1))
    out["copy_flags"] = np.ascontiguousarray(np.concatenate([np.asarray(ws[j]["copy_flags"], dtype=np.uint8) for j in pick]))
    if small is None:
        small = [oracle_lib.check_copy(w, r, 0, w["copy"].shape[1] - 2) for w in ws]
    t = Tiled(out, pick, offsets, *_lower_bound(small, pick, offsets, np.ones(n_copies, dtype=bool)))
    t.r = r
    return t
