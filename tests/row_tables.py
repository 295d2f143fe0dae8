"""The six row circuits (bytecode, state, exp, public inputs, tx, sig) in one shape, for the strided, lookup-order and
borrowed-storage tests (test_gpu_row_tiled.py, test_row_lookup_order.py, test_gpu_row_lookup.py,
test_gpu_borrowed.py).

A witness is a dict: "m" the circuit's matrix uint64[n_cols][n_rows][4], "flags" its row flags (None: none), one
entry per lookup table the checker reads (TABLES), and "r" (keccak challenge limbs) or "clen" (the public-inputs
circuit length) where the circuit has them.  `oracle` and `emu` check such a dict.  The reference's tables are sets and
every one of these lookups names every column of its table, so no reordering or duplication can make one ambiguous."""
import os
import re

import emu_lib
import golden_util
import oracle_lib
import table_perturb as tp
from oracle_lib import same  # noqa: F401  (arrays == the oracle's, with the differing ids in the message)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = ("bytecode", "state", "exp", "pi", "tx", "sig")
TABLES = {"bytecode": ("push", "keccak"), "state": ("mpt",), "exp": (), "pi": ("keccak", "gas"), "tx": ("keccak",),
          "sig": ("keccak",)}
LOOKUP_FAMILIES = tuple(f for f in FAMILIES if TABLES[f])
MACRO = {"bytecode": "ZK_BYTECODE_CONSTRAINTS", "state": "ZK_STATE_CONSTRAINTS", "pi": "ZK_PI_CONSTRAINTS",
         "tx": "ZK_TX_CONSTRAINTS", "sig": "ZK_SIG_CONSTRAINTS", "exp": "ZK_EXP_CONSTRAINTS"}
# the lookups of these tables name every column: a duplicate row can never make them ambiguous
NEVER = {"state": ("ST_STO_MPT_AMBIG", "ST_ACC_MPT_AMBIG"), "pi": ("PI_TX_GAS_AMBIG",)}


def constraint_ids(family):
    """{constraint name: id} of a circuit, in the order of its X-macro in include/zk_constraints.h"""
    text = open(os.path.join(ROOT, "include", "zk_constraints.h")).read()
    body = text.split(f"#define {MACRO[family]}(X)", 1)[1].split("#define ", 1)[0]
    return {name: i for i, name in enumerate(re.findall(r"X\((\w+),", body))}


def vectors(family, every=1):
    """(label, witness dict) of every `every`-th golden vector of a family; each dict owns its arrays"""
    if family == "bytecode":
        for name, k, cols, push, kec, r, _, _ in golden_util.bytecode_vectors():
            if k % every == 0:
                yield f"{name}[{k}]", {"m": cols, "flags": None, "push": push, "keccak": kec, "r": r}
    elif family == "state":
        for name, k, s, f, m, _, _ in golden_util.state_vectors():
            if k % every == 0:
                yield f"{name}[{k}]", {"m": s, "flags": f, "mpt": m}
    elif family == "exp":
        for name, k, r, _, _ in golden_util.exp_vectors():
            if k % every == 0:
                yield f"{name}[{k}]", {"m": r, "flags": None}
    elif family == "pi":
        for name, k, R, K, G, clen, _, _ in golden_util.pi_vectors():  # the arrays are reused: copy them
            if k % every == 0:
                yield f"{name}[{k}]", {"m": R.copy(), "flags": None, "keccak": K.copy(), "gas": G.copy(), "clen": clen}
    else:
        gen = golden_util.tx_vectors() if family == "tx" else golden_util.sig_vectors()
        for k, rows, flags, kec, r, _, _ in gen:
            if k % every == 0:
                yield f"{family}[{k}]", {"m": rows, "flags": flags, "keccak": kec, "r": r}


def oracle(family, w, row_begin=0, row_end=None):
    m, f = w["m"], w["flags"]
    if family == "bytecode":
        return oracle_lib.check_bytecode(m, w["push"], w["keccak"], w["r"], row_begin, row_end)
    if family == "state":
        return oracle_lib.check_state(m, f, w["mpt"], row_begin, row_end)
    if family == "exp":
        return oracle_lib.check_exp(m, row_begin, row_end)
    if family == "pi":
        return oracle_lib.check_pi(m, w["keccak"], w["gas"], w["clen"], row_begin=row_begin, row_end=row_end)
    fn = oracle_lib.check_tx if family == "tx" else oracle_lib.check_sig
    return fn(m, f, w["keccak"], w["r"], row_begin, row_end)


def emu(family, w, challenge=None):
    """the product's row checker run serially on the CPU over the whole witness, trimmed to the oracle's constraint
    count"""
    m, f = w["m"], w["flags"]
    if family == "bytecode":
        ff, fc = emu_lib.check_bytecode(m, w["push"], w["keccak"], w["r"], challenge=challenge)
    elif family == "state":
        ff, fc = emu_lib.check_state(m, f, w["mpt"], challenge=challenge)
    elif family == "exp":
        ff, fc = emu_lib.check_exp(m)
    elif family == "pi":
        ff, fc = emu_lib.check_pi(m, w["keccak"], w["gas"], w["clen"], challenge=challenge)
    else:
        fn = emu_lib.check_tx if family == "tx" else emu_lib.check_sig
        ff, fc = fn(m, f, w["keccak"], w["r"], challenge=challenge)
    n = len(constraint_ids(family))
    return ff[:n], fc[:n]


def transformed(w, table, seed):
    """(kind, witness) for each transform of one table of a witness: its rows in a seeded random order, three
    identical copies of seeded rows, and for every column two copies of seeded rows with that column's cell changed"""
    t = w[table]
    yield "permuted", dict(w, **{table: tp.permute(t, None, seed)[0]})
    yield "identical", dict(w, **{table: tp.with_identical_duplicates(t, None, k=3, seed=seed)[0]})
    for c in range(t.shape[0]):
        yield f"near col {c}", dict(w, **{table: tp.with_near_duplicates(t, None, col=c, k=2, seed=seed + c)[0]})
