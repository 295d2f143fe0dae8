"""Inputs of the device exp-circuit builder (zk_assign_exp_circuit, csrc/assign.cu) and what the host mirror of the
reference's builder produces for them: ExpCircuit.add_event per (base, exponent, identifier), fill_dummy_events, and the
exp table of Tables(exp_circuit=...) (evm_circuit.main.exp_table_rows).  Shared by test_assign_exp_emu.py (CPU) and
test_gpu_assign_exp.py."""
import os

import numpy as np

from zkevm_specs_b200 import packing
from zkevm_specs_b200.evm_circuit.main import exp_table_rows
from zkevm_specs_b200.exp_circuit import ExpCircuit, exp_row
from zkevm_specs_b200.util.arithmetic import FR_MODULUS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX = (1 << 256) - 1
# the constant fill_dummy_events row as an exp-table row (is_step = 1 there, table.py:654-671)
PAD_TABLE_ROW = (1, 0, 0, 1, 0, 0, 0, 1, 0, 1, 0)


def cell(limbs) -> int:
    return sum(int(x) << (64 * k) for k, x in enumerate(limbs))


def events_from_rows(rows):
    """the add_event calls behind circuit rows uint64[21][n][4]: an event starts at a step row that is row 0 or follows an
    is_last row, and its first row holds (base, exponent = x, identifier)"""
    out = []
    for r in range(rows.shape[1]):
        if cell(rows[1, r]) == 1 and (r == 0 or cell(rows[3, r - 1]) == 1):
            out.append((cell(rows[4, r]) + (cell(rows[5, r]) << 128), cell(rows[6, r]) + (cell(rows[7, r]) << 128),
                        cell(rows[2, r])))
    return out


def golden_events():
    """yield (scenario, events, golden rows uint64[21][n][4]) of tests/golden/exp.npz"""
    z = np.load(os.path.join(GOLDEN, "exp.npz"))
    for name in z["names"]:
        rows = z[f"{name}/rows"]
        yield str(name), events_from_rows(rows), rows


def events_from_table(tab):
    """the add_event calls behind an exp table uint64[11][n][4] (evm19.npz): per (identifier, base), the row with the
    largest exponent"""
    best = {}
    for r in range(tab.shape[1]):
        c = [cell(tab[k, r]) for k in range(11)]
        base = c[3] + (c[4] << 64) + (c[5] << 128) + (c[6] << 192)
        x = c[7] + (c[8] << 128)
        key = (c[1], base)
        best[key] = max(best.get(key, 0), x)
    return [(base, x, ident) for (ident, base), x in best.items()]


def table_set(tab):
    return {tuple(cell(tab[k, r]) for k in range(tab.shape[0])) for r in range(tab.shape[1])}


def mirror(events, n_rows_min=0):
    """(rows uint64[21][n][4], exp-table row set, event rows) of the host mirror: add_event per event, then the dummy
    row up to n_rows_min rows"""
    c = ExpCircuit()
    for base, x, ident in events:
        c.add_event(base, x, ident)
    used = len(c.rows)
    c.OFFSET_INCREMENT, c.max_exp_steps = 1, n_rows_min  # fill_dummy_events up to exactly n_rows_min rows
    c.fill_dummy_events()
    return packing.matrix_from_ints([exp_row(r) for r in c.rows], 21), {tuple(r) for r in exp_table_rows(c.rows)}, used


def random_events(n, seed, exp_bits=256):
    rng = np.random.default_rng(seed)
    big = lambda bits: int.from_bytes(rng.bytes(32), "little") >> (256 - bits)  # noqa: E731
    return [(big(256), big(int(rng.integers(1, exp_bits + 1))), int(rng.integers(1, 1 << 20))) for _ in range(n)]


def cases():
    """yield (label, events, n_rows_min)"""
    for name, ev, rows in golden_events():
        yield f"golden {name}", ev, rows.shape[1]
    b = 0xC0FFEE ** 9 % (1 << 256)
    for x in (0, 1, 2, 3, 1 << 255, MAX):
        yield f"exponent {x:#x}", [(b, x, 7)], 0
    for base in (0, 1, 1 << 128, MAX):
        yield f"base {base:#x}", [(base, 0x1F0F, 3), (base, MAX, 4), (base, 2, 5)], 0
    yield "identifier p - 1", [(b, 1023, FR_MODULUS - 1), (b + 1, 6, FR_MODULUS - 1)], 0
    ev = [(b, 101, 12), (3, 5, 77), (MAX, 3, 9)]
    used = sum(n_rows(x) for _, x, _ in ev)
    for label, n in (("below", used - 3), ("equal", used), ("above", used + 40)):
        yield f"pad {label} the used rows", ev, n
    yield "zero events", [], 0
    yield "zero events, padded", [], 11
    yield "exponents 0 / 1 only, padded", [(b, 0, 1), (b, 1, 2)], 3
    yield "seeded random batch", random_events(40, seed=5), 4000


def n_rows(x: int) -> int:
    return 0 if x < 2 else (x.bit_length() - 1) + (bin(x).count("1") - 1)
