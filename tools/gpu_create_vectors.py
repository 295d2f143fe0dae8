"""ErrorOutOfGasCREATE, ErrorOutOfGasSloadSstore and CREATE / CREATE2 vectors (tests/golden/evm26.npz, evm25.npz, evm24.npz) through the C-ABI on cuda:0 against the oracle, array for array.
Small enough to run under compute-sanitizer."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import importlib

import golden_util  # noqa: E402
import oracle_lib  # noqa: E402
from test_oracle_evm import fixed_table_matrix  # noqa: E402

native = importlib.import_module("zkevm-specs_b200.native")
evm_main = importlib.import_module("zkevm-specs_b200.evm_circuit.main")

limit = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 30
ctx = native.default_context()
fixed = fixed_table_matrix()
evm_main.upload_fixed_table(ctx)
ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
ctx.upload_table(native.TABLE_EXP, np.zeros((11, 0, 4), dtype=np.uint64))
ctx.upload_table(native.TABLE_TX, np.zeros((5, 0, 4), dtype=np.uint64))
ctx.upload_table(native.TABLE_BLOCK, np.zeros((4, 0, 4), dtype=np.uint64))
n = 0
import itertools  # noqa: E402

for name, k, w, exp_row, exp_exc in itertools.chain(golden_util.evm28_vectors(), golden_util.evm27_vectors(), golden_util.evm26_vectors(), golden_util.evm25_vectors(), golden_util.evm24_vectors()):
    if n >= limit:
        break
    ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
    ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
    ctx.upload_table(native.TABLE_COPY, w["copy"])
    if "tx_flags" in w:
        ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
    else:
        ctx.upload_table(native.TABLE_TX, w["tx"] if "tx" in w else np.zeros((5, 0, 4), dtype=np.uint64))
    ctx.upload_table(native.TABLE_STEP_AUX, w["aux"] if "aux" in w else np.zeros((3, 0, 4), dtype=np.uint64))
    ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
    ff, fc = ctx.check(native.CIRCUIT_EVM, 0, w["steps"].shape[1] - 1, 0, 0)
    off, ofc = oracle_lib.check_evm_x(w, fixed)
    assert np.array_equal(ff, off) and np.array_equal(fc, ofc), f"{name}[{k}] differs from oracle"
    n += 1
print(f"step-aux vectors ok: {n} cuda == oracle")
