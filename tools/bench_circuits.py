"""Supplementary measurements (not the bench.py contract): BASELINE.json's cfg3 / cfg4 / cfg5 on one
H100 — device time, rows/s and achieved GB/s (canonical algorithmic bytes, SURVEY.md §8d) of every
row circuit, each pass including its lookup-index work, for canonical and packed storage:
  state circuit  cfg3: 2^18 rows;  cfg5 share: 2^21 rows
  copy circuit   cfg4: 2^20 rows;  cfg5 share: 2^19 rows
  bytecode circuit     cfg5 share: 2^19 rows
  evm circuit          cfg5 share: 2^20 steps (bench.py's workload)
and the cfg5 "super circuit" aggregate (sum of rows / sum of device time; each circuit is checked
against its own tables, DESIGN.md section 7).  One JSON line per measurement on stdout."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zkevm_specs_b200 import native, synth  # noqa: E402
from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix  # noqa: E402


def measure(ctx, circuit, row_end, flags, reps=20):
    ctx.enable_timing(True)
    idx, chk = [], []
    for _ in range(reps + 3):
        ctx.invalidate_indexes()
        ctx.check_async(circuit, 0, row_end, 0, flags)
        a, b = ctx.last_timing()
        idx.append(a)
        chk.append(b)
    ctx.enable_timing(False)
    ff, fc = ctx.fetch_result(circuit)
    assert (ff == native.PASS).all(), native.first_failure(ff, circuit)
    return float(np.mean(idx[3:])), float(np.mean(chk[3:]))


def line(name, storage, n, i_ms, c_ms, byt, peak, **extra):
    d = {"circuit": name, "storage": storage, "rows": n, "index_ms": i_ms, "check_ms": c_ms,
         "rows_per_s": n / ((i_ms + c_ms) / 1e3), "algorithmic_bytes": byt, "achieved_gbs": byt / (c_ms / 1e3) / 1e9,
         "frac_of_measured_hbm": byt / (c_ms / 1e3) / 1e9 / peak, **extra}
    print(json.dumps(d), flush=True)
    return d


def main():
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 6650.0
    ctx = native.Context(0)
    agg = {}
    for storage in ("canonical", "packed"):
        ctx.packed_uploads = "min" if storage == "packed" else None
        super_rows = super_ms = 0.0
        for tag, n_state in (("cfg3", 1 << 18), ("cfg5", 1 << 21)):
            w = synth.state_rows(n_state, seed=3)
            ctx.upload_table(native.TABLE_MPT, w["mpt"])
            ctx.upload_columns(native.CIRCUIT_STATE, w["rows"], flags=w["flags"])
            n = w["rows"].shape[1]
            i_ms, c_ms = measure(ctx, native.CIRCUIT_STATE, n, native.FLAG_WRAP)
            line(f"state ({tag})", storage, n, i_ms, c_ms, 32 * (n * 57 + w["mpt"].shape[1] * 12), peak)
            if tag == "cfg5":
                super_rows, super_ms = super_rows + n, super_ms + i_ms + c_ms
        for tag, n_events in (("cfg4", 512), ("cfg5", 256)):
            w = synth.copy_events(n_events, 1024, seed=4)
            ctx.set_challenge(native.CHALLENGE_KECCAK, sum(int(w["r"][k]) << (64 * k) for k in range(4)))
            ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
            ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
            ctx.upload_table(native.TABLE_TX, w["tx"], flags=w["tx_flags"])
            ctx.upload_columns(native.CIRCUIT_COPY, w["copy"], flags=w["copy_flags"])
            n = w["copy"].shape[1]
            i_ms, c_ms = measure(ctx, native.CIRCUIT_COPY, n, native.FLAG_WRAP)
            line(f"copy ({tag})", storage, n, i_ms, c_ms, 32 * (n * 20 + w["rw"].shape[1] * 14 + w["tx"].shape[1] * 5), peak)
            if tag == "cfg5":
                super_rows, super_ms = super_rows + n, super_ms + i_ms + c_ms
        w = synth.bytecode_circuit_rows(19, 8)
        ctx.set_challenge(native.CHALLENGE_KECCAK, sum(int(w["r"][k]) << (64 * k) for k in range(4)))
        ctx.upload_table(native.TABLE_PUSH, w["push"])
        ctx.upload_table(native.TABLE_KECCAK, w["keccak"])
        ctx.upload_columns(native.CIRCUIT_BYTECODE, w["rows"])
        n = w["rows"].shape[1]
        i_ms, c_ms = measure(ctx, native.CIRCUIT_BYTECODE, n, native.FLAG_WRAP)
        line("bytecode (cfg5)", storage, n, i_ms, c_ms, 32 * n * 12, peak)
        super_rows, super_ms = super_rows + n, super_ms + i_ms + c_ms
        w = synth.evm_trace(1 << 18, seed=2)
        ctx.upload_table(native.TABLE_FIXED, fixed_table_matrix())
        ctx.upload_table(native.TABLE_COPY, np.zeros((14, 0, 4), dtype=np.uint64))
        ctx.upload_table(native.TABLE_KECCAK, np.zeros((5, 0, 4), dtype=np.uint64))
        ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
        ctx.upload_table(native.TABLE_RW, w["rw"])
        ctx.upload_columns(native.CIRCUIT_EVM, w["steps"])
        n = w["n_steps"]
        i_ms, c_ms = measure(ctx, native.CIRCUIT_EVM, n, 0)
        line("evm (cfg5)", storage, n, i_ms, c_ms,
             32 * (n * 13 + w["rw"].shape[1] * 14 + w["bytecode"].shape[1] * 6), peak)
        super_rows, super_ms = super_rows + n, super_ms + i_ms + c_ms
        agg[storage] = {"circuit": "super circuit (cfg5: evm 2^20 + state 2^21 + copy 2^19 + bytecode 2^19)",
                        "storage": storage, "rows": int(super_rows), "device_ms": super_ms,
                        "rows_per_s": super_rows / (super_ms / 1e3)}
        print(json.dumps(agg[storage]), flush=True)


if __name__ == "__main__":
    main()
