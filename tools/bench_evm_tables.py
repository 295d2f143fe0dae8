"""Supplementary measurement (not the bench.py contract): the EVM circuit's tx table and copy table built on the device
(zk_assign_tx_table from 11 cells + the call data per transaction; zk_assign_copy_table from the resident copy circuit)
against the host path they replace (Transaction.table_assignments / Tables._copy_circuit_to_table, then the packer).
Workloads:
  tx_2_18       64 txs sharing 2^18 call-data bytes
  tx_2_20       64 txs sharing 2^20 call-data bytes
  tx_one_2_20   one tx owning 2^20 call-data bytes
  tx_4096x256   4,096 txs of 256 bytes
  copy_2_20     the copy table of a 2^20-row copy circuit assigned by zk_assign_copy_circuit (512 events of 1,024 bytes)
Per workload one JSON line: table rows; the whole call (CUDA events around it, host validation and the pageable H2D
copies included, after warm-up; the copy-table call synchronises once); each kernel's device time (torch.profiler, a run
of its own); the bytes that cross PCIe against the canonical upload of the same table (32 B per cell + 1 flag byte per
row); for the tx table, the copy check that follows (a 2-event copy circuit whose TxCalldata rows look the table up: its
lookup-index build over the table and its check kernel, zk_last_timing); and the host path's time on a bounded sample
(rows of the first txs up to 2^16 call-data bytes, or the first 2^14 circuit rows), a CPU figure.  The card's name, power
limit and maximum SM clock are read in the same run.
    python tools/bench_evm_tables.py [--reps 20] [--warmup 3]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zkevm_specs_b200 import assign, native, packing, synth  # noqa: E402
from zkevm_specs_b200.evm_circuit.table import CopyCircuitRow, Tables  # noqa: E402
from zkevm_specs_b200.evm_circuit.typing import Transaction  # noqa: E402
from zkevm_specs_b200.util.arithmetic import FQ, Word, WordOrValue  # noqa: E402


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def kernel_times(run, names):
    """device microseconds per call of each kernel whose name contains one of `names`, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    reps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            run()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if any(n in e.key for n in names):
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            name = e.key.split("(")[0].replace("void ", "").replace("zk::", "")
            out[name] = out.get(name, 0.0) + us / reps
    return out


def timed(run, reps, warmup):
    import torch

    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), min(ms)


def seeded_txs(n_txs, length, seed):
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, n_txs * length, dtype=np.uint8)
    data[rng.random(data.shape[0]) < 0.3] = 0
    return [Transaction(k + 1, nonce=k, gas=1 << 20, caller_address=0xCAFE + k, callee_address=0xBEEF,
                        call_data=data[k * length:(k + 1) * length].tobytes()) for k in range(n_txs)]


def host_tx_path(txs):
    """what upload_tables does with a tx set: the mirror's rows, their cells and their Word flags"""
    rows = list(set(r for t in txs for r in t.table_assignments()))
    m = packing.pack(rows, packing.tx_table_row, 5)
    f = np.array([packing.word_flag(r.value) for r in rows], dtype=np.uint8)
    return m, f


def measure_tx(ctx, name, n_txs, length, reps, warmup, stream):
    txs = seeded_txs(n_txs, length, seed=n_txs)
    rec, cd, offs = assign.tx_records(txs)
    run = lambda: ctx.assign_tx_table(rec, cd, offs, stream=stream)  # noqa: E731
    med, mn = timed(run, reps, warmup)
    kt = kernel_times(run, ("k_assign_tx",))
    run()
    rows = ctx.table_rows(native.TABLE_TX)
    # the copy check that follows: a small copy circuit whose TxCalldata rows look the table up (verdict not used)
    w = synth.copy_events(2, 64)
    ctx.upload_table(native.TABLE_RW, w["rw"], flags=w["rw_flags"])
    ctx.upload_table(native.TABLE_BYTECODE, w["bytecode"])
    ctx.upload_columns(native.CIRCUIT_COPY, w["copy"], flags=w["copy_flags"])
    ctx.enable_timing(True)
    idx, chk = [], []
    for _ in range(warmup + reps):
        run()
        ctx.check_async(native.CIRCUIT_COPY, 0, w["copy"].shape[1], 0, native.FLAG_WRAP)
        i, c = ctx.last_timing()
        idx.append(i)
        chk.append(c)
    ctx.enable_timing(False)
    ctx.fetch_result(native.CIRCUIT_COPY)
    sample, total = [], 0
    for t in txs:
        if sample and total + len(t.call_data) > 1 << 16:
            break
        sample.append(t)
        total += len(t.call_data)
    t0 = time.perf_counter()
    m, _ = host_tx_path(sample)
    host_s = time.perf_counter() - t0
    return {"workload": name, "txs": n_txs, "call_data_bytes": int(offs[-1]), "rows": rows,
            "assign_ms_median": med, "assign_ms_min": mn, "kernel_us": kt,
            "h2d_bytes": rec.nbytes + int(offs[-1]) + offs.nbytes, "canonical_bytes": rows * (5 * 32 + 1),
            "copy_check_index_ms_median": statistics.median(idx[warmup:]), "copy_check_kernel_ms_median": statistics.median(chk[warmup:]),
            "host_sample_rows": m.shape[1], "host_sample_cpu_s": host_s}


def measure_copy(ctx, reps, warmup, stream):
    w = synth.copy_events(512, 1024)
    ctx.set_challenge(native.CHALLENGE_KECCAK, w["r_int"])
    ctx.assign_copy_circuit(w["events"], w["data"])
    run = lambda: ctx.assign_copy_table(stream=stream)  # noqa: E731
    med, mn = timed(run, reps, warmup)
    kt = kernel_times(run, ("k_copy_table", "CountScan"))
    rows = ctx.table_rows(native.TABLE_COPY)
    c = w["copy"][:, :1 << 14]
    fl = w["copy_flags"][:1 << 14]
    objs = []  # the mirror's CopyCircuitRow objects of the sample (what CopyCircuit.rows holds); not timed
    for r in range(c.shape[1]):
        f = [FQ(packing.cell_to_int(c[k, r])) for k in range(20)]
        objs.append(CopyCircuitRow(f[0], f[1], f[2], WordOrValue(Word((f[3], f[4]))) if fl[r] else WordOrValue(f[3]), *f[5:]))
    t0 = time.perf_counter()
    host_rows = packing.pack(Tables._copy_circuit_to_table(objs), packing.copy_table_row, 14)
    host_s = time.perf_counter() - t0
    return {"workload": "copy_2_20", "circuit_rows": int(w["copy"].shape[1]), "rows": rows,
            "assign_ms_median": med, "assign_ms_min": mn, "kernel_us": kt,
            "pcie_bytes": 16, "canonical_bytes": rows * 14 * 32,
            "host_sample_circuit_rows": int(c.shape[1]), "host_sample_table_rows": int(host_rows.shape[1]),
            "host_sample_cpu_s": host_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the device and has no CPU fallback")
    info = card()
    print(json.dumps(info), flush=True)
    ctx = native.Context(0)
    stream = torch.cuda.current_stream().cuda_stream
    for name, n_txs, length in (("tx_2_18", 64, 1 << 12), ("tx_2_20", 64, 1 << 14), ("tx_one_2_20", 1, 1 << 20),
                                ("tx_4096x256", 4096, 256)):
        print(json.dumps({**measure_tx(ctx, name, n_txs, length, args.reps, args.warmup, stream), **info}), flush=True)
    print(json.dumps({**measure_copy(ctx, args.reps, args.warmup, stream), **info}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
