"""Supplementary measurement (not the bench.py contract): the exponentiation circuit assigned on the device
(zk_assign_exp_circuit: ExpCircuit.add_event per EXP event + fill_dummy_events, and the exp table) against the host
mirror's Python loop, on seeded events for two workloads of 2^20 rows:
  exp256  uniformly random 256-bit exponents (~382 rows per event)
  exp64   uniformly random exponents below 2^64 (~94 rows per event)
Per workload one JSON line: the device assignment time (CUDA events around the whole call, host preparation and the
H2D copy included, after warm-up), the device time of each of its two kernels (torch.profiler, a run of its own), the
k_check_exp time on the assigned narrow rows, the bytes that cross PCIe (96 B per event + the row offsets) against the
672 B per row of the canonical upload, and the host mirror's ExpCircuit.add_event time for the same events, a CPU
figure.  The card's name, power limit and maximum SM clock are read in the same run and printed with the results.
    python tools/bench_exp_assign.py [--rows 1048576] [--reps 20] [--mirror-events N]"""
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
from zkevm_specs_b200 import assign, native  # noqa: E402
from zkevm_specs_b200.exp_circuit import ExpCircuit  # noqa: E402


def event_rows(x: int) -> int:
    return 0 if x < 2 else (x.bit_length() - 1) + (bin(x).count("1") - 1)


def workload(n_rows: int, exp_bits: int, seed: int):
    """seeded (base, exponent, identifier) events whose rows fill at most n_rows"""
    rng = np.random.default_rng(seed)
    events, used = [], 0
    while True:
        base = int.from_bytes(rng.bytes(32), "little")
        x = int.from_bytes(rng.bytes(32), "little") >> (256 - exp_bits)
        if used + event_rows(x) > n_rows:
            return events, used
        events.append((base, x, len(events) + 1))
        used += event_rows(x)


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def kernel_times(ctx, ev, n_rows, stream):
    """device microseconds per call of each kernel of the assignment, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    reps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.assign_exp_circuit(ev, n_rows, stream=stream)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "k_assign_exp" in e.key:
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            name = "chain" if "chain" in e.key else "rows"
            out[f"{name}_kernel_us"] = us / reps
    return out


def measure(ctx, name, exp_bits, n_rows, reps, warmup, mirror_events, seed):
    import torch

    events, used = workload(n_rows, exp_bits, seed)
    ev = assign.exp_events(events)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(warmup):
        ctx.assign_exp_circuit(ev, n_rows, stream=stream)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ctx.assign_exp_circuit(ev, n_rows, stream=stream)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    kt = kernel_times(ctx, ev, n_rows, stream)
    ctx.enable_timing(True)
    chk = []
    for _ in range(warmup + reps):
        ctx.check_async(native.CIRCUIT_EXP, 0, n_rows, 0, native.FLAG_WRAP)
        chk.append(ctx.last_timing()[1])
    ctx.enable_timing(False)
    ff, _ = ctx.fetch_result(native.CIRCUIT_EXP)
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_EXP)
    sub = events if mirror_events is None else events[:mirror_events]
    t = time.perf_counter()
    c = ExpCircuit()
    for base, x, ident in sub:
        c.add_event(base, x, ident)
    mirror_s = time.perf_counter() - t
    return {"workload": name, "rows": n_rows, "event_rows": used, "events": len(events),
            "assign_ms_median": statistics.median(ms), "assign_ms_min": min(ms), **kt,
            "check_exp_ms_median": statistics.median(chk[warmup:]),
            "h2d_bytes": ev.nbytes + 8 * (len(events) + 1), "h2d_event_bytes": ev.nbytes, "canonical_bytes": 672 * n_rows,
            "host_mirror_cpu_s": mirror_s, "host_mirror_cpu_rows": len(c.rows), "host_mirror_cpu_events": len(sub)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mirror-events", type=int, default=None, help="time the host mirror on the first N events only")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the device and has no CPU fallback")
    info = card()
    print(json.dumps(info), flush=True)
    ctx = native.Context(0)
    for name, bits, seed in (("exp256", 256, 1), ("exp64", 64, 2)):
        print(json.dumps({**measure(ctx, name, bits, args.rows, args.reps, args.warmup, args.mirror_events, seed), **info}),
              flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
