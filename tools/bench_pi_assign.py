"""Supplementary measurement (not the bench.py contract): the public-inputs circuit assigned on the device
(zk_assign_pi_circuit: public_data2witness from the raw public-input stream, with its keccak and calldata gas tables)
against the host mirror's Python loop, on seeded public data for two workloads:
  bench    bench.py --workload pi's shape: 48 txs in 64 slots, 2^18 calldata bytes, 16 withdrawals (292,998 rows)
  cd2_20   the same with 2^20 calldata bytes (1,079,430 rows; the host mirror is timed on the bench shape only)
Per workload one JSON line: the whole call (CUDA events around it, host validation and the pageable H2D copy included,
after warm-up; the call waits for the digest), each kernel's device time (torch.profiler, a run of its own) with the
single-thread sponge reported on its own, the k_check_pi time on the assigned narrow rows, the bytes that cross PCIe
(the stream + the staged calldata offsets) against the 896 B per row of the canonical upload, and the host mirror's
public_data2witness time, a CPU figure.  The card's name, power limit and maximum SM clock are read in the same run.
    python tools/bench_pi_assign.py [--reps 20] [--warmup 3] [--skip-mirror]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zkevm_specs_b200 import native, synth  # noqa: E402
from zkevm_specs_b200 import pi_circuit as pc  # noqa: E402


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def kernel_times(ctx, args, stream):
    """device microseconds per call of each kernel of the assignment, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    reps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.assign_pi_circuit(*args, stream=stream)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "k_assign_pi" in e.key:
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            name = e.key.split("(")[0].replace("void ", "").replace("zk::", "")
            out[name] = out.get(name, 0.0) + us / reps
    return {"kernel_us": out, "sponge_us": sum(v for k, v in out.items() if "sponge" in k),
            "other_kernels_us": sum(v for k, v in out.items() if "sponge" not in k)}


def measure(ctx, name, max_cd, reps, warmup, mirror):
    import torch

    mt, mw = 64, 16
    pd = synth.pi_public_data(48, max_cd, mw, seed=7)
    raw = pc.raw_public_inputs(pd, mt, max_cd, mw)
    n = len(raw)
    ctx.set_challenge(native.CHALLENGE_PI_KECCAK, pc.keccak_rand.n)
    ctx.set_challenge(native.CHALLENGE_PI_BYTE_BASE, pc.byte_pow_base.n)
    args = (mt, max_cd, mw, raw)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(warmup):
        ctx.assign_pi_circuit(*args, stream=stream)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ctx.assign_pi_circuit(*args, stream=stream)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    kt = kernel_times(ctx, args, stream)
    ctx.assign_pi_circuit(*args, stream=stream)
    ctx.enable_timing(True)
    chk = []
    for _ in range(warmup + reps):
        ctx.check_async(native.CIRCUIT_PI, 0, n, 0, native.FLAG_WRAP)
        chk.append(ctx.last_timing()[1])
    ctx.enable_timing(False)
    ff, _ = ctx.fetch_result(native.CIRCUIT_PI)
    assert (ff == native.PASS).all(), native.first_failure(ff, native.CIRCUIT_PI)
    out = {"workload": name, "rows": n, "max_txs": mt, "max_calldata_bytes": max_cd, "max_withdrawals": mw,
           "assign_ms_median": statistics.median(ms), "assign_ms_min": min(ms), **kt,
           "sponge_permutations": n // 136 + 1, "check_pi_ms_median": statistics.median(chk[warmup:]),
           "h2d_bytes": n + 8 * (mt + 1), "canonical_bytes": 896 * n}
    if mirror:
        t = time.perf_counter()
        w = pc.public_data2witness(pd, mt, max_cd, mw)
        out["host_mirror_cpu_s"] = time.perf_counter() - t
        assert w.circuit_len == n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-mirror", action="store_true", help="do not time the host mirror")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the device and has no CPU fallback")
    info = card()
    print(json.dumps(info), flush=True)
    ctx = native.Context(0)
    for name, max_cd in (("bench", 1 << 18), ("cd2_20", 1 << 20)):
        mirror = not args.skip_mirror and name == "bench"  # the mirror takes minutes at 2^20
        print(json.dumps({**measure(ctx, name, max_cd, args.reps, args.warmup, mirror), **info}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
