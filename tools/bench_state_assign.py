"""Supplementary measurement (not the bench.py contract): the state circuit assigned on the device with its roots and MPT
table computed there (zk_assign_state_circuit_mpt, 13 cells per operation) against op2row on the device with roots and
the MPT table computed on the host (zk_assign_state_circuit, 15 cells per operation, + zk_upload_table of the MPT
table).  Three workloads:
  synth18   synth.state_rows(2^18), the bench.py state shape
  synth21   synth.state_rows(2^21)
  unsorted  2^20 unsorted operations over 2^16 keys, each Storage key touched under several tx ids
Per workload one JSON line: the time of each path (CUDA events around the call, the H2D copies and host preparation
included, after warm-up, the two paths alternated), the k_check_state time after each, the bytes each path sends over
PCIe, and the number of MPT updates.  Both paths must give equal rows, equal MPT tables and equal check verdicts
(asserted; the unsorted list fails the circuit's ordering constraints by design).  The card's name, power limit and
maximum SM clock are read in the same run and printed with the results.
    python tools/bench_state_assign.py [--reps 10] [--warmup 3]"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zkevm_specs_b200 import assign, native, packing, synth  # noqa: E402


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def unsorted_workload(n: int, n_keys: int, seed: int):
    """(ops13, flags, roots, mpt): n unsorted ops, a quarter Memory, the rest Storage / Account over n_keys keys, with
    the roots and the MPT table computed on the host (first touches by np.unique, next MPT op by searchsorted)"""
    rng = np.random.default_rng(seed)
    key = rng.integers(0, n_keys, n)
    acc = key % 5 == 0
    tag = np.where(acc, 6, 4)
    tag[rng.random(n) < 0.25] = 2
    ops = np.zeros((13, n, 4), dtype=np.uint64)
    ops[0, :, 0] = np.arange(n)
    ops[1, :, 0] = rng.integers(0, 2, n)
    ops[2, :, 0] = tag
    ops[3, :, 0] = rng.integers(1, 9, n)
    ops[4, :, 0] = 0x1000 + key // 8
    ops[5, :, 0] = np.where(acc, 1 + key % 4, 0)
    ops[6, :, 0] = np.where(acc, 0, key * 0x9E3779B9)
    ops[7, :, 0] = np.where(acc, 0, key % 3)
    ops[8, :, 0] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    ops[10, :, 0] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    ops[12, :, 0] = 1
    flags = np.zeros(n, dtype=np.uint8)
    pos = np.nonzero((tag == 4) | (tag == 6))[0]
    keys = np.stack([ops[c, pos, 0] for c in (4, 5, 6, 7)], axis=1)
    _, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)
    rank = np.empty(len(order), dtype=np.int64)
    rank[order] = np.arange(len(order))
    j = np.searchsorted(pos, np.arange(n), side="right")
    roots = np.full(n, 3 + 5 * len(order), dtype=np.uint64)
    roots[j < len(pos)] = 3 + 5 * rank[inv.reshape(-1)][j[j < len(pos)]]
    src = pos[first[order]]
    U = len(order)
    mpt = np.zeros((12, U, 4), dtype=np.uint64)
    mpt[0, :, 0], mpt[2, :, 0], mpt[3, :, 0] = ops[4, src, 0], ops[6, src, 0], ops[7, src, 0]
    mpt[1, :, 0] = np.where(tag[src] == 4, 6, ops[5, src, 0])
    mpt[4, :, 0] = 3 + 5 * (np.arange(U) + 1)
    mpt[6, :, 0] = 3 + 5 * np.arange(U)
    mpt[8, :, 0], mpt[10, :, 0] = ops[8, src, 0], ops[10, src, 0]
    return ops, flags, roots, mpt


def ops15_of(ops13, roots):
    """the 15 cells of zk_assign_state_circuit: the 13 with root lo, hi inserted before the selector"""
    r = np.zeros((2, ops13.shape[1], 4), dtype=np.uint64)
    r[0, :, 0] = roots
    return np.concatenate([ops13[:12], r, ops13[12:]], axis=0)


def digest(ctx):
    rows, fl = ctx.download_columns(native.CIRCUIT_STATE)
    h = hashlib.sha256(rows.tobytes()).hexdigest() + hashlib.sha256(fl.tobytes()).hexdigest()
    del rows
    t = ctx.download_table(native.TABLE_MPT)
    return h, sorted(tuple(int(x) for x in t[:, r, :].reshape(-1)) for r in range(t.shape[1]))


def timed(fn):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def check_ms(ctx, n, reps):
    ctx.enable_timing(True)
    out = []
    for _ in range(reps):
        ctx.check_async(native.CIRCUIT_STATE, 0, n, 0, native.FLAG_WRAP)
        out.append(ctx.last_timing()[1])
    ctx.enable_timing(False)
    ff, fc = ctx.fetch_result(native.CIRCUIT_STATE)
    return statistics.median(out[1:]), (ff.tolist(), fc.tolist())


def measure(ctx, name, ops13, flags, roots, mpt, reps, warmup):
    import torch

    n = ops13.shape[1]
    stream = torch.cuda.current_stream().cuda_stream
    pm13 = packing.pack_matrix(ops13)
    pm15 = packing.pack_matrix(ops15_of(ops13, roots))
    pmt = packing.pack_matrix(mpt)

    def host_roots():
        ctx.assign_state_circuit(pm15, flags=flags, stream=stream)
        ctx.upload_table_packed(native.TABLE_MPT, pmt, stream=stream)

    def device_roots():
        assign.assign_state_circuit_mpt(ctx, pm13, flags, stream=stream)

    host_roots()
    torch.cuda.synchronize()
    want = digest(ctx)
    chk_host, verdict = check_ms(ctx, n, reps + 1)
    device_roots()
    assert digest(ctx) == want, name
    chk_dev, verdict_dev = check_ms(ctx, n, reps + 1)
    assert verdict_dev == verdict, name
    for _ in range(warmup):
        host_roots()
        device_roots()
    t_host, t_dev = [], []
    for _ in range(reps):
        t_host.append(timed(host_roots))
        t_dev.append(timed(device_roots))
    return {"workload": name, "ops": n, "mpt_updates": mpt.shape[1],
            "host_roots_assign_ms_median": statistics.median(t_host), "host_roots_assign_ms_min": min(t_host),
            "device_roots_assign_ms_median": statistics.median(t_dev), "device_roots_assign_ms_min": min(t_dev),
            "check_state_ms_after_host_roots": chk_host, "check_state_ms_after_device_roots": chk_dev,
            "check_passes": all(f == native.PASS for f in verdict[0]),
            "h2d_bytes_host_roots": pm15.nbytes + n + pmt.nbytes, "h2d_bytes_device_roots": pm13.nbytes + 2 * n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the device and has no CPU fallback")
    info = card()
    print(json.dumps(info), flush=True)
    ctx = native.Context(0)
    for name, n in (("synth18", 1 << 18), ("synth21", 1 << 21)):
        w = synth.state_rows(n)
        ops13 = assign.state_op13_from_rows(w["rows"])
        roots = w["rows"][54, :, 0].copy()
        del w["rows"]
        print(json.dumps({**measure(ctx, name, ops13, w["flags"], roots, w["mpt"], args.reps, args.warmup), **info}), flush=True)
    ops13, flags, roots, mpt = unsorted_workload(1 << 20, 1 << 16, seed=9)
    print(json.dumps({**measure(ctx, "unsorted", ops13, flags, roots, mpt, args.reps, args.warmup), **info}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
