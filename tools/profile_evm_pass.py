"""Per-kernel listing of the bench's main EVM pass (2^20 cfg2 steps, adaptive packed storage) with torch.profiler.

    python tools/profile_evm_pass.py --out DIR [--passes 20] [--groups 262144]

Runs the same upload and hot path as `bench.py` (invalidate every index, then one EVM check), back to back on one
stream, under torch.profiler with CUDA activities.  A one-element torch kernel between passes marks the pass
boundaries; it is left out of the listing.  Writes DIR/evm_pass_kernels.txt:
  - every device operation of one pass in the middle of the run: start (us from the pass's first operation),
    duration, gap from the latest end of the operations before it (negative: it overlaps them, as the hot kernels
    on their own streams do);
  - per operation name: count per pass and mean duration over all profiled passes;
  - index phase (everything before k_evm_sort), check phase (the rest), the step sort (k_evm_sort's duration and
    the gap from its start to the first hot kernel's start), hot phase (first start to last end of k_evm_push_* and
    k_evm_gadget) and the pass span.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--passes", type=int, default=20)
    ap.add_argument("--groups", type=int, default=1 << 18)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from zkevm_specs_b200 import native, packing, synth
    from zkevm_specs_b200.evm_circuit.table import fixed_table_matrix

    torch.cuda.set_device(0)
    ctx = native.Context(0)
    stream = torch.cuda.current_stream().cuda_stream
    w = synth.evm_trace(args.groups, seed=2)
    n = w["n_steps"]
    ctx.upload_table(native.TABLE_FIXED, fixed_table_matrix(), stream=stream)
    ctx.upload_bytecode_table_from_code(**w["bytecode_src"], stream=stream)
    ctx.upload_table_packed(native.TABLE_RW, packing.pack_matrix(w["rw"]), stream=stream)
    ctx.upload_columns_packed(native.CIRCUIT_EVM, packing.pack_matrix(w["steps"]), stream=stream)
    marker = torch.zeros(1, device="cuda")

    def hot_path():
        ctx.invalidate_indexes()
        ctx.check_async(native.CIRCUIT_EVM, 0, n, 0, 0, stream)

    for _ in range(5):
        hot_path()
    ff, _ = ctx.fetch_result(native.CIRCUIT_EVM, stream)
    assert (ff == native.PASS).all()
    torch.cuda.synchronize()
    l0 = ctx.launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.passes):
            marker.add_(1)
            hot_path()
        marker.add_(1)
        torch.cuda.synchronize()
    launches = (ctx.launch_count() - l0) / args.passes
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "evm_pass.pt.trace.json")
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))["traceEvents"]
    os.remove(trace)
    ops = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")),
                 key=lambda e: e["ts"])
    passes, cur = [], None
    for e in ops:
        name = e["name"]
        if "at::native" in name:  # the marker
            if cur:
                passes.append(cur)
            cur = []
            continue
        if cur is not None:
            short = name.split("(")[0].replace("void ", "").replace("zk::", "")
            cur.append((short, float(e["ts"]), float(e["dur"])))
    passes = [p for p in passes if p]

    lines = [f"{args.passes} passes of {n} steps; library launches per pass {launches:.1f}", ""]
    mid = passes[len(passes) // 2]
    t0, prev_end = mid[0][1], mid[0][1]
    lines.append(f"{'start_us':>9} {'dur_us':>8} {'gap_us':>7}  op (gap < 0: overlap)")
    for name, ts, dur in mid:
        lines.append(f"{ts - t0:9.1f} {dur:8.1f} {ts - prev_end:7.1f}  {name}")
        prev_end = max(prev_end, ts + dur)
    stats = {}
    idx_ms, chk_ms, hot_ms, span_ms, sort_us, to_hot_us = [], [], [], [], [], []
    is_hot = lambda name: name.startswith(("k_evm_push", "k_evm_gadget"))  # noqa: E731
    for p in passes:
        seen = {}
        for name, ts, dur in p:
            s = stats.setdefault(name, [0, 0.0])
            s[0] += 1
            s[1] += dur
            seen[name] = 1
        start = p[0][1]
        end = max(ts + d for _, ts, d in p)
        srt = next(((ts, d) for name, ts, d in p if name.startswith("k_evm_sort")), (end, 0.0))
        idx_ms.append((srt[0] - start) / 1e3)
        chk_ms.append((end - srt[0]) / 1e3)
        hot = [(ts, ts + d) for name, ts, d in p if is_hot(name)]
        if hot:
            hot_ms.append((max(e for _, e in hot) - min(s for s, _ in hot)) / 1e3)
            sort_us.append(srt[1])
            to_hot_us.append(min(s for s, _ in hot) - srt[0])
        span_ms.append((end - start) / 1e3)
    lines += ["", f"{'per_pass':>8} {'mean_us':>8}  op"]
    for name, (c, tot) in sorted(stats.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"{c / len(passes):8.2f} {tot / c:8.1f}  {name}")
    mean = lambda xs: sum(xs) / len(xs)  # noqa: E731
    lines += ["", f"index phase (first op -> k_evm_sort start): {mean(idx_ms):.4f} ms",
              f"check phase (k_evm_sort start -> last op end): {mean(chk_ms):.4f} ms",
              f"step sort: k_evm_sort {mean(sort_us) if sort_us else 0:.1f} us, its start -> first hot kernel start "
              f"{mean(to_hot_us) if to_hot_us else 0:.1f} us",
              f"hot phase (first hot kernel start -> last hot kernel end): {mean(hot_ms) if hot_ms else 0:.4f} ms",
              f"pass span: {mean(span_ms):.4f} ms over {len(passes)} passes"]
    with open(os.path.join(args.out, "evm_pass_kernels.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
