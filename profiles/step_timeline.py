"""Kernel timeline of the replayed config-2 SVI step (`bench.py`'s `glm+graph` path, N = 1e6, D = 32, 64 particles).

torch.profiler with CUDA activities around a few graph replays, L2 flushed between steps as in `bench.py`.  For
every kernel of a step: its start and end relative to the step's first kernel, its duration and the idle gap
before it; then the median of each over the profiled steps.  Writes one JSON file and prints a table.

usage: python profiles/step_timeline.py [--steps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bench
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(1234)
    X, y = bench.make_data(dev)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    svi = bench.build_svi("glm+graph", bench.PARTICLES)
    for _ in range(10):
        svi.step_async(X, y)
    torch.cuda.synchronize(dev)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            flush.zero_()
            svi.step_async(X, y)
        torch.cuda.synchronize(dev)
    kern = sorted(((e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA and "Memset" not in e.name
                   and "Memcpy" not in e.name), key=lambda t: t[0])
    # a step = the kernels between two flushes (the flush is the one elementwise fill over 64 Mi floats)
    flush_idx = [i for i, k in enumerate(kern) if "fill" in k[2].lower() and k[1] - k[0] > 20]
    steps = []
    for i0, i1 in zip(flush_idx, flush_idx[1:] + [len(kern)]):
        ks = kern[i0 + 1:i1]
        if not ks:
            continue
        t0 = ks[0][0]
        rows, prev_end = [], None
        for s, e, n in ks:
            rows.append({"name": n[:90], "start_us": s - t0, "end_us": e - t0, "dur_us": e - s,
                         "gap_before_us": 0.0 if prev_end is None else s - prev_end})
            prev_end = e
        steps.append(rows)
    steps = steps[1:]      # the first one may straddle the profiler's start
    n_nodes = statistics.mode(len(r) for r in steps)
    steps = [r for r in steps if len(r) == n_nodes]
    med = []
    for j in range(n_nodes):
        col = [r[j] for r in steps]
        med.append({"name": col[0]["name"],
                    **{k: round(statistics.median(c[k] for c in col), 2)
                       for k in ("start_us", "end_us", "dur_us", "gap_before_us")}})
    span = statistics.median(r[-1]["end_us"] for r in steps)
    res = {"gpu": torch.cuda.get_device_name(dev), "steps": len(steps), "kernels_per_step": n_nodes,
           "span_us_median": round(span, 2), "nodes": med}
    try:
        import subprocess
        res["power_limit_and_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 -- diagnostic only
        res["power_limit_and_clock"] = repr(e)[:80]
    for r in med:
        print("%8.2f %8.2f %8.2f  gap %6.2f  %s" % (r["start_us"], r["end_us"], r["dur_us"], r["gap_before_us"],
                                                  r["name"][:70]))
    print("span %.2f us over %d steps, %d kernels per step" % (span, len(steps), n_nodes))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "step_timeline.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
