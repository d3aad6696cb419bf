"""Cost of distribution gauges (lh_snapshot_ingest_arrays, MetricSystem.RegisterDeviceDistribution), on the GPU:
  kernel   time of k_ingest_arrays on the snapshot stream (torch.profiler CUDA activity, summed over one call's
           launches), for 1 / 64 / 1 024 arrays of 1 Ki / 64 Ki / 1 Mi elements in float32, bfloat16 and float64; mean
           over --reps snapshots, and the bytes read over that time as GB/s and as a share of the H100 SXM data sheet's
           3.35 TB/s of HBM3 bandwidth (the kernel is bound by its shared-memory counting, not by those bytes)
  collect  host time of collectRawMetrics + processMetrics (MetricSystem collect_and_process) on two systems with the
           same 64 histogram names, one of them with 64 distributions of 4 096 float32 elements registered; the two
           alternate, median of --reps
Prints the card's name and power limit first.

    python tools/device_distribution_probe.py [--reps 21] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def kernel_us(torch, eng, arrays, reps):
    """Mean over reps snapshots of the summed k_ingest_arrays time of one lh_snapshot_ingest_arrays call, and the
    launches of one call."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        eng.snapshot(np.zeros(0), export=False, arrays=arrays)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.snapshot(np.zeros(0), export=False, arrays=arrays)
        torch.cuda.synchronize()
    rows = [r for r in prof.key_averages() if "k_ingest_arrays" in r.key]
    total = sum(getattr(r, "device_time_total", None) or getattr(r, "cuda_time_total", 0.0) for r in rows)
    count = sum(r.count for r in rows)
    assert count and count % reps == 0, (count, reps)
    return total / reps, count // reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    with lh.Engine(device=0, max_histograms=1024, max_counters=1) as eng:
        for dt, name in ((torch.float32, "f32"), (torch.bfloat16, "bf16"), (torch.float64, "f64")):
            for n_arrays in (1, 64, 1024):
                for n in (1 << 10, 1 << 16, 1 << 20):
                    if n_arrays * n > (1 << 28):
                        continue
                    x = (torch.rand(n_arrays * n, device="cuda:0", dtype=torch.float64) * 1e6).to(dt)
                    arrays = [(i, x[i * n:(i + 1) * n]) for i in range(n_arrays)]
                    us, launches = kernel_us(torch, eng, arrays, a.reps)
                    gbs = x.numel() * x.element_size() / (us * 1e-6) / 1e9
                    key = "kernel %s %dx%d" % (name, n_arrays, n)
                    res[key] = {"us": us, "GB/s": gbs, "of_hbm": gbs * 1e9 / HBM_BYTES_PER_S, "launches": launches,
                                "Gsamples/s": x.numel() / (us * 1e-6) / 1e9}
                    print("%-26s %10.1f us  %7.1f GB/s (%4.1f %% of 3.35 TB/s)  %6.2f G samples/s  %d launch(es)"
                          % (key, us, gbs, 100 * res[key]["of_hbm"], res[key]["Gsamples/s"], launches), flush=True)
                    del x

    from loghisto_b200.metric_system import MetricSystem
    systems = [MetricSystem(1.0, False, max_histograms=160, max_counters=8) for _ in range(2)]
    try:
        names = ["n%02d" % i for i in range(64)]
        vals = np.full(64, 3.0)
        dists = torch.rand(64, 4096, device="cuda:0", dtype=torch.float32)
        for i in range(64):
            systems[1].RegisterDeviceDistribution("d%02d" % i, dists[i])
        times = [[], []]
        for rep in range(a.reps + 3):
            for k, ms in enumerate(systems):
                for nm in names:
                    ms.HistogramMany(nm, vals)
                t0 = time.perf_counter()
                ms.collect_and_process()
                if rep >= 3:
                    times[k].append((time.perf_counter() - t0) * 1e3)
        for k, label in enumerate(("without distributions", "with 64 distributions of 4096")):
            res["collect_ms " + label] = statistics.median(times[k])
            print("collect_and_process %-32s %8.3f ms (median of %d; min %.3f, max %.3f)"
                  % (label, res["collect_ms " + label], len(times[k]), min(times[k]), max(times[k])), flush=True)
    finally:
        for ms in systems:
            ms.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
