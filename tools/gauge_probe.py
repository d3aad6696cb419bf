"""Cost of device gauges (lh_gauges_read, MetricSystem.RegisterDeviceGauge), on the GPU:
  read     host time of one lh_gauges_read of n = 1, 64, 1024 and 8192 float32 gauges (the call ends in a wait for its
           launches), median of --reps after a warm-up
  collect  host time of collectRawMetrics + processMetrics (MetricSystem collect_and_process) on two systems with the
           same 64 histogram names, one of them with 64 device gauges registered; the two alternate, median of --reps
Prints the card's name and power limit first.

    python tools/gauge_probe.py [--reps 51] [--json out.json]
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
from loghisto_b200 import _lib as L  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=51)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    g = torch.rand(8192, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with lh.Engine(device=0, max_histograms=1, max_counters=1) as eng:
        for n in (1, 64, 1024, 8192):
            srcs = (L.lh_gauge_src * n)(*[L.lh_gauge_src(g.data_ptr() + 4 * i, L.LH_GAUGE_F32, 0) for i in range(n)])
            out = np.zeros(n)
            times = []
            for rep in range(a.reps + 3):
                t0 = time.perf_counter()
                eng._check(eng.lib.lh_gauges_read(eng.h, srcs, n, out.ctypes.data))
                if rep >= 3:
                    times.append((time.perf_counter() - t0) * 1e6)
            assert (out == g[:n].double().cpu().numpy()).all()
            res["read_us n=%d" % n] = statistics.median(times)
            print("lh_gauges_read n=%5d: %8.1f us (median of %d; min %.1f, max %.1f)"
                  % (n, res["read_us n=%d" % n], len(times), min(times), max(times)), flush=True)

    from loghisto_b200.metric_system import MetricSystem
    systems = [MetricSystem(1.0, False, max_histograms=64, max_counters=8) for _ in range(2)]
    try:
        names = ["n%02d" % i for i in range(64)]
        vals = np.full(64, 3.0)
        for i in range(64):
            systems[1].RegisterDeviceGauge("g%02d" % i, g[i])
        times = {0: [], 64: []}
        for rep in range(a.reps + 1):
            for k, ms in ((0, systems[0]), (64, systems[1])):   # alternate: the same work without and with gauges
                for nm in names:
                    ms.HistogramMany(nm, vals)
                t0 = time.perf_counter()
                raw, _ = ms.collect_and_process()
                dt = (time.perf_counter() - t0) * 1e3
                assert len(raw["Gauges"]) == k
                if rep:   # the first round warms up
                    times[k].append(dt)
        for k in (0, 64):
            res["collect_ms gauges=%d" % k] = statistics.median(times[k])
            print("collect_and_process with %2d device gauges: %.3f ms (median of %d)"
                  % (k, res["collect_ms gauges=%d" % k], len(times[k])), flush=True)
    finally:
        for ms in systems:
            ms.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
