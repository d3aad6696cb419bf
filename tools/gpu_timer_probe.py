"""What a GPU timer (MetricSystem.StartGpuTimer / Stop, lh_gpu_timer_*) costs and the shortest span it reports.

Prints one JSON line with the card and its power limit and three figures, all through the Python MetricSystem:
  floor        start then Stop with nothing between, durations written by the stop kernel (ns): a distribution, on an
               idle stream (each mark runs as soon as the host issues it) and on a busy one (the marks queue behind a
               spin and run back to back);
  added_us     stream time a start/stop pair adds around a fixed sequence of kernels (torch elementwise ops), from
               CUDA events on the stream, rounds with and without the timer alternating: median difference;
  host_us      host time of one StartGpuTimer + Stop pair (ctypes call overhead included), over a loop.
Needs build().

    python tools/gpu_timer_probe.py [--reps 2000] [--rounds 400]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--ops", type=int, default=8, help="kernels in the timed sequence")
    args = ap.parse_args()
    import torch
    from loghisto_b200 import build
    from loghisto_b200.metric_system import MetricSystem

    name, power = card()
    ms = MetricSystem(3600.0, False, max_histograms=16, max_counters=4)
    st = torch.cuda.Stream()

    # 1. empty-span floor
    out = torch.zeros(args.reps, dtype=torch.int64, device="cuda")
    for i in range(args.reps):
        ms.StartGpuTimer("floor", st).Stop(out=out[i:i + 1])
    torch.cuda.synchronize()
    floor = out.cpu().numpy()[args.reps // 10:]        # the first tenth warms up
    # ... and with the stream busy (a 200 us spin enqueued before each start), so that the two marks run back to back
    # on the device instead of each as soon as the host issues it
    build.build_device_client()
    spin = C.CDLL(build.TIMER_CLIENT_LIB)
    spin.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    for i in range(args.reps):
        assert spin.gtc_spin(200_000, st.cuda_stream) == 0
        ms.StartGpuTimer("floor_queued", st).Stop(out=out[i:i + 1])
    torch.cuda.synchronize()
    floor_q = out.cpu().numpy()[args.reps // 10:]

    # 2. stream time added around a fixed kernel sequence
    x = torch.ones(1 << 20, device="cuda")

    def seq():
        for _ in range(args.ops):
            x.mul_(1.0000001)
    with torch.cuda.stream(st):
        for _ in range(20):
            seq()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(2 * args.rounds)]
        for r in range(2 * args.rounds):
            a, b = ev[r]
            a.record(st)
            if r % 2:
                with ms.gpu_timer("seq", st):
                    seq()
            else:
                seq()
            b.record(st)
    torch.cuda.synchronize()
    ms_times = np.array([a.elapsed_time(b) for a, b in ev]) * 1e3   # us
    plain, timed = ms_times[0::2], ms_times[1::2]

    # 3. host time per StartGpuTimer + Stop
    n = args.reps
    t0 = time.perf_counter()
    for _ in range(n):
        ms.StartGpuTimer("host", st).Stop()
    host_us = (time.perf_counter() - t0) / n * 1e6
    torch.cuda.synchronize()
    ms.close()

    def dist(a):
        return {"n": int(a.size), "min": int(a.min()), "p50": float(np.percentile(a, 50)), "p90": float(np.percentile(a, 90)),
                "p99": float(np.percentile(a, 99)), "max": int(a.max())}
    print(json.dumps({
        "probe": "gpu_timer", "gpu": name, "power_limit": power,
        "floor_ns": dist(floor), "floor_queued_ns": dist(floor_q),
        "seq": {"ops": args.ops, "rounds": args.rounds, "plain_us_median": float(np.median(plain)),
                "timed_us_median": float(np.median(timed)), "added_us": float(np.median(timed) - np.median(plain))},
        "host_us_per_start_stop": host_us,
    }))


if __name__ == "__main__":
    main()
