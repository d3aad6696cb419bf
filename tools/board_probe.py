"""Cost of device subscriptions (lh_board_*, lh_snapshot_publish), on the GPU:
  publish   the k_board_publish launch of lh_snapshot_publish for 1, 64 and 1024 histogram rows at np = 3 and 32, CUDA
            events on the snapshot stream around --batch publishes of the same reduction (ms per publish)
  read      the k_board_read launch of lh_board_read for the same boards, events on a stream of its own
  row       lh::read_histogram from one thread of a kernel (tests/board_read_client.cu), %globaltimer over 10 000 reads
            of one row (ns per row read)
  collect   host time of collectRawMetrics + processMetrics (MetricSystem collect_and_process) on two systems with the
            same 1024 names, every name holding samples, one of them with a subscription of all 1024 names open; the
            two alternate, median of --reps each
Every variant is warmed up; kernel figures are the median of --reps.  Prints the card's name and power limit first.

    python tools/board_probe.py [--reps 9] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402
from loghisto_b200 import build  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def events_ms(torch, stream, fn, reps, batch):
    """median over reps of (ms between two events on `stream` around `batch` calls of fn) / batch, after a warm-up.
    The stream is held by a sleep kernel while the window is enqueued, so the window is back-to-back device time, not
    the host's issue rate."""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            torch.cuda._sleep(40_000_000)
        a.record(stream)
        for _ in range(batch):
            fn()
        b.record(stream)
        b.synchronize()
        out.append(a.elapsed_time(b) / batch)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    client = C.CDLL(build.BOARD_CLIENT_LIB)
    client.brc_read_cost.argtypes = [C.POINTER(lh._lib.lh_board), C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
    H = 1024
    with lh.Engine(device=0, max_histograms=H, max_counters=8) as eng:
        ids = (np.arange(2_000_000) % H).astype(np.uint16)
        eng.ingest_keyed_f64_u16_host(ids, np.random.default_rng(1).lognormal(3.0, 1.0, ids.size))
        eng.snapshot_begin()
        snap = torch.cuda.ExternalStream(eng.snapshot_device().stream)
        side = torch.cuda.Stream()
        for npct in (3, 32):
            eng.snapshot_reduce(np.linspace(0.01, 1.0, npct))
            for k in (1, 64, 1024):
                with eng.board(k, 0) as b:
                    hid = list(range(k))
                    pub = events_ms(torch, snap, lambda: b.publish(hid), a.reps, a.batch)
                    out = torch.empty(b.board.bytes, dtype=torch.uint8, device="cuda")
                    rd = events_ms(torch, side, lambda: b.read(out, stream=side), a.reps, a.batch)
                    res["publish_ms np=%d k=%d" % (npct, k)] = pub
                    res["read_ms np=%d k=%d" % (npct, k)] = rd
                    print("np %2d  rows %4d  publish %.4f ms  read %.4f ms" % (npct, k, pub, rd), flush=True)
                    if k == 1024 and npct == 32:
                        d = torch.zeros(2, dtype=torch.int64, device="cuda")
                        costs = []
                        for _ in range(a.reps):
                            assert client.brc_read_cost(C.byref(b.board), 513, 10_000, d.data_ptr(), side.cuda_stream) == 0
                            side.synchronize()
                            costs.append(int(d[0].item()) / 10_000)
                        res["read_histogram_ns_per_row"] = statistics.median(costs)
                        print("lh::read_histogram  %.1f ns per row (one thread)" % res["read_histogram_ns_per_row"], flush=True)
        eng.snapshot_end()

    from loghisto_b200.metric_system import MetricSystem
    systems = [MetricSystem(1.0, False, max_histograms=H, max_counters=8) for _ in range(2)]
    try:
        names = ["n%04d" % i for i in range(H)]
        vals = np.full(64, 3.0)   # one bucket per name: the Python side of collect_and_process stays small
        for ms in systems:
            ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p99": 0.99, "%s_max": 1.0})
        sub = systems[1].device_subscription(histograms=names)   # open for the whole run
        times = {0: [], 1: []}
        for rep in range(a.reps + 1):
            for subs in (0, 1):   # alternate: the same work on a system without and one with the subscription
                ms = systems[subs]
                for nm in names:
                    ms.HistogramMany(nm, vals)
                t0 = time.perf_counter()
                ms.collect_and_process()
                dt = (time.perf_counter() - t0) * 1e3
                if rep:   # the first round warms up
                    times[subs].append(dt)
        sub.close()
        for subs in (0, 1):
            res["collect_ms subs=%d" % subs] = statistics.median(times[subs])
            print("collect_and_process with %d subscription(s) of %d names: %.3f ms (median of %d)"
                  % (subs, H, res["collect_ms subs=%d" % subs], len(times[subs])), flush=True)
    finally:
        for ms in systems:
            ms.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
