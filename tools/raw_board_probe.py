"""Cost of raw device subscriptions (lh_raw_board_*, lh_snapshot_publish_raw, lh_raw_percentiles / lh_raw_ranks), on
the GPU:
  publish   the k_raw_publish launch of lh_snapshot_publish_raw for 1, 64 and 1 024 rows, window-only rows (every
            count inside the fast window) and dense rows (one count outside it), at precision 100 and 250: CUDA events
            on the snapshot stream around --batch publishes of the same snapshot (ms per publish)
  query     lh_raw_percentiles and lh_raw_ranks over 2^20 (row, input) pairs spread over 64 rows, events on a stream of
            their own (ms per call and queries/s)
  one       lh::raw_percentile from one thread of a kernel (tests/raw_read_client.cu), %globaltimer over 10 000 queries
            of one row (ns per query)
  collect   host time of collectRawMetrics + processMetrics (MetricSystem collect_and_process) on two systems with the
            same 1 024 names, every name holding samples, one of them with a raw subscription of 64 names open; the two
            alternate, each going first in every other round, median of --reps each; then again with the subscription
            on the other system
Every variant is warmed up; kernel figures are the median of --reps.  Prints the card's name and power limit first.

    python tools/raw_board_probe.py [--reps 9] [--json out.json]
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
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    client = C.CDLL(build.RAW_CLIENT_LIB)
    client.rrc_cost.argtypes = [C.POINTER(lh._lib.lh_raw_board), C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
    H = 1024
    side = torch.cuda.Stream()
    for precision in (100, 250):
        with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng:
            ids = (np.arange(4_000_000) % H).astype(np.uint16)
            eng.ingest_keyed_f64_u16_host(ids, np.random.default_rng(1).lognormal(3.0, 1.0, ids.size))
            for form in ("window", "dense"):
                if form == "dense":   # one count at the most negative key: every row needs all 65 536 cells
                    eng.merge_counts_host(np.arange(H, dtype=np.uint32), np.full(H, -32768, np.int16),
                                          np.ones(H, np.uint64))
                eng.snapshot_begin()
                snap = torch.cuda.ExternalStream(eng.snapshot_device().stream)
                for k in (1, 64, 1024):
                    with eng.raw_board(k) as b:
                        hid = list(range(k))
                        ms = events_ms(torch, snap, lambda: b.publish(hid), a.reps, a.batch)
                        res["publish_ms p=%d %s k=%d" % (precision, form, k)] = ms
                        print("precision %3d  %-6s  rows %4d  publish %.4f ms" % (precision, form, k, ms), flush=True)
                        if precision == 100 and form == "window" and k == 64:
                            b.publish(hid)
                            torch.cuda.synchronize()
                            n = 1 << 20
                            rng = np.random.default_rng(2)
                            rows = torch.from_numpy(rng.integers(0, 64, n).astype(np.int32)).cuda()
                            ps = torch.from_numpy(rng.random(n)).cuda()
                            vs = torch.from_numpy(rng.lognormal(3.0, 1.0, n)).cuda()
                            for what, fn in (("percentiles", lambda: b.percentiles(ps, rows=rows, stream=side)),
                                             ("ranks", lambda: b.ranks(vs, rows=rows, stream=side))):
                                qms = events_ms(torch, side, fn, a.reps, a.batch)
                                res["%s_ms n=2^20 rows=64" % what] = qms
                                print("lh_raw_%s  2^20 queries over 64 rows: %.4f ms  (%.3g queries/s)"
                                      % (what, qms, n / (qms * 1e-3)), flush=True)
                            d = torch.zeros(2, dtype=torch.int64, device="cuda")
                            costs = []
                            for _ in range(a.reps):
                                assert client.rrc_cost(C.byref(b.board), 17, 10_000, d.data_ptr(), side.cuda_stream) == 0
                                side.synchronize()
                                costs.append(int(d[0].item()) / 10_000)
                            res["raw_percentile_ns"] = statistics.median(costs)
                            print("lh::raw_percentile  %.1f ns per query (one thread)" % res["raw_percentile_ns"], flush=True)
                eng.snapshot_end()

    from loghisto_b200.metric_system import MetricSystem
    systems = [MetricSystem(1.0, False, max_histograms=H, max_counters=8) for _ in range(2)]
    try:
        names = ["n%04d" % i for i in range(H)]
        vals = np.full(64, 3.0)
        for ms in systems:
            ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p99": 0.99, "%s_max": 1.0})
        for holder in (1, 0):   # the subscription on one system, then on the other: a control for the systems
            sub = systems[holder].raw_device_subscription(histograms=names[:64])
            times = {0: [], 1: []}
            for rep in range(a.reps + 1):
                for i in ((0, 1) if rep % 2 else (1, 0)):   # alternate which system goes first
                    ms = systems[i]
                    for nm in names:
                        ms.HistogramMany(nm, vals)
                    t0 = time.perf_counter()
                    ms.collect_and_process()
                    dt = (time.perf_counter() - t0) * 1e3
                    if rep:   # the first round warms up
                        times[i].append(dt)
            sub.close()
            for i in (0, 1):
                subs = int(i == holder)
                key = "collect_ms system=%d raw_subs=%d" % (i, subs)
                res[key] = statistics.median(times[i])
                print("collect_and_process of %d names on system %d with %d raw subscription(s) of 64 names: %.3f ms "
                      "(median of %d)" % (H, i, subs, res[key], len(times[i])), flush=True)
    finally:
        for ms in systems:
            ms.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
