"""Cost of window raw device subscriptions (lh_raw_board_create_window, MetricSystem raw_device_subscription(window=)),
on the GPU:
  collect   host time of collectRawMetrics + processMetrics (MetricSystem collect_and_process) on four systems with the
            same names, every name holding samples: no raw subscription, a plain one (window 1), and windows of 2 and
            60 collections, each subscription over k = 1, 64 and 1 024 of the names.  The systems alternate, the order
            rotating every round; median of --reps after a warm-up round
  publish   device time of one publish (k_raw_publish vs k_raw_publish_window) of k = 1, 64 and 1 024 window-only rows
            (one count at each edge of the fast window, merged before every snapshot) at precision 100 in steady state, one publish per snapshot, CUDA events on the snapshot stream held by a sleep kernel while
            the publish is enqueued; median of --reps.  With the bytes each form moves over the live key range (plain:
            read the interval, write the running counts; window: also read the outgoing slot and the sum, write both,
            read the sum again) as GB/s
  memory    device memory per row of each board, from the layout and from cudaMemGetInfo around its creation
Prints the card's name and power limit first.

    python tools/raw_window_probe.py [--reps 9] [--json out.json]
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

WINDOWS = (1, 2, 60)
ROWS = (1, 64, 1024)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def layout_bytes_per_row(window):
    """Device memory of one row: header, running counts and id table; a window board adds its sum row, slot counts,
    slot levels and slots (include/loghisto_b200.h)."""
    plain = 32 + 65536 * 8 + 4
    return plain if window == 1 else plain + (window + 1) * 65536 * 8 + 8 + window


def publish_ms(torch, eng, board, hid, reps, win):
    """Median device time of one publish, each in a snapshot of its own, after window + 1 untimed ones (so that every
    slot holds an interval and the timed publishes read the outgoing one, as in steady state)."""
    out = []
    warm = board.window + 1
    k = board.k
    rows = np.repeat(np.arange(k, dtype=np.uint32), 2)
    edges = np.tile(np.array([-(win - 1), win - 1], np.int16), k)   # every row's live range: the whole fast window
    for rep in range(warm + reps):
        eng.merge_counts_host(rows, edges, np.ones(2 * k, np.uint64))
        eng.snapshot_begin()
        snap = torch.cuda.ExternalStream(eng.snapshot_device().stream)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(snap):
            torch.cuda._sleep(20_000_000)
        a.record(snap)
        board.publish(hid)
        b.record(snap)
        b.synchronize()
        eng.snapshot_end()
        if rep >= warm:
            out.append(a.elapsed_time(b))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)

    # memory and device time per publish
    H = max(ROWS)
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=100) as eng:
        win = int(100 * np.log(2.0 ** 63) + 0.5) + 1    # the fast window at precision 100: 4 368 keys each side
        n = 2 * win - 1
        for k in ROWS:
            hid = list(range(k))
            base = None
            for w in WINDOWS:
                torch.cuda.synchronize()
                free0 = torch.cuda.mem_get_info()[0]
                with eng.raw_board(k, window=w) as b:
                    torch.cuda.synchronize()
                    used = free0 - torch.cuda.mem_get_info()[0]
                    res["bytes_per_row layout w=%d" % w] = layout_bytes_per_row(w)
                    res["bytes_per_row measured k=%d w=%d" % (k, w)] = used / k
                    ms = publish_ms(torch, eng, b, hid, a.reps, win)
                    moved = k * n * 8 * (2 if w == 1 else 7)
                    res["publish_ms k=%d w=%d" % (k, w)] = ms
                    base = ms if w == 1 else base
                    print("rows %4d  window %2d  publish %.4f ms (%.2fx plain, %.1f GB/s over %d live keys per row)  "
                          "memory per row %.1f MiB (layout %.1f MiB)"
                          % (k, w, ms, ms / base, moved / (ms * 1e-3) / 1e9, n, used / k / 2 ** 20,
                             layout_bytes_per_row(w) / 2 ** 20), flush=True)

    # host time of collect_and_process
    from loghisto_b200.metric_system import MetricSystem
    names = ["n%04d" % i for i in range(H)]
    vals = np.full(64, 3.0)
    for k in ROWS:
        systems = [MetricSystem(1.0, False, max_histograms=H, max_counters=8) for _ in range(len(WINDOWS) + 1)]
        subs = []
        try:
            for ms in systems:
                ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p99": 0.99})
            subs = [systems[i + 1].raw_device_subscription(histograms=names[:k], window=w) for i, w in enumerate(WINDOWS)]
            times = [[] for _ in systems]
            for rep in range(a.reps + 1):
                order = list(range(len(systems)))
                order = order[rep % len(order):] + order[:rep % len(order)]
                for i in order:
                    ms = systems[i]
                    for nm in names:
                        ms.HistogramMany(nm, vals)
                    t0 = time.perf_counter()
                    ms.collect_and_process()
                    dt = (time.perf_counter() - t0) * 1e3
                    if rep:
                        times[i].append(dt)
            for i, t in enumerate(times):
                what = "none" if i == 0 else "window=%d" % WINDOWS[i - 1]
                res["collect_ms k=%d %s" % (k, what)] = statistics.median(t)
                print("collect_and_process of %d names, raw subscription of %4d names: %-9s %.3f ms (median of %d)"
                      % (H, k, what, statistics.median(t), len(t)), flush=True)
        finally:
            for s in subs:
                s.close()
            for ms in systems:
                ms.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
