"""Cost of the captured graph recorder calls, on the GPU, with CUDA events:
  keyed     GraphRecorder.keyed of n (uint16 id, float64) pairs, k = 16 and 1024 local ids, n = 2^20 and 2^27, captured
            and replayed, against lh_ingest_keyed_f64_u16 of the same arrays outside a graph (its route included)
  counters  GraphRecorder.counters of n (uint16 id, uint64) pairs into kc = 16 and 1024 counters, captured and replayed,
            against lh_counter_add_u16 of the same arrays
  timer     replay time of a graph of 16 small torch kernels, with and without one start / stop pair around them
Everything runs on one stream; every variant is warmed up and the figure is the median of --reps.  Prints the card's
name, power limit and maximum SM clock first.

    python tools/graph_capture_probe.py [--reps 11] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(torch, stream, fn, reps):
    """median ms of fn() between two events on `stream` (current while fn runs), after two warm-up calls"""
    with torch.cuda.stream(stream):
        fn()
        fn()
        torch.cuda.synchronize()
        out = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            e1.synchronize()
            out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def capture(torch, fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        fn()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--json")
    a = ap.parse_args()
    import torch
    print("card:", card(), "| torch:", torch.cuda.get_device_name(0), flush=True)
    s = torch.cuda.Stream()
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(7)
    with lh.Engine(device=0, max_histograms=1024, max_counters=1024) as eng:
        for n_log in (20, 27):
            n = 1 << n_log
            vals = torch.exp(torch.randn(n, dtype=torch.float64, device="cuda", generator=gen) * 3)
            amounts = torch.randint(0, 1 << 20, (n,), dtype=torch.int64, device="cuda", generator=gen)
            for k in (16, 1024):
                ids = torch.randint(0, k, (n,), dtype=torch.int32, device="cuda", generator=gen).to(torch.int16).view(torch.uint16)
                with eng.graph_recorder(list(range(k)), list(range(k))) as gr:
                    gk = capture(torch, lambda: gr.keyed(ids, vals))
                    gc = capture(torch, lambda: gr.counters(ids, amounts))
                    t_gk = timed(torch, s, gk.replay, a.reps)
                    t_ek = timed(torch, s, lambda: eng.ingest_keyed_f64_u16(ids.data_ptr(), vals.data_ptr(), n, s.cuda_stream), a.reps)
                    route = eng.keyed_kernel_name()
                    t_gc = timed(torch, s, gc.replay, a.reps)
                    t_ec = timed(torch, s, lambda: eng.counter_add_u16(ids.data_ptr(), amounts.data_ptr(), n, s.cuda_stream), a.reps)
                    torch.cuda.synchronize()
                eng.snapshot([0.5])
                for what, tg, te, eager in (("keyed", t_gk, t_ek, "lh_ingest_keyed_f64_u16 (%s)" % route),
                                            ("counters", t_gc, t_ec, "lh_counter_add_u16")):
                    r = {"call": what, "k": k, "n": n, "captured_ms": tg, "eager_ms": te,
                         "captured_Gps": n / tg / 1e6, "eager_Gps": n / te / 1e6, "eager": eager}
                    rows.append(r)
                    print("%-8s k=%4d n=2^%d  captured %8.3f ms (%6.1f G/s)   %s %8.3f ms (%6.1f G/s)" % (
                        what, k, n_log, tg, r["captured_Gps"], eager, te, r["eager_Gps"]), flush=True)
            del vals, amounts, ids
            torch.cuda.empty_cache()
        x = torch.zeros(1 << 16, device="cuda")
        with eng.graph_recorder([0]) as gr:
            def body():
                for _ in range(16):
                    x.add_(1.0)
            g0 = capture(torch, body)

            def timed_body():
                gr.start_timer(0)
                body()
                gr.stop_timer(0)
            g1 = capture(torch, timed_body)
            t = {0: [], 1: []}
            for _ in range(5):                      # alternate the two graphs, 200 replays per round
                for which, g in ((0, g0), (1, g1)):
                    t[which].append(timed(torch, s, lambda: [g.replay() for _ in range(200)], 1) / 200 * 1e3)
            r = {"call": "timer", "replay_us": statistics.median(t[0]), "replay_with_span_us": statistics.median(t[1])}
            rows.append(r)
            print("timer    replay of 16 kernels %.2f us, with a start/stop pair %.2f us (+%.2f us)" % (
                r["replay_us"], r["replay_with_span_us"], r["replay_with_span_us"] - r["replay_us"]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
