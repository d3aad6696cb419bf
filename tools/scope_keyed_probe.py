"""Cost of the mapped (record-scope) keyed and counter calls, on the GPU, with CUDA events, against the raw calls on
the same arrays (the map is the identity, so both record the same thing):
  keyed     lh_ingest_keyed_mapped_u16 (float64) against lh_ingest_keyed_f64_u16: k = 1024 at n = 2^27 and 2^30 on
            streams U and L; k = 8 and 32 at n = 2^27, where the mapped call plans on k ids and the raw one on 1024
  counters  lh_counter_add_mapped_u16 against lh_counter_add_u16, kc = 16 and 1024, n = 2^27
Every pair is warmed up, then timed in --rounds rounds that alternate which call goes first; the figure is the median.
The map is built once, outside the timed window, and the ABI is called directly, as RecordScope does with its ids.
Each row names the kernel each call ran.  Prints the card's name, power limit and maximum SM clock first.

    python tools/scope_keyed_probe.py [--rounds 9] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def alternate(torch, s, fns, rounds):
    """median ms of each fn between two events on stream s, the fns alternating round by round, after a warm-up"""
    for f in fns:
        f()
    torch.cuda.synchronize()
    out = [[] for _ in fns]
    for rd in range(rounds):
        order = list(enumerate(fns))
        for i, f in (order if rd % 2 == 0 else order[::-1]):       # the first call of a round alternates too
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            f()
            e1.record(s)
            e1.synchronize()
            out[i].append(e0.elapsed_time(e1))
    return [statistics.median(x) for x in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--json")
    a = ap.parse_args()
    import torch
    print("card:", card(), "| torch:", torch.cuda.get_device_name(0), flush=True)
    s = torch.cuda.Stream()
    sp = s.cuda_stream
    rows = []
    keyed_cases = [(1024, 27, lh.STREAM_U), (1024, 27, lh.STREAM_L), (1024, 30, lh.STREAM_U), (1024, 30, lh.STREAM_L),
                   (8, 27, lh.STREAM_U), (32, 27, lh.STREAM_U)]
    with lh.Engine(device=0, max_histograms=1024, max_counters=1024) as eng:
        for k, n_log, kind in keyed_cases:
            n = 1 << n_log
            vals = eng.gen_stream(kind, n, lh.DEFAULT_SEED)
            ids = eng.gen_ids_u16(0, n, k, lh.DEFAULT_SEED)
            m = (C.c_uint32 * k)(*range(k))
            names = {}

            def mapped():
                eng._check(eng.lib.lh_ingest_keyed_mapped_u16(eng.h, m, k, ids.ptr, vals.ptr, 0, n, sp))
                names["mapped"] = eng.keyed_kernel_name()

            def raw():
                eng.ingest_keyed_f64_u16(ids.ptr, vals.ptr, n, sp)
                names["raw"] = eng.keyed_kernel_name()
            tm, tr = alternate(torch, s, [mapped, raw], a.rounds)
            eng.snapshot([0.5])
            r = {"call": "keyed", "k": k, "n": n, "stream": "U" if kind == lh.STREAM_U else "L", "mapped_ms": tm,
                 "raw_ms": tr, "raw_over_mapped": tr / tm, "mapped_kernel": names["mapped"], "raw_kernel": names["raw"]}
            rows.append(r)
            print("keyed    k=%4d n=2^%d %s  mapped %8.3f ms (%s)  raw %8.3f ms (%s)  raw/mapped %.3f" % (
                k, n_log, r["stream"], tm, names["mapped"], tr, names["raw"], tr / tm), flush=True)
            del vals, ids
        n = 1 << 27
        amounts = eng.gen_stream(lh.STREAM_AMOUNTS, n, lh.DEFAULT_SEED)
        for kc in (16, 1024):
            ids = eng.gen_ids_u16(0, n, kc, lh.DEFAULT_SEED)
            m = (C.c_uint32 * kc)(*range(kc))
            tm, tr = alternate(torch, s, [lambda: eng._check(eng.lib.lh_counter_add_mapped_u16(eng.h, m, kc, ids.ptr, amounts.ptr, n, sp)),
                                          lambda: eng.counter_add_u16(ids.ptr, amounts.ptr, n, sp)], a.rounds)
            eng.snapshot([0.5])
            r = {"call": "counters", "k": kc, "n": n, "mapped_ms": tm, "raw_ms": tr, "raw_over_mapped": tr / tm}
            rows.append(r)
            print("counters k=%4d n=2^27    mapped %8.3f ms  raw %8.3f ms  raw/mapped %.3f" % (kc, tm, tr, tr / tm), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
