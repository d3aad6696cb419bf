"""Times every K1 kernel variant (and the keyed / counter kernels) on device-resident synthetic streams.

Development tool: one JSON line per (variant, stream, grid multiple) is appended to --out.
Usage: python tools/k1_sweep.py [--n 1000000000] [--variants 0,5] [--streams U,L] [--iters 5] [--out file]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import loghisto_b200 as lh

KINDS = {"U": 0, "L": 1, "S": 2, "C": 3, "Z": 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000_000)
    ap.add_argument("--variants", default="all")
    ap.add_argument("--streams", default="U,L")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--grid-mults", default="1")
    ap.add_argument("--keyed", type=int, default=0, help="also time the keyed kernel with this many histograms")
    ap.add_argument("--out", default="k1_sweep.jsonl")
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    out = open(a.out, "a")
    H = max(a.keyed, 1)
    eng = lh.Engine(device=0, max_histograms=H, max_counters=1024)
    names = eng.k1_variants()
    variants = ([i for i, nm in enumerate(names) if not nm.startswith("probe")] if a.variants == "all"
                else [int(x) for x in a.variants.split(",")])
    d = eng.alloc(a.n, np.float64)
    for sname in a.streams.split(","):
        eng.gen_stream(KINDS[sname], a.n, lh.DEFAULT_SEED, out=d)
        eng.sync()
        ref_counts = None
        for gm in [int(x) for x in a.grid_mults.split(",")]:
            eng.tune("k1_grid_mult", gm)
            for vi in variants:
                eng.tune("k1", vi)
                times = []
                for it in range(a.iters + 2):
                    eng.ingest_f64(0, d, a.n)
                    ms = eng.last_kernel_ms()
                    if it >= 2:
                        times.append(ms)
                red, sp = eng.snapshot([0.5, 0.99])
                ok = int(red.counts[0]) == a.n * (a.iters + 2)
                h = (tuple(sp.keys.tolist()), tuple(sp.counts.tolist()))
                if ref_counts is None:
                    ref_counts = h
                same = h == ref_counts
                best, med = min(times), sorted(times)[len(times) // 2]
                rec = {"kernel": names[vi], "variant": vi, "stream": sname, "n": a.n, "grid_mult": gm,
                       "ms_best": best, "ms_median": med, "gsamples_s": a.n / med / 1e6,
                       "gb_s": a.n * 8 / med / 1e6, "count_ok": ok, "same_as_first": same}
                print(json.dumps(rec), flush=True)
                out.write(json.dumps(rec) + "\n")
        eng.tune("k1_grid_mult", 1)
    if a.keyed:
        nk = min(a.n, 500_000_000)
        for idkind in (0, 1):
            ids = eng.gen_ids_u16(idkind, nk, a.keyed, lh.DEFAULT_SEED)
            eng.gen_stream(KINDS["U"], nk, lh.DEFAULT_SEED, out=d)
            for mode, bps in ((1, 8), (2, 8), (2, 10), (2, 18), (2, 20)):
                eng.tune("keyed_mode", mode)
                eng.tune("keyed_blocks_per_sm", 8)
                if mode == 2:
                    eng.tune("kp_shape", 1 if bps >= 18 else 0)
                    eng.tune("kp_chunk", {8: 16 << 20, 10: 32 << 20, 18: 16 << 20, 20: 32 << 20}[bps])
                times = []
                for it in range(a.iters + 2):
                    eng.ingest_keyed_f64_u16(ids, d, nk)
                    ms = eng.last_kernel_ms()
                    if it >= 2:
                        times.append(ms)
                red, _ = eng.snapshot([0.5], export=False)
                med = sorted(times)[len(times) // 2]
                rec = {"kernel": "keyed_f64_u16", "ids": idkind, "H": a.keyed, "n": nk, "mode": mode,
                       "kp_chunk": {8: 16 << 20, 10: 32 << 20, 18: 16 << 20, 20: 32 << 20}[bps] if mode == 2 else None,
                       "kp_shape": (1 if bps >= 18 else 0) if mode == 2 else None,
                       "ms_median": med, "gsamples_s": nk / med / 1e6, "gb_s": nk * 10 / med / 1e6,
                       "count_ok": int(red.counts.sum()) == nk * (a.iters + 2)}
                print(json.dumps(rec), flush=True)
                out.write(json.dumps(rec) + "\n")
            ids.free()
    # counters: C = 1024 ids, random and single-id (worst-case contention)
    nc = min(a.n, 400_000_000)
    amounts = eng.alloc(nc, np.uint64)
    # amounts: reuse raw splitmix bits (kind 5 = raw u64)
    eng._check(eng.lib.lh_gen_stream_f64(eng.h, 5, lh.DEFAULT_SEED, 0, nc, amounts.ptr, 0))
    for idkind, nid in ((0, 1024), (0, 1)):
        ids = eng.gen_ids_u16(idkind, nc, nid, lh.DEFAULT_SEED)
        times = []
        for it in range(a.iters + 2):
            eng.counter_add_u16(ids, amounts, nc)
            ms = eng.last_kernel_ms()
            if it >= 2:
                times.append(ms)
        _, sp = eng.snapshot([0.5])
        med = sorted(times)[len(times) // 2]
        rec = {"kernel": "counter_add_u16", "n_ids": nid, "n": nc, "ms_median": med, "gops_s": nc / med / 1e6,
               "gb_s": nc * 10 / med / 1e6}
        print(json.dumps(rec), flush=True)
        out.write(json.dumps(rec) + "\n")
        ids.free()
    amounts.free()
    d.free()
    eng.close()


if __name__ == "__main__":
    main()
