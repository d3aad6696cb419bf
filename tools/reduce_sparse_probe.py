"""Cost of lh_reduce_sparse_host at the size of a cross-host aggregation: 16 hosts' exports of 1024 histograms
(stream U, precision 100), concatenated per name, reduced with 8 percentiles.

Prints one JSON line: the card and its power limit, the input (segments, entries, bytes), the whole call's wall time
(host clock around the synchronous call: H2D of the input, kernels, D2H of the results, host copies), the device time
of its kernels (k_scatter_segments + k_reduce + k_sparse_epilogue + k_clear_touched, summed from torch.profiler's
CUDA kernel records of one call), and entries per second for both.

    python tools/reduce_sparse_probe.py [--hosts 16] [--histograms 1024] [--samples 4194304] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import loghisto_b200 as lh  # noqa: E402

PS = [0.0, 0.5, 0.75, 0.9, 0.99, 0.999, 0.9999, 1.0]
KERNELS = ("k_scatter_segments", "k_reduce", "k_sparse_epilogue", "k_clear_touched")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hosts", type=int, default=16)
    ap.add_argument("--histograms", type=int, default=1024)
    ap.add_argument("--samples", type=int, default=1 << 22, help="samples per host export")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    H = a.histograms
    sps = []
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        for e in range(a.hosts):
            d_v = eng.gen_stream(lh.STREAM_U, a.samples, lh.DEFAULT_SEED + 17 * e)
            d_i = eng.gen_ids_u16(0, a.samples, H, lh.DEFAULT_SEED + 17 * e)
            eng.ingest_keyed_f64_u16(d_i, d_v, a.samples)
            sps.append(eng.snapshot([], export=True)[1])
    sizes, keys, counts = [], [], []          # segment h: histogram h of every export, one after the other
    for h in range(H):
        for sp in sps:
            x, y = int(sp.offsets[h]), int(sp.offsets[h + 1])
            keys.append(sp.keys[x:y])
            counts.append(sp.counts[x:y])
        sizes.append(sum(int(sp.offsets[h + 1]) - int(sp.offsets[h]) for sp in sps))
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    keys, counts = np.concatenate(keys), np.concatenate(counts)
    entries = int(offsets[-1])

    with lh.Engine(device=0, max_histograms=1, max_counters=1) as eng:
        eng.reduce_sparse(offsets, keys, counts, PS)            # warm-up: scratch allocation, module load
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            red = eng.reduce_sparse(offsets, keys, counts, PS)
            walls.append(time.perf_counter() - t0)
        assert int(red.counts.sum()) == a.hosts * a.samples
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.reduce_sparse(offsets, keys, counts, PS)
            torch.cuda.synchronize()
        dev_us = {k: 0.0 for k in KERNELS}
        for ev in prof.key_averages():
            for k in KERNELS:
                if k + "(" in ev.key or ev.key.endswith(k):
                    dev_us[k] += ev.device_time_total
    name, power = card()
    wall = float(np.median(walls))
    dev_ms = sum(dev_us.values()) / 1e3
    print(json.dumps({
        "probe": "reduce_sparse", "gpu": name, "power_limit": power,
        "segments": H, "hosts": a.hosts, "entries": entries, "input_bytes": int(offsets.nbytes + keys.nbytes + counts.nbytes),
        "wall_ms_median": round(wall * 1e3, 3), "wall_ms_all": [round(w * 1e3, 3) for w in walls],
        "device_ms": round(dev_ms, 3), "device_ms_by_kernel": {k: round(v / 1e3, 3) for k, v in dev_us.items()},
        "entries_per_s_wall": entries / wall, "entries_per_s_device": entries / (dev_ms / 1e3) if dev_ms else None,
    }))


if __name__ == "__main__":
    main()
