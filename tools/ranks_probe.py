"""Cost of job-wide MetricSystem collections (MetricSystem.join_ranks), one thread per rank, rank r on device
r % device_count():

  * collect_and_process of joined systems against unjoined ones, at world 2 and 4, with 64 and 1 024 names per rank
    (every name shared, 20 samples each per interval), host time per collection, median over the rounds;
  * the row-mapped K5 (lh_snapshot_allreduce_rows) against the identity K5 (lh_snapshot_allreduce) on the same arrays,
    device time from lh_comm_allreduce_ms, median;
  * the host-gather workaround: every rank's collected raw set pickled, gathered and merged, then processMetrics of
    the union on one system (host time, median).

Prints one JSON line with the card's name and power limit.  Usage: python tools/ranks_probe.py [--rounds N]"""
import argparse
import json
import os
import pickle
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def on_ranks(world, fn):
    out = [None] * world
    ts = [threading.Thread(target=lambda r=r: out.__setitem__(r, fn(r))) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


class Exchange:
    def __init__(self, world):
        self.slots, self.barrier = [None] * world, threading.Barrier(world)

    def for_rank(self, r):
        def allgather(mine):
            self.slots[r] = bytes(mine)
            self.barrier.wait()
            out = list(self.slots)
            self.barrier.wait()
            return out
        return allgather


def collections(world, n_names, joined, rounds, ndev):
    from loghisto_b200.metric_system import MetricSystem
    systems = [MetricSystem(3600.0, device=r % ndev, max_histograms=max(n_names, 64), max_counters=64)
               for r in range(world)]
    if joined:
        ex = Exchange(world)
        on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r)))
    names = ["name.%04d" % i for i in range(n_names)]
    vals = np.linspace(1.0, 1e6, 20)
    times, raws = [], None
    for i in range(rounds + 1):
        for ms in systems:
            for n in names:
                ms.HistogramMany(n, vals)

        def one(r):
            t0 = time.perf_counter()
            raw, _ = systems[r].collect_and_process()
            return time.perf_counter() - t0, raw
        res = on_ranks(world, one)
        if i:
            times.append(max(t for t, _ in res))
        raws = [raw for _, raw in res]
    for ms in systems:
        ms.close()
    return statistics.median(times) * 1e3, raws


def host_gather(raws, rounds):
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(3600.0, max_histograms=64, max_counters=64)
    times = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        parts = [pickle.loads(pickle.dumps(r)) for r in raws]
        union = {"Histograms": {}, "Counters": {}, "Rates": {}}
        for p in parts:
            for n, m in p["Histograms"].items():
                u = union["Histograms"].setdefault(n, {})
                for k, c in m.items():
                    u[k] = u.get(k, 0) + c
        ms.processMetrics(union)
        times.append(time.perf_counter() - t0)
    ms.close()
    return statistics.median(times) * 1e3


def k5_forms(ndev, rounds, H=1024, precision=100):
    import loghisto_b200 as lh
    world = 2
    engs = [lh.Engine(device=r % ndev, max_histograms=H, max_counters=16, precision=precision) for r in range(world)]
    handles = b"".join(e.comm_export() for e in engs)
    for r, e in enumerate(engs):
        e.comm_import(r, world, handles)
    rng = np.random.default_rng(1)
    ident_h = np.tile(np.arange(H, dtype=np.uint32), (world, 1))
    ident_c = np.tile(np.arange(16, dtype=np.uint32), (world, 1))
    ms = {"identity": [], "mapped": []}
    for i in range(2 * rounds + 2):
        mapped = i % 2 == 1
        for e in engs:
            e.merge_counts_host(rng.integers(0, H, 1 << 16).astype(np.uint32),
                                rng.integers(-4000, 4000, 1 << 16).astype(np.int16), np.ones(1 << 16, np.uint64))
            e.sync()
        for e in engs:
            e.snapshot_begin()
        if mapped:
            fr = [e.snapshot_rows()[2] for e in engs]
            seq = max(e.comm_info()["allreduces"] for e in engs) + 1
            seqs = [e.snapshot_allreduce_rows(seq, fr, ident_h, ident_c) for e in engs]
        else:
            seqs = [e.snapshot_allreduce(True) for e in engs]
        t = max(e.comm_allreduce_ms(s) for e, s in zip(engs, seqs))
        for e in engs:
            e.snapshot_end()
            e.sync()
        if i >= 2:
            ms["mapped" if mapped else "identity"].append(t)
    for e in engs:
        e.close()
    return {k: statistics.median(v) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    import torch
    ndev = torch.cuda.device_count()
    if ndev < 1:
        raise SystemExit("ranks_probe needs a GPU")
    res = {"card": card(), "devices": ndev, "collect_ms": {}, "host_gather_ms": {}}
    for world in (2, 4):
        for n in (64, 1024):
            key = "world%d_names%d" % (world, n)
            un, raws = collections(world, n, False, a.rounds, ndev)
            jo, _ = collections(world, n, True, a.rounds, ndev)
            res["collect_ms"][key] = {"unjoined": un, "joined": jo}
            res["host_gather_ms"][key] = host_gather(raws, a.rounds)
    res["k5_ms_H1024"] = k5_forms(ndev, a.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
