"""Cost of job-wide MetricSystem collections through the caller's all-reduce (join_ranks(..., allreduce)):

  * k_rows_pack / k_rows_unpack device time (CUDA events on the snapshot stream around lh_snapshot_pack_rows, which
    includes its row-table upload, and lh_snapshot_unpack_rows), median over the rounds, for 1, 64 and 1 024 window
    rows and 64 dense rows at precisions 100 and 250, with the bytes each moves (payload read + written) per second;
  * collect_and_process host time per collection, slowest rank, median over the rounds, at world 2 and 4 with 64 and
    1 024 names per rank (every name shared, 20 samples each): the peer path, this path with an in-process all-reduce
    (ranks as threads), and this path through distributed.rank_allreduce over a gloo group (ranks as processes).
    Every rank runs on device r % device_count().

Prints one JSON line with the card's name and power limit.  Usage: python tools/ranks_allreduce_probe.py [--rounds N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def win_of(precision):
    import math
    return math.floor(precision * 63 * math.log(2) + 0.5) + 1


def kernel_times(rows, dense, precision, rounds):
    """(pack ms, unpack ms, payload words) for `rows` rows of one context, window-only or dense."""
    import torch
    import loghisto_b200 as lh
    e = lh.Engine(device=0, max_histograms=max(rows, 1), max_counters=4, precision=precision)
    try:
        ids = np.repeat(np.arange(rows, dtype=np.uint32), 4)
        keys = np.tile(np.array([1, 200, -300, 30000 if dense else 4], np.int16), rows)
        counts = np.ones(ids.size, np.uint64)
        hr = np.arange(rows, dtype=np.uint32)
        levels = np.full(rows, 3 if dense else 1, np.uint8)
        pack, unpack, words = [], [], 0
        for i in range(rounds + 2):
            e.merge_counts_host(ids, keys, counts)
            e.sync()
            e.snapshot_begin()
            if i == 0:
                _, _, words, sptr = e.snapshot_pack_rows(hr, levels, np.zeros(0, np.uint32))
                s = torch.cuda.ExternalStream(sptr, device=torch.device("cuda", 0))
            else:
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record(s)
                e.snapshot_pack_rows(hr, levels, np.zeros(0, np.uint32))
                ev[1].record(s)
                e.snapshot_unpack_rows(True)
                ev[2].record(s)
                ev[2].synchronize()
                if i >= 2:
                    pack.append(ev[0].elapsed_time(ev[1]))
                    unpack.append(ev[1].elapsed_time(ev[2]))
            e.snapshot_end()
        return statistics.median(pack), statistics.median(unpack), words
    finally:
        e.close()


class ThreadReduce:
    def __init__(self, world):
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)

    def for_rank(self, r):
        import torch
        from loghisto_b200.distributed import _CudaView

        def allreduce(send, recv, n, stream):
            ts, tr = torch.as_tensor(_CudaView(send, n)), torch.as_tensor(_CudaView(recv, n))
            s = torch.cuda.ExternalStream(stream, device=ts.device)
            s.synchronize()
            self.slots[r] = ts.cpu().numpy().view(np.uint64)
            self.barrier.wait()
            total = np.zeros(n, np.uint64)
            for x in self.slots:
                total += x
            self.barrier.wait()
            with torch.cuda.stream(s):
                tr.copy_(torch.from_numpy(total.view(np.int64)).pin_memory(), non_blocking=True)
            s.synchronize()
        return allreduce


def feed(ms, names, r, rng):
    for n in names:
        ms.HistogramMany(n, rng.lognormal(3, 2, 20))
    ms.Counter("steps", r + 1)


def threads_host_ms(world, n_names, transport, rounds):
    import torch
    from test_gpu_ranks import Exchange
    from loghisto_b200.metric_system import MetricSystem
    ndev = torch.cuda.device_count()
    H = max(64, 2 * n_names)
    systems = [MetricSystem(3600.0, device=r % ndev, max_histograms=H, max_counters=8, precision=100)
               for r in range(world)]
    ex, red = Exchange(world), ThreadReduce(world)
    names = ["name.%04d" % i for i in range(n_names)]

    def run(r):
        if transport == "peer":
            systems[r].join_ranks(r, world, ex.for_rank(r))
        else:
            systems[r].join_ranks(r, world, ex.for_rank(r), red.for_rank(r))
        rng = np.random.default_rng(r)
        times = []
        for i in range(rounds + 1):
            feed(systems[r], names, r, rng)
            t0 = time.perf_counter()
            systems[r].collect_and_process()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        return times
    out = [None] * world
    ts = [threading.Thread(target=lambda r=r: out.__setitem__(r, run(r))) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for ms in systems:
        ms.close()
    return statistics.median(max(t[i] for t in out) for i in range(rounds))


def _gloo_rank(rank, world, n_names, rounds, path, q):
    import torch
    import torch.distributed as dist
    from loghisto_b200.distributed import rank_allgather, rank_allreduce
    from loghisto_b200.metric_system import MetricSystem
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method="file://" + path, rank=rank, world_size=world)
    try:
        gather, group = dist.new_group(backend="gloo"), dist.new_group(backend="gloo")
        ms = MetricSystem(3600.0, device=dev, max_histograms=max(64, 2 * n_names), max_counters=8, precision=100)
        ms.join_ranks(rank, world, rank_allgather(gather), rank_allreduce(group))
        names = ["name.%04d" % i for i in range(n_names)]
        rng = np.random.default_rng(rank)
        times = []
        for i in range(rounds + 1):
            feed(ms, names, rank, rng)
            dist.barrier(group=gather)
            t0 = time.perf_counter()
            ms.collect_and_process()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        q.put((rank, times, ms.ranks_info()["status"]))
        ms.close()
    finally:
        dist.destroy_process_group()


def gloo_host_ms(world, n_names, rounds):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as d:
        ps = [ctx.Process(target=_gloo_rank, args=(r, world, n_names, rounds, os.path.join(d, "store"), q))
              for r in range(world)]
        try:
            for p in ps:
                p.start()
            res = [q.get(timeout=600) for _ in range(world)]
        finally:
            for p in ps:
                p.join(timeout=60)
                if p.is_alive():
                    p.terminate()
                    p.join(timeout=30)
    assert all(st == 0 for _, _, st in res), res
    times = [t for _, t, _ in res]
    return statistics.median(max(t[i] for t in times) for i in range(rounds))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    out = {"card": card(), "kernels": [], "collect_ms": []}
    for precision in (100, 250):
        for rows, dense in ((1, False), (64, False), (1024, False), (64, True)):
            pk, up, words = kernel_times(rows, dense, precision, args.rounds)
            moved = 2 * 8 * words
            out["kernels"].append({"precision": precision, "rows": rows, "dense": dense, "payload_bytes": 8 * words,
                                   "pack_ms": round(pk, 4), "unpack_ms": round(up, 4),
                                   "pack_GBps": round(moved / pk / 1e6, 1), "unpack_GBps": round(moved / up / 1e6, 1)})
    for world in (2, 4):
        for n_names in (64, 1024):
            row = {"world": world, "names": n_names}
            for transport in ("peer", "allreduce_threads"):
                row[transport] = round(threads_host_ms(world, n_names, transport, args.rounds), 3)
            row["allreduce_gloo_processes"] = round(gloo_host_ms(world, n_names, args.rounds), 3)
            out["collect_ms"].append(row)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
