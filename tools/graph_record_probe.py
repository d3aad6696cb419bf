"""Cost of recording through graph recorders (lh_graph_recorder_*), on the GPU, with CUDA events:
  replay   a kernel recording 64 M samples through lh::BlockRecorder (tests/graph_record_client.cu, 4096-slot table)
           into a graph recorder's rows, captured and replayed, against the same kernel launched eagerly in a record
           scope; the record code is the same, so the two should match
  drain    the k_graph_drain launch of lh_snapshot_begin for k = 1, 64 and 1024 rows, window-only (flag 1) and
           full-row (flag 3), events around lh_snapshot_begin on the snapshot stream
  ingest   GraphRecorder ingest of 4096 x 1024 and 64 x 4 M float64 arrays captured and replayed, against the device
           time (lh_kernel_ms) of eager lh_ingest_batch (RecordScope.histograms) of the same arrays
Replays and kernels run on a stream of their own, and a record scope is opened and ended outside the timed window.
Every variant is warmed up; the reported figure is the median of --reps.  Prints the card's name and power limit first.

    python tools/graph_record_probe.py [--reps 9] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402
from loghisto_b200 import _lib, build  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(torch, stream, fn, reps):
    """median ms of fn() (issued with `stream` current) between two events on `stream`, after one warm-up call"""
    with torch.cuda.stream(stream):
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


def client():
    lib = C.CDLL(build.GRAPH_CLIENT_LIB)
    lib.grc_prepare.argtypes = [C.c_uint32, C.c_uint32]
    lib.grc_block_record.argtypes = [C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32,
                                     C.c_size_t, C.c_void_p]
    lib.grc_set_device.argtypes = [C.c_int]
    assert lib.grc_set_device(0) == 0
    assert lib.grc_prepare(100 * 1024, 4096) == 0   # BlockHistogram at precision 200 takes 68 KiB
    return lib


def replay_cost(torch, cl, reps):
    n, H, chunk = 64 << 20, 64, 1 << 16
    with lh.Engine(device=0, max_histograms=H) as eng:
        d = eng.gen_stream(lh.STREAM_L, n, lh.DEFAULT_SEED)
        ids = (torch.arange(n, device="cuda", dtype=torch.int64) % H).to(torch.int32)
        vals = d.ptr
        torch.cuda.synchronize()
        gr = eng.graph_recorder(list(range(H)))
        cur = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=cur):
            assert cl.grc_block_record(C.byref(gr.recorder), ids.data_ptr(), vals, n, 4096, chunk, cur.cuda_stream) == 0
        res = {}
        for _ in range(2):   # alternate; the scope is opened and ended outside the timed window
            res["graph_replay_ms"] = timed(torch, cur, g.replay, reps)
            rec = eng.record_begin(cur.cuda_stream)
            res["record_scope_ms"] = timed(torch, cur, lambda: cl.grc_block_record(
                C.byref(rec), ids.data_ptr(), vals, n, 4096, chunk, cur.cuda_stream), reps)
            eng.record_end(rec)
            eng.snapshot([0.5])
        gr.close()
        eng.snapshot([0.5])
        res["samples"] = n
        return res


def drain_times(torch, reps):
    out = []
    with lh.Engine(device=0, max_histograms=1024) as eng:
        eng.snapshot([0.5])
        eng.snapshot_begin()
        snap = torch.cuda.ExternalStream(eng.snapshot_device().stream)
        eng.snapshot_end()
        win = torch.from_numpy(np.array([1.0, 5.0, -3.0, 1e6], dtype=np.float64)).cuda()
        full = torch.from_numpy(np.array([1.0, 1e20, -1e20, 1e30], dtype=np.float64)).cuda()   # keys past the window
        torch.cuda.synchronize()
        for k in (1, 64, 1024):
            for kind, arr in (("window", win), ("full", full)):
                gr = eng.graph_recorder(list(range(k)))
                items = [(i, arr) for i in range(k)]
                ms = []
                for r in range(reps + 1):
                    gr.ingest(items, stream=0)
                    eng.sync()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(snap)
                    eng.snapshot_begin()
                    e1.record(snap)
                    e1.synchronize()
                    eng.snapshot_end()
                    if r:
                        ms.append(e0.elapsed_time(e1))
                gr.close(stream=0)
                eng.snapshot([0.5])
                out.append({"rows": k, "flags": kind, "drain_ms": statistics.median(ms)})
    return out


def ingest_cost(torch, reps):
    out = []
    for N, L_ in ((4096, 1024), (64, 4 << 20)):
        with lh.Engine(device=0, max_histograms=N) as eng:
            d = eng.gen_stream(lh.STREAM_U, N * L_, lh.DEFAULT_SEED)
            flat = torch.as_tensor(d, device="cuda")
            arrays = [flat[i * L_:(i + 1) * L_] for i in range(N)]
            items = [(i, a) for i, a in enumerate(arrays)]
            torch.cuda.synchronize()
            gr = eng.graph_recorder(list(range(N)))
            cur = torch.cuda.Stream()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=cur):
                gr.ingest(items)
            res = {"items": N, "length": L_}
            for _ in range(2):
                res["graph_replay_ms"] = timed(torch, cur, g.replay, reps)
                # eager: device time of the call's write bracket (lh_kernel_ms), the Python marshalling excluded
                kms = []
                for r in range(reps + 1):
                    eng.ingest_batch(items, stream=cur.cuda_stream)
                    eng.sync()
                    if r:
                        kms.append(eng.last_kernel_ms())
                res["eager_batch_kernel_ms"] = statistics.median(kms)
                eng.snapshot([0.5])
            gr.close()
            eng.snapshot([0.5])
            out.append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    res["replay"] = replay_cost(torch, client(), a.reps)
    print("replay:", res["replay"], flush=True)
    res["drain"] = drain_times(torch, a.reps)
    for r in res["drain"]:
        print("drain:", r, flush=True)
    res["ingest"] = ingest_cost(torch, a.reps)
    for r in res["ingest"]:
        print("ingest:", r, flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
