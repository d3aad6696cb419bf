"""Cost of ingesting N device arrays under N histogram ids, three ways, on the same samples:
  batch   one lh_ingest_batch
  single  one lh_ingest_f64 per item
  keyed   one lh_ingest_keyed_f64_u32 over a materialised id array (the id array is built before the timed window)
  batch_py  Engine.ingest_batch, the Python API over the same items (array checks and marshalling included)
The first three call the C ABI directly through ctypes, so their host time is the library's plus one ctypes call each.
For each: host time of the call sequence ending in a synchronise, device time (lh_kernel_ms: the one sequence number
of batch / keyed; CUDA events around the sequence on the ingest stream for all three), and samples per second.  Every
shape is warmed up, then the variants alternate.  Stream U and L at precision 100; item counts 1 ... 4096, item lengths
64 ... 4 M, capped at --max-samples per shape.  Prints the card's name and power limit first.

    python tools/batch_ingest_probe.py [--reps 7] [--max-samples 268435456] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--max-samples", type=int, default=1 << 28)
    ap.add_argument("--counts", default="1,8,64,512,4096")
    ap.add_argument("--lengths", default="64,1024,16384,262144,4194304")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    print("card:", card(), flush=True)
    counts = [int(x) for x in a.counts.split(",")]
    lengths = [int(x) for x in a.lengths.split(",")]
    H = max(counts)
    rows = []
    with lh.Engine(device=0, max_histograms=H) as e:
        ist = torch.cuda.ExternalStream(e.ingest_stream)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for kind, sname in ((lh.STREAM_U, "U"), (lh.STREAM_L, "L")):
            for L_ in lengths:
                for N in counts:
                    total = N * L_
                    if total > a.max_samples:
                        continue
                    d = e.gen_stream(kind, total, lh.DEFAULT_SEED)
                    ids = torch.arange(N, dtype=torch.int32, device="cuda:0").repeat_interleave(L_)
                    torch.cuda.synchronize()
                    e.sync()
                    items = [(i, _View(d, i * L_, L_)) for i in range(N)]
                    ptrs = [d.offset(i * L_) for i in range(N)]

                    arr = (lh._lib.lh_batch_item * N)(*[lh._lib.lh_batch_item(ptrs[i], L_, i, 0) for i in range(N)])
                    lib, h = e.lib, e.h

                    def batch():          # the C call on a prepared item table
                        lib.lh_ingest_batch(h, arr, N, None)

                    def single():
                        for i in range(N):
                            lib.lh_ingest_f64(h, i, ptrs[i], L_, None)

                    def keyed():
                        lib.lh_ingest_keyed_f64_u32(h, ids.data_ptr(), d.ptr, total, None)

                    def batch_py():       # Engine.ingest_batch: the Python API, item checks and marshalling included
                        e.ingest_batch(items)

                    variants = {"batch": batch, "single": single, "keyed": keyed, "batch_py": batch_py}
                    res = {k: {"host_ms": [], "stream_ms": [], "kernel_ms": []} for k in variants}
                    for k, fn in variants.items():      # warm-up
                        fn()
                    e.sync()
                    for r in range(a.reps):
                        for k, fn in variants.items():
                            e.sync()
                            seq0 = e.ingest_seq()
                            t0 = time.perf_counter()
                            ev0.record(ist)
                            fn()
                            ev1.record(ist)
                            e.sync()
                            t1 = time.perf_counter()
                            res[k]["host_ms"].append((t1 - t0) * 1e3)
                            res[k]["stream_ms"].append(ev0.elapsed_time(ev1))
                            seqs = e.ingest_seq() - seq0
                            if seqs <= 16:
                                res[k]["kernel_ms"].append(sum(e.kernel_ms(q) for q in range(seq0 + 1, seq0 + seqs + 1)))
                        e.snapshot_begin()
                        e.snapshot_end()
                    row = {"stream": sname, "items": N, "length": L_, "samples": total}
                    for k in variants:
                        hm = float(np.median(res[k]["host_ms"]))
                        sm = float(np.median(res[k]["stream_ms"]))
                        km = float(np.median(res[k]["kernel_ms"])) if res[k]["kernel_ms"] else None
                        row[k] = {"host_ms": hm, "stream_ms": sm, "kernel_ms": km, "gsps_host": total / hm / 1e6}
                    rows.append(row)
                    print("%s N=%5d len=%8d | %s" % (sname, N, L_, " | ".join(
                        "%s host %.4f stream %.4f kern %s ms %.2f GS/s" % (
                            k, row[k]["host_ms"], row[k]["stream_ms"],
                            "%.4f" % row[k]["kernel_ms"] if row[k]["kernel_ms"] is not None else "n/a", row[k]["gsps_host"])
                        for k in variants)), flush=True)
                    del items, ptrs, ids, arr
                    d.free()
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


class _View:
    """n float64 of a DeviceArray from element `off`, as a __cuda_array_interface__ object."""

    def __init__(self, d, off, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (d.offset(off), False),
                                         "version": 3}


if __name__ == "__main__":
    main()
