"""Cost of lh_ingest_arrays (Engine.ingest_arrays) on the GPU against the float64 path, per dtype.

Throughput: for float32, int32, bfloat16 and float16 samples of streams U and L (the float64 streams converted with
torch's .to), 2^30 samples (1.07e9) per call, it reports
  arrays     one lh_ingest_arrays of the narrow array (a K1 form, the item being past its threshold), device time of
             the call's kernels (lh_kernel_ms: CUDA events on the ingest stream);
  f64        one lh_ingest_f64 of the same values held as float64, device time likewise;
  workaround x.double() then lh_ingest_f64 of the result, both on one non-default torch stream, timed end to end with
             CUDA events recorded on that stream before the cast and after the ingest;
with samples/s and the share of 3.35 TB/s (the H100 SXM data sheet) that each form's algorithmic bytes take: 4 B per
sample for float32 / int32, 2 B for the 16-bit dtypes, 8 B for float64, and for the workaround the narrow read, the
float64 write and its re-read.  Variants alternate after a warm-up; the median of --reps calls is printed.

Threshold sweep: for float32 and bfloat16 items of 2^18 .. 2^24 samples, the device time of the short-item kernel
(the item cut into pieces below the threshold under one id, which k_ingest_arrays takes as one concatenation) and,
from the threshold up, of the routed call (a K1 form).  Below the threshold no call reaches the narrow K1 forms.

The card's name, power limit and maximum SM clock are printed in the same run.
Usage: python tools/array_ingest_probe.py [--reps 5] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import loghisto_b200 as lh  # noqa: E402

HBM = 3.35e12
N = 1 << 30


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


class _View:
    def __init__(self, d, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (d.offset(0), False), "version": 3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    rows = []
    with lh.Engine(device=0, max_histograms=4) as e:
        for sname, stream in (("U", lh.STREAM_U), ("L", lh.STREAM_L)):
            d = e.gen_stream(stream, N, lh.DEFAULT_SEED)
            x64 = torch.as_tensor(_View(d, N), device="cuda:0").clone()
            d.free()
            for dname, dt, nbytes in (("float32", torch.float32, 4), ("int32", torch.int32, 4),
                                      ("bfloat16", torch.bfloat16, 2), ("float16", torch.float16, 2)):
                x = x64.to(dt) if dt != torch.int32 else x64.clamp(-2.0 ** 31, 2.0 ** 31 - 1).to(dt)
                ref = x.double()
                torch.cuda.synchronize()
                ws = torch.cuda.Stream()   # non-default: its handle reaches lh_ingest_f64, which then runs on it
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                times = {"arrays": [], "f64": [], "workaround": []}

                def arrays():
                    e.ingest_arrays([(0, x)])
                    e.sync()
                    return e.kernel_ms(e.ingest_seq())

                def f64():
                    e.ingest_f64(1, ref.data_ptr(), N)
                    e.sync()
                    return e.kernel_ms(e.ingest_seq())

                def workaround():
                    with torch.cuda.stream(ws):
                        ev0.record(ws)
                        y = x.double()                            # allocated and written on ws
                        e.ingest_f64(2, y.data_ptr(), N, ws)      # stream-ordered after the cast
                        ev1.record(ws)
                    ev1.synchronize()
                    del y                                         # after the ingest has read it
                    return ev0.elapsed_time(ev1)

                for f in (arrays, f64, workaround):   # warm-up
                    f()
                for _ in range(a.reps):
                    for k, f in (("arrays", arrays), ("f64", f64), ("workaround", workaround)):
                        times[k].append(f())
                e.snapshot([0.5])
                algo = {"arrays": nbytes, "f64": 8, "workaround": nbytes + 8 + 8}
                for k, v in times.items():
                    ms = float(np.median(v))
                    r = {"stream": sname, "dtype": dname, "variant": k, "ms": round(ms, 4),
                         "gsamples_per_s": round(N / ms / 1e6, 1),
                         "hbm_share": round(N * algo[k] / HBM / (ms / 1e3), 3)}
                    rows.append(r)
                    print(json.dumps(r), flush=True)
                del x, ref
            del x64
            torch.cuda.empty_cache()
    sweep = []
    with lh.Engine(device=0, max_histograms=2) as e:
        x64 = torch.randn(1 << 24, device="cuda:0", dtype=torch.float64).mul_(6).exp_()
        for dname, dt in (("float32", torch.float32), ("bfloat16", torch.bfloat16)):
            x = x64.to(dt)
            torch.cuda.synchronize()
            piece = (1 << 20) - 1   # below both narrow thresholds
            for lg in range(18, 25):
                n = 1 << lg
                forms = {"short": [(0, x[o:min(o + piece, n)]) for o in range(0, n, piece)]}
                if n >= (1 << 20):
                    forms["routed"] = [(0, x[:n])]
                t = {k: [] for k in forms}
                for rep in range(a.reps + 1):
                    for k, items in forms.items():
                        e.ingest_arrays(items)
                        e.sync()
                        if rep:
                            t[k].append(e.kernel_ms(e.ingest_seq()))
                for k, v in t.items():
                    r = {"sweep": dname, "n": n, "route": k, "ms": round(float(np.median(v)), 4),
                         "gsamples_per_s": round(n / float(np.median(v)) / 1e6, 1)}
                    sweep.append(r)
                    print(json.dumps(r), flush=True)
                e.snapshot([0.5])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "array_ingest_probe.json"), "w") as f:
            json.dump({"card": card(), "n": N, "rows": rows, "sweep": sweep}, f, indent=1)


if __name__ == "__main__":
    main()
