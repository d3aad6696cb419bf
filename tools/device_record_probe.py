"""Records per second of the device record API (include/loghisto_b200_device.cuh) next to the materialised path.

For streams U and L and H = 1, 16 and 1024 histograms, on the same n samples:
  materialised  lh_gen_stream_f64 (+ lh_gen_ids_u16 at H > 1) writes the samples to HBM, then lh_ingest_f64 (H = 1) or
                lh_ingest_keyed_f64_u16 reads them back; reported for the ingest alone and with the materialising write
  record        lh::record from the client kernel of tests/device_record_client.cu, one call per sample
  block         lh::BlockHistogram from the same client, one histogram per CTA (65536 samples per CTA)
  block_rec     lh::BlockRecorder from tests/block_recorder_client.cu: a 4096-entry table, 65536 samples per CTA, one
                flush at the end
The client kernels read their values (8 B) and ids (4 B, record and block_rec at H > 1; per-CTA for block) from HBM, so their rates
are those of a producer that has its samples in memory already; one that computes them in registers skips that read.
Every time is CUDA events on the recording / ingest stream, median of --reps after one warm-up.  Prints the card and
its power limit, then one JSON line per configuration.

    python tools/device_record_probe.py [--n 67108864] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import loghisto_b200 as lh  # noqa: E402
from loghisto_b200 import _lib, build  # noqa: E402

CHUNK = 65536
TABLE_ENTRIES = 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def client():
    lib = C.CDLL(build.build_device_client())
    rp, vp, sz = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t
    lib.lhc_record.argtypes = [rp, vp, vp, sz, vp]
    lib.lhc_block.argtypes = [rp, vp, vp, sz, sz, vp]
    lib.lhc_record.restype = lib.lhc_block.restype = C.c_int
    br = C.CDLL(build.BLOCK_CLIENT_LIB)
    br.brc_record.argtypes = [rp, vp, vp, sz, sz, C.c_uint32, C.c_int, vp]
    br.brc_record.restype = C.c_int
    return lib, br


def timed(stream, fn, reps):
    """median device time (ms) of fn() over reps runs after one warm-up; events on `stream`"""
    ms = []
    for i in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        if i:
            ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 26)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    n = a.n
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "n": n}), flush=True)
    cl, br = client()
    torch.cuda.init()
    for H in (1, 16, 1024):
        with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
            stream = torch.cuda.ExternalStream(eng.ingest_stream)
            s = eng.ingest_stream
            d_v = eng.alloc(n, np.float64)
            d_i16 = eng.alloc(n, np.uint16)
            d_i32 = eng.alloc(n, np.uint32) if H > 1 else None
            nblk = (n + CHUNK - 1) // CHUNK
            d_blk = eng.upload((np.arange(nblk) % H).astype(np.uint32))
            for kind, sname in ((lh.STREAM_U, "U"), (lh.STREAM_L, "L")):
                def gen():
                    eng.gen_stream(kind, n, lh.DEFAULT_SEED, out=d_v, stream=s)
                    if H > 1:
                        eng.gen_ids_u16(0, n, H, lh.DEFAULT_SEED, out=d_i16, stream=s)
                gen()
                if H > 1:
                    ids = d_i16.to_host().astype(np.uint32)
                    eng._check(eng.lib.lh_memcpy_h2d(eng.h, d_i32.ptr, ids.ctypes.data, ids.nbytes))

                def ingest():
                    if H == 1:
                        eng.ingest_f64(0, d_v, n, stream=s)
                    else:
                        eng.ingest_keyed_f64_u16(d_i16, d_v, n, stream=s)

                def record():
                    with eng.recording(s) as rec:
                        assert cl.lhc_record(C.byref(rec), d_i32.ptr if d_i32 else None, d_v.ptr, n, s) == 0

                def block():
                    with eng.recording(s) as rec:
                        assert cl.lhc_block(C.byref(rec), d_blk.ptr, d_v.ptr, n, CHUNK, s) == 0

                def block_rec():
                    with eng.recording(s) as rec:
                        assert br.brc_record(C.byref(rec), d_i32.ptr if d_i32 else None, d_v.ptr, n, CHUNK, TABLE_ENTRIES,
                                             0, s) == 0

                res = {}
                for label, fn in (("gen", gen), ("ingest", ingest), ("record", record), ("block", block),
                                  ("block_rec", block_rec)):
                    res[label] = timed(stream, fn, a.reps)
                    eng.snapshot([], export=False)      # keep every interval small; not timed
                out = {"stream": sname, "H": H, "n": n, "card": name, "power_limit": power,
                       "ms": {k: round(v, 4) for k, v in res.items()},
                       "records_per_s": {
                           "ingest_only": n / res["ingest"] * 1e3,
                           "gen_plus_ingest": n / (res["gen"] + res["ingest"]) * 1e3,
                           "record": n / res["record"] * 1e3,
                           "block_histogram": n / res["block"] * 1e3,
                           "block_recorder": n / res["block_rec"] * 1e3}}
                print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
