"""Update granularity of %globaltimer, the clock of lh::start_timer / lh::stop (include/loghisto_b200_device.cuh).

One GPU thread reads the timer back to back and keeps the values at which it changed; the steps between them are the
timer's granularity as a kernel sees it.  Needs build() (tests/_build/libnamed_record_client.so).

    python tools/globaltimer_probe.py [--changes 4096]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--changes", type=int, default=4096)
    args = ap.parse_args()
    import torch
    from loghisto_b200 import build
    lib = C.CDLL(build.NAMED_CLIENT_LIB)
    lib.nrc_globaltimer_probe.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p]
    lib.nrc_globaltimer_probe.restype = C.c_int
    out = torch.zeros(args.changes, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    assert lib.nrc_globaltimer_probe(out.data_ptr(), args.changes, 1 << 26, 0) == 0
    torch.cuda.synchronize()
    t = out.cpu().numpy()
    t = t[t != 0]
    steps = np.diff(t)
    vals, counts = np.unique(steps, return_counts=True)
    top = sorted(zip(counts.tolist(), vals.tolist()), reverse=True)[:5]
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(0), "changes": int(t.size),
        "step_ns_min": int(steps.min()), "step_ns_median": float(np.median(steps)), "step_ns_max": int(steps.max()),
        "most_common_steps_ns": [{"ns": v, "count": c} for c, v in top],
    }))


if __name__ == "__main__":
    main()
