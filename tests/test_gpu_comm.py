"""Multi-GPU snapshot behind the C ABI (lh_comm_* / lh_snapshot_allreduce): the peer-memory all-reduce kernel must
give every rank exactly the histogram a single GPU would have produced over the whole stream (SURVEY.md section 8e).

  * two contexts in ONE process (raw peer pointers): runs on a single-GPU box too -- both "ranks" then share
    device 0, which still exercises the arrive / depart protocol, the flag-driven cell sets and the reduced views;
  * one process per GPU (CUDA IPC mappings) through torchrun when the box has >= 2 GPUs.
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PS = [0.0, 0.5, 0.75, 0.9, 0.95, 0.99, 0.999, 0.9999, 1.0]
SEED = 0x10C415C0


def dense_from_sparse(sp, hid):
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in sp.histogram(hid).items():
        out[k & 0xFFFF] = c
    return out


def test_two_contexts_one_process(oracle):
    import torch
    import loghisto_b200 as lh
    from loghisto_b200.distributed import shard_range
    world = 2
    devs = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    H, C, n_total = 5, 8, 3_000_001
    engs = [lh.Engine(device=d, max_histograms=H, max_counters=C) for d in devs]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, world, handles)
        for interval in range(3):
            vals = oracle.gen_stream(lh.STREAM_S, n_total, SEED + interval)
            ids = oracle.gen_ids(0, n_total, H - 1, SEED + interval)            # histogram H-1 stays untouched
            want = np.zeros((H, 65536), dtype=np.uint64)
            want[: H - 1] = oracle.ingest_keyed(ids, vals, H - 1)
            want[2] += oracle.ingest(vals)
            for r, e in enumerate(engs):
                a, b = shard_range(r, world, n_total)
                d = e.upload(vals[a:b])
                di = e.upload(ids[a:b].astype(np.uint16))
                e.ingest_keyed_f64_u16(di, d, b - a)
                e.ingest_f64(2, d, b - a)
                e.counter_add_u16_host(np.array([1, 7], np.uint16), np.array([r + 1 + interval, 2 ** 63 + 3], np.uint64))
            # collective: begin + all-reduce on every rank first (the kernels wait for each other on the device)
            seqs = []
            for e in engs:
                e.snapshot_begin()
                seqs.append(e.snapshot_allreduce(counters=True))
            for r, e in enumerate(engs):
                red = e.snapshot_reduce(PS)
                sp = e.snapshot_export()
                e.snapshot_end()
                assert e.comm_info()["status"] == 0
                assert e.comm_allreduce_ms(seqs[r]) > 0
                for h in range(H):
                    assert (dense_from_sparse(sp, h) == want[h]).all(), (interval, r, h)
                    ref = oracle.process_histogram(want[h], PS)
                    assert int(red.counts[h]) == ref["total"]
                    if ref["total"]:
                        assert (red.pkeys[h] == ref["pkeys"]).all()
                assert int(sp.counter_deltas[1]) == sum(r2 + 1 + interval for r2 in range(world))
                assert int(sp.counter_deltas[7]) == (world * (2 ** 63 + 3)) % 2 ** 64
        # an empty interval stays empty on every rank, and the reduced arrays were cleared
        for e in engs:
            e.snapshot_begin()
            e.snapshot_allreduce()
        for e in engs:
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
            e.snapshot_end()
            assert int(red.counts.sum()) == 0 and int(sp.offsets[-1]) == 0
        info = engs[0].comm_info()
        assert info["world"] == 2 and info["allreduces"] == 4
    finally:
        for e in engs:
            e.close()


def test_two_contexts_many_histograms_two_shot(oracle):
    """H = 48 histograms: the payload is above the 1 MiB threshold, so each rank sums its share of the (histogram,
    chunk) items and PUSHES the sums into every rank's reduced array (reduce-scatter + all-gather in one kernel).
    Histogram 3 also gets out-of-window values on one rank only (dense flag on one side)."""
    import torch
    import loghisto_b200 as lh
    from loghisto_b200.distributed import shard_range
    world = 2
    devs = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    H, n_total = 48, 2_000_003
    engs = [lh.Engine(device=d, max_histograms=H, max_counters=4) for d in devs]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, world, handles)
        for interval in range(2):
            vals = oracle.gen_stream(lh.STREAM_S, n_total, SEED + 10 + interval)
            ids = oracle.gen_ids(0, n_total, H - 2, SEED + 10 + interval)        # the last two histograms stay untouched
            huge = np.array([1e300, -1e300, 3e200, -7e250], dtype=np.float64)    # keys far outside the window
            want = np.zeros((H, 65536), dtype=np.uint64)
            want[: H - 2] = oracle.ingest_keyed(ids, vals, H - 2)
            want[3] += oracle.ingest(huge)
            for r, e in enumerate(engs):
                a, b = shard_range(r, world, n_total)
                e.ingest_keyed_f64_u16(e.upload(ids[a:b].astype(np.uint16)), e.upload(vals[a:b]), b - a)
            engs[1].ingest_f64(3, engs[1].upload(huge), len(huge))
            for e in engs:
                e.snapshot_begin()
                e.snapshot_allreduce()
            for r, e in enumerate(engs):
                red = e.snapshot_reduce(PS)
                sp = e.snapshot_export()
                e.snapshot_end()
                assert e.comm_info()["status"] == 0
                for h in range(H):
                    assert (dense_from_sparse(sp, h) == want[h]).all(), (interval, r, h)
                    ref = oracle.process_histogram(want[h], PS)
                    assert int(red.counts[h]) == ref["total"]
                    if ref["total"]:
                        assert (red.pkeys[h] == ref["pkeys"]).all()
            assert engs[0].comm_last_bytes() > 0
    finally:
        for e in engs:
            e.close()


def test_allreduce_requires_import():
    import loghisto_b200 as lh
    with lh.Engine(device=0) as e:
        e.snapshot_begin()
        with pytest.raises(lh.LhError):
            e.snapshot_allreduce()
        e.snapshot_end()


@pytest.mark.parametrize("H", [3, 40])        # one-shot and two-shot (push) forms of the all-reduce, over CUDA IPC mappings
def test_one_process_per_gpu_peer_collective(H):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = min(n, 8)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "_multi_gpu_worker.py"), "peer", str(H)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


def test_c_host_drives_two_ranks_without_python(tmp_path):
    """tests/c_comm_client.c: a C11 program (pthreads, no Python / torch / NCCL) shards a stream over 2 contexts and
    must see the single-context histogram on every rank after lh_snapshot_allreduce."""
    import torch
    from loghisto_b200 import build
    build.build()
    libdir = os.path.dirname(build.LIB)
    exe = str(tmp_path / "c_comm_client")
    subprocess.run(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c_comm_client.c"), "-o", exe, "-L", libdir, "-lloghisto_b200",
                    "-Wl,-rpath," + libdir, "-lpthread"], check=True)
    ngpu = min(torch.cuda.device_count(), 8)
    for ranks in sorted({2, max(2, ngpu)}):
        res = subprocess.run([exe, str(ranks), "4000001", str(ngpu)], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0 and "C_COMM_OK" in res.stdout, res.stdout + res.stderr
