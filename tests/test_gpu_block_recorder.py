"""lh::BlockRecorder (include/loghisto_b200_device.cuh): any number of histograms from one CTA through a shared-memory
combining table keyed by the exact (id, bucket) of each sample.

The kernels live in tests/block_recorder_client.cu, a separate CUDA library built by build() that knows the engine only
through its public headers.  Bar: every bucket equal to the oracle whatever the table size (a full table sends samples
straight to the rows), reductions and exports identical to lh_ingest_keyed_f64_u32 of the same pairs, exact dropped
tallies, and the same metrics as the oracle's port of metrics.go when recording under MetricSystem names."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_device_record import PS, SEED, STREAMS, dense_all, edge_inputs, stream_with_edges, want_keyed

pytestmark = pytest.mark.gpu

PRECISIONS = [50, 100, 200]
UNBOUND = 0xFFFFFFFF


def bad_ids(H):
    """Dropped and counted; 65536 + 3 must never alias onto id 3."""
    return (H + 7, 65536 + 3, UNBOUND)


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def client():
    from loghisto_b200 import _lib, build
    assert os.path.exists(build.BLOCK_CLIENT_LIB), "build() did not produce " + build.BLOCK_CLIENT_LIB
    lib = C.CDLL(build.BLOCK_CLIENT_LIB)
    rp, vp, sz, u32 = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t, C.c_uint32
    lib.brc_set_device.argtypes = [C.c_int]
    lib.brc_record.argtypes = [rp, vp, vp, sz, sz, u32, C.c_int, vp]
    for name in ("brc_record_subset", "brc_record_ns", "brc_stop"):
        getattr(lib, name).argtypes = [rp, vp, vp, sz, sz, u32, vp]
    for name in ("brc_set_device", "brc_record", "brc_record_subset", "brc_record_ns", "brc_stop"):
        getattr(lib, name).restype = C.c_int
    assert lib.brc_set_device(0) == 0
    return lib


def launch(client, fn, rec, stream, *args):
    assert getattr(client, fn)(C.byref(rec), *args, stream) == 0, fn


def with_bad_ids(ids, H):
    ids = ids.copy()
    for j, bad in enumerate(bad_ids(H)):
        ids[j::101 + 2 * j] = bad
    return ids


def keys_of(oracle, vals, precision):
    return oracle.compress_many(vals, precision).view(np.uint16).astype(np.int64)


def record_and_check(lh, oracle, client, vals, ids, H, precision, chunk, entries, mid_flush=1):
    """One BlockRecorder launch over (ids, vals): every bucket == the oracle, dropped == the bad ids."""
    want = want_keyed(oracle, ids, vals, H, precision)
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng:
        d_v, d_i = eng.upload(vals), eng.upload(ids)
        with eng.recording() as rec:
            launch(client, "brc_record", rec, eng.ingest_stream, d_i.ptr, d_v.ptr, vals.size, chunk, entries, mid_flush)
        red, sp = eng.snapshot(PS)
        eng.sync()
        got = dense_all(sp, H)
        for h in range(H):
            assert (got[h] == want[h]).all(), (precision, entries, h)
        assert eng.stats()["dropped"] == int((ids >= H).sum())
        return red, sp


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("stream", list(STREAMS))
def test_block_recorder_matches_oracle_and_keyed_ingest(lh, oracle, client, precision, stream):
    """Every bucket == the oracle (thresholds +-3 ulp and the epsilon band included); ids H + 7, 65536 + 3 and
    0xFFFFFFFF raise `dropped` by exactly their number; reductions and exports are byte-identical to
    lh_ingest_keyed_f64_u32 of the same pairs."""
    H, kind = 37, STREAMS[stream]
    vals = stream_with_edges(oracle, kind, precision)
    n = vals.size
    ids = with_bad_ids(oracle.gen_ids(0, n, H, SEED ^ precision ^ 0xB7).astype(np.uint32), H)
    bad = int((ids >= H).sum())
    want = want_keyed(oracle, ids, vals, H, precision)
    with lh.Engine(device=0, max_histograms=H, max_counters=4, precision=precision) as eng:
        d_v, d_i = eng.upload(vals), eng.upload(ids)
        with eng.recording() as rec:
            launch(client, "brc_record", rec, eng.ingest_stream, d_i.ptr, d_v.ptr, n, 8191, 1024, 1)
        red_d, sp_d = eng.snapshot(PS)
        eng.sync()
        dropped_d = eng.stats()["dropped"]
        got = dense_all(sp_d, H)
        for h in range(H):
            assert (got[h] == want[h]).all(), (precision, stream, h)
        assert dropped_d == bad
        eng.ingest_keyed_f64_u32(d_i, d_v, n)
        red_k, sp_k = eng.snapshot(PS)
        eng.sync()
        assert eng.stats()["dropped"] - dropped_d == bad
        for a, b in ((red_d.counts, red_k.counts), (red_d.sums, red_k.sums), (red_d.avgs, red_k.avgs),
                     (red_d.pkeys, red_k.pkeys), (red_d.pvals, red_k.pvals),
                     (sp_d.offsets, sp_k.offsets), (sp_d.keys, sp_k.keys), (sp_d.counts, sp_k.counts),
                     (sp_d.counter_deltas, sp_k.counter_deltas)):
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (precision, stream)


@pytest.mark.parametrize("entries", [0, 16, 32, 1024, 8192])
@pytest.mark.parametrize("H,stream", [(37, "L"), (1024, "U")])
def test_table_pressure(lh, oracle, client, entries, H, stream):
    """Tables of no slots (every sample takes the direct path) up to 8192 slots (96 KiB of shared memory) on the same
    input.  At H = 1024 on stream U each CTA sees far more distinct (id, bucket) pairs than the largest table holds, so
    most samples find the table full; every bucket stays exact."""
    chunk = 65536
    vals = stream_with_edges(oracle, STREAMS[stream], 100)
    ids = with_bad_ids(oracle.gen_ids(0, vals.size, H, SEED ^ H).astype(np.uint32), H)
    if H == 1024:
        ok = ids[:chunk] < H
        pairs = np.unique(ids[:chunk][ok].astype(np.int64) << 16 | keys_of(oracle, vals[:chunk][ok], 100)).size
        assert pairs > 4 * 8192, pairs
    record_and_check(lh, oracle, client, vals, ids, H, 100, chunk, entries, mid_flush=0)


@pytest.mark.parametrize("mid_flush", [0, 1], ids=["one_flush", "two_flushes"])
def test_hot_cell_from_a_full_grid(lh, oracle, client, mid_flush):
    """Every lane of every CTA records the same value into one id: one slot per CTA takes every count, and the total
    is exact whether the CTA flushes once or twice."""
    n = 132 * 8 * 256 * 5
    chunk = 4096
    vals = np.full(n, 4.2e5, dtype=np.float64)
    key = int(oracle.compress(4.2e5)) & 0xFFFF
    with lh.Engine(device=0, max_histograms=2) as eng:
        d_v = eng.upload(vals)
        with eng.recording() as rec:
            launch(client, "brc_record", rec, eng.ingest_stream, None, d_v.ptr, n, chunk, 64, mid_flush)
        red, sp = eng.snapshot(PS)
        assert sp.histogram(0) == {key - 65536 if key >= 32768 else key: n}
        assert int(red.counts[0]) == n and int(red.counts[1]) == 0


@pytest.mark.parametrize("entries", [32, 4096])
def test_flush_reuse(lh, oracle, client, entries):
    """Two flushes per CTA over many ids: the table is reused after the first flush and nothing is counted twice."""
    H = 300
    vals = np.concatenate([oracle.gen_stream(lh.STREAM_S, 700_001, SEED ^ 3), edge_inputs(100)])
    ids = with_bad_ids(oracle.gen_ids(0, vals.size, H, SEED ^ 3).astype(np.uint32), H)
    record_and_check(lh, oracle, client, vals, ids, H, 100, 20_000, entries, mid_flush=1)


def test_divergent_subset_counts_only_the_recording_lanes(lh, oracle, client):
    H = 11
    vals = np.concatenate([oracle.gen_stream(lh.STREAM_S, 1_000_003, SEED), edge_inputs(100)])
    n = vals.size
    ids = with_bad_ids(oracle.gen_ids(0, n, H, SEED).astype(np.uint32), H)
    mask = (vals.view(np.uint64) & np.uint64(1)) == 1
    assert 0.2 < mask.mean() < 0.8
    want = oracle.ingest_keyed(ids[mask & (ids < H)], vals[mask & (ids < H)], H)
    with lh.Engine(device=0, max_histograms=H) as eng:
        d_v, d_i = eng.upload(vals), eng.upload(ids)
        with eng.recording() as rec:
            launch(client, "brc_record_subset", rec, eng.ingest_stream, d_i.ptr, d_v.ptr, n, 16384, 512)
        _, sp = eng.snapshot(PS)
        eng.sync()
        assert (dense_all(sp, H) == want).all()
        assert eng.stats()["dropped"] == int((mask & (ids >= H)).sum())


def test_record_ns_matches_timer_ingest(lh, oracle, client):
    """float64(ns), round-to-nearest-even, through the table == lh_ingest_keyed_i64ns_u16 of the same ns."""
    H = 5
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, 600_001, SEED).view(np.int64).copy()
    ns[::3] *= -1
    big = np.array([2 ** 53 + 1, 2 ** 53 + 3, 2 ** 60 + 12345, 2 ** 62 - 1, 2 ** 63 - 1, -(2 ** 63), -(2 ** 53) - 1,
                    -(2 ** 61) - 777], dtype=np.int64)
    ns = np.concatenate([ns, np.repeat(big, 3)])
    n = ns.size
    ids = oracle.gen_ids(0, n, H, SEED ^ 1).astype(np.uint32)
    ids[::31] = H + 2
    keep = ids < H
    want = oracle.ingest_keyed_i64(ids[keep], ns[keep], H)
    with lh.Engine(device=0, max_histograms=H) as eng:
        d_n, d_i = eng.upload(ns), eng.upload(ids)
        with eng.recording() as rec:
            launch(client, "brc_record_ns", rec, eng.ingest_stream, d_i.ptr, d_n.ptr, n, 8192, 256)
        red_d, sp_d = eng.snapshot(PS)
        eng.sync()
        assert (dense_all(sp_d, H) == want).all()
        assert eng.stats()["dropped"] == int((~keep).sum())
        eng.ingest_keyed_i64ns_u16(eng.upload(ids.astype(np.uint16)), d_n, n)
        red_k, sp_k = eng.snapshot(PS)
        assert (dense_all(sp_k, H) == dense_all(sp_d, H)).all()
        assert red_d.pkeys.tobytes() == red_k.pkeys.tobytes() and red_d.sums.tobytes() == red_k.sums.tobytes()


def test_stop_records_the_durations_it_returns(lh, oracle, client):
    """stop() on tokens started in the same kernel: the durations it returned, ingested as Timer samples into the next
    interval, give the buckets of the interval stop() recorded into."""
    H = 6
    n = 40_000
    ids = oracle.gen_ids(0, n, H, SEED ^ 9).astype(np.uint32)
    ids[::53] = H + 1
    with lh.Engine(device=0, max_histograms=H) as eng:
        d_i, d_out = eng.upload(ids), eng.alloc(n, np.int64)
        with eng.recording() as rec:
            launch(client, "brc_stop", rec, eng.ingest_stream, d_i.ptr, d_out.ptr, n, 2048, 128)
        _, sp_d = eng.snapshot(PS)
        eng.sync()
        ns = d_out.to_host()
        assert (ns >= 0).all() and ns.max() >= 16 * 100, (ns.min(), ns.max())
        dropped_d = eng.stats()["dropped"]
        assert dropped_d == int((ids >= H).sum())
        eng.ingest_keyed_i64ns_u16(eng.upload(ids.astype(np.uint16)), d_out, n)
        _, sp_k = eng.snapshot(PS)
        eng.sync()
        assert (dense_all(sp_d, H) == dense_all(sp_k, H)).all()
        assert int(dense_all(sp_d, H).sum()) == int((ids < H).sum())
        assert eng.stats()["dropped"] - dropped_d == dropped_d


def test_ids_past_16_bits_keep_their_rows(lh, oracle, client, torch):
    """Valid ids 65536 + k and k in one table, recorded through a recorder over a bucket array of 65540 rows: each
    lands in its own row (the table's tag holds the whole id).  Only the touched rows are backed by zeroed memory
    that is read back; the recorder's precision block and dropped tally come from a real scope."""
    from loghisto_b200 import _lib
    H, row = 65540, 65536
    n = 300_000
    vals = oracle.gen_stream(lh.STREAM_S, n, SEED ^ 5)
    k = oracle.gen_ids(0, n, 4, SEED ^ 5).astype(np.uint32)
    ids = np.where(np.arange(n) % 2 == 0, k, k + 65536).astype(np.uint32)
    buckets = torch.empty(H * row, dtype=torch.int64, device="cuda")          # 32 GiB + 2 MiB, never read in full
    low, high = buckets[: 4 * row], buckets[65536 * row:]                   # rows 0..3 and 65536..65539
    low.zero_()
    high.zero_()
    flags = torch.zeros(H, dtype=torch.int32, device="cuda")
    try:
        with lh.Engine(device=0, max_histograms=1) as eng:
            with eng.recording() as rec:
                wide = _lib.lh_recorder.from_buffer_copy(rec)
                wide.d_buckets, wide.d_flags = buckets.data_ptr(), flags.data_ptr()
                wide.max_histograms = H
                d_v, d_i = eng.upload(vals), eng.upload(ids)
                launch(client, "brc_record", wide, eng.ingest_stream, d_i.ptr, d_v.ptr, n, 32768, 2048, 1)
                eng.sync()
            assert eng.stats()["dropped"] == 0
        torch.cuda.synchronize()
        got = np.concatenate([low.cpu().numpy(), high.cpu().numpy()]).view(np.uint64).reshape(8, row)
        keys = keys_of(oracle, vals, 100)
        for j, hid in enumerate(list(range(4)) + [65536 + i for i in range(4)]):
            want = np.bincount(keys[ids == hid], minlength=row).astype(np.uint64)
            assert (got[j] == want).all(), hid
        f = flags.cpu().numpy()
        assert (f[[0, 1, 2, 3, 65536, 65537, 65538, 65539]] != 0).all() and np.count_nonzero(f) == 8
    finally:
        del buckets, low, high
        torch.cuda.empty_cache()


def test_under_metric_system_names(oracle, client, torch):
    """Three names bound by MetricSystem.recording, recorded through BlockRecorder under s.histogram_ids, plus host
    Histogram() calls on the same names: collectRawMetrics / processMetrics equal the oracle's port of metrics.go over
    two intervals."""
    import importlib.util
    from loghisto_b200.metric_system import MetricSystem
    spec = importlib.util.spec_from_file_location("name_recycling_cases",
                                                  os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                               "_name_recycling_cases.py"))
    cases = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cases)
    names = ["rpc_latency", "payload_bytes", "queue_depth"]
    rng = np.random.default_rng(17)
    ms = MetricSystem(1e-6, False, max_histograms=8, max_counters=8)
    ref = oracle.OracleMetricSystem()
    st = torch.cuda.Stream()
    try:
        for interval in range(2):
            n = 12_000 + 999 * interval
            which = rng.integers(0, 3, n)
            vals = np.exp(rng.uniform(-4, 22, n)) * np.where(which == 2, -1.0, 1.0)
            for i in range(n):
                ref.Histogram(names[which[i]], float(vals[i]))
            for nm in names:
                for v in np.exp(rng.uniform(-4, 22, 5)):
                    ms.Histogram(nm, float(v))
                    ref.Histogram(nm, float(v))
            d_v = torch.from_numpy(vals).cuda()
            with ms.recording(st, histograms=names) as s:
                hid = np.array([s.histogram_ids[nm] for nm in names], dtype=np.uint32)
                assert (hid != UNBOUND).all()
                d_i = torch.from_numpy(hid[which].view(np.int32)).cuda()
                st.wait_stream(torch.cuda.current_stream())
                launch(client, "brc_record", s.recorder, st.cuda_stream, d_i.data_ptr(), d_v.data_ptr(), n, 3000, 64, 1)
            st.synchronize()
            raw, m = ms.collect_and_process()
            rraw, rm = ref.collect_and_process()
            assert set(raw["Histograms"]) == set(names)
            cases._compare_interval(raw, m, rraw, rm)
        assert ms.dropped() == 0
    finally:
        ref.close()
        ms.close()
