"""Recording from CUDA code (include/loghisto_b200_device.cuh) through record scopes (lh_record_begin / lh_record_end).

The kernels live in tests/device_record_client.cu, a separate CUDA library built by build() that knows the engine only
through its public headers.  Bar: every bucket of every histogram equal to the oracle and to the host-issued ingest of
the same samples, identical reductions and exports, exact dropped tallies, and the snapshot ordering of the scopes."""
import ctypes as C
import functools
import os
import threading
import time

import numpy as np
import pytest

from _ingest_routes import thresholds

pytestmark = pytest.mark.gpu

SEED = 0x5EC0DE
PS = [0.0, 0.5, 0.75, 0.9, 0.95, 0.99, 0.999, 0.9999, 1.0]
PRECISIONS = [50, 100, 200]
LH_ERR_INVALID, LH_ERR_STATE = -1, -5


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def client():
    from loghisto_b200 import _lib, build
    assert os.path.exists(build.CLIENT_LIB), "build() did not produce " + build.CLIENT_LIB
    lib = C.CDLL(build.CLIENT_LIB)
    rp, vp, sz = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t
    for name in ("lhc_record", "lhc_record_subset", "lhc_record_ns", "lhc_count"):
        getattr(lib, name).argtypes = [rp, vp, vp, sz, vp]
        getattr(lib, name).restype = C.c_int
    lib.lhc_block.argtypes = [rp, vp, vp, sz, sz, vp]
    lib.lhc_block.restype = C.c_int
    lib.lhc_set_device.argtypes = [C.c_int]
    lib.lhc_set_device.restype = C.c_int
    return lib


def launch(client, fn, eng, rec, *args):
    """One client launch on the scope's stream (the engine's ingest stream)."""
    assert client.lhc_set_device(eng.device) == 0
    assert getattr(client, fn)(C.byref(rec), *args, eng.ingest_stream) == 0, fn


def dense_all(sp, H):
    out = np.zeros((H, 65536), dtype=np.uint64)
    hid = np.repeat(np.arange(H), np.diff(sp.offsets.astype(np.int64)))
    out[hid, sp.keys.view(np.uint16)] = sp.counts
    return out


def want_keyed(oracle, ids, vals, H, precision):
    keep = ids < H
    out = np.zeros((H, 65536), dtype=np.uint64)
    np.add.at(out, (ids[keep], oracle.compress_many(vals[keep], precision).view(np.uint16)), 1)
    return out


@functools.lru_cache(maxsize=None)
def edge_inputs(precision):
    """Every bucket threshold of the finite range +-3 ulp, both signs, and the inputs just inside and outside the
    epsilon band around every boundary of the fast window (where an estimator error would flip a bucket)."""
    from oracle import oracle
    kmax = int(np.floor(precision * np.log1p(1.7976931348623157e308) + 0.5))
    T = thresholds(oracle, precision, kmax)
    bits = (T[:, None].astype(np.int64) + np.arange(-3, 4, dtype=np.int64)[None, :]).reshape(-1).astype(np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(0x8000000000000000)])
    win = int(np.floor(precision * 63 * np.log(2.0) + 0.5)) + 1
    Tw = T[: win - 1].view(np.float64)
    Tw = Tw[Tw > 0.02]
    eps = 2.0 ** -12 * max(1.0, precision / 100.0)
    band = []
    for mult in (0.6, 0.9, 1.1, 1.5, 3.0):
        dv = (1.0 + Tw) * (mult * eps) / precision
        band += [Tw + dv, Tw - dv, -(Tw + dv), -(Tw - dv)]
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 2.0 ** 63, -2.0 ** 63, 1e300, -1e-300], dtype=np.float64)
    return np.concatenate([bits.view(np.float64)] + band + [special])


def stream_with_edges(oracle, kind, precision, n=400_000):
    vals = np.concatenate([oracle.gen_stream(kind, n, SEED ^ kind ^ precision), edge_inputs(precision)])
    return np.ascontiguousarray(vals)


STREAMS = {"U": 0, "L": 1, "S": 2, "N": 8}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("stream", list(STREAMS))
def test_record_matches_oracle_and_keyed_ingest(lh, oracle, client, precision, stream):
    """record() over (ids, values) == the oracle, bucket for bucket, and == lh_ingest_keyed_f64_u16 of the same pairs:
    identical arrays, reductions and exports; ids >= H change `dropped` by exactly their number."""
    H, kind = 37, STREAMS[stream]
    vals = stream_with_edges(oracle, kind, precision)
    n = vals.size
    ids = oracle.gen_ids(0, n, H, SEED ^ precision).astype(np.uint32)
    ids[::101] = H + 7                                   # out of range: dropped and counted
    bad = int((ids >= H).sum())
    want = want_keyed(oracle, ids, vals, H, precision)
    with lh.Engine(device=0, max_histograms=H, max_counters=4, precision=precision) as eng:
        d_v, d_i32, d_i16 = eng.upload(vals), eng.upload(ids), eng.upload(ids.astype(np.uint16))
        with eng.recording() as rec:
            assert rec.max_histograms == H and rec.block_smem_bytes == (2 * (int(np.floor(precision * 63 * np.log(2.0) + 0.5)) + 1) + 8) * 4
            launch(client, "lhc_record", eng, rec, d_i32.ptr, d_v.ptr, n)
        red_d, sp_d = eng.snapshot(PS)
        eng.sync()
        dropped_d = eng.stats()["dropped"]
        got = dense_all(sp_d, H)
        for h in range(H):
            assert (got[h] == want[h]).all(), (precision, stream, h)
        assert dropped_d == bad
        eng.ingest_keyed_f64_u16(d_i16, d_v, n)
        red_k, sp_k = eng.snapshot(PS)
        eng.sync()
        assert eng.stats()["dropped"] - dropped_d == bad
        for a, b in ((red_d.counts, red_k.counts), (red_d.sums, red_k.sums), (red_d.avgs, red_k.avgs),
                     (red_d.pkeys, red_k.pkeys), (red_d.pvals, red_k.pvals),
                     (sp_d.offsets, sp_k.offsets), (sp_d.keys, sp_k.keys), (sp_d.counts, sp_k.counts),
                     (sp_d.counter_deltas, sp_k.counter_deltas)):
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (precision, stream)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("stream", list(STREAMS))
def test_block_histogram_matches_oracle(lh, oracle, client, precision, stream):
    """BlockHistogram, one histogram per CTA (flushed twice per CTA): every bucket == the oracle's ingest of the CTA's
    samples; CTAs bound to an id >= H drop exactly their samples."""
    H, kind, chunk = 19, STREAMS[stream], 4099
    vals = stream_with_edges(oracle, kind, precision)
    n = vals.size
    nblk = (n + chunk - 1) // chunk
    block_ids = oracle.gen_ids(0, nblk, H, SEED ^ 0xB10C ^ precision).astype(np.uint32)
    block_ids[::13] = H + 1
    ids = np.repeat(block_ids, chunk)[:n]
    want = want_keyed(oracle, ids, vals, H, precision)
    with lh.Engine(device=0, max_histograms=H, precision=precision) as eng:
        d_v, d_b = eng.upload(vals), eng.upload(block_ids)
        with eng.recording() as rec:
            launch(client, "lhc_block", eng, rec, d_b.ptr, d_v.ptr, n, chunk)
        red, sp = eng.snapshot(PS)
        eng.sync()
        got = dense_all(sp, H)
        for h in range(H):
            assert (got[h] == want[h]).all(), (precision, stream, h)
            ref = oracle.process_histogram(want[h], PS, precision)
            assert int(red.counts[h]) == ref["total"]
            if ref["total"]:
                assert (red.pkeys[h] == ref["pkeys"]).all()
        assert eng.stats()["dropped"] == int((ids >= H).sum())


def test_divergent_record_counts_only_the_recording_lanes(lh, oracle, client):
    H = 11
    vals = np.concatenate([oracle.gen_stream(lh.STREAM_S, 1_000_003, SEED), edge_inputs(100)])
    n = vals.size
    ids = oracle.gen_ids(0, n, H, SEED).astype(np.uint32)
    ids[::57] = H
    mask = (vals.view(np.uint64) & np.uint64(1)) == 1
    assert 0.2 < mask.mean() < 0.8
    want = oracle.ingest_keyed(ids[mask & (ids < H)], vals[mask & (ids < H)], H)
    with lh.Engine(device=0, max_histograms=H) as eng:
        d_v, d_i = eng.upload(vals), eng.upload(ids)
        with eng.recording() as rec:
            launch(client, "lhc_record_subset", eng, rec, d_i.ptr, d_v.ptr, n)
        _, sp = eng.snapshot(PS)
        eng.sync()
        assert (dense_all(sp, H) == want).all()
        assert eng.stats()["dropped"] == int((mask & (ids >= H)).sum())


def test_record_ns_matches_timer_ingest(lh, oracle, client):
    """float64(ns) with round-to-nearest-even: negative durations and values above 2^53 included."""
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
            launch(client, "lhc_record_ns", eng, rec, d_i.ptr, d_n.ptr, n)
        red_d, sp_d = eng.snapshot(PS)
        eng.sync()
        assert (dense_all(sp_d, H) == want).all()
        assert eng.stats()["dropped"] == int((~keep).sum())
        eng.ingest_keyed_i64ns_u16(eng.upload(ids.astype(np.uint16)), d_n, n)
        red_k, sp_k = eng.snapshot(PS)
        assert (dense_all(sp_k, H) == want).all()
        assert red_d.pkeys.tobytes() == red_k.pkeys.tobytes() and red_d.sums.tobytes() == red_k.sums.tobytes()


def test_count_matches_counter_add(lh, oracle, client):
    """Wrapping uint64 adds, ids >= C dropped and counted."""
    Cn = 9
    n = 300_007
    rng = np.random.default_rng(SEED)
    ids = rng.integers(0, Cn + 3, n).astype(np.uint32)
    amounts = rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + np.uint64(1)   # wraps many times
    keep = ids < Cn
    want = oracle.counter_add(ids[keep], amounts[keep], Cn)
    with lh.Engine(device=0, max_histograms=1, max_counters=Cn) as eng:
        d_i, d_a = eng.upload(ids), eng.upload(amounts)
        with eng.recording() as rec:
            launch(client, "lhc_count", eng, rec, d_i.ptr, d_a.ptr, n)
        _, sp = eng.snapshot(PS)
        eng.sync()
        assert (sp.counter_deltas == want).all()
        assert eng.stats()["dropped"] == int((~keep).sum())
        eng.counter_add_u16(eng.upload(ids.astype(np.uint16)), d_a, n)
        _, sp2 = eng.snapshot(PS)
        assert (sp2.counter_deltas == want).all()


def test_constant_stream_from_a_full_grid(lh, oracle, client):
    """Every lane of every warp records the same value: the warp combining must add exactly n to one bucket."""
    n = 132 * 8 * 256 * 5
    vals = np.full(n, 4.2e5, dtype=np.float64)
    key = int(oracle.compress(4.2e5)) & 0xFFFF
    with lh.Engine(device=0, max_histograms=2) as eng:
        d_v = eng.upload(vals)
        with eng.recording() as rec:
            launch(client, "lhc_record", eng, rec, None, d_v.ptr, n)
        red, sp = eng.snapshot(PS)
        assert sp.histogram(0) == {key - 65536 if key >= 32768 else key: n}
        assert int(red.counts[0]) == n and int(red.counts[1]) == 0


def test_snapshot_waits_for_open_scopes(lh, oracle, client):
    """Thread A holds a scope for ~300 ms after launching its records; thread B's lh_snapshot_begin returns only after
    A's lh_record_end and its snapshot holds all of A's records.  A scope opened after B's flip, and ingest calls
    issued meanwhile, return at once and land in the next interval."""
    H = 4
    a_vals = oracle.gen_stream(lh.STREAM_L, 500_000, SEED)
    d_vals = oracle.gen_stream(lh.STREAM_U, 300_000, SEED)
    c_vals = oracle.gen_stream(lh.STREAM_S, 200_000, SEED)
    with lh.Engine(device=0, max_histograms=H) as eng:
        d_a, d_d, d_c = eng.upload(a_vals), eng.upload(d_vals), eng.upload(c_vals)
        ids_a = eng.upload(np.zeros(a_vals.size, np.uint32))
        ids_d = eng.upload(np.ones(d_vals.size, np.uint32))
        ids_c = eng.upload(np.full(c_vals.size, 2, np.uint16))
        t = {}
        a_open = threading.Event()
        errors = []

        def thread_a():
            try:
                rec = eng.record_begin()
                launch(client, "lhc_record", eng, rec, ids_a.ptr, d_a.ptr, a_vals.size)
                a_open.set()
                time.sleep(0.3)
                t["a_end"] = time.monotonic()
                eng.record_end(rec)
            except Exception as e:          # pragma: no cover - reported below
                errors.append(e)
                a_open.set()

        def thread_b():
            try:
                eng.snapshot_begin()
                t["b_ret"] = time.monotonic()
            except Exception as e:          # pragma: no cover
                errors.append(e)

        ta = threading.Thread(target=thread_a)
        ta.start()
        assert a_open.wait(10)
        tb = threading.Thread(target=thread_b)
        tb.start()
        time.sleep(0.08)                       # B has flipped the buffers and waits for A
        assert "b_ret" not in t
        with eng.recording() as rec:           # opened after the flip: next interval
            launch(client, "lhc_record", eng, rec, ids_d.ptr, d_d.ptr, d_vals.size)
        eng.ingest_keyed_f64_u16(ids_c, d_c, c_vals.size)
        t["c_ret"] = time.monotonic()
        ta.join(10)
        tb.join(10)
        assert not ta.is_alive() and not tb.is_alive() and not errors, errors
        assert t["c_ret"] < t["a_end"], "scopes and ingest after the flip must not wait for the open scope"
        assert t["b_ret"] >= t["a_end"], "lh_snapshot_begin returned before the scope ended"
        red = eng.snapshot_reduce(PS)
        sp = eng.snapshot_export()
        eng.snapshot_end()
        got = dense_all(sp, H)
        assert (got[0] == oracle.ingest(a_vals)).all() and int(red.counts.sum()) == a_vals.size
        _, sp2 = eng.snapshot(PS)
        got2 = dense_all(sp2, H)
        assert int(got2[0].sum()) == 0
        assert (got2[1] == oracle.ingest(d_vals)).all() and (got2[2] == oracle.ingest(c_vals)).all()


def test_scope_error_paths(lh, client):
    with lh.Engine(device=0, max_histograms=2) as eng:
        rec = eng.record_begin()
        assert eng.lib.lh_snapshot_begin(eng.h) == LH_ERR_STATE       # this thread holds the scope: no deadlock
        assert eng.lib.lh_destroy(eng.h) == LH_ERR_STATE              # scopes open
        eng.record_end(rec)
        assert eng.lib.lh_record_end(eng.h, C.byref(rec)) == LH_ERR_INVALID
        bogus = type(rec)()
        bogus.scope = 12345
        assert eng.lib.lh_record_end(eng.h, C.byref(bogus)) == LH_ERR_INVALID
        # with no scope open the snapshot behaves as before
        red, _ = eng.snapshot(PS)
        assert int(red.counts.sum()) == 0


def test_records_on_two_contexts_allreduce(lh, oracle, client):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    H, n = 6, 1_000_003
    vals = oracle.gen_stream(lh.STREAM_S, n, SEED ^ 2)
    ids = oracle.gen_ids(0, n, H, SEED ^ 2).astype(np.uint32)
    want = oracle.ingest_keyed(ids, vals, H)
    engs = [lh.Engine(device=d, max_histograms=H) for d in (0, 1)]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, 2, handles)
        half = n // 2
        for r, e in enumerate(engs):
            a, b = (0, half) if r == 0 else (half, n)
            d_v, d_i = e.upload(vals[a:b]), e.upload(ids[a:b])
            with e.recording() as rec:
                launch(client, "lhc_record", e, rec, d_i.ptr, d_v.ptr, b - a)
        for e in engs:
            e.snapshot_begin()
            e.snapshot_allreduce()
        for e in engs:
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
            e.snapshot_end()
            assert e.comm_info()["status"] == 0
            assert (dense_all(sp, H) == want).all()
            assert (red.counts == want.sum(axis=1)).all()
    finally:
        for e in engs:
            e.close()
