"""Ingest from several streams into one context, and from several live contexts of different precisions and H on one
device, against the oracle.

Streams are held back by bounded spins of different lengths (tests/gpu_timer_client.cu, built by build()), so that
kernels run in another order than they were issued and kernels of different streams overlap.  Every check is exact:
every bucket of every histogram the interval touched, the counts, percentile keys and values of the reduction, every
counter and the dropped tally."""
import ctypes as C
import threading

import numpy as np
import pytest

import _ingest_routes as R
from _op_sequences import PS, Want, check, check_reduced

pytestmark = pytest.mark.gpu

SEED = 0x5EA4ED
MS = 1_000_000                     # one millisecond of spin, in ns
SPECIALS = np.array([np.inf, -np.inf, np.nan, 2.0 ** 63, -(2.0 ** 64), 0.0, -0.0, 5e-324, 1e300], np.float64)
AMOUNTS = np.array([2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, 1 << 63], np.uint64)   # carry out of either half


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def spin():
    """spin(ns, stream): enqueue one bounded spin of at least `ns` on a torch stream."""
    from loghisto_b200 import build
    lib = C.CDLL(build.TIMER_CLIENT_LIB)
    lib.gtc_set_device.argtypes = [C.c_int]
    lib.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    lib.gtc_set_device.restype = lib.gtc_spin.restype = C.c_int
    assert lib.gtc_set_device(0) == 0

    def run(ns, stream):
        assert lib.gtc_spin(int(ns), stream.cuda_stream) == 0
    return run


def values(oracle, n, seed):
    """Stream S, with every 7th sample from stream N (random sign: the exact route), every 5th from stream L and a
    special value (non-finite, past 2^63, zeros, subnormal) every 1009th."""
    v = oracle.gen_stream(oracle.STREAM_S, n, seed)
    v[::7] = oracle.gen_stream(oracle.STREAM_N, n, seed + 1)[::7]
    v[3::5] = oracle.gen_stream(oracle.STREAM_L, n, seed + 2)[3::5]
    v[2::1009] = SPECIALS[np.arange(v[2::1009].size) % SPECIALS.size]
    return v


def nanos(oracle, n, seed):
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, seed).view(np.int64).copy()
    ns[::5] *= -1
    return ns


def keyed_ids(oracle, n, H, seed):
    """(u16 ids, u32 ids) that drop the same samples: u16 ids H and 65535, u32 ids 65536 + H - 1, 2^31 and 2^32 - 1."""
    ids = oracle.gen_ids(0, n, H, seed).astype(np.uint32)
    return (R.with_bad_ids(ids, np.array([H, 65535], np.uint32), 997).astype(np.uint16),
            R.with_bad_ids(ids, R.high_ids(H, H - 1), 997))


def counter_batch(n, C, seed):
    """(u16 ids, u32 ids, amounts): one hot counter, ids past C in both widths, amounts that carry."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, min(C, 65536), n).astype(np.uint32)
    ids[::3] = 5
    amounts = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    amounts[::2] = AMOUNTS[np.arange(amounts[::2].size) % AMOUNTS.size]
    ids16 = R.with_bad_ids(ids, np.array([65535], np.uint32), 89)
    ids32 = R.with_bad_ids(ids, R.high_ids(min(C, 65536), 5), 89)
    return ids16.astype(np.uint16), ids32, amounts


def timed_since(e, seq0):
    """Every ingest sequence number after seq0 has a finite, positive kernel time; returns the last one.  The library
    keeps the last 16 pairs of events, so callers check at most that many at a time."""
    seq = e.ingest_seq()
    assert 0 < seq - seq0 <= 16, (seq0, seq)
    for q in range(seq0 + 1, seq + 1):
        ms = e.kernel_ms(q)
        assert np.isfinite(ms) and ms > 0, (q, ms)
    return seq


def k1_indices(e):
    return [i for i, name in enumerate(e.k1_variants()) if not name.startswith("probe")]


# ------------------------------------------------------------------------------------------------ one context, 4 streams
@pytest.mark.parametrize("H,keyed_mode,C", [(5, 0, 8192), (300, 1, 8193)])
def test_every_route_from_four_streams(lh, oracle, torch, spin, sms, H, keyed_mode, C):
    """K1 (every variant, into one histogram and into distinct ones), keyed (small at H = 5, vector at H = 300), both
    counter kernels, GPU timer stops and host-fed calls, issued round-robin on 4 streams each held by a spin of a
    different length, with host-fed calls on the ingest stream in between: one snapshot holds exactly their union."""
    precision, n1, nk, nc = 100, 1_000_003, (1 << 20) + 3, 100_003
    kernel = R.keyed_route(H, nk, precision, sms, keyed_mode=keyed_mode).kernel
    assert kernel == (R.SMALL if H == 5 else R.VEC)
    assert R.counter_route(C, nc).kernel == (R.COUNTER_SMEM if C <= R.CONST["K2_SMEM_COUNTERS"] else R.COUNTER_GLOBAL)
    vals, ns = values(oracle, nk + 4, SEED ^ H), nanos(oracle, nk + 4, SEED ^ H)
    ids16, ids32 = keyed_ids(oracle, nk + 4, H, SEED ^ H)
    cids16, cids32, amounts = counter_batch(nc + 4, C, SEED ^ C)
    streams = [torch.cuda.Stream() for _ in range(4)]

    def hold(rnd):
        for i, st in enumerate(streams):
            spin((2 + 2 * ((i + rnd) % 4)) * MS, st)

    with lh.Engine(device=0, max_histograms=H, max_counters=C, staging_bytes=4 << 20) as e:
        e.tune("keyed_mode", keyed_mode)
        d_v, d_n, d_i16, d_i32 = e.upload(vals), e.upload(ns), e.upload(ids16), e.upload(ids32)
        d_c16, d_c32, d_a = e.upload(cids16), e.upload(cids32), e.upload(amounts)
        d_t = torch.zeros(8, dtype=torch.int64, device="cuda:0")
        torch.cuda.synchronize()
        want = Want(oracle, H, C, precision)
        before, seq = e.stats()["dropped"], e.ingest_seq()
        for rnd in range(2):
            # K1: every variant into histogram 1 and into a histogram of its own, from 4 streams
            hold(rnd)
            for j, vi in enumerate(k1_indices(e)):
                e.tune("k1", vi)
                off = (j + rnd) % 4
                e.ingest_f64(1, d_v.offset(off), n1, streams[j % 4])
                want.single(1, vals[off:off + n1])
                e.ingest_f64((2 + j) % H, d_v.offset(3 - off), n1 - j, streams[(j + 1) % 4])
                want.single((2 + j) % H, vals[3 - off:3 - off + n1 - j])
            e.ingest_f64_host(0, vals[:70_001])
            want.single(0, vals[:70_001])
            seq = timed_since(e, seq)
            # keyed: every id width and value type, the pair, a misaligned piece, and host-fed samples
            hold(rnd + 1)
            k = rnd * 2
            for name, call, id_bytes, ids, vv in (
                    ("f64_u16", lambda st: e.ingest_keyed_f64_u16(d_i16, d_v, nk, st), 2, ids16, vals),
                    ("f64_u32", lambda st: e.ingest_keyed_f64_u32(d_i32, d_v, nk, st), 4, ids32, vals),
                    ("i64ns_u16", lambda st: e.ingest_keyed_i64ns_u16(d_i16, d_n, nk, st), 2, ids16, ns)):
                call(streams[k % 4])
                k += 1
                assert e.keyed_kernel_name() == R.keyed_route(H, nk, precision, sms, id_bytes=id_bytes,
                                                              keyed_mode=keyed_mode).kernel, name
                want.hist(ids[:nk], vv[:nk].astype(np.float64))
            e.ingest_keyed_pair_u16(d_i16, d_v, nk, d_i16, d_n, nk, streams[k % 4])
            assert e.keyed_kernel_name() == kernel
            want.hist(ids16[:nk], vals[:nk])
            want.hist(ids16[:nk], ns[:nk].astype(np.float64))
            e.ingest_keyed_f64_u16(d_i16.offset(1), d_v.offset(2), 200_001, streams[(k + 1) % 4])
            assert e.keyed_kernel_name() == R.SCALAR                      # ids 2-byte aligned only: the scalar kernel
            want.hist(ids16[1:200_002], vals[2:200_003])
            e.ingest_keyed_f64_u16_host(ids16[:90_001], vals[:90_001])
            want.hist(ids16[:90_001], vals[:90_001])
            seq = timed_since(e, seq)
            # counters: vector body with ragged ends, misaligned, u32 ids past 16 bits; host-fed
            hold(rnd + 2)
            for j, (off, m) in enumerate(((0, nc), (1, nc - 1), (3, 20_000))):
                e.counter_add_u16(d_c16.offset(off), d_a.offset(off), m, streams[j % 4])
                want.counter(cids16[off:off + m], amounts[off:off + m])
                e.counter_add_u32(d_c32.offset(off), d_a.offset(off), m, streams[(j + 2) % 4])
                want.counter(cids32[off:off + m], amounts[off:off + m])
            e.counter_add_u16_host(cids16[:5_000], amounts[:5_000])
            want.counter(cids16[:5_000], amounts[:5_000])
            seq = timed_since(e, seq)
            # GPU timers: start and stop on each stream around a spin; the durations go to histogram 3
            hold(rnd + 3)
            for i, st in enumerate(streams):
                t = e.gpu_timer_start(st)
                spin((i + 1) * 100_000, st)
                e.gpu_timer_stop(t, 3, st, d_out=d_t[4 * rnd + i:4 * rnd + i + 1])
                e.gpu_timer_release(t)
            e.ingest_f64_host(4, vals[5:40_005])
            want.single(4, vals[5:40_005])
            seq = timed_since(e, seq)
        red, sp = e.snapshot(PS)
        durs = d_t.cpu().numpy()
        assert (durs >= np.tile((np.arange(4) + 1) * 100_000, 2)).all(), durs
        want.single(3, durs.astype(np.float64))
        check(e, want, ("four streams", H), before, snap=(red, sp))
        for x in (d_v, d_n, d_i16, d_i32, d_c16, d_c32, d_a):
            x.free()


# ------------------------------------------------------------------------------------- interval boundaries, stalled streams
def issue_batch(e, oracle, want, st, vals, ids, cids, amounts, hid):
    """K1 into `hid`, keyed and counters from the host arrays (uploaded first) on stream `st`; returns the buffers."""
    bufs = [e.upload(vals), e.upload(ids), e.upload(cids), e.upload(amounts)]
    d_v, d_i, d_c, d_a = bufs
    e.ingest_f64(hid, d_v, vals.size, st)
    want.single(hid, vals)
    e.ingest_keyed_f64_u16(d_i, d_v, vals.size, st)
    want.hist(ids, vals)
    e.counter_add_u16(d_c, d_a, cids.size, st)
    want.counter(cids, amounts)
    return bufs


def test_interval_boundaries_with_stalled_streams(lh, oracle, torch, spin):
    """Batch X on a stalled stream, snapshot_begin, then batch Y on the same still-stalled stream and on a second
    one: the first interval holds X alone and the next Y alone.  Then the same with the reduction of each interval
    collected only after the next interval's ingest has been issued (snapshot_reduce_async)."""
    H, C, n = 6, 16, 300_007
    vals = values(oracle, 8 * n, SEED ^ 0x1B)
    ids, _ = keyed_ids(oracle, 8 * n, H, SEED ^ 0x1B)
    cids, _, amounts = counter_batch(8 * n, C, SEED ^ 0x1C)

    def part(i):
        s = slice(i * n, (i + 1) * n - i)          # ragged lengths
        return vals[s], ids[s], cids[s], amounts[s]

    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with lh.Engine(device=0, max_histograms=H, max_counters=C) as e:
        before = e.stats()["dropped"]
        x, y = Want(oracle, H, C), Want(oracle, H, C)
        spin(30 * MS, A)
        bufs = issue_batch(e, oracle, x, A, *part(0), hid=1)
        e.snapshot_begin()
        bufs += issue_batch(e, oracle, y, A, *part(1), hid=2)
        spin(3 * MS, B)
        bufs += issue_batch(e, oracle, y, B, *part(2), hid=1)
        try:
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
        finally:
            e.snapshot_end()
        check(e, x, "X", snap=(red, sp))
        check(e, y, "Y")
        assert e.stats()["dropped"] - before == x.dropped + y.dropped
        # pipelined: interval k's reduction is collected after interval k+1's ingest was issued
        wants, handles = [], []
        for i in range(4):
            w = Want(oracle, H, C)
            spin((4 + 3 * i) * MS, A)
            spin((10 - 2 * i) * MS, B)
            bufs += issue_batch(e, oracle, w, A, *part(3 + i), hid=i % H)
            if i % 2:
                bufs += issue_batch(e, oracle, w, B, *part(7), hid=(i + 3) % H)
            e.snapshot_begin()
            handles.append(e.snapshot_reduce_async(PS))
            e.snapshot_end()
            wants.append(w)
            if i:
                check_reduced(e.snapshot_result(handles[i - 1]), wants[i - 1], ("pipelined", i - 1))
        check_reduced(e.snapshot_result(handles[-1]), wants[-1], ("pipelined", 3))
        for d in bufs:
            d.free()


# ------------------------------------------------------------------------------------- hot-window guard across streams
@pytest.mark.parametrize("keyed_mode,H", [(0, 2), (1, 301)])
def test_hot_window_guard_across_streams(lh, oracle, torch, spin, sms, keyed_mode, H):
    """Stream A, held by a spin, takes 3 calls of N = 2^30 + 2^20 constant samples; stream B then takes one.  The host
    tally of the uint32 hot window reaches the guard at B's call, so B drains the window first: that drain must come
    after A's kernels, or 4 N > 2^32 samples pile up in one uint32 cell.  keyed_mode 0 at H = 2 runs the shared-memory
    kernel; keyed_mode 1 at H = 301 the L2-atomic kernel with one copy of the window (every sample on one cell)."""
    N = (1 << 30) + (1 << 20)
    plan = R.hot_window_plan([N] * 4)
    assert all("fold" not in ev for ev in plan[:3]) and plan[3][0] == "fold"
    assert 4 * N > 1 << 32
    kernel = R.keyed_route(H, N, 100, sms, keyed_mode=keyed_mode).kernel
    assert kernel == (R.SMALL, R.VEC)[keyed_mode]
    if keyed_mode == 1:
        assert H * 2 * R.window(100) * 4 * 2 > 20 << 20          # hot_replicas = 1 (lh_create keeps the copies in 20 MB)
    sentinels = np.array([0, 12_345, N // 2, N - 1], np.int64)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        e.tune("keyed_mode", keyed_mode)
        d_v, d_i = None, None
        try:
            d_v = e.gen_stream(lh.STREAM_C, N, SEED)                         # 8.6 GB
            d_i = torch.zeros(N, dtype=torch.int16, device="cuda:0")         # every id 0 ...
            d_i[torch.as_tensor(sentinels, device="cuda:0")] = 1             # ... but a few in histogram 1
            torch.cuda.synchronize()
            e.sync()
            spin(100 * MS, A)
            for _ in range(3):
                e.ingest_keyed_f64_u16(d_i, d_v, N, A)
            e.ingest_keyed_f64_u16(d_i, d_v, N, B)
            assert e.keyed_kernel_name() == kernel
            red, sp = e.snapshot(PS)
        finally:                                                              # 10.7 GB: give it back even on a failure
            if d_v is not None:
                e.sync()
                d_v.free()
            del d_i
            torch.cuda.empty_cache()
    key = int(oracle.compress(float(oracle.gen_stream(oracle.STREAM_C, 1, SEED)[0])))
    in1 = 4 * sentinels.size
    assert sp.histogram(0) == {key: 4 * N - in1}
    assert sp.histogram(1) == {key: in1}
    assert int(red.counts[0]) == 4 * N - in1 and int(red.counts[1]) == in1 and int(red.counts.sum()) == 4 * N


# ------------------------------------------------------------------------------------- write-combining on two streams
@pytest.mark.parametrize("kp_chunk", ["default", "65536", "switch"])
def test_write_combining_from_two_streams(lh, oracle, torch, spin, sms, kp_chunk):
    """H = 1024: every keyed call takes the write-combining kernel, whose record queues and grid-barrier word belong to
    the context.  Calls of every id width, the int64 form and the fused pair alternate between two spun streams.
    65536-sample chunks make a launch cross many grid barriers; "switch" changes the chunk size (so the queues are
    re-allocated) while the other stream's launches are still queued."""
    H, precision, n = 1024, 100, (8 << 20) + 5
    chunk = {"default": R.DEFAULTS["kp_chunk"], "65536": 65536, "switch": 65536}[kp_chunk]
    route = R.keyed_route(H, n, precision, sms, kp_chunk=chunk)
    assert route.kernel == R.WC and R.pair_route(H, n, n, precision, sms, kp_chunk=chunk).kernel == R.WC
    if kp_chunk != "default":
        assert route.wc.nchunks > 8
    vals, ns = values(oracle, n, SEED ^ 0x4C), nanos(oracle, n, SEED ^ 0x4C)
    ids16, ids32 = keyed_ids(oracle, n, H, SEED ^ 0x4C)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        if kp_chunk == "65536":
            e.tune("kp_chunk", 65536)
        d_v, d_n, d_i16, d_i32 = e.upload(vals), e.upload(ns), e.upload(ids16), e.upload(ids32)
        torch.cuda.synchronize()
        before = e.stats()["dropped"]
        rounds = 3
        for rnd in range(rounds):
            spin((2 + 3 * rnd) * MS, A)
            spin((8 - 3 * rnd) * MS, B)
            one, other = (A, B) if rnd % 2 == 0 else (B, A)
            e.ingest_keyed_f64_u16(d_i16, d_v, n, one)
            assert e.keyed_kernel_name() == R.WC
            e.ingest_keyed_f64_u32(d_i32, d_v, n, other)
            assert e.keyed_kernel_name() == R.WC
            if kp_chunk == "switch" and rnd == 0:
                e.tune("kp_chunk", 65536)
            e.ingest_keyed_i64ns_u16(d_i16, d_n, n, one)
            assert e.keyed_kernel_name() == R.WC
            e.ingest_keyed_pair_u16(d_i16, d_v, n, d_i16, d_n, n, other)
            assert e.keyed_kernel_name() == R.WC
        want = Want(oracle, H, 1, precision)
        want.hist(ids16, vals, times=3 * rounds)          # f64_u16, f64_u32 (same drops) and the pair's float64 half
        want.hist(ids16, ns.astype(np.float64), times=2 * rounds)
        check(e, want, ("two streams", kp_chunk), before)
        for x in (d_v, d_n, d_i16, d_i32):
            x.free()


# ------------------------------------------------------------------------------------- contexts of different precisions
def ingest_and_check(e, oracle, precision, sms, seed):
    """K1 with every variant, keyed (the shared-memory kernel) and counters on `e`, checked at its precision."""
    H, C, n = e.H, e.C, 200_003
    vals = values(oracle, n + 3, seed)
    ids16, _ = keyed_ids(oracle, n, H, seed)
    cids, _, amounts = counter_batch(n, C, seed)
    want = Want(oracle, H, C, precision)
    before = e.stats()["dropped"]
    d_v, d_i, d_c, d_a = e.upload(vals), e.upload(ids16), e.upload(cids), e.upload(amounts)
    for j, vi in enumerate(k1_indices(e)):
        e.tune("k1", vi)
        e.ingest_f64(j % H, d_v.offset(j % 4), n - j)
        want.single(j % H, vals[j % 4:j % 4 + n - j])
    e.ingest_keyed_f64_u16(d_i, d_v, n)
    assert e.keyed_kernel_name() == R.keyed_route(H, n, precision, sms).kernel == R.SMALL
    want.hist(ids16, vals[:n])
    e.counter_add_u16(d_c, d_a, n)
    want.counter(cids, amounts)
    check(e, want, ("precision", precision), before)
    for x in (d_v, d_i, d_c, d_a):
        x.free()


def test_older_context_of_higher_precision(lh, oracle, sms):
    """A context at precision 100, then one at 50, both alive: the first one's launches (which need more shared
    memory than the second's) still run, and both match the oracle at their own precision."""
    with lh.Engine(device=0, max_histograms=3, max_counters=8, precision=100) as old:
        with lh.Engine(device=0, max_histograms=3, max_counters=8, precision=50) as new:
            ingest_and_check(old, oracle, 100, sms, SEED ^ 100)
            ingest_and_check(new, oracle, 50, sms, SEED ^ 50)
            ingest_and_check(old, oracle, 100, sms, SEED ^ 101)


def test_contexts_of_every_precision_alive_together(lh, oracle, sms):
    """Contexts at precisions 1 ... 250, including those on either side of where lh_create substitutes a smaller K1
    ring, all created first, from the highest precision down (each one needs less shared memory than every older one);
    then each ingests and is checked, in creation order and in reverse."""
    edges = set(R.k1_substitution_precisions().values())
    precisions = sorted({1, 50, 100, 102, 103, 200, 250} | edges | {p - 1 for p in edges}, reverse=True)
    engines = []
    try:
        for p in precisions:
            engines.append((p, lh.Engine(device=0, max_histograms=3, max_counters=8, precision=p)))
        for order in (engines, engines[::-1]):
            for p, e in order:
                ingest_and_check(e, oracle, p, sms, SEED ^ (p * 7))
    finally:
        for _, e in engines:
            e.close()


# ------------------------------------------------------------------------------------- contexts in threads
def test_contexts_in_threads(lh, oracle, torch, spin, sms):
    """4 threads, each with its own context, stream and configuration (the last one on the write-combining kernel),
    run K1, keyed and counter ingest and take a snapshot per round; every interval matches the oracle at that context's
    precision.  Meanwhile a fifth thread creates, uses and destroys contexts of other precisions."""
    configs = [(100, 3, 0), (50, 11, 0), (200, 40, 0), (100, 1024, 2)]     # (precision, H, keyed_mode)
    rounds, n, stride, C = 4, 400_003, 400_016, 16      # each round's slice starts 32-byte aligned
    errors = []
    stop = threading.Event()
    data = []
    for k, (precision, H, mode) in enumerate(configs):
        vals = values(oracle, rounds * stride, SEED ^ (k + 1))
        ids, _ = keyed_ids(oracle, rounds * stride, H, SEED ^ (k + 1))
        cids, _, amounts = counter_batch(rounds * stride, C, SEED ^ (k + 1))
        data.append((vals, ids, cids, amounts))

    def worker(k):
        precision, H, mode = configs[k]
        vals, ids, cids, amounts = data[k]
        kernel = R.keyed_route(H, n, precision, sms, keyed_mode=mode).kernel
        try:
            st = torch.cuda.Stream()
            with lh.Engine(device=0, max_histograms=H, max_counters=C, precision=precision) as e:
                e.tune("keyed_mode", mode)
                d_v, d_i, d_c, d_a = e.upload(vals), e.upload(ids), e.upload(cids), e.upload(amounts)
                for r in range(rounds):
                    a = r * stride
                    want = Want(oracle, H, C, precision)
                    before = e.stats()["dropped"]
                    spin((1 + k + r) * MS, st)
                    e.ingest_f64(r % H, d_v.offset(a), n, st)
                    want.single(r % H, vals[a:a + n])
                    e.ingest_keyed_f64_u16(d_i.offset(a), d_v.offset(a), n, st)
                    assert e.keyed_kernel_name() == kernel, (k, r)
                    want.hist(ids[a:a + n], vals[a:a + n])
                    e.counter_add_u16(d_c.offset(a), d_a.offset(a), n, st)
                    want.counter(cids[a:a + n], amounts[a:a + n])
                    check(e, want, ("thread", k, r), before)
                for x in (d_v, d_i, d_c, d_a):
                    x.free()
        except BaseException as ex:   # pragma: no cover - reported below
            errors.append((k, ex))

    def churn():
        i = 0
        try:
            while not stop.is_set() or i < 2:
                p = (7, 250, 103)[i % 3]
                with lh.Engine(device=0, max_histograms=2, max_counters=1, precision=p) as e:
                    v = values(oracle, 50_001, SEED ^ i)
                    d = e.upload(v)
                    e.ingest_f64(1, d, v.size)
                    _, sp = e.snapshot(PS)
                    got = np.zeros(65536, np.uint64)
                    for key, c in sp.histogram(1).items():
                        got[key & 0xFFFF] = c
                    assert (got == oracle.ingest(v, precision=p)).all(), ("churn", p)
                    d.free()
                i += 1
        except BaseException as ex:   # pragma: no cover - reported below
            errors.append(("churn", ex))

    assert R.keyed_route(1024, n, 100, sms, keyed_mode=2).kernel == R.WC
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(len(configs))]
    ch = threading.Thread(target=churn)
    ch.start()
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    stop.set()
    ch.join()
    assert not errors, errors


# ------------------------------------------------------------------------------------- two MetricSystems
def test_metric_systems_of_different_precisions(oracle, torch):
    """A MetricSystem at the reference's precision, then one at precision 50: a record scope's histogram() on the
    older one still works and matches the oracle's port of metrics.go; the newer one matches the oracle at 50."""
    from loghisto_b200.metric_system import MetricSystem
    from _name_recycling_cases import _compare_interval
    vals = oracle.gen_stream(oracle.STREAM_S, 20_011, SEED ^ 7)
    vals[::3] = oracle.gen_stream(oracle.STREAM_N, 20_011, SEED ^ 8)[::3]
    t = torch.from_numpy(vals).cuda()
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    old = MetricSystem(1e-6, False, max_histograms=8, max_counters=4)
    new = MetricSystem(1e-6, False, max_histograms=8, max_counters=4, precision=50)
    ref = oracle.OracleMetricSystem()
    try:
        with old.recording(st, histograms=["payload"]) as s:
            s.histogram("payload", t)
        for v in vals:
            ref.Histogram("payload", float(v))
        raw, m = old.collect_and_process()
        rraw, rm = ref.collect_and_process()
        _compare_interval(raw, m, rraw, rm)
        with new.recording(st, histograms=["payload"]) as s:
            s.histogram("payload", t)
        raw, _ = new.collect_and_process()
        got = np.zeros(65536, np.uint64)
        for key, c in raw["Histograms"]["payload"].items():
            got[int(key) & 0xFFFF] = c
        assert (got == oracle.ingest(vals, precision=50)).all()
        assert old.dropped() == 0 and new.dropped() == 0
    finally:
        ref.close()
        new.close()
        old.close()
