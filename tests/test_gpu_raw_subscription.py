"""Raw device subscriptions (lh_raw_board_*, lh_snapshot_publish_raw, lh_raw_percentiles / lh_raw_ranks,
MetricSystem::NewRawDeviceSubscription): each collection's running bucket counts published into device memory, with
exact percentile, rank and bucket queries from kernels, from the query calls and from captured graphs.

The querying kernels live in tests/raw_read_client.cu, a separate CUDA library built by build() that knows the engine
only through its public headers.  Bar: percentiles equal lh_snapshot_reduce and the exact reference of
tests/_reduce_cases.py bit for bit, bucket counts equal the export, ranks equal running sums of the export up to the
oracle's compress(v), answers through names equal the collection's RawMetricSet and processMetrics, readers beside
hundreds of collections never see a torn answer, captured queries follow the latest publish, and a collection without
a raw subscription issues the same work as before."""
import ctypes as C
import math
import os
import time

import numpy as np
import pytest

import _reduce_cases as rc

pytestmark = pytest.mark.gpu

INT32_MIN = -(1 << 31)
UNBOUND = 0xFFFFFFFF
LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = -1, -5, -6
SEED = 0x5A3B1E


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
    assert os.path.exists(build.RAW_CLIENT_LIB), "build() did not produce " + build.RAW_CLIENT_LIB
    lib = C.CDLL(build.RAW_CLIENT_LIB)
    bp, vp, u32 = C.POINTER(_lib.lh_raw_board), C.c_void_p, C.c_uint32
    lib.rrc_percentiles.argtypes = [bp, vp, vp, u32, vp, vp, vp, vp]
    lib.rrc_ranks.argtypes = [bp, vp, vp, u32, vp, vp, vp, vp]
    lib.rrc_bucket_counts.argtypes = [bp, vp, vp, u32, vp, vp, vp]
    lib.rrc_torn_start.argtypes = [bp, C.c_double, C.c_double, vp, vp, vp, C.c_int, C.c_uint64, vp, vp]
    lib.rrc_cost.argtypes = [bp, u32, C.c_int, vp, vp]
    for name in ("rrc_percentiles", "rrc_ranks", "rrc_bucket_counts", "rrc_torn_start", "rrc_cost"):
        getattr(lib, name).restype = C.c_int
    return lib


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def cuda(torch, a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def host(torch, *ts):
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in ts]


def kernel_percentiles(torch, client, board, rows, ps):
    r, p = cuda(torch, rows, np.uint32), cuda(torch, ps, np.float64)
    keys = torch.empty(len(rows), dtype=torch.int32, device="cuda")
    vals = torch.empty(len(rows), dtype=torch.float64, device="cuda")
    pub = torch.empty(len(rows), dtype=torch.int64, device="cuda")
    assert client.rrc_percentiles(C.byref(board), r.data_ptr(), p.data_ptr(), len(rows), keys.data_ptr(),
                                  vals.data_ptr(), pub.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    return host(torch, keys, vals, pub)


def kernel_ranks(torch, client, board, rows, values):
    r, v = cuda(torch, rows, np.uint32), cuda(torch, values, np.float64)
    ranks, totals, pub = (torch.empty(len(rows), dtype=torch.int64, device="cuda") for _ in range(3))
    assert client.rrc_ranks(C.byref(board), r.data_ptr(), v.data_ptr(), len(rows), ranks.data_ptr(), totals.data_ptr(),
                            pub.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    return host(torch, ranks, totals, pub)


def kernel_bucket_counts(torch, client, board, rows, keys):
    r, k = cuda(torch, rows, np.uint32), cuda(torch, keys, np.int32)
    counts, pub = (torch.empty(len(rows), dtype=torch.int64, device="cuda") for _ in range(2))
    assert client.rrc_bucket_counts(C.byref(board), r.data_ptr(), k.data_ptr(), len(rows), counts.data_ptr(),
                                    pub.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    return host(torch, counts, pub)


def reference_keys(ref, ps):
    """Reference.percentile for every p at once: the first bucket in the reference's order whose ratio reaches p (the
    ratios are not monotone once the running count wraps at 2^64, and 0/0.0 is NaN, which reaches nothing)."""
    ps = np.asarray(ps, dtype=np.float64)
    if not ref.nnz:
        return np.full(ps.size, INT32_MIN, np.int32)
    best = np.fmax.accumulate(np.where(np.isnan(ref.ratios), -np.inf, ref.ratios))   # the largest ratio so far
    i = np.searchsorted(best, ps, side="left")
    order = np.array(ref.order + [INT32_MIN], dtype=np.int64)
    i[np.isnan(ps)] = ref.nnz
    return order[np.minimum(i, ref.nnz)].astype(np.int32)


def dense_export(sp, H):
    d = np.zeros((H, 65536), dtype=np.uint64)
    for h in range(H):
        a, b = int(sp.offsets[h]), int(sp.offsets[h + 1])
        d[h, sp.keys[a:b].astype(np.int64) + 32768] = sp.counts[a:b]
    return d


def rank_values(precision, w):
    """Values at and one ulp beside the bucket boundaries around the fast window's edges and 0, both signs, and the
    special values."""
    out = []
    for k in (1, 2, w - 2, w - 1, w, w + 1, 2 * w):
        v = math.expm1((k - 0.5) / precision)
        if math.isfinite(v):
            out += [math.nextafter(v, -math.inf), v, math.nextafter(v, math.inf)]
    out += [-v for v in out]
    out += [math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, 2.0 ** 63, -(2.0 ** 63), math.nextafter(2.0 ** 63, 0),
            2.0 ** 63 * 1.5, 1e300, -1e300, 2.0 ** 64]
    return np.array(out, dtype=np.float64)


@pytest.mark.parametrize("precision", rc.PRECISIONS)
def test_exact_on_constructed_histograms(lh, oracle, torch, client, precision):
    """Every case of tests/_reduce_cases.py in its own row: percentiles for the special ps, the crossings and one ulp
    beside them and 10^4 random ps equal lh_snapshot_reduce (batches of 32) and the reference bit for bit, from the grid
    call, the pair call and a kernel; every key's bucket count equals the export; ranks equal the export's running
    sums.  The last row is unbound and row k answers as empty, with publish number 0.  The cases of make_cases, then
    those whose counts wrap at 2^64 (running counts mod 2^64, as np.cumsum of uint64 gives them)."""
    table = oracle.decompress_table(precision)
    plain = rc.make_cases(precision, table, SEED)
    wrapped = rc.make_wrapped_cases(precision, table, SEED)
    for cases, pool in ((plain, rc.percentile_pool(plain, table, SEED)),
                        (wrapped, rc.wrapped_percentile_pool(wrapped, table, SEED))):
        exact_on_cases(lh, oracle, torch, client, table, precision, cases, pool)


def exact_on_cases(lh, oracle, torch, client, table, precision, cases, pool):
    H = 64
    assert len(cases) < H
    refs = [rc.Reference(c["hist"], table, c["name"]) for c in cases] + [rc.Reference({}, table, "untouched")] * (H - len(cases))
    refs[H - 1] = rc.Reference({}, table, "unbound")
    rng = np.random.default_rng(SEED + precision)
    ps = np.array(pool + list(rng.random(10_000) * 1.1 - 0.05), dtype=np.float64)
    ids, keys, counts = rc.merge_triples(cases)
    hid = list(range(H - 1)) + [UNBOUND]
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng, eng.raw_board(H) as rb:
        eng.merge_counts_host(ids, keys, counts)
        eng.snapshot_begin()
        try:
            rb.publish(hid)
            sp = eng.snapshot_export()
            want_k = np.empty((H, ps.size), np.int32)
            want_v = np.empty((H, ps.size), np.float64)
            for b0 in range(0, ps.size, 32):
                red = eng.snapshot_reduce(list(ps[b0:b0 + 32]))
                want_k[:, b0:b0 + 32] = red.pkeys
                want_v[:, b0:b0 + 32] = red.pvals
        finally:
            eng.snapshot_end()
        want_k[H - 1], want_v[H - 1] = INT32_MIN, math.nan
        for h, ref in enumerate(refs):
            assert (reference_keys(ref, ps) == want_k[h]).all(), (precision, h, ref.name)
        # grid call (Python), pair call (C ABI) and a kernel
        gk, gv, gp = host(torch, *rb.percentiles(cuda(torch, ps)))
        assert (gk == want_k).all() and (bits(gv) == bits(want_v)).all() and (gp == 1).all()
        rows = np.concatenate([np.repeat(np.arange(H), 64), [H, H + 7]]).astype(np.uint32)
        pp = np.concatenate([np.tile(ps[:64], H), [0.5, 0.5]])
        wk = np.concatenate([want_k[:, :64].ravel(), [INT32_MIN] * 2])
        wv = np.concatenate([want_v[:, :64].ravel(), [math.nan] * 2])
        ck, cv, cp = host(torch, *rb.percentiles(cuda(torch, pp), rows=cuda(torch, rows)))
        kk, kv, kp = kernel_percentiles(torch, client, rb.board, rows, pp)
        for k_, v_, p_ in ((ck, cv, cp), (kk, kv, kp)):
            assert (k_ == wk).all() and (bits(v_) == bits(wv)).all()
            assert (p_[:-2] == 1).all() and (p_[-2:] == 0).all()
        # bucket counts of every key of every row
        dense = dense_export(sp, H)
        rows = np.repeat(np.arange(H), 65536).astype(np.uint32)
        allkeys = np.tile(np.arange(-32768, 32768), H).astype(np.int32)
        bc, bp = kernel_bucket_counts(torch, client, rb.board, rows, allkeys)
        assert (bc.view(np.uint64) == dense.ravel()).all() and (bp == 1).all()
        # ranks
        vals = rank_values(precision, rc.window(precision))
        key = oracle.compress_many(vals, precision).astype(np.int64) + 32768
        cum = np.cumsum(dense, axis=1, dtype=np.uint64)
        want_r = cum[:, key]
        gr, gt, gp = host(torch, *rb.ranks(cuda(torch, vals)))
        assert (gr.view(np.uint64) == want_r).all() and (gt.view(np.uint64) == cum[:, -1]).all() and (gp == 1).all()
        rows = np.repeat(np.arange(H), vals.size).astype(np.uint32)
        vv = np.tile(vals, H)
        for r_, t_, p_ in (host(torch, *rb.ranks(cuda(torch, vv), rows=cuda(torch, rows))),
                           kernel_ranks(torch, client, rb.board, rows, vv)):
            assert (r_.view(np.uint64) == want_r.ravel()).all()
            assert (t_.view(np.uint64) == np.repeat(cum[:, -1], vals.size)).all() and (p_ == 1).all()


def test_queries_before_the_first_publish(lh, oracle, torch, client):
    """A new board answers as empty rows of publish 0 before anything is published, even when its memory held another
    board's running counts: ranks and totals 0 (NaN, +-Inf, +-0 and other values of bucket 0 included), bucket counts 0
    for every key, percentiles INT32_MIN / NaN."""
    H = 8
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        ids = (np.arange(80_000) % H).astype(np.uint16)
        vals = np.concatenate([np.zeros(40_000), oracle.gen_stream(lh.STREAM_U, 40_000, 11)])
        for _ in range(3):   # boards of the same size, published and freed: their cells go back to the pool
            eng.ingest_keyed_f64_u16_host(ids, vals)
            with eng.raw_board(H) as old:
                eng.snapshot_begin()
                old.publish(list(range(H)))
                eng.snapshot_end()
                r, t, p = host(torch, *old.ranks(cuda(torch, [0.0])))
                assert (r >= 5_000).all() and (t == 10_000).all() and (p == 1).all()   # key-0 cells non-zero
            eng.sync()
        with eng.raw_board(H) as rb:
            values = np.array([0.0, -0.0, math.nan, math.inf, -math.inf, 0.4e-2, -0.4e-2, 1.0, 1e300, -5.0])
            r, t, p = host(torch, *rb.ranks(cuda(torch, values)))
            assert (r == 0).all() and (t == 0).all() and (p == 0).all()
            rows = np.repeat(np.arange(H), values.size).astype(np.uint32)
            kr, kt, kp = kernel_ranks(torch, client, rb.board, rows, np.tile(values, H))
            assert (kr == 0).all() and (kt == 0).all() and (kp == 0).all()
            rows = np.repeat(np.arange(H), 65536).astype(np.uint32)
            bc, bp = kernel_bucket_counts(torch, client, rb.board, rows, np.tile(np.arange(-32768, 32768), H))
            assert (bc == 0).all() and (bp == 0).all()
            k, v, p = host(torch, *rb.percentiles(cuda(torch, [-1.0, 0.0, 0.5, 1.0])))
            assert (k == INT32_MIN).all() and np.isnan(v).all() and (p == 0).all()


LABELS = dict([("%%s_q%02d" % j, p) for j, p in enumerate([0.0, 1.0, 1.5, float("nan"), -0.5, 1e-300, 0.5, 0.99, 0.999])])


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_answers_through_names(lh, oracle, torch, client, precision):
    """Streams U / L / S through Histogram, a record scope and a graph recorder; names absent in some collections,
    never seen, recycled away (their id reused by churn names) and back: percentiles equal processMetrics' labels and
    ranks the running sums of the collection's Histograms."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4, precision=precision)
    labels = sorted(LABELS.items())
    ps_t = cuda(torch, [p for _, p in labels])
    try:
        ms.SpecifyPercentiles(LABELS)
        names = ["h0", "h1", "h2", "hr", "never"]
        with ms.raw_device_subscription(histograms=names) as sub, ms.graph_recorder(histograms=["h2"]) as g:
            assert sub.rows == {nm: i for i, nm in enumerate(names)}
            k0, _, p0 = host(torch, *sub.percentiles(ps_t))
            assert (k0 == INT32_MIN).all() and (p0 == 0).all()
            for j in range(9):
                kind = (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S)[j % 3]
                if j % 4 != 3:
                    ms.HistogramMany("h0", oracle.gen_stream(kind, 500 + 13 * j, 1000 * j))
                if j % 4 != 1:
                    x = cuda(torch, oracle.gen_stream(kind, 700 + 7 * j, 1000 * j + 1))
                    with ms.recording(torch.cuda.current_stream(), histograms=["h1"]) as s:
                        s.histogram("h1", x)
                if j % 3 != 2:
                    g.histograms({"h2": cuda(torch, oracle.gen_stream(kind, 300 + j, 1000 * j + 2))})
                    torch.cuda.synchronize()
                if j in (0, 7, 8):   # "hr" idles through collections 1..6: its id is freed and taken by churn names
                    ms.HistogramMany("hr", oracle.gen_stream(kind, 300, 77 + j))
                for t in range(3):
                    ms.Histogram("tmp%d_%d" % (j, t), 1.0 + t)
                raw, metrics = ms.collect_and_process()
                hs = raw["Histograms"]
                values = np.concatenate([oracle.gen_stream(kind, 40, 5 + j), [math.nan, math.inf, -math.inf, 0.0, -1.0]])
                keys, vals, pub = host(torch, *sub.percentiles(ps_t))
                ranks, totals, rpub = host(torch, *sub.ranks(cuda(torch, values)))
                assert (pub == j + 1).all() and (rpub == j + 1).all()
                vkeys = oracle.compress_many(values, precision)
                for i, nm in enumerate(names):
                    h = hs.get(nm)
                    if h is None:
                        assert (keys[i] == INT32_MIN).all() and np.isnan(vals[i]).all()
                        assert (ranks[i] == 0).all() and totals[i] == 0
                        continue
                    assert int(totals[i]) == sum(h.values())
                    for c, (label, _) in enumerate(labels):
                        name = label.replace("%s", nm, 1)
                        if keys[i, c] == INT32_MIN:
                            assert name not in metrics
                        else:
                            assert bits(vals[i, c]) == bits(metrics[name])
                    hk = np.array(sorted(h), dtype=np.int64)
                    hc = np.array([h[x] for x in sorted(h)], dtype=np.uint64)
                    cs = np.cumsum(hc, dtype=np.uint64)
                    idx = np.searchsorted(hk, vkeys.astype(np.int64), side="right")
                    want = np.where(idx > 0, cs[np.maximum(idx - 1, 0)], 0)
                    assert (ranks[i].view(np.uint64) == want).all(), (precision, j, nm)
                assert "never" not in hs and ("hr" in hs) == (j in (0, 7, 8))
    finally:
        ms.close()


def test_big_board_stages_ids(lh, oracle, torch):
    """A board of 4 104 rows (more ids than one parameter block) maps every row to its id; rows bound to one id twice
    agree."""
    H = 4104
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng, eng.raw_board(H) as rb:
        rng = np.random.default_rng(7)
        ids = rng.integers(0, H, 300_000).astype(np.uint16)
        eng.ingest_keyed_f64_u16_host(ids, oracle.gen_stream(lh.STREAM_L, ids.size, 9))
        hid = np.arange(H - 1, -1, -1).astype(np.uint32)   # row i -> id H-1-i
        hid[5] = UNBOUND
        hid[4100] = hid[4101]
        eng.snapshot_begin()
        try:
            rb.publish(hid)
            red = eng.snapshot_reduce([0.0, 0.5, 0.99, 1.0])
        finally:
            eng.snapshot_end()
        ps = cuda(torch, [0.0, 0.5, 0.99, 1.0])
        k, v, p = host(torch, *rb.percentiles(ps))
        bound = hid != UNBOUND
        assert (k[bound] == red.pkeys[hid[bound]]).all() and (bits(v[bound]) == bits(red.pvals[hid[bound]])).all()
        assert (k[5] == INT32_MIN).all() and (p == 1).all()
        _, t, _ = host(torch, *rb.ranks(cuda(torch, [1.0])))
        assert (t.view(np.uint64)[bound] == red.counts[hid[bound]]).all() and t[5] == 0


def test_two_contexts_allreduce(lh, oracle, torch):
    """Two contexts on one GPU all-reduced: each raw board holds the summed counts."""
    H = 6
    engs = [lh.Engine(device=0, max_histograms=H, max_counters=1) for _ in range(2)]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, 2, handles)
        boards = [e.raw_board(H) for e in engs]
        dense = np.zeros((H, 65536), np.uint64)
        for r, e in enumerate(engs):
            ids = (np.arange(20_000) % H).astype(np.uint16)
            vals = oracle.gen_stream(lh.STREAM_U if r else lh.STREAM_L, ids.size, 40 + r)
            e.ingest_keyed_f64_u16_host(ids, vals)
            np.add.at(dense, (ids.astype(np.int64), oracle.compress_many(vals).astype(np.int64) + 32768), 1)
        for e in engs:
            e.sync()
        for e in engs:
            e.snapshot_begin()
            e.snapshot_allreduce(False)
        reds = []
        for e, b in zip(engs, boards):
            b.publish(list(range(H)))
            reds.append(e.snapshot_reduce([0.25, 0.5, 0.9]))
            e.snapshot_end()
        cum = np.cumsum(dense, axis=1, dtype=np.uint64)
        vals = np.linspace(-3, 3000, 257)
        key = oracle.compress_many(vals).astype(np.int64) + 32768
        for red, b in zip(reds, boards):
            k, v, _ = host(torch, *b.percentiles(cuda(torch, [0.25, 0.5, 0.9])))
            assert (k == red.pkeys).all() and (bits(v) == bits(red.pvals)).all()
            r, t, _ = host(torch, *b.ranks(cuda(torch, vals)))
            assert (r.view(np.uint64) == cum[:, key]).all() and (t.view(np.uint64) == cum[:, -1]).all()
            assert int(t.sum()) == 40_000
        for b in boards:
            b.close()
    finally:
        for e in engs:
            e.close()


def test_captured_queries_follow_latest_publish(oracle, torch):
    """.percentiles and .ranks captured in one torch.cuda.graph and replayed after each of three collections: every
    replay answers from the latest publish, and its publish number advances."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4)
    try:
        ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p99": 0.99})
        with ms.raw_device_subscription(histograms=["lat", "idle"]) as sub:
            ps = cuda(torch, [0.5, 0.99])
            budget = cuda(torch, [50.0])
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                keys, vals, pub = sub.percentiles(ps)
                ranks, totals, rpub = sub.ranks(budget)
                share = ranks[:, 0].double() / totals.double()
            for j in range(1, 4):
                x = np.linspace(1.0, 100.0 * j, 1000)
                ms.HistogramMany("lat", x)
                raw, metrics = ms.collect_and_process()
                g.replay()
                k, v, p, r, t, rp, sh = host(torch, keys, vals, pub, ranks, totals, rpub, share)
                assert (p == j).all() and (rp == j).all()
                assert bits(v[0, 0]) == bits(metrics["lat_p50"]) and bits(v[0, 1]) == bits(metrics["lat_p99"])
                assert (k[1] == INT32_MIN).all() and t[1] == 0
                kb = int(oracle.compress(50.0))
                want = sum(c for key, c in raw["Histograms"]["lat"].items() if key <= kb)
                assert int(r[0, 0]) == want and int(t[0]) == 1000 and sh[0] == want / 1000
    finally:
        ms.close()


def test_no_torn_answers(oracle, torch, client):
    """A reader kernel on a few CTAs queries row 0 for a fixed %globaltimer budget while the host runs 200 collections
    that alternate two histograms with different totals: every answer is one of the two, of the publish it names."""
    from loghisto_b200.metric_system import MetricSystem
    n = 200
    ms = MetricSystem(1.0, False, max_histograms=16, max_counters=4)
    a = np.concatenate([np.full(100, 1.5), np.full(50, 1000.0), np.linspace(-5e6, 5e6, 4001)])
    b = np.full(30, 7.0)
    v = 10.0
    kv = int(oracle.compress(v))

    def expect(x):
        k = oracle.compress_many(x).astype(np.int64)
        srt = np.sort(k)
        return x.size, int((k <= kv).sum()), int(srt[(x.size + 1) // 2 - 1])   # p50: first key reaching ceil(n/2)

    ea, eb = expect(a), expect(b)
    try:
        with ms.raw_device_subscription(histograms=["t", "never"]) as sub:
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            stats = torch.zeros(5, dtype=torch.int64, device="cuda")
            stats[3] = -1
            side = torch.cuda.Stream()
            torch.cuda.synchronize()
            tot = (C.c_uint64 * 2)(ea[0], eb[0])
            rk = (C.c_uint64 * 2)(ea[1], eb[1])
            ky = (C.c_int32 * 2)(ea[2], eb[2])
            assert client.rrc_torn_start(C.byref(sub.board), v, 0.5, tot, rk, ky, max(sms // 4, 1), 4_000_000_000,
                                         stats.data_ptr(), side.cuda_stream) == 0
            t0 = time.monotonic()
            for j in range(1, n + 1):
                ms.HistogramMany("t", a if j % 2 else b)
                ms.collect_and_process()
            host_s = time.monotonic() - t0
            side.synchronize()
            reads, bad, hi, lo, changes = [int(x) for x in stats.cpu().numpy().view(np.uint64)]
            assert bad == 0, (reads, bad, hi, lo, changes)
            assert reads > 0 and hi > lo >= 1 and changes > 0, (reads, hi, lo, changes)
            if host_s < 2.0:
                assert hi == n
    finally:
        ms.close()


def test_no_change_without_a_raw_subscription(oracle):
    """A collection issues one more launch while a raw subscription is open, and the same launches as before once it
    is closed."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4)
    try:
        ms.SpecifyPercentiles({"%s_p50": 0.5})

        def collect():
            ms.HistogramMany("a", oracle.gen_stream(0, 1000, 3))
            before = ms.stats()["kernel_launches"]
            ms.collect_and_process()
            return ms.stats()["kernel_launches"] - before

        plain = [collect() for _ in range(3)]
        with ms.raw_device_subscription(histograms=["a", "b"]):
            with_sub = [collect() for _ in range(3)]
        after = [collect() for _ in range(3)]
        assert plain == after and len(set(plain)) == 1
        assert with_sub == [plain[0] + 1] * 3
    finally:
        ms.close()


def test_validation(lh, torch):
    """Every refusal returns its status and enqueues nothing: k 0 or > H, ids out of range, publish outside a
    snapshot, NULL or misaligned query arrays, destroyed and foreign handles; n == 0 enqueues nothing."""
    from loghisto_b200 import _lib as L
    with lh.Engine(device=0, max_histograms=4, max_counters=1) as eng, lh.Engine(device=0, max_histograms=4) as other:
        lib = eng.lib
        b = L.lh_raw_board()
        before = eng.stats()["kernel_launches"]
        assert lib.lh_raw_board_create(eng.h, 0, C.byref(b)) == LH_ERR_INVALID
        assert lib.lh_raw_board_create(eng.h, 5, C.byref(b)) == LH_ERR_RANGE
        assert lib.lh_raw_board_create(eng.h, 1, None) == LH_ERR_INVALID
        rb = eng.raw_board(4)
        assert rb.board.k == 4 and rb.board.d_decomp
        bb = C.byref(rb.board)
        assert lib.lh_snapshot_publish_raw(eng.h, bb, None) == LH_ERR_STATE          # no snapshot
        rows = torch.zeros(8, dtype=torch.int32, device="cuda")
        f = torch.zeros(16, dtype=torch.float64, device="cuda")
        i32 = torch.zeros(16, dtype=torch.int32, device="cuda")
        u = torch.zeros(16, dtype=torch.int64, device="cuda")
        r, x, k, v, pu = rows.data_ptr(), f.data_ptr(), i32.data_ptr(), f.data_ptr() + 64, u.data_ptr()
        for args in ((None, x, 4, k, v, pu), (r, None, 4, k, v, pu), (r, x, 4, None, v, pu), (r, x, 4, k, None, pu),
                     (r, x, 4, k, v, None), (r + 2, x, 4, k, v, pu), (r, x + 4, 4, k, v, pu), (r, x, 4, k + 2, v, pu),
                     (r, x, 4, k, v + 4, pu), (r, x, 4, k, v, pu + 4)):
            assert lib.lh_raw_percentiles(eng.h, bb, *args, None) == LH_ERR_INVALID, args
            assert lib.lh_raw_ranks(eng.h, bb, *args[:3], u.data_ptr() if args[3] == k else args[3],
                                    args[4], args[5], None) == LH_ERR_INVALID, args
        assert lib.lh_raw_percentiles_grid(eng.h, bb, None, 2, k, v, pu, None) == LH_ERR_INVALID
        assert lib.lh_raw_ranks_grid(eng.h, bb, x, 2, pu, v, pu + 4, None) == LH_ERR_INVALID
        assert lib.lh_raw_percentiles(eng.h, bb, None, None, 0, None, None, None, None) == 0   # n == 0
        assert lib.lh_raw_percentiles_grid(eng.h, bb, None, 0, None, None, None, None) == 0
        assert lib.lh_raw_percentiles(other.h, bb, r, x, 4, k, v, pu, None) == LH_ERR_INVALID  # foreign
        eng.snapshot_begin()
        assert lib.lh_snapshot_publish_raw(eng.h, bb, (C.c_uint32 * 4)(0, 1, 4, 2)) == LH_ERR_RANGE
        assert lib.lh_snapshot_publish_raw(other.h, bb, None) == LH_ERR_INVALID
        launches = eng.stats()["kernel_launches"]
        assert lib.lh_snapshot_publish_raw(eng.h, bb, (C.c_uint32 * 4)(0, UNBOUND, 3, 2)) == 0   # no reduction needed
        assert eng.stats()["kernel_launches"] == launches + 1
        eng.snapshot_end()
        assert lib.lh_snapshot_publish_raw(eng.h, bb, None) == LH_ERR_STATE          # snapshot ended
        assert lib.lh_raw_board_destroy(other.h, bb) == LH_ERR_INVALID
        saved = L.lh_raw_board.from_buffer_copy(rb.board)
        rb.close()
        sb = C.byref(saved)
        launches = eng.stats()["kernel_launches"]
        assert lib.lh_raw_board_destroy(eng.h, sb) == LH_ERR_INVALID
        assert lib.lh_raw_percentiles(eng.h, sb, r, x, 4, k, v, pu, None) == LH_ERR_INVALID
        assert lib.lh_raw_ranks_grid(eng.h, sb, x, 1, pu, pu + 8, pu + 16, None) == LH_ERR_INVALID
        eng.snapshot_begin()
        assert lib.lh_snapshot_publish_raw(eng.h, sb, None) == LH_ERR_INVALID
        eng.snapshot_end()
        assert eng.stats()["kernel_launches"] - launches == 1                         # the clear of the snapshot only
        assert launches - before == 2                                                # the publish, one snapshot's clear
        with pytest.raises(TypeError):
            eng.raw_board(1).percentiles(torch.zeros(2, dtype=torch.float32, device="cuda"))
        eng.raw_board(2)   # freed by lh_destroy
