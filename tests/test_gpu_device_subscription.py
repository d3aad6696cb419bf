"""Device subscriptions (lh_board_*, lh_snapshot_publish, MetricSystem::NewDeviceSubscription): every collection's
processed metrics published into device memory, read by kernels (lh::read_histogram / lh::read_counter) and by a
captured lh_board_read.

The reading kernels live in tests/board_read_client.cu, a separate CUDA library built by build() that knows the engine
only through its public headers.  Bar: the rows equal the host's processMetrics values for the same collection bit for
bit (NaN-aware), counter rows equal Rates / Counters, readers running beside hundreds of collections never see a torn
row, captured reads reflect the latest publish at each replay, and a collection without a subscription issues the same
work as before."""
import ctypes as C
import os
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INT32_MIN = -(1 << 31)
UNBOUND = 0xFFFFFFFF
LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = -1, -5, -6
P = 32
HIST_ROW = np.dtype([("count", "<u8"), ("sum", "<f8"), ("avg", "<f8"), ("present", "<u4"), ("reserved", "<u4"),
                     ("pvals", "<f8", (P,)), ("pkeys", "<i4", (P,))])
CTR_ROW = np.dtype([("rate", "<u8"), ("total", "<u8"), ("present", "<u4"), ("reserved", "<u4")])


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
    assert os.path.exists(build.BOARD_CLIENT_LIB), "build() did not produce " + build.BOARD_CLIENT_LIB
    lib = C.CDLL(build.BOARD_CLIENT_LIB)
    bp, vp = C.POINTER(_lib.lh_board), C.c_void_p
    lib.brc_read_rows.argtypes = [bp, vp, vp, vp, vp]
    lib.brc_torn_start.argtypes = [bp, C.c_int, C.c_uint64, vp, vp]
    lib.brc_read_cost.argtypes = [bp, C.c_uint32, C.c_int, vp, vp]
    for name in ("brc_read_rows", "brc_torn_start", "brc_read_cost"):
        getattr(lib, name).restype = C.c_int
    return lib


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def to_host(torch, views):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in views.items()}


def kernel_rows(torch, client, board):
    """Every row of `board` read in a kernel through lh::read_histogram / lh::read_counter: (hist rows, counter rows,
    publish number per row)."""
    k, kc = board.k, board.kc
    h = torch.zeros(max(k, 1) * HIST_ROW.itemsize, dtype=torch.uint8, device="cuda")
    c = torch.zeros(max(kc, 1) * CTR_ROW.itemsize, dtype=torch.uint8, device="cuda")
    pub = torch.zeros(max(k + kc, 1), dtype=torch.int64, device="cuda")
    assert client.brc_read_rows(C.byref(board), h.data_ptr(), c.data_ptr(), pub.data_ptr(),
                                torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    return (h.cpu().numpy().view(HIST_ROW)[:k], c.cpu().numpy().view(CTR_ROW)[:kc], pub.cpu().numpy()[:k + kc])


def assert_kernel_matches_image(hr, cr, pub, v):
    """The in-kernel reads equal the lh_board_read image, and every row is of the image's publish."""
    assert (pub == int(v["collection"])).all()
    assert (hr["count"] == v["count"].view(np.uint64)).all()
    assert (bits(hr["sum"]) == bits(v["sum"])).all() and (bits(hr["avg"]) == bits(v["avg"])).all()
    assert (hr["present"] == v["present"]).all()
    assert (bits(hr["pvals"]) == bits(v["pvals"])).all() and (hr["pkeys"] == v["pkeys"]).all()
    assert (cr["rate"] == v["rate"].view(np.uint64)).all() and (cr["total"] == v["total"].view(np.uint64)).all()
    assert (cr["present"] == v["counter_present"]).all()


def assert_untouched(v, i):
    assert v["present"][i] == 0 and v["count"][i] == 0 and bits(v["sum"][i]) == 0 and np.isnan(v["avg"][i])
    assert (v["pkeys"][i] == INT32_MIN).all() and np.isnan(v["pvals"][i]).all()


def assert_matches_metrics(v, hnames, cnames, raw, metrics, labels):
    """Board rows (host copies of read()) against processMetrics' dict for the same collection, bit for bit."""
    npct = len(labels)
    assert int(v["np"]) == npct
    assert (bits(v["percentiles"][:npct]) == bits([p for _, p in labels])).all() and np.isnan(v["percentiles"][npct:]).all()
    for i, nm in enumerate(hnames):
        if nm not in raw["Histograms"]:
            assert_untouched(v, i)
            assert nm + "_count" not in metrics
            continue
        assert v["present"][i] == 1
        assert float(v["count"].view(np.uint64)[i]) == metrics[nm + "_count"]
        assert bits(v["sum"][i]) == bits(metrics[nm + "_sum"]) and bits(v["avg"][i]) == bits(metrics[nm + "_avg"])
        for j, (label, _) in enumerate(labels):
            key = label.replace("%s", nm, 1)
            if v["pkeys"][i, j] == INT32_MIN:
                assert key not in metrics and np.isnan(v["pvals"][i, j])
            else:
                assert bits(v["pvals"][i, j]) == bits(metrics[key])
        assert (v["pkeys"][i, npct:] == INT32_MIN).all() and np.isnan(v["pvals"][i, npct:]).all()
    for i, nm in enumerate(cnames):
        if nm in raw["Rates"]:
            assert v["counter_present"][i] == 1 and int(v["rate"].view(np.uint64)[i]) == raw["Rates"][nm]
        else:
            assert v["counter_present"][i] == 0 and v["rate"][i] == 0
        assert int(v["total"].view(np.uint64)[i]) == raw["Counters"].get(nm, 0)


LABEL_SETS = [
    {},
    {"%s_p50": 0.5, "%s_p99": 0.99, "%s_max": 1.0},
    dict([("%%s_q%02d" % j, p) for j, p in enumerate(
        [0.0, 1.0, 1.5, float("nan"), -0.5, 1e-300] + [j / 26.0 for j in range(26)])]),
]


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_rows_equal_processed_metrics(lh, oracle, torch, client, precision):
    """Streams U / L / S, label sets with np = 0, 3 and 32 changed between collections, names absent in some
    collections, never seen, recycled away (their id reused by other names) and recycled back."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4, precision=precision)
    try:
        hnames = ["h0", "h1", "h2", "hr", "never"]
        cnames = ["c0", "c1", "cr", "cnever"]
        with ms.device_subscription(histograms=hnames, counters=cnames) as sub:
            assert sub.histogram_rows == {nm: i for i, nm in enumerate(hnames)}
            assert sub.counter_rows == {nm: i for i, nm in enumerate(cnames)}
            v = to_host(torch, sub.read())
            assert int(v["collection"]) == 0 and (v["present"] == 0).all() and (v["counter_present"] == 0).all()
            for j in range(9):
                labels = LABEL_SETS[j % 3]
                ms.SpecifyPercentiles(labels)
                kind = (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S)[j % 3]
                for i, nm in enumerate(hnames[:3]):
                    if (i + j) % 4 != 3:
                        ms.HistogramMany(nm, oracle.gen_stream(kind, 500 + 97 * i + 13 * j, 1000 * j + i))
                if j in (0, 7, 8):   # "hr" idles through collections 1..6: its id is freed and taken by churn names
                    ms.HistogramMany("hr", oracle.gen_stream(kind, 300, 77 + j))
                for t in range(3):   # churn that fills the table
                    ms.Histogram("tmp%d_%d" % (j, t), 1.0 + t)
                    ms.Counter("ctmp%d_%d" % (j, t), 1)
                ms.Counter("c0", j + 1)
                if j % 2:
                    ms.Counter("c1", 0)   # in Rates with a zero delta
                if j in (0, 8):
                    ms.Counter("cr", 5)
                raw, metrics = ms.collect_and_process()
                v = to_host(torch, sub.read())
                assert int(v["collection"]) == j + 1
                assert_matches_metrics(v, hnames, cnames, raw, metrics, sorted(labels.items()))
                assert_kernel_matches_image(*kernel_rows(torch, client, sub.board), v)
    finally:
        ms.close()


def test_engine_sync_async_and_big_board(lh, oracle, torch, client):
    """Publishes after lh_snapshot_reduce and after lh_snapshot_reduce_async (before lh_snapshot_result) equal the
    reduction; a board of 4 096 + 8 rows (more than one parameter block) maps every row to its id."""
    H, C_ = 4096, 8
    ps = [0.0, 0.5, 0.99, 1.0, 2.0]
    with lh.Engine(device=0, max_histograms=H, max_counters=C_) as eng:
        rng = np.random.default_rng(5)
        ids = rng.integers(0, H, 400_000).astype(np.uint16)
        vals = oracle.gen_stream(lh.STREAM_L, ids.size, 9)
        amounts = rng.integers(1, 1000, 64).astype(np.uint64)
        cids = rng.integers(0, C_, 64).astype(np.uint16)
        hid = np.arange(H - 1, -1, -1).astype(np.uint32)   # row i -> id H-1-i
        hid[7] = UNBOUND
        cid = np.array([3, 2, UNBOUND, 0, 7, 6, 5, 4], dtype=np.uint32)
        totals = np.arange(C_, dtype=np.uint64) * 1000 + 1
        with eng.board(H, C_) as b:
            for mode in ("sync", "async"):
                eng.ingest_keyed_f64_u16_host(ids, vals)
                eng.counter_add_u16_host(cids, amounts)
                eng.snapshot_begin()
                if mode == "sync":
                    red = eng.snapshot_reduce(ps)
                    b.publish(hid, cid, totals)
                else:
                    h = eng.snapshot_reduce_async(ps)
                    b.publish(hid, cid, totals)
                    red = eng.snapshot_result(h)
                deltas = eng.snapshot_export().counter_deltas.copy()
                eng.snapshot_end()
                v = to_host(torch, b.read())
                bound = hid != UNBOUND
                t = hid[bound]
                assert (v["count"].view(np.uint64)[bound] == red.counts[t]).all()
                assert (bits(v["sum"][bound]) == bits(red.sums[t])).all()
                assert (bits(v["avg"][bound]) == bits(red.avgs[t])).all()
                assert (v["pkeys"][bound, :len(ps)] == red.pkeys[t]).all()
                assert (bits(v["pvals"][bound, :len(ps)]) == bits(red.pvals[t])).all()
                assert (v["present"][bound] == (red.counts[t] != 0)).all()
                assert_untouched(v, 7)
                cb = cid != UNBOUND
                assert (v["rate"].view(np.uint64)[cb] == deltas[cid[cb]]).all() and (v["counter_present"] == cb).all()
                assert v["rate"][2] == 0 and (v["total"].view(np.uint64) == totals).all()
                assert_kernel_matches_image(*kernel_rows(torch, client, b.board), v)
            assert int(v["collection"]) == 2


def test_two_contexts_allreduce(lh, oracle, torch, client):
    """Two contexts on one GPU all-reduced: each board equals the reduction of the summed snapshot."""
    H, C_ = 6, 3
    ps = [0.5, 0.9]
    engs = [lh.Engine(device=0, max_histograms=H, max_counters=C_) for _ in range(2)]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, 2, handles)
        boards = [e.board(H, C_) for e in engs]
        for r, e in enumerate(engs):
            ids = np.arange(20_000, dtype=np.uint16) % H
            e.ingest_keyed_f64_u16_host(ids, oracle.gen_stream(lh.STREAM_U, ids.size, 40 + r))
            e.counter_add_u16_host(np.arange(C_, dtype=np.uint16), np.full(C_, 3 + r, dtype=np.uint64))
        for e in engs:
            e.sync()
        for e in engs:
            e.snapshot_begin()
            e.snapshot_allreduce(True)
        reds = []
        for e, b in zip(engs, boards):
            reds.append(e.snapshot_reduce(ps))
            b.publish(list(range(H)), list(range(C_)), None)
            e.snapshot_end()
        for red, b in zip(reds, boards):
            v = to_host(torch, b.read())
            assert (v["count"].view(np.uint64) == red.counts).all() and red.counts.sum() == 40_000
            assert (bits(v["sum"]) == bits(red.sums)).all()
            assert (bits(v["pvals"][:, :2]) == bits(red.pvals)).all()
            assert (v["rate"] == 7).all() and (v["total"] == 0).all()
        for b in boards:
            b.close()
    finally:
        for e in engs:
            e.close()


def test_validation(lh, torch):
    """State, range, foreign and destroyed handles, empty boards: each returns its status and enqueues nothing."""
    from loghisto_b200 import _lib as L
    with lh.Engine(device=0, max_histograms=4, max_counters=2) as eng, lh.Engine(device=0, max_histograms=4) as other:
        lib = eng.lib
        b = L.lh_board()
        assert lib.lh_board_create(eng.h, 0, 0, C.byref(b)) == LH_ERR_INVALID
        assert lib.lh_board_create(eng.h, 5, 0, C.byref(b)) == LH_ERR_RANGE
        assert lib.lh_board_create(eng.h, 1, 3, C.byref(b)) == LH_ERR_RANGE
        board = eng.board(4, 2)
        bb = C.byref(board.board)
        out = torch.zeros(board.board.bytes, dtype=torch.uint8, device="cuda")
        assert lib.lh_snapshot_publish(eng.h, bb, None, None, None) == LH_ERR_STATE   # no snapshot
        eng.snapshot_begin()
        assert lib.lh_snapshot_publish(eng.h, bb, None, None, None) == LH_ERR_STATE   # no reduction yet
        eng.snapshot_export()                                                          # not a reduction either
        assert lib.lh_snapshot_publish(eng.h, bb, None, None, None) == LH_ERR_STATE
        eng.snapshot_reduce([0.5])
        bad = (C.c_uint32 * 4)(0, 1, 4, 2)
        assert lib.lh_snapshot_publish(eng.h, bb, bad, None, None) == LH_ERR_RANGE
        bad_c = (C.c_uint32 * 2)(0, 2)
        assert lib.lh_snapshot_publish(eng.h, bb, None, bad_c, None) == LH_ERR_RANGE
        ok = (C.c_uint32 * 4)(0, UNBOUND, 3, 2)
        assert lib.lh_snapshot_publish(eng.h, bb, ok, None, None) == 0
        assert lib.lh_snapshot_publish(other.h, bb, None, None, None) == LH_ERR_INVALID   # foreign
        assert lib.lh_board_read(other.h, bb, out.data_ptr(), None) == LH_ERR_INVALID
        assert lib.lh_board_read(eng.h, bb, out.data_ptr() + 4, None) == LH_ERR_INVALID   # misaligned
        eng.snapshot_end()
        assert lib.lh_snapshot_publish(eng.h, bb, None, None, None) == LH_ERR_STATE   # snapshot ended
        before = eng.stats()["kernel_launches"]
        assert lib.lh_board_destroy(other.h, bb) == LH_ERR_INVALID
        saved = L.lh_board.from_buffer_copy(board.board)
        board.close()
        sb = C.byref(saved)
        assert lib.lh_board_destroy(eng.h, sb) == LH_ERR_INVALID
        assert lib.lh_board_read(eng.h, sb, out.data_ptr(), None) == LH_ERR_INVALID
        eng.snapshot_begin()
        eng.snapshot_reduce([])
        assert lib.lh_snapshot_publish(eng.h, sb, None, None, None) == LH_ERR_INVALID
        eng.snapshot_end()
        assert eng.stats()["kernel_launches"] - before == 2   # K3 and the clear of the second snapshot only
        left = eng.board(1, 1)   # freed by lh_destroy
        assert left.board.bytes == 288 + 416 + 24


def test_no_torn_reads(torch, client):
    """A reader kernel on fewer CTAs than SMs loops over every row for a fixed %globaltimer budget while the host runs
    200 collections; collection j gives every name j samples of one value (counter j): no row read mixes publishes."""
    from loghisto_b200.metric_system import MetricSystem
    k, kc, n = 48, 8, 200
    ms = MetricSystem(1.0, False, max_histograms=64, max_counters=16)
    try:
        ms.SpecifyPercentiles({"%s_p50": 0.5})
        hnames, cnames = ["t%d" % i for i in range(k)], ["n%d" % i for i in range(kc)]
        with ms.device_subscription(histograms=hnames, counters=cnames) as sub:
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            stats = torch.zeros(5, dtype=torch.int64, device="cuda")
            side = torch.cuda.Stream()
            torch.cuda.synchronize()
            budget = 4_000_000_000
            assert client.brc_torn_start(C.byref(sub.board), sms // 4, budget, stats.data_ptr(), side.cuda_stream) == 0
            t0 = time.monotonic()
            for j in range(1, n + 1):
                vj = np.full(j, 1.5 + 0.37 * j)
                for nm in hnames:
                    ms.HistogramMany(nm, vj)
                for nm in cnames:
                    ms.Counter(nm, j)
                ms.collect_and_process()
            host_s = time.monotonic() - t0
            side.synchronize()
            reads, bad, hi, lo, changes = [int(x) for x in stats.cpu().numpy().view(np.uint64)]
            assert bad == 0, (reads, bad, hi, lo, changes)
            assert reads > 0 and hi > lo >= 1 and changes > 0, (reads, hi, lo, changes)
            if host_s < 2.0:   # every publish happened well inside the reader's budget
                assert hi == n
    finally:
        ms.close()


def test_captured_read_follows_latest_publish(torch):
    """sub.read(out) and torch ops on its pvals captured in one CUDA graph: each replay reflects the latest collection."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4)
    try:
        ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p99": 0.99})
        with ms.device_subscription(histograms=["lat", "idle"], counters=["req"]) as sub:
            out = torch.zeros(sub.board.bytes, dtype=torch.uint8, device="cuda")
            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                v = sub.read(out)
                y = v["pvals"][:, :2] * 2.0
                n = v["collection"] + 0
            for j in range(1, 4):
                ms.HistogramMany("lat", np.linspace(1.0, 100.0 * j, 1000))
                ms.Counter("req", j)
                raw, metrics = ms.collect_and_process()
                g.replay()
                torch.cuda.synchronize()
                assert int(n.item()) == j
                got = y.cpu().numpy()
                assert bits(got[0, 0]) == bits(2.0 * metrics["lat_p50"]) and bits(got[0, 1]) == bits(2.0 * metrics["lat_p99"])
                assert np.isnan(got[1]).all()
                assert int(v["rate"][0].item()) == j and int(v["total"][0].item()) == j * (j + 1) // 2
    finally:
        ms.close()


def test_no_change_without_a_subscription(lh, oracle):
    """Collections with no board, and after a board was created and destroyed, issue the same kernel launches."""
    with lh.Engine(device=0, max_histograms=16, max_counters=4) as eng:
        ids = (np.arange(10_000) % 16).astype(np.uint16)
        vals = oracle.gen_stream(lh.STREAM_U, ids.size, 3)

        def collect():
            eng.ingest_keyed_f64_u16_host(ids, vals)
            eng.sync()
            before = eng.stats()["kernel_launches"]
            eng.snapshot_begin()
            eng.snapshot_reduce([0.5, 0.99])
            eng.snapshot_export()
            eng.snapshot_end()
            return eng.stats()["kernel_launches"] - before

        plain = [collect() for _ in range(3)]
        eng.board(16, 4).close()
        after = [collect() for _ in range(3)]
        assert plain == after and len(set(plain)) == 1
