"""Window boards (lh_raw_board_create_window, MetricSystem::NewRawDeviceSubscription(names, window)): every row answers
for the sum of its last `window` publishes.

Bar: after every publish, a window board equals, bit for bit (headers, cells inside the published range, every key's
bucket count through tests/raw_read_client.cu, the grid queries), a plain board of a second context that was fed the
sparse exports of the row's last `window` intervals through lh_merge_counts_host; its percentiles also equal the exact
reference of tests/_reduce_cases.py on the summed histogram.  The cases cover every slot reused, dense intervals and
wrapped sums entering and leaving, staged ids, names absent and recycled, captured replays, readers beside collections,
all-reduced contexts and joined ranks, the refusals and the launch count."""
import collections
import ctypes as C
import math
import threading
import time

import numpy as np
import pytest

import _reduce_cases as rc

pytestmark = pytest.mark.gpu

INT32_MIN = -(1 << 31)
UNBOUND = 0xFFFFFFFF
LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = -1, -5, -6
WRAPPED = 65536
PS = np.array(rc.SPECIAL_PS + [0.001, 0.1, 0.25, 0.75, 0.9, 0.999, 0.9999], dtype=np.float64)
VALUES = np.array([-1e300, -2.0 ** 63, -5.0, -1.0, 0.0, 0.5, 1.0, 3.0, 10.0, 1e3, 1e6, 2.0 ** 63, 1e300, math.inf,
                   -math.inf, math.nan], dtype=np.float64)


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
    import os
    from loghisto_b200 import _lib, build
    assert os.path.exists(build.RAW_CLIENT_LIB), "build() did not produce " + build.RAW_CLIENT_LIB
    lib = C.CDLL(build.RAW_CLIENT_LIB)
    bp, vp, u32 = C.POINTER(_lib.lh_raw_board), C.c_void_p, C.c_uint32
    lib.rrc_percentiles.argtypes = [bp, vp, vp, u32, vp, vp, vp, vp]
    lib.rrc_bucket_counts.argtypes = [bp, vp, vp, u32, vp, vp, vp]
    lib.rrc_torn_start.argtypes = [bp, C.c_double, C.c_double, vp, vp, vp, C.c_int, C.c_uint64, vp, vp]
    for name in ("rrc_percentiles", "rrc_bucket_counts", "rrc_torn_start"):
        getattr(lib, name).restype = C.c_int
    return lib


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def cuda(torch, a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def host(torch, *ts):
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in ts]


def reference_keys(ref, ps):
    """Reference.percentile for every p at once (as tests/test_gpu_raw_subscription.py states it)."""
    ps = np.asarray(ps, dtype=np.float64)
    if not ref.nnz:
        return np.full(ps.size, INT32_MIN, np.int32)
    best = np.fmax.accumulate(np.where(np.isnan(ref.ratios), -np.inf, ref.ratios))
    i = np.searchsorted(best, ps, side="left")
    order = np.array(ref.order + [INT32_MIN], dtype=np.int64)
    i[np.isnan(ps)] = ref.nnz
    return order[np.minimum(i, ref.nnz)].astype(np.int32)


def key_hi(h):
    """A header's key_hi without the wrapped mark."""
    v = int(h["key_hi"])
    return v - WRAPPED if v > 32767 else v


def read_board(eng, board, cells=True):
    """(headers [k] structured, cells [k, 65536] uint64 or None) of a board, after everything issued."""
    from loghisto_b200 import _lib as L
    eng.sync()
    k = board.k
    raw = np.zeros(L.LH_RAW_CELLS_OFFSET(k) + (k * 65536 * 8 if cells else 0), np.uint8)
    eng._check(eng.lib.lh_memcpy_d2h(eng.h, raw.ctypes.data, board.d_rows, raw.nbytes))
    hdr = np.frombuffer(raw[:k * 32].tobytes(), dtype=[("seq", "<u8"), ("publishes", "<u8"), ("total", "<u8"),
                                                        ("key_lo", "<i4"), ("key_hi", "<i4")])
    if not cells:
        return hdr, None
    return hdr, raw[L.LH_RAW_CELLS_OFFSET(k):].view(np.uint64).reshape(k, 65536)


def assert_boards_equal(torch, client, eng_a, a, eng_b, b, all_keys=True, what=""):
    """Window board a equals plain board b: headers, cells inside each row's range, grid queries, bucket counts."""
    ha, ca = read_board(eng_a, a.board, all_keys)
    hb, cb = read_board(eng_b, b.board, all_keys)
    assert (ha == hb).all(), (what, ha, hb)
    for r in range(a.k if all_keys else 0):
        lo, hi = int(ha[r]["key_lo"]), key_hi(ha[r])
        if lo <= hi:
            assert (ca[r, lo + 32768:hi + 32769] == cb[r, lo + 32768:hi + 32769]).all(), (what, r)
    ps = cuda(torch, PS)
    for x, y in zip(host(torch, *a.percentiles(ps)), host(torch, *b.percentiles(ps))):
        assert (x.view(np.uint64) == y.view(np.uint64)).all() if x.dtype == np.float64 else (x == y).all(), what
    vs = cuda(torch, VALUES)
    for x, y in zip(host(torch, *a.ranks(vs)), host(torch, *b.ranks(vs))):
        assert (x == y).all(), what
    if all_keys:
        k = a.k
        rows = cuda(torch, np.repeat(np.arange(k), 65536), np.uint32)
        keys = cuda(torch, np.tile(np.arange(-32768, 32768), k), np.int32)
        out = []
        for bd in (a.board, b.board):
            counts, pub = (torch.empty(k * 65536, dtype=torch.int64, device="cuda") for _ in range(2))
            assert client.rrc_bucket_counts(C.byref(bd), rows.data_ptr(), keys.data_ptr(), k * 65536, counts.data_ptr(),
                                            pub.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
            out.append(host(torch, counts, pub))
        assert (out[0][0] == out[1][0]).all() and (out[0][1] == out[1][1]).all(), what
    return ha


class MergedReference:
    """A second context whose plain board is published, at every step, from the merge of the sparse exports of each
    row's last `window` intervals (lh_merge_counts_host), one row per histogram id."""

    def __init__(self, lh, k, window, precision=0):
        self.eng = lh.Engine(device=0, max_histograms=k, max_counters=1, precision=precision)
        self.board = self.eng.raw_board(k)
        self.window = window
        self.k = k
        self.last = collections.deque(maxlen=window)   # per interval: (ids, keys, counts) triples by row

    def interval(self, sp, hid):
        """Record one interval: row r's entering counts are histogram hid[r] of export sp (UNBOUND: nothing)."""
        ids, keys, counts = [], [], []
        for r, h in enumerate(hid):
            if h == UNBOUND:
                continue
            a, b = int(sp.offsets[h]), int(sp.offsets[h + 1])
            ids.append(np.full(b - a, r, np.uint32))
            keys.append(np.asarray(sp.keys[a:b], np.int16))
            counts.append(np.asarray(sp.counts[a:b], np.uint64))
        cat = (lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt))
        self.last.append((cat(ids, np.uint32), cat(keys, np.int16), cat(counts, np.uint64)))

    def publish(self):
        ids = np.concatenate([t[0] for t in self.last])
        if ids.size:
            self.eng.merge_counts_host(ids, np.concatenate([t[1] for t in self.last]),
                                       np.concatenate([t[2] for t in self.last]))
        self.eng.snapshot_begin()
        try:
            self.board.publish(list(range(self.k)))
        finally:
            self.eng.snapshot_end()

    def hist(self, r):
        """Row r's window histogram {key: count mod 2^64}."""
        d = {}
        for ids, keys, counts in self.last:
            for key, c in zip(keys[ids == r].tolist(), counts[ids == r].tolist()):
                d[key] = (d.get(key, 0) + c) % 2 ** 64
        return d

    def close(self):
        self.board.close()
        self.eng.close()


H = 8
GIANT = 2 ** 63


def feed_step(eng, oracle, lh, t, w, precision, cases, rng):
    """Interval t of the source context: histogram ids 0..H-1, one behaviour each (see test_window_equals_merged)."""
    period = w + 3
    ids, keys, counts = [], [], []

    def triples(h, d):
        for key, c in d.items():
            ids.append(h)
            keys.append(key)
            counts.append(c)
    streams = (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S)
    for h in range(3):
        if h == 1 and t % 3 == 2:
            continue                                  # absent: untouched this interval
        x = oracle.gen_stream(streams[h], 1000 + 37 * h, 1000 * t + h)
        if h == 0 and t % (2 * w + 1) == 2:           # dense: a key outside the fast window, and +-Inf / NaN
            x = np.concatenate([x, [2.0 ** 63 * 1.5, -1e300, math.inf, -math.inf, math.nan]])
        eng.ingest_keyed_f64_u16_host(np.full(x.size, h, np.uint16), x)
    triples(3, cases[t % len(cases)]["hist"])         # constructed cases, wrapped ones among them
    if t % period in (0, 1):                          # two giants at one key: their window sums to 0
        triples(4, {17: GIANT})
    if t % period in (0, 1):                          # a window of both (at two keys) wraps; it stops when one leaves
        triples(5, {-3 + t % period: GIANT + 3, 40: 5})
    else:
        triples(5, {40: 1 + t % 4})
    eng.ingest_keyed_f64_u16_host(np.full(50, 6, np.uint16), rng.lognormal(2, 3, 50))
    if ids:
        eng.merge_counts_host(np.array(ids, np.uint32), np.array(keys, np.int16), np.array(counts, np.uint64))


@pytest.mark.parametrize("precision", rc.PRECISIONS)
@pytest.mark.parametrize("w", [1, 2, 3, 7, 64])
def test_window_equals_merged(lh, oracle, torch, client, w, precision):
    """Over 3w + 2 publishes (every slot reused), rows bound to scattered ids: streams U / L / S (L absent every third
    interval, S dense throughout, U dense in intervals 2 and 2w + 3, so that its range widens and narrows), constructed and wrapped cases of tests/_reduce_cases.py, two giant 2^63 counts
    whose window sums to 0, giants at two keys that wrap the window only while both are in it, a row unbound every other
    interval and a row never touched.  Each publish equals the merged reference; at w = 1 the window board also
    equals a plain board of the same context cell for cell; percentiles equal the exact reference."""
    table = oracle.decompress_table(precision)
    cases = rc.make_cases(precision, table, 11) + rc.make_wrapped_cases(precision, table, 11)
    rng = np.random.default_rng(precision * 1000 + w)
    ref = MergedReference(lh, H, w, precision)
    perm = [(3 * r + 1) % H for r in range(H)]        # row r <- id perm[r]; id 7 (never touched) is row 2
    try:
        with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng, \
                eng.raw_board(H, window=w) as wb, eng.raw_board(H) as plain:
            assert wb.window == w and wb.board.k == H
            seen_wrap = seen_zero = seen_narrow = False
            widths = []
            steps = 3 * w + 2
            for t in range(1, steps + 1):
                feed_step(eng, oracle, lh, t, w, precision, cases, rng)
                hid = [perm[r] if not (perm[r] == 6 and t % 2) else UNBOUND for r in range(H)]
                eng.snapshot_begin()
                try:
                    wb.publish(hid)
                    if w == 1:
                        plain.publish(hid)
                    sp = eng.snapshot_export()
                finally:
                    eng.snapshot_end()
                ref.interval(sp, hid)
                ref.publish()
                every_key = w < 64 or t % 16 == 0 or t == steps
                hdr = assert_boards_equal(torch, client, eng, wb, ref.eng, ref.board, every_key, (w, precision, t))
                assert (hdr["publishes"] == t).all()
                if w == 1:
                    hp, cp = read_board(eng, plain.board)
                    hw, cw = read_board(eng, wb.board)
                    assert (hp[["total", "key_lo", "key_hi"]] == hw[["total", "key_lo", "key_hi"]]).all()
                    for r in range(H):
                        lo, hi = int(hw[r]["key_lo"]), key_hi(hw[r])
                        if lo <= hi:
                            assert (cp[r, lo + 32768:hi + 32769] == cw[r, lo + 32768:hi + 32769]).all()
                seen_wrap |= bool(hdr[perm.index(5)]["key_hi"] > 32767)
                seen_zero |= bool(hdr[perm.index(4)]["total"] == 0 and hdr[perm.index(4)]["key_lo"] < 0)
                widths.append(key_hi(hdr[perm.index(0)]) - int(hdr[perm.index(0)]["key_lo"]))
                if len(widths) > 1 and widths[-1] < widths[-2]:
                    seen_narrow = True
                if t in (steps // 2, steps):          # the exact reference on every row's window
                    k, v, _ = host(torch, *wb.percentiles(cuda(torch, PS)))
                    for r in range(H):
                        want = reference_keys(rc.Reference(ref.hist(r), table), PS)
                        assert (k[r] == want).all(), (w, precision, t, r)
            assert seen_narrow and 65535 in widths
            if w >= 2:
                assert seen_wrap and seen_zero
    finally:
        ref.close()


def test_staged_ids(lh, oracle, torch, client):
    """A window board of 4 104 rows (ids staged by k_raw_stage) at w = 2 over seven publishes equals the merged
    reference; rows map to reversed ids, one unbound and two bound to one id."""
    k = 4104
    ref = MergedReference(lh, k, 2)
    try:
        with lh.Engine(device=0, max_histograms=k, max_counters=1) as eng, eng.raw_board(k, window=2) as wb:
            hid = np.arange(k - 1, -1, -1).astype(np.uint32)
            hid[5] = UNBOUND
            hid[4100] = hid[4101]
            for t in range(7):
                rng = np.random.default_rng(t)
                ids = rng.integers(0, k // (1 + t % 3), 200_000).astype(np.uint16)
                eng.ingest_keyed_f64_u16_host(ids, oracle.gen_stream(lh.STREAM_L, ids.size, 9 + t))
                eng.snapshot_begin()
                try:
                    wb.publish(hid)
                    sp = eng.snapshot_export()
                finally:
                    eng.snapshot_end()
                ref.interval(sp, hid.tolist())
                ref.publish()
                assert_boards_equal(torch, client, eng, wb, ref.eng, ref.board, all_keys=False, what=t)
    finally:
        ref.close()


def test_two_contexts_allreduce(lh, oracle, torch, client):
    """Two contexts on one GPU all-reduced at every step: each window board equals the merge of the all-reduced
    intervals."""
    k = 6
    engs = [lh.Engine(device=0, max_histograms=k, max_counters=1) for _ in range(2)]
    ref = MergedReference(lh, k, 3)
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, 2, handles)
        boards = [e.raw_board(k, window=3) for e in engs]
        for t in range(8):
            for r, e in enumerate(engs):
                ids = (np.arange(5000 + 100 * t) % (k - t % 2)).astype(np.uint16)
                vals = oracle.gen_stream(lh.STREAM_U if r else lh.STREAM_L, ids.size, 40 + 2 * t + r)
                if t == 2 and r == 1:
                    vals[:3] = [1e300, -1e300, 2.0 ** 64]
                e.ingest_keyed_f64_u16_host(ids, vals)
            for e in engs:
                e.sync()
            for e in engs:
                e.snapshot_begin()
                e.snapshot_allreduce(False)
            sps = []
            for e, b in zip(engs, boards):
                b.publish(list(range(k)))
                sps.append(e.snapshot_export())
                e.snapshot_end()
            ref.interval(sps[0], list(range(k)))
            ref.publish()
            for e, b in zip(engs, boards):
                assert_boards_equal(torch, client, e, b, ref.eng, ref.board, all_keys=t % 3 == 0, what=t)
        for b in boards:
            b.close()
    finally:
        ref.close()
        for e in engs:
            e.close()


def window_of(history, name, w):
    d = {}
    for raw in history[-w:]:
        for key, c in raw["Histograms"].get(name, {}).items():
            d[key] = (d.get(key, 0) + c) % 2 ** 64
    return d


def check_names(torch, oracle, table, sub, history, names, ps_t, val_t, keys, vals, pub, ranks, totals, rpub):
    """Answers (already computed, e.g. by a graph replay) against the exact reference on each name's window."""
    k, v, p, rk, tot, rp = host(torch, keys, vals, pub, ranks, totals, rpub)
    ps, values = ps_t.cpu().numpy(), val_t.cpu().numpy()
    assert (p == len(history)).all() and (rp == len(history)).all()
    kv = oracle.compress_many(values).astype(np.int64)
    for i, nm in enumerate(names):
        d = window_of(history, nm, sub.window)
        want = reference_keys(rc.Reference(d, table), ps)
        assert (k[i] == want).all(), (nm, len(history))
        wv = np.array([table[x & 0xFFFF] if x != INT32_MIN else math.nan for x in want])
        assert (bits(v[i]) == bits(wv)).all()
        assert int(tot[i]) % 2 ** 64 == sum(d.values()) % 2 ** 64
        for j in range(values.size):
            assert int(rk[i, j]) % 2 ** 64 == sum(c for key, c in d.items() if key <= kv[j]) % 2 ** 64


def test_names_through_every_route_and_captured_replay(oracle, torch):
    """A MetricSystem with window subscriptions at 1, 2 and 5 over 14 collections.  "lat" is fed by Histogram() on
    stream U, "tok" by a record scope's keyed samples on stream L and "gr" by graph-recorder replays on stream S; "idle"
    is absent in most collections, "churn" is recycled away by other names and comes back, "never" is never seen.
    Percentiles and ranks captured in one torch.cuda.graph and replayed after each collection equal the exact
    reference on each name's last w collections of the RawMetricSet, and follow the latest publish."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(3600.0, False, max_histograms=8, max_counters=2)
    table = oracle.decompress_table(100)
    names = ["lat", "tok", "gr", "idle", "churn", "never"]
    history = []
    try:
        subs = [ms.raw_device_subscription(histograms=names, window=w) for w in (1, 2, 5)]
        assert [s.window for s in subs] == [1, 2, 5]
        with ms.graph_recorder(histograms=["gr"]) as g:
            gx = torch.tensor(oracle.gen_stream(oracle.STREAM_S, 3000, 5), dtype=torch.float64, device="cuda")
            gid = torch.zeros(gx.numel(), dtype=torch.int32, device="cuda")
            side = torch.cuda.Stream()
            gg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gg, stream=side):
                g.keyed(gid, gx)
            ps_t = cuda(torch, PS)
            val_t = cuda(torch, VALUES)
            torch.cuda.synchronize()
            q = torch.cuda.CUDAGraph()
            outs = []
            with torch.cuda.graph(q):
                for s in subs:
                    outs.append(s.percentiles(ps_t) + s.ranks(val_t))
            for j in range(1, 15):
                ms.HistogramMany("lat", oracle.gen_stream(oracle.STREAM_U, 2000, 100 + j))
                x = torch.tensor(oracle.gen_stream(oracle.STREAM_L, 4000, 200 + j), device="cuda")
                torch.cuda.synchronize()
                with ms.recording(histograms=["tok"]) as sc:
                    sc.keyed(torch.zeros(x.numel(), dtype=torch.int32, device="cuda"), x)
                torch.cuda.synchronize()
                for _ in range(j % 3):
                    gg.replay()
                torch.cuda.synchronize()
                if j % 4 == 1:
                    ms.Histogram("idle", 10.0 * j)
                if j in (1, 2, 12):
                    ms.HistogramMany("churn", np.full(7, 3.0 * j))
                if 3 <= j <= 9:                       # other names push "churn" out of the table meanwhile
                    for i in range(3):
                        ms.Histogram("other.%d.%d" % (j, i), 1.0)
                raw, _ = ms.collect_and_process()
                history.append(raw)
                q.replay()
                for s, o in zip(subs, outs):
                    check_names(torch, oracle, table, s, history, names, ps_t, val_t, *o)
        assert "churn" not in history[6]["Histograms"] and "churn" in history[11]["Histograms"]
        for s in subs:
            s.close()
    finally:
        ms.close()


def test_no_torn_answers(oracle, torch, client):
    """A reader kernel queries row 0 of a w = 3 subscription while the host runs 200 collections alternating
    histograms a and b: the window alternates between a + b + a (odd publishes) and b + a + b (even ones), and every
    answer is the one of the publish it names."""
    from loghisto_b200.metric_system import MetricSystem
    n = 200
    ms = MetricSystem(1.0, False, max_histograms=16, max_counters=4)
    a = np.concatenate([np.full(100, 1.5), np.full(50, 1000.0), np.linspace(-5e6, 5e6, 4001)])
    b = np.full(30, 7.0)
    v = 10.0
    kv = int(oracle.compress(v))

    def expect(x):
        k = np.sort(oracle.compress_many(x).astype(np.int64))
        return x.size, int((k <= kv).sum()), int(k[(x.size + 1) // 2 - 1])

    ea, eb = expect(np.concatenate([a, b, a])), expect(np.concatenate([b, a, b]))
    try:
        with ms.raw_device_subscription(histograms=["t", "never"], window=3) as sub:
            for j in range(1, 4):                     # publishes 1 and 2 hold partial windows: read from 3 on
                ms.HistogramMany("t", a if j % 2 else b)
                ms.collect_and_process()
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
            for j in range(4, n + 4):
                ms.HistogramMany("t", a if j % 2 else b)
                ms.collect_and_process()
            host_s = time.monotonic() - t0
            side.synchronize()
            reads, bad, hi, lo, changes = [int(x) for x in stats.cpu().numpy().view(np.uint64)]
            assert bad == 0, (reads, bad, hi, lo, changes)
            assert reads > 0 and hi > lo >= 3 and changes > 0, (reads, hi, lo, changes)
            if host_s < 2.0:
                assert hi == n + 3
    finally:
        ms.close()


class Exchange:
    """An all-gather between rank threads (as tests/test_gpu_ranks.py runs them)."""

    def __init__(self, world):
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)

    def for_rank(self, r):
        def allgather(mine):
            self.slots[r] = bytes(mine)
            self.barrier.wait(timeout=120)
            out = list(self.slots)
            self.barrier.wait(timeout=120)
            return out
        return allgather


def on_ranks(world, fn):
    out, errs = [None] * world, []

    def run(r):
        try:
            out[r] = fn(r)
        except BaseException as e:   # pragma: no cover - reported below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_joined_ranks(oracle, torch, world):
    """JoinRanks at world 2 and 3, one thread per rank on one GPU: every rank's w = 3 subscription answers for the
    job-wide intervals of its names' last three collections (names private to a rank, names present on some ranks in
    some collections, a name never seen)."""
    from loghisto_b200.metric_system import MetricSystem
    ndev = torch.cuda.device_count()
    ex = Exchange(world)
    systems = [MetricSystem(3600.0, device=r % ndev, max_histograms=32, max_counters=4) for r in range(world)]
    table = oracle.decompress_table(100)
    names = ["shared", "r0", "come_go", "never"]
    history = []
    try:
        on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r)))
        subs = [ms.raw_device_subscription(histograms=names, window=3) for ms in systems]
        for j in range(8):
            for r, ms in enumerate(systems):
                ms.HistogramMany("shared", oracle.gen_stream(oracle.STREAM_U, 500 + 10 * r, 10 * j + r))
                if r == 0:
                    ms.HistogramMany("r0", oracle.gen_stream(oracle.STREAM_L, 300, 70 + j))
                if (j + r) % 3 == 0:
                    ms.HistogramMany("come_go", np.array([1e100, 2.0 * j, -3.0]))
            got = on_ranks(world, lambda r: systems[r].collect_and_process())
            for raw, _ in got[1:]:
                assert raw["Histograms"] == got[0][0]["Histograms"]
            history.append(got[0][0])
            for r, (ms, s) in enumerate(zip(systems, subs)):
                with torch.cuda.device(r % ndev):
                    ps_t = torch.tensor(PS, device="cuda")
                    val_t = torch.tensor(VALUES, device="cuda")
                    check_names(torch, oracle, table, s, history, names, ps_t, val_t, *(s.percentiles(ps_t) +
                                                                                       s.ranks(val_t)))
        for s in subs:
            s.close()
    finally:
        for ms in systems:
            ms.close()


def test_validation(lh):
    """Window 0 and above LH_RAW_MAX_WINDOW, a foreign or destroyed handle and a second publish in one snapshot are
    refused with their statuses; headers stay as they were and nothing is enqueued.  The Python layer refuses a bad
    window before any call."""
    from loghisto_b200 import _lib as L
    with lh.Engine(device=0, max_histograms=4, max_counters=1) as eng, lh.Engine(device=0, max_histograms=4) as other:
        lib = eng.lib
        b = L.lh_raw_board()
        before = eng.stats()["kernel_launches"]
        assert lib.lh_raw_board_create_window(eng.h, 2, 0, C.byref(b)) == LH_ERR_INVALID
        assert lib.lh_raw_board_create_window(eng.h, 2, L.LH_RAW_MAX_WINDOW + 1, C.byref(b)) == LH_ERR_RANGE
        assert lib.lh_raw_board_create_window(eng.h, 0, 2, C.byref(b)) == LH_ERR_INVALID
        assert lib.lh_raw_board_create_window(eng.h, 5, 2, C.byref(b)) == LH_ERR_RANGE
        assert lib.lh_raw_board_create_window(eng.h, 1, 2, None) == LH_ERR_INVALID
        for bad, err in ((0, ValueError), (-1, ValueError), (2.0, TypeError), ("2", TypeError), (True, TypeError),
                         (None, TypeError)):
            with pytest.raises(err):
                eng.raw_board(2, window=bad)
        assert eng.stats()["kernel_launches"] == before
        with eng.raw_board(1, window=L.LH_RAW_MAX_WINDOW) as big:   # the maximum is accepted (one row: 2 GiB)
            assert big.window == L.LH_RAW_MAX_WINDOW
        rb = eng.raw_board(4, window=3)
        bb = C.byref(rb.board)
        eng.ingest_keyed_f64_u16_host(np.arange(40, dtype=np.uint16) % 4, np.arange(40.0))
        eng.snapshot_begin()
        assert lib.lh_snapshot_publish_raw(other.h, bb, None) == LH_ERR_INVALID
        assert lib.lh_snapshot_publish_raw(eng.h, bb, (C.c_uint32 * 4)(0, 1, 4, 2)) == LH_ERR_RANGE
        launches = eng.stats()["kernel_launches"]
        rb.publish([0, 1, 2, 3])
        assert eng.stats()["kernel_launches"] == launches + 1
        h1, _ = read_board(eng, rb.board)
        assert lib.lh_snapshot_publish_raw(eng.h, bb, None) == LH_ERR_STATE         # second publish, same snapshot
        assert eng.stats()["kernel_launches"] == launches + 1
        eng.snapshot_end()
        h2, _ = read_board(eng, rb.board)
        assert (h1 == h2).all() and (h1["publishes"] == 1).all() and (h1["total"] == 10).all()
        assert lib.lh_snapshot_publish_raw(eng.h, bb, None) == LH_ERR_STATE         # no snapshot
        eng.snapshot_begin()
        rb.publish(None)                                                              # the next snapshot takes one
        eng.snapshot_end()
        h3, _ = read_board(eng, rb.board)
        assert (h3["publishes"] == 2).all() and (h3["total"] == 10).all()
        saved = L.lh_raw_board.from_buffer_copy(rb.board)
        rb.close()
        eng.snapshot_begin()
        launches = eng.stats()["kernel_launches"]
        assert lib.lh_snapshot_publish_raw(eng.h, C.byref(saved), None) == LH_ERR_INVALID
        assert lib.lh_raw_board_destroy(eng.h, C.byref(saved)) == LH_ERR_INVALID
        assert eng.stats()["kernel_launches"] == launches
        eng.snapshot_end()


def test_one_launch_per_collection(oracle):
    """A collection issues one more launch per open raw subscription, window or not, and none once they are closed."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4)
    try:
        def collect():
            ms.HistogramMany("a", oracle.gen_stream(0, 1000, 3))
            before = ms.stats()["kernel_launches"]
            ms.collect_and_process()
            return ms.stats()["kernel_launches"] - before

        plain = [collect() for _ in range(3)]
        with ms.raw_device_subscription(histograms=["a", "b"], window=4):
            one = [collect() for _ in range(6)]
            with ms.raw_device_subscription(histograms=["a"]), ms.raw_device_subscription(histograms=["b"], window=2):
                three = [collect() for _ in range(3)]
        after = [collect() for _ in range(3)]
        assert plain == after and len(set(plain)) == 1
        assert one == [plain[0] + 1] * 6 and three == [plain[0] + 3] * 3
    finally:
        ms.close()
