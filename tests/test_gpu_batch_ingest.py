"""lh_ingest_batch (Engine.ingest_batch) and RecordScope.histograms on the real library: many device arrays, each under
its own histogram id, in one call.  Every bucket of every histogram is checked against the CPU oracle and against the
same items issued one call each (lh_ingest_f64, and lh_ingest_keyed_i64ns_u16 with a constant id array) on a second
context.  The routing constants (kBatchK1Min, BI_PIECE, BI_MAX_ITEMS) are read from the CUDA sources."""
import ctypes as C
import threading

import numpy as np
import pytest

import _ingest_routes as R

pytestmark = pytest.mark.gpu

SEED = 0xBA7C4
PS = [0.0, 0.5, 0.99, 1.0]
MS = 1_000_000                     # one millisecond of spin, in ns
SPECIALS = np.array([np.inf, -np.inf, np.nan, -np.nan, 2.0 ** 63, -(2.0 ** 64), 1e300, 0.0, -0.0, 5e-324], np.float64)
I64_EDGES = np.array([0, -1, -1000, np.iinfo(np.int64).min, np.iinfo(np.int64).max, 1, (1 << 53) + 1], np.int64)
F64, I64NS = 0, 1


def _constants():
    k = R._src("lh_kernels.cuh")
    a = R._src("lh_api.cu")
    return {"piece": R._int_expr(k, r"constexpr uint32_t BI_PIECE = ([^;]+);", {}),
            "items": R._int_expr(k, r"constexpr int BI_MAX_ITEMS = ([^;]+);", {}),
            "k1_min": R._int_expr(a, r"constexpr size_t kBatchK1Min = ([^;]+);", {})}


K = _constants()


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def spin():
    """spin(ns, stream): enqueue one bounded spin of at least `ns` on a torch stream (tests/gpu_timer_client.cu)."""
    from loghisto_b200 import build
    lib = C.CDLL(build.TIMER_CLIENT_LIB)
    lib.gtc_set_device.argtypes = [C.c_int]
    lib.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    lib.gtc_set_device.restype = lib.gtc_spin.restype = C.c_int
    assert lib.gtc_set_device(0) == 0

    def run(ns, stream):
        assert lib.gtc_spin(int(ns), stream.cuda_stream) == 0
    return run


class Want:
    """(id * 65536 + key) -> count of one interval, keys from the oracle at the context's precision."""

    def __init__(self, oracle, H, precision=100):
        self.oracle, self.H, self.precision = oracle, H, precision
        self.parts = []

    def add(self, hid, vals):
        vals = np.asarray(vals)
        if vals.dtype == np.int64:
            dense = self.oracle.ingest_keyed_i64(np.zeros(vals.size, np.uint32), vals, 1)[0] if self.precision == 100 else \
                self.oracle.ingest(vals.astype(np.float64), precision=self.precision)
            keys = np.nonzero(dense)[0]
            self.parts.append((hid * 65536 + keys.astype(np.int64), dense[keys]))
            return
        keys = self.oracle.compress_many(vals.astype(np.float64), self.precision).view(np.uint16).astype(np.int64)
        u, c = np.unique(keys, return_counts=True)
        self.parts.append((hid * 65536 + u, c.astype(np.uint64)))

    def sparse(self):
        return merge(self.parts)


def merge(parts):
    if not parts:
        return np.zeros(0, np.int64), np.zeros(0, np.uint64)
    u, inv = np.unique(np.concatenate([p[0] for p in parts]), return_inverse=True)
    c = np.zeros(u.size, np.uint64)
    np.add.at(c, inv, np.concatenate([p[1] for p in parts]).astype(np.uint64))
    return u, c


def flat(sp, H):
    """(id * 65536 + key, count) of an export."""
    ids = np.repeat(np.arange(H, dtype=np.int64), np.diff(sp.offsets.astype(np.int64)))
    return merge([(ids * 65536 + sp.keys.view(np.uint16).astype(np.int64), sp.counts)])


def same(a, b, what):
    assert a[0].size == b[0].size and (a[0] == b[0]).all(), (what, a[0].size, b[0].size)
    assert (a[1] == b[1]).all(), (what, np.nonzero(a[1] != b[1])[0][:5])


def expected_launches(items):
    """kernel_launches of one batch without the sample cap: one per F64 item of at least kBatchK1Min samples (K1 splits
    only above 2^31 samples per CTA), plus the batch kernel's launches of BI_MAX_ITEMS items each."""
    k1 = sum(1 for _, n, kind in items if kind == F64 and n >= K["k1_min"])
    rest = sum(1 for _, n, kind in items if n and not (kind == F64 and n >= K["k1_min"]))
    return k1 + (rest + K["items"] - 1) // K["items"]


def issue(e, torch_bufs, items, stream=None):
    """items: (id, offset, n, kind) over the float64 / int64 device buffers; one ingest_batch."""
    e.ingest_batch([(hid, torch_bufs[kind][off:off + n]) for hid, off, n, kind in items], stream)


def one_by_one(e, torch_bufs, torch, items):
    for hid, off, n, kind in items:
        if not n:
            continue
        if kind == F64:
            e.ingest_f64(hid, torch_bufs[F64][off:off + n].data_ptr(), n)
        else:
            ids = torch.full((n,), hid, dtype=torch.int16, device="cuda:0")
            torch.cuda.synchronize()
            e.ingest_keyed_i64ns_u16(ids.data_ptr(), torch_bufs[I64NS][off:off + n].data_ptr(), n)
            e.sync()


def host_values(oracle, n, seed):
    """Streams U, L and S in turn, with special values and the epsilon band spread over them."""
    v = oracle.gen_stream(oracle.STREAM_U, n, seed)
    v[1::3] = oracle.gen_stream(oracle.STREAM_L, n, seed + 1)[1::3]
    v[2::3] = oracle.gen_stream(oracle.STREAM_S, n, seed + 2)[2::3]
    v[5::997] = SPECIALS[np.arange(v[5::997].size) % SPECIALS.size]
    band = R.epsilon_band_values(oracle, 100)
    m = min(band.size, n // 4)
    v[n // 2:n // 2 + m] = band[:m]
    return v


def host_nanos(oracle, n, seed):
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, seed).view(np.int64).copy()
    ns[::5] *= -1
    ns[3::101] = I64_EDGES[np.arange(ns[3::101].size) % I64_EDGES.size]
    return ns


def shape_items(H, total):
    """Items of every length of interest, at 8 / 16 / 24 bytes past 32-byte alignment, ids 0 and H - 1 and repeats."""
    P, K1 = K["piece"], K["k1_min"]
    lengths = [0, 1, 2, 3, 4, 5, 31, 32, 33, P - 1, P, P + 1, 4099, K1 - 1, K1, K1 + 3]
    items, off = [], 0
    for i, n in enumerate(lengths):
        for kind in (F64, I64NS):
            if kind == I64NS and n > 5 * P:
                n = n // 7
            shift = (1, 2, 3, 4)[(i + kind) % 4]             # 8, 16, 24 and 32 bytes past a 32-byte boundary
            start = (off + 3) // 4 * 4 + shift
            hid = (0, H - 1, i % H, 1)[(i + kind) % 4]
            items.append((hid, start, n, kind))
            off = start + n
    assert off < total
    return items


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_item_shapes_match_the_oracle_and_single_calls(lh, oracle, torch, precision):
    H = 7
    items = shape_items(H, 4 << 20)
    total = 4 << 20
    vals, ns = host_values(oracle, total, SEED ^ precision), host_nanos(oracle, total, SEED + precision)
    bufs = {F64: torch.from_numpy(vals).cuda(), I64NS: torch.from_numpy(ns).cuda()}
    want = Want(oracle, H, precision)
    for hid, off, n, kind in items:
        want.add(hid, (vals if kind == F64 else ns)[off:off + n])
    with lh.Engine(device=0, max_histograms=H, precision=precision) as e, \
            lh.Engine(device=0, max_histograms=H, precision=precision) as ref:
        torch.cuda.synchronize()
        st0, seq0 = e.stats(), e.ingest_seq()
        issue(e, bufs, items)
        st1 = e.stats()
        assert e.ingest_seq() == seq0 + 1
        e.sync()
        assert np.isfinite(e.kernel_ms(seq0 + 1)) and e.kernel_ms(seq0 + 1) > 0
        assert st1["samples"] - st0["samples"] == sum(n for _, _, n, _ in items)
        assert st1["kernel_launches"] - st0["kernel_launches"] == expected_launches([(h, n, k) for h, _, n, k in items])
        one_by_one(ref, bufs, torch, items)
        got = flat(e.snapshot(PS)[1], H)
        same(got, want.sparse(), ("oracle", precision))
        same(got, flat(ref.snapshot(PS)[1], H), ("single calls", precision))


def test_table_overflow_is_exact(lh, oracle, torch):
    """Each CTA sees far more distinct (id, bucket) pairs than its table has slots: 2048 short items of stream U over
    H = 1024, and 1024 items of stream U of varied length."""
    H = 1024
    rng = np.random.default_rng(SEED)
    vals = oracle.gen_stream(oracle.STREAM_U, 3 << 20, SEED)
    d = torch.from_numpy(vals).cuda()
    for lens in (np.full(2048, 40), rng.integers(1, 3000, 1024)):
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
        items = [(int(i % H), int(o), int(n)) for i, (o, n) in enumerate(zip(offs, lens))]
        want = Want(oracle, H)
        for hid, o, n in items:
            want.add(hid, vals[o:o + n])
        with lh.Engine(device=0, max_histograms=H) as e:
            before = e.stats()["kernel_launches"]
            e.ingest_batch([(hid, d[o:o + n]) for hid, o, n in items])
            assert e.stats()["kernel_launches"] - before == expected_launches([(h, n, F64) for h, _, n in items])
            same(flat(e.snapshot(PS)[1], H), want.sparse(), ("overflow", lens.size))


def test_more_items_than_one_parameter_block(lh, oracle, torch):
    H = 97
    rng = np.random.default_rng(SEED + 1)
    lens = rng.integers(0, 300, 5000)
    vals, ns = host_values(oracle, int(lens.sum()), SEED + 2), host_nanos(oracle, int(lens.sum()), SEED + 3)
    bufs = {F64: torch.from_numpy(vals).cuda(), I64NS: torch.from_numpy(ns).cuda()}
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    items = [(int(rng.integers(0, H)), int(o), int(n), int(i % 3 == 0)) for i, (o, n) in enumerate(zip(offs, lens))]
    want = Want(oracle, H)
    for hid, off, n, kind in items:
        want.add(hid, (vals if kind == F64 else ns)[off:off + n])
    with lh.Engine(device=0, max_histograms=H) as e:
        st0, seq0 = e.stats(), e.ingest_seq()
        issue(e, bufs, items)
        st1 = e.stats()
        assert e.ingest_seq() == seq0 + 1
        launches = st1["kernel_launches"] - st0["kernel_launches"]
        assert launches == expected_launches([(h, n, k) for h, _, n, k in items]) and launches >= 4
        same(flat(e.snapshot(PS)[1], H), want.sparse(), "5000 items")


def test_full_size_batch(lh, oracle):
    """About 1e9 samples of stream U in 4096 items of varied length over H = 1024 ids (long items through K1), checked
    bucket for bucket with the oracle's streaming checker."""
    H, n_items = 1024, 4096
    rng = np.random.default_rng(SEED + 4)
    lens = rng.integers(1, 2 * 240_000, n_items)
    lens[::64] = K["k1_min"] + rng.integers(0, 1 << 20, lens[::64].size)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    total = int(lens.sum())
    assert 0.9e9 < total < 1.2e9
    with lh.Engine(device=0, max_histograms=H) as e:
        d = e.gen_stream(lh.STREAM_U, total, lh.DEFAULT_SEED)
        before = e.stats()
        e.ingest_batch([(i % H, _Slice(d, int(o), int(n))) for i, (o, n) in enumerate(zip(offs, lens))])
        after = e.stats()
        assert after["samples"] - before["samples"] == total
        assert after["kernel_launches"] - before["kernel_launches"] == \
            expected_launches([(0, int(n), F64) for n in lens])
        e.snapshot_begin()
        try:
            for hid in range(H):
                want = np.zeros(65536, np.uint64)
                for i in range(hid, n_items, H):
                    oracle.stream_ingest(oracle.STREAM_U, int(lens[i]), lh.DEFAULT_SEED, int(offs[i]), want)
                got = e.snapshot_copy_histogram(hid)
                assert (got == want).all(), (hid, np.nonzero(got != want)[0][:5])
        finally:
            e.snapshot_end()
        d.free()


class _Slice:
    """n float64 of a DeviceArray from element `off`, as a __cuda_array_interface__ object."""

    def __init__(self, d, off, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (d.offset(off), False),
                                         "version": 3}


def test_validation_changes_nothing(lh, oracle, torch):
    H = 4
    good = torch.arange(1, 65, dtype=torch.float64, device="cuda:0")
    gns = torch.arange(1, 65, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    with lh.Engine(device=0, max_histograms=H) as e:
        e.ingest_f64(2, good.data_ptr(), 3)
        e.sync()
        base = (e.stats(), e.ingest_seq())
        L = e.lib
        Item = lh._lib.lh_batch_item

        def call(*items, n_items=None, ptr=True):
            arr = (Item * max(len(items), 1))(*[Item(*it) for it in items])
            return L.lh_ingest_batch(e.h, arr if ptr else None, len(items) if n_items is None else n_items, None)
        ok = (good.data_ptr(), 64, 1, F64)
        cases = [
            (lh._lib.LH_ERR_INVALID, dict(n_items=3, ptr=False)),
            (lh._lib.LH_ERR_INVALID, (ok, (0, 5, 0, F64))),
            (lh._lib.LH_ERR_INVALID, (ok, (good.data_ptr() + 4, 5, 0, F64))),
            (lh._lib.LH_ERR_INVALID, (ok, (gns.data_ptr() + 2, 5, 0, I64NS))),
            (lh._lib.LH_ERR_INVALID, (ok, (good.data_ptr(), 5, 0, 2))),
            (lh._lib.LH_ERR_INVALID, (ok, (0, 0, 0, 7))),
            (lh._lib.LH_ERR_RANGE, (ok, (good.data_ptr(), 5, H, F64))),
            (lh._lib.LH_ERR_RANGE, ((good.data_ptr(), 5, 0xFFFFFFFF, F64), ok)),
        ]
        for status, c in cases:
            got = call(**c) if isinstance(c, dict) else call(*c)
            assert got == status, (c, got)
            assert (e.stats(), e.ingest_seq()) == base, c
        # no samples: LH_OK, no bracket, no launch (bad ids and pointers of empty items are not looked at)
        assert call() == 0
        assert call((0, 0, H + 5, F64), (good.data_ptr() + 1, 0, 0, I64NS)) == 0
        e.ingest_batch([])
        e.ingest_batch([(0, good[:0]), (3, gns[:0])])
        assert (e.stats(), e.ingest_seq()) == base
        with pytest.raises(lh.LhError) as ex:
            e.ingest_batch([(0, good), (H, good)])
        assert ex.value.status == lh._lib.LH_ERR_RANGE
        assert (e.stats(), e.ingest_seq()) == base
        want = Want(oracle, H)
        want.add(2, good[:3].cpu().numpy())
        same(flat(e.snapshot(PS)[1], H), want.sparse(), "after refused calls")


def test_batch_on_a_stalled_stream_lands_in_its_interval(lh, oracle, torch, spin):
    H = 8
    vals = host_values(oracle, 200_000, SEED + 5)
    d = torch.from_numpy(vals).cuda()
    items = [(i % H, d[i * 1000:(i + 1) * 1000 + i]) for i in range(150)]
    want = Want(oracle, H)
    for i in range(150):
        want.add(i % H, vals[i * 1000:(i + 1) * 1000 + i])
    with lh.Engine(device=0, max_histograms=H) as e:
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        spin(30 * MS, st)
        e.ingest_batch(items, st)
        e.snapshot_begin()
        try:
            got = flat(e.snapshot_export(), H)
        finally:
            e.snapshot_end()
        same(got, want.sparse(), "stalled stream")
        assert flat(e.snapshot(PS)[1], H)[0].size == 0


def test_four_streams_and_a_snapshot_thread(lh, oracle, torch, spin):
    H, rounds = 64, 12
    vals, ns = host_values(oracle, 1 << 20, SEED + 6), host_nanos(oracle, 1 << 20, SEED + 7)
    bufs = {F64: torch.from_numpy(vals).cuda(), I64NS: torch.from_numpy(ns).cuda()}
    rng = np.random.default_rng(SEED + 8)
    plans = []
    for t in range(4):
        plan = []
        for r in range(rounds):
            items = []
            for _ in range(int(rng.integers(1, 40))):
                n = int(rng.integers(0, 20_000))
                off = int(rng.integers(0, (1 << 20) - n))
                items.append((int(rng.integers(0, H)), off, n, int(rng.integers(0, 2))))
            plan.append(items)
        plans.append(plan)
    want = Want(oracle, H)
    for plan in plans:
        for items in plan:
            for hid, off, n, kind in items:
                want.add(hid, (vals if kind == F64 else ns)[off:off + n])
    with lh.Engine(device=0, max_histograms=H) as e:
        torch.cuda.synchronize()
        streams = [torch.cuda.Stream() for _ in range(4)]
        got, stop, errors = [], threading.Event(), []

        def snapper():
            try:
                while not stop.is_set():
                    got.append(flat(e.snapshot(PS)[1], H))
            except BaseException as ex:
                errors.append(ex)

        def writer(t):
            try:
                for r, items in enumerate(plans[t]):
                    spin((1 + (t + r) % 4) * MS // 2, streams[t])
                    issue(e, bufs, items, streams[t])
            except BaseException as ex:
                errors.append(ex)

        th = [threading.Thread(target=writer, args=(t,)) for t in range(4)]
        snap = threading.Thread(target=snapper)
        snap.start()
        for x in th:
            x.start()
        for x in th:
            x.join()
        stop.set()
        snap.join()
        assert not errors, errors
        got.append(flat(e.snapshot(PS)[1], H))
        same(merge(got), want.sparse(), "four streams")


def test_metric_system_histograms(lh, oracle, torch):
    from loghisto_b200.metric_system import MetricSystem
    vals = host_values(oracle, 300_000, SEED + 9)
    ns = host_nanos(oracle, 50_000, SEED + 10)
    d, dn = torch.from_numpy(vals).cuda(), torch.from_numpy(ns).cuda()
    torch.cuda.synchronize()
    ms = MetricSystem(1e-6, False, max_histograms=8, max_counters=4)
    small = MetricSystem(1e-6, False, max_histograms=2, max_counters=2)
    ref = oracle.OracleMetricSystem()
    try:
        st = torch.cuda.Stream()
        with ms.recording(st, histograms=["lat", "size", "ns"]) as s:
            s.histograms({"lat": d[:1000], "size": d[1000:151_000], "ns": dn})
            s.histograms([("lat", d[151_000:151_007]), ("lat", d[200_000:300_000]), ("size", d[5:6])])
        for a, b, nm in ((0, 1000, "lat"), (1000, 151_000, "size"), (151_000, 151_007, "lat"), (200_000, 300_000, "lat"),
                         (5, 6, "size")):
            for v in vals[a:b]:
                ref.Histogram(nm, float(v))
        for x in ns:
            ref.Histogram("ns", float(x))
        st.synchronize()
        raw, m = ms.collect_and_process()
        rraw, rm = ref.collect_and_process()
        assert raw["Histograms"] == rraw["Histograms"]
        for k in rm:
            if k in m and k.split("_")[0] in ("lat", "size", "ns") and not k.endswith(("_sum", "_avg")):
                assert m[k] == rm[k], k
        assert ms.dropped() == 0
        # a name that found no free id: its samples are dropped and counted, the others recorded
        for nm in ("a", "b"):
            small.Histogram(nm, 1.0)
        with small.recording(st, histograms=["late", "a"]) as s:
            assert s.histogram_ids["late"] == s.UNBOUND
            s.histograms([("late", d[:123]), ("a", d[:10]), ("late", dn[:7])])
        st.synchronize()
        raw, _ = small.collect_and_process()
        assert "late" not in raw["Histograms"]
        assert sum(raw["Histograms"]["a"].values()) == 11
        assert small.dropped() == 130
        with ms.recording(st, histograms=["lat"]) as s:
            with pytest.raises(KeyError):
                s.histograms({"nope": d[:3]})
            with pytest.raises(TypeError):
                s.histograms({"lat": d[:3].float()})
    finally:
        ms.close()
        small.close()
        ref.close()


def test_engine_type_checks(lh, torch):
    with lh.Engine(device=0, max_histograms=2) as e:
        for bad in (torch.zeros(4, dtype=torch.float64), torch.zeros(4, dtype=torch.float32, device="cuda:0"),
                    torch.zeros((4, 2), dtype=torch.float64, device="cuda:0")[:, 0], np.zeros(4)):
            with pytest.raises(TypeError):
                e.ingest_batch([(0, bad)])
        assert e.ingest_seq() == 0
