"""lh_ingest_arrays / lh_graph_recorder_ingest_arrays (Engine.ingest_arrays, RecordScope.arrays, GraphRecorder.arrays)
on the real library: device arrays of float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64 recorded without a
float64 copy.  Every histogram is compared bucket for bucket with the CPU oracle fed the values as numpy's
astype(float64), on every route: the short-item kernel, K1 (float64), its 4-byte form (float32, int32) and its 16-bit
key-table form (float16, bfloat16).  The routing thresholds are read from the CUDA sources."""
import ctypes as C
import threading

import numpy as np
import pytest

import _ingest_routes as R

pytestmark = pytest.mark.gpu

SEED = 0xA77A5
PS = [0.0, 0.5, 0.99, 1.0]
PRECISIONS = [1, 50, 100, 200, 250]
F64, F32, F16, BF16, I64, I32, U64 = range(7)
TORCH = {F64: "float64", F32: "float32", F16: "float16", BF16: "bfloat16", I64: "int64", I32: "int32", U64: "uint64"}
SIZE = {F64: 8, F32: 4, F16: 2, BF16: 2, I64: 8, I32: 4, U64: 8}
MS = 1_000_000                     # one millisecond of spin, in ns


def _constants():
    a = R._src("lh_api.cu")
    k1 = R._int_expr(a, r"constexpr size_t kBatchK1Min = ([^;]+);", {})
    four = R._int_expr(a, r"constexpr size_t kArraysK1Min4 = ([^;]+);", {})
    two = R._int_expr(a, r"constexpr size_t kArraysK1Min2 = ([^;]+);", {})
    return {F64: k1, F32: four, I32: four, F16: two, BF16: two}


THRESHOLD = _constants()


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


def as_f64(bits, dtype):
    """float64(x) of raw element bits as Go converts them (numpy: exact for floats and int32, nearest even for 64-bit
    integers)."""
    with np.errstate(invalid="ignore"):   # NaN patterns
        return _as_f64(bits, dtype)


def _as_f64(bits, dtype):
    if dtype == F64:
        return bits.view(np.float64).copy()
    if dtype == F32:
        return bits.view(np.float32).astype(np.float64)
    if dtype == F16:
        return bits.view(np.float16).astype(np.float64)
    if dtype == BF16:
        return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    if dtype == I64:
        return bits.view(np.int64).astype(np.float64)
    if dtype == I32:
        return bits.view(np.int32).astype(np.float64)
    return bits.view(np.uint64).astype(np.float64)


def device(torch, bits, dtype, off=0):
    """The raw bits on cuda:0 as a tensor of `dtype`, `off` elements past the start of its allocation."""
    t = torch.empty(bits.size + off, dtype=getattr(torch, TORCH[dtype]), device="cuda:0")
    raw = {8: torch.int64, 4: torch.int32, 2: torch.int16}[SIZE[dtype]]
    t.view(raw)[off:] = torch.from_numpy(bits.view({8: np.int64, 4: np.int32, 2: np.int16}[SIZE[dtype]])).cuda()
    return t[off:]


def dense(oracle, vals, precision):
    return oracle.ingest(np.ascontiguousarray(vals, np.float64), precision=precision)


def rows(e, ids):
    e.snapshot_begin()
    try:
        return {h: e.snapshot_copy_histogram(h) for h in ids}
    finally:
        e.snapshot_end()


def check(e, want, what):
    got = rows(e, list(want))
    for h, w in want.items():
        assert (got[h] == w).all(), (what, h, np.nonzero(got[h] != w)[0][:5])


def all_16bit():
    return np.arange(65536, dtype=np.uint32).astype(np.uint16)


def f32_boundaries(precision):
    """float32(T[k]) and its two float32 neighbours for every bucket boundary T[k] of the fast window at `precision`
    (T[k] = e^((k - 1/2) / precision) - 1, where compress steps from k - 1 to k), both signs."""
    win = int(np.floor(precision * 63.0 * np.log(2.0) + 0.5)) + 1
    t = np.expm1((np.arange(1, win, dtype=np.float64) - 0.5) / precision)
    with np.errstate(over="ignore"):
        t32 = t.astype(np.float32)
    t32 = t32[np.isfinite(t32)]
    near = np.concatenate([t32, np.nextafter(t32, np.float32(np.inf)), np.nextafter(t32, np.float32(-np.inf))])
    return np.concatenate([near, -near]).view(np.uint32)


def f32_patterns(oracle, rng, precision):
    """The float32 checks, most telling first: every fast-window boundary of the context's precision and of 50 / 100 /
    200 (at, above and below), the epsilon band as float32, streams U / L / S as float32, the specials (+-0,
    subnormals, +-FLT_MAX, Inf, NaN) and 10^6 random bit patterns."""
    fl = np.finfo(np.float32)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, fl.max, -fl.max, fl.tiny, -fl.tiny, fl.smallest_subnormal,
                         -fl.smallest_subnormal, 1.0, -1.0], np.float32).view(np.uint32)
    rnd = rng.integers(0, 1 << 32, 10 ** 6, dtype=np.uint64).astype(np.uint32)
    n = 1 << 18
    streams = np.concatenate([oracle.gen_stream(k, n, SEED + k) for k in (oracle.STREAM_U, oracle.STREAM_L, oracle.STREAM_S)])
    with np.errstate(over="ignore"):
        streams = streams.astype(np.float32).view(np.uint32)
    bounds = np.concatenate([f32_boundaries(p) for p in sorted({precision, 50, 100, 200})])
    with np.errstate(over="ignore"):
        band = R.epsilon_band_values(oracle, precision).astype(np.float32).view(np.uint32)
    return np.concatenate([bounds, band, streams, specials, rnd])


def int_patterns(dtype):
    if dtype == I32:
        v = np.array([0, 1, -1, 2 ** 31 - 1, -2 ** 31, 2 ** 24 + 1, -(2 ** 24 + 1), 1000, -1000], np.int64)
        return v.astype(np.int32).view(np.uint32)
    ties = [2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, 2 ** 53 + 3, 2 ** 63 - 1, 2 ** 63 - 512, 2 ** 63 - 513, 2 ** 63 - 1024,
            2 ** 54 + 2, 2 ** 54 + 6, 0, 1]
    if dtype == I64:
        neg = [-x for x in ties if x] + [-2 ** 63, -1]
        return np.array(ties + neg, np.int64).view(np.uint64)
    big = [2 ** 64 - 1, 2 ** 64 - 1024, 2 ** 64 - 1025, 2 ** 64 - 2048, 2 ** 63, 2 ** 63 + 1024, 2 ** 63 + 1025]
    return np.array(ties + big, np.uint64)


def tile(bits, n):
    return np.resize(bits, n)


def patterns(oracle, dtype, precision):
    rng = np.random.default_rng([SEED, dtype, precision])
    if dtype in (F16, BF16):
        return all_16bit()
    if dtype == F32:
        return f32_patterns(oracle, rng, precision)
    if dtype == F64:
        v = R.epsilon_band_values(oracle, precision)
        return np.concatenate([v, np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, 5e-324, 2.0 ** 63, -2.0 ** 70])]).view(np.uint64)
    return int_patterns(dtype)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_every_dtype_on_both_routes_matches_the_oracle(lh, oracle, torch, precision):
    """Each dtype's patterns as a short item (k_ingest_arrays) and tiled past its K1 threshold (when it has one), at
    every natural misalignment against 32 bytes, in one call: every row equals the oracle's."""
    H = 16
    items, want = [], {}
    hid = 0
    short = min(THRESHOLD.values()) - 1
    for dtype in range(7):
        pats = patterns(oracle, dtype, precision)
        # every pattern on the short route (pieces below the threshold under one id) ...
        off = (hid * 3) % (32 // SIZE[dtype])
        d = device(torch, pats, dtype, off)
        items += [(hid, d[o:o + short]) for o in range(0, pats.size, short)]
        want[hid] = dense(oracle, as_f64(pats, dtype), precision)
        hid += 1
        # ... and every pattern again in one item past the threshold (tiled up to it when shorter)
        if dtype in THRESHOLD:
            bits = tile(pats, max(THRESHOLD[dtype] + 7, pats.size))
            off = (hid * 3) % (32 // SIZE[dtype])
            items.append((hid, device(torch, bits, dtype, off)))
            want[hid] = dense(oracle, as_f64(bits, dtype), precision)
            hid += 1
    assert hid <= H
    with lh.Engine(device=0, max_histograms=H, precision=precision) as e:
        torch.cuda.synchronize()
        st0, seq0 = e.stats(), e.ingest_seq()
        e.ingest_arrays(items)
        st1 = e.stats()
        assert e.ingest_seq() == seq0 + 1
        assert st1["samples"] - st0["samples"] == sum(t.numel() for _, t in items)
        assert st1["kernel_launches"] - st0["kernel_launches"] == 1 + len(THRESHOLD)
        check(e, want, ("routes", precision))


@pytest.mark.parametrize("dtype", [F32, I32, F16, BF16, F64])
def test_threshold_boundaries_and_misalignment(lh, oracle, torch, dtype):
    """Lengths threshold - 1, threshold and threshold + 7 at every natural misalignment against 32 bytes: one launch
    per item on K1 and one k_ingest_arrays launch for the short ones; every row equals the oracle's."""
    t = THRESHOLD[dtype]
    rng = np.random.default_rng([SEED, dtype, 7])
    base = patterns(oracle, dtype, 100)
    offs = list(range(32 // SIZE[dtype]))
    items, want, long_items, hid = [], {}, 0, 0
    for n in (t - 1, t, t + 7):
        for off in offs:
            bits = tile(base[rng.permutation(base.size)], n)
            items.append((hid, device(torch, bits, dtype, off)))
            want[hid] = dense(oracle, as_f64(bits, dtype), 100)
            long_items += n >= t
            hid += 1
    with lh.Engine(device=0, max_histograms=hid) as e:
        torch.cuda.synchronize()
        l0 = e.stats()["kernel_launches"]
        e.ingest_arrays(items)
        assert e.stats()["kernel_launches"] - l0 == long_items + 1
        check(e, want, ("thresholds", dtype))


def test_graph_recorder_every_16bit_pattern_and_f32(lh, oracle, torch):
    """Captured in torch.cuda.graph, replayed 0..3 times between collections: every float16 and bfloat16 pattern on
    both routes and float32 patterns past the 4-byte threshold, under local ids mapped to context ids."""
    H = 8
    hmap = [7, 3, 5, 1, 6]
    bits16 = all_16bit()
    specs = [(F16, bits16), (BF16, bits16), (F16, tile(bits16, THRESHOLD[F16] + 9)),
             (BF16, tile(bits16, THRESHOLD[BF16] + 9)),
             (F32, f32_patterns(oracle, np.random.default_rng(1), 100))]
    specs[-1] = (F32, tile(specs[-1][1], max(THRESHOLD[F32] + 3, specs[-1][1].size)))
    for precision in (1, 100, 250):
        with lh.Engine(device=0, max_histograms=H, precision=precision) as e:
            items = [(i, device(torch, b, d, i % 3)) for i, (d, b) in enumerate(specs)]
            want = {hmap[i]: dense(oracle, as_f64(b, d), precision) for i, (d, b) in enumerate(specs)}
            with e.graph_recorder(hmap) as gr:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=torch.cuda.Stream()):
                    gr.ingest_arrays(items)
                torch.cuda.synchronize()
                for reps in (0, 1, 3):
                    for _ in range(reps):
                        g.replay()
                    torch.cuda.synchronize()
                    got = rows(e, list(want))   # snapshot_begin drains the replays into the interval it freezes
                    for h, w in want.items():
                        assert (got[h] == w * np.uint64(reps)).all(), (precision, reps, h)


def test_i64_and_f64_equal_ingest_batch(lh, oracle, torch):
    """An I64 item counts as lh_ingest_batch's LH_VALUES_I64NS on the same memory, an F64 item as LH_VALUES_F64."""
    n = THRESHOLD[F64] + 5
    rng = np.random.default_rng(SEED + 3)
    ns = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    edges = int_patterns(I64).view(np.int64)
    ns[:edges.size] = edges
    vals = oracle.gen_stream(oracle.STREAM_U, n, SEED)
    d_ns, d_v = torch.from_numpy(ns).cuda(), torch.from_numpy(vals).cuda()
    torch.cuda.synchronize()
    for m in (37, n):
        with lh.Engine(device=0, max_histograms=2) as a, lh.Engine(device=0, max_histograms=2) as b:
            a.ingest_arrays([(0, d_ns[:m]), (1, d_v[:m])])
            b.ingest_batch([(0, d_ns[:m]), (1, d_v[:m])])
            ra, rb = rows(a, [0, 1]), rows(b, [0, 1])
            for h in (0, 1):
                assert (ra[h] == rb[h]).all(), (m, h)


def test_many_items_split_across_launches(lh, oracle, torch):
    """1 025 short items of mixed dtypes (two launches of the short-item kernel), ids repeated and aliased memory."""
    H = 64
    rng = np.random.default_rng(SEED + 4)
    items, want = [], {h: np.zeros(65536, np.uint64) for h in range(H)}
    pools = {d: (patterns(oracle, d, 100), None) for d in range(7)}
    for d in range(7):
        pools[d] = (pools[d][0], device(torch, tile(pools[d][0], 5000), d))
    for i in range(1025):
        d = int(rng.integers(0, 7))
        off, n = int(rng.integers(0, 4000)), int(rng.integers(1, 900))
        hid = int(rng.integers(0, H))
        items.append((hid, pools[d][1][off:off + n]))
        want[hid] += dense(oracle, as_f64(tile(pools[d][0], 5000)[off:off + n], d), 100)
    with lh.Engine(device=0, max_histograms=H) as e:
        torch.cuda.synchronize()
        l0 = e.stats()["kernel_launches"]
        e.ingest_arrays(items)
        assert e.stats()["kernel_launches"] - l0 == 2
        check(e, want, "1025 items")


def test_large_items(lh, oracle, torch):
    """A 2^28-element float32 item, and about 1e9 bfloat16 samples over 64 ids, bucket for bucket."""
    n = 1 << 28
    g = torch.Generator(device="cuda:0").manual_seed(5)
    x = (torch.randn(n, device="cuda:0", generator=g) * 30).exp_().to(torch.float32)
    x[::3] *= -1
    torch.cuda.synchronize()
    with lh.Engine(device=0, max_histograms=64) as e:
        e.ingest_arrays([(0, x)])
        want = dense(oracle, x.cpu().numpy().astype(np.float64), 100)
        check(e, {0: want}, "2^28 float32")
        del x
        per = 15_625_000
        y = torch.randn(per, device="cuda:0", generator=g).mul_(8).exp_().to(torch.bfloat16)
        y[1::2] *= -1
        yb = y.view(torch.int16).cpu().numpy().view(np.uint16)
        one = dense(oracle, as_f64(yb, BF16), 100)
        torch.cuda.synchronize()
        e.ingest_arrays([(h, y) for h in range(64)])
        check(e, {h: one for h in range(64)}, "1e9 bfloat16")


def test_refusals_launch_nothing(lh, torch):
    import loghisto_b200._lib as L
    good = torch.ones(64, dtype=torch.float32, device="cuda:0")
    with lh.Engine(device=0, max_histograms=4) as e:
        torch.cuda.synchronize()
        st0, seq0 = e.stats(), e.ingest_seq()
        lib = e.lib

        def call(srcs):
            arr = (L.lh_array_src * max(len(srcs), 1))(*srcs)
            return lib.lh_ingest_arrays(e.h, arr, len(srcs), None)
        p = good.data_ptr()
        assert call([L.lh_array_src(p, 64, 1, 0), L.lh_array_src(p, 4, 7, 0)]) == L.LH_ERR_INVALID     # dtype
        assert call([L.lh_array_src(p, 64, 1, 0), L.lh_array_src(0, 4, 1, 0)]) == L.LH_ERR_INVALID     # NULL
        assert call([L.lh_array_src(p, 64, 1, 0), L.lh_array_src(p + 2, 4, 1, 0)]) == L.LH_ERR_INVALID  # misaligned
        assert call([L.lh_array_src(p, 64, 1, 0), L.lh_array_src(p + 4, 4, 0, 0)]) == L.LH_ERR_INVALID  # f64 at 4 B
        assert call([L.lh_array_src(p, 64, 1, 0), L.lh_array_src(p, 4, 1, 4)]) == L.LH_ERR_RANGE
        assert lib.lh_ingest_arrays(e.h, None, 3, None) == L.LH_ERR_INVALID
        assert call([L.lh_array_src(0, 0, 1, 99)]) == L.LH_OK                                          # n == 0: skipped
        with pytest.raises(TypeError):
            e.ingest_arrays([(0, good), (1, good.cpu())])
        with pytest.raises(TypeError):
            e.ingest_arrays([(0, good), (1, torch.ones(4, 2, device="cuda:0").t())])
        with pytest.raises(TypeError):
            e.ingest_arrays([(0, torch.ones(4, dtype=torch.int16, device="cuda:0"))])
        st1 = e.stats()
        assert st1["kernel_launches"] == st0["kernel_launches"] and st1["samples"] == st0["samples"]
        assert e.ingest_seq() == seq0


def test_metric_system_scopes_and_graph_recorders(lh, oracle, torch):
    """RecordScope.arrays and GraphRecorder.arrays under names: each collection equals the oracle's buckets of the
    values as float64; an unbound name's samples are dropped and counted."""
    from loghisto_b200.metric_system import MetricSystem
    c = oracle.compress
    ms = MetricSystem(3600, max_histograms=3, max_counters=1)
    try:
        a = torch.tensor([1.5, -2.5, 1e9, 0.0], dtype=torch.float32, device="cuda:0")
        b = torch.tensor([3, -7, 3], dtype=torch.int32, device="cuda:0")
        h = torch.tensor([0.5, 65504.0], dtype=torch.bfloat16, device="cuda:0")
        torch.cuda.synchronize()
        with ms.graph_recorder(histograms=["g"]) as g:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=torch.cuda.Stream()):
                g.arrays({"g": h})
            torch.cuda.synchronize()
            with pytest.raises(KeyError):
                g.arrays({"nope": h})
            for reps in (0, 2):
                with ms.recording(histograms=["lat", "tok"]) as s:
                    s.arrays([("lat", a), ("tok", b), ("lat", a[:1])])
                    with pytest.raises(KeyError):
                        s.arrays({"zzz": a})
                    with pytest.raises(TypeError):
                        s.arrays({"lat": a.double().cpu()})
                for _ in range(reps):
                    graph.replay()
                torch.cuda.synchronize()
                raw, _ = ms.collect_and_process()
                want_lat = {}
                for v in (1.5, -2.5, 1e9, 0.0, 1.5):
                    want_lat[c(v)] = want_lat.get(c(v), 0) + 1
                want = {"lat": want_lat, "tok": {c(3.0): 2, c(-7.0): 1}}
                if reps:
                    want["g"] = {c(0.5): reps, c(65504.0): reps}
                assert raw["Histograms"] == want, reps
            with ms.recording(histograms=["x1", "x2", "x3", "x4"]) as s:   # only 3 ids: some name is unbound
                unbound = sum(1 for i in s.histogram_ids.values() if i == 0xFFFFFFFF)
                d0 = ms.dropped()
                s.arrays([(nm, b) for nm in ("x1", "x2", "x3", "x4")])
            torch.cuda.synchronize()
            assert unbound >= 1 and ms.dropped() - d0 == 3 * unbound
    finally:
        ms.close()


def dense_export(sp, H):
    """[H, 65536] bucket counts of a snapshot export."""
    out = np.zeros((H, 65536), np.uint64)
    ids = np.repeat(np.arange(H, dtype=np.int64), np.diff(sp.offsets.astype(np.int64)))
    np.add.at(out, (ids, sp.keys.view(np.uint16).astype(np.int64)), sp.counts.astype(np.uint64))
    return out


def mixed_pool(oracle, torch, n):
    """{dtype: (host bits, device tensor)} of n elements per dtype: its patterns tiled."""
    return {d: (b, device(torch, b, d)) for d in range(7) for b in [tile(patterns(oracle, d, 100), n)]}


def test_arrays_on_a_stalled_stream_land_in_their_interval(lh, oracle, torch, spin):
    """A call issued behind a 30 ms spin on its stream, snapshot right after: every sample, long items of the narrow K1
    forms included, is in the interval the call was made in, and none in the next."""
    H = 8
    pool = mixed_pool(oracle, torch, (1 << 20) + 100)
    items, want = [], np.zeros((H, 65536), np.uint64)
    for i in range(60):
        d = i % 7
        n = THRESHOLD[d] + 3 if (i % 10 == 0 and d in THRESHOLD) else 1000 + i
        items.append((i % H, pool[d][1][i:i + n]))
        want[i % H] += dense(oracle, as_f64(pool[d][0][i:i + n], d), 100)
    with lh.Engine(device=0, max_histograms=H) as e:
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        spin(30 * MS, st)
        e.ingest_arrays(items, st)
        e.snapshot_begin()
        try:
            got = dense_export(e.snapshot_export(), H)
        finally:
            e.snapshot_end()
        assert (got == want).all(), np.argwhere(got != want)[:5]
        assert dense_export(e.snapshot(PS)[1], H).sum() == 0


def test_four_streams_and_a_snapshot_thread(lh, oracle, torch, spin):
    """Four threads issue calls on their own streams behind short spins while a fifth snapshots in a loop: the sum of
    every interval equals the oracle's, so no sample is lost or counted twice across the brackets."""
    H, rounds = 64, 12
    pool = mixed_pool(oracle, torch, (1 << 20) + 50_000)
    rng = np.random.default_rng(SEED + 8)
    plans, want = [], np.zeros((H, 65536), np.uint64)
    for t in range(4):
        plan = []
        for r in range(rounds):
            items = []
            for j in range(int(rng.integers(1, 40))):
                d = int(rng.integers(0, 7))
                long_ = r == t and j == 0 and d in THRESHOLD
                n = THRESHOLD[d] + 5 if long_ else int(rng.integers(0, 20_000))
                off = int(rng.integers(0, pool[d][0].size - n))
                hid = int(rng.integers(0, H))
                items.append((hid, d, off, n))
                want[hid] += dense(oracle, as_f64(pool[d][0][off:off + n], d), 100)
            plan.append(items)
        plans.append(plan)
    with lh.Engine(device=0, max_histograms=H) as e:
        torch.cuda.synchronize()
        streams = [torch.cuda.Stream() for _ in range(4)]
        got, stop, errors = np.zeros((H, 65536), np.uint64), threading.Event(), []

        def snapper():
            try:
                while not stop.is_set():
                    got[...] += dense_export(e.snapshot(PS)[1], H)
            except BaseException as ex:
                errors.append(ex)

        def writer(t):
            try:
                for r, items in enumerate(plans[t]):
                    spin((1 + (t + r) % 4) * MS // 2, streams[t])
                    e.ingest_arrays([(hid, pool[d][1][off:off + n]) for hid, d, off, n in items], streams[t])
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
        got += dense_export(e.snapshot(PS)[1], H)
        assert (got == want).all(), np.argwhere(got != want)[:5]
