"""Distribution gauges (lh_snapshot_ingest_arrays, MetricSystem::RegisterDeviceDistribution): every element of a
device array recorded as Histogram(name, float64(x)) into the interval each collection collects, by k_ingest_arrays on
the snapshot stream.

Bar: bucket counts and the reduction equal the oracle fed numpy astype(float64) of the array at precisions 50 / 100 /
200; sizes from 0 to 2^28 and tables over several launches count exactly; every refusal launches nothing and the
ABI-level ones are made outside a snapshot, where only validation can refuse with LH_ERR_INVALID / LH_ERR_RANGE; the
state check refuses before begin and after a read; in a MetricSystem each interval carries the array's contents at its
collection, joined with Histogram, scope and graph-recorder samples of the name, a collection never waits for a
caller stream, a concurrent writer never tears an element, and collections without distributions issue the launches
they issued before."""
import ctypes as C
import functools
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LH_OK, LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = 0, -1, -5, -6
F64, F32, F16, BF16, I64, I32, U64 = range(7)
BI_PIECE, BI_MAX_ITEMS = 2048, 1024
PS = [0.5, 0.9, 0.99]


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def spin():
    """spin(ns, stream): one bounded spin of at least `ns` on a torch stream (tests/gpu_timer_client.cu)."""
    from loghisto_b200 import build
    lib = C.CDLL(build.TIMER_CLIENT_LIB)
    lib.gtc_set_device.argtypes = [C.c_int]
    lib.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    lib.gtc_set_device.restype = lib.gtc_spin.restype = C.c_int
    assert lib.gtc_set_device(0) == 0

    def run(ns, stream):
        assert lib.gtc_spin(int(ns), stream.cuda_stream) == 0
    return run


@pytest.fixture(scope="module")
def gwc():
    from loghisto_b200 import build
    lib = C.CDLL(build.GAUGE_CLIENT_LIB)
    lib.gwc_set.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p]
    lib.gwc_flip.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_int, C.c_uint64, C.c_void_p]
    lib.gwc_set.restype = lib.gwc_flip.restype = C.c_int
    return lib


def dense(sp, h):
    out = np.zeros(65536, np.uint64)
    lo, hi = int(sp.offsets[h]), int(sp.offsets[h + 1])
    out[sp.keys[lo:hi].astype(np.int64) & 0xFFFF] = sp.counts[lo:hi]
    return out


def host_f64(torch, t):
    """numpy astype(float64) of a tensor's elements (bfloat16 through float32, which widens it exactly)."""
    c = t.detach().cpu().reshape(-1)
    if c.dtype == torch.bfloat16:
        c = c.float()
    if c.dtype == torch.uint64:
        return c.view(torch.int64).numpy().view(np.uint64).astype(np.float64)
    return c.numpy().astype(np.float64)


@functools.lru_cache(maxsize=None)
def magnitudes(precision):
    from oracle import oracle
    return np.abs(oracle.decompress_table(float(precision)))


def check_rows(oracle, red, sp, want, precision):
    """Each row h of the snapshot equals the oracle's histogram of want[h] (float64 values), bucket for bucket, and
    its reduction equals the oracle's processHistograms: count, percentile keys and values exactly, the sum up to the
    rounding of a sum taken in another order (1e-12 of the sum of magnitudes; NaN and infinities as they are)."""
    for h, vals in enumerate(want):
        exp = oracle.ingest(vals, precision=float(precision))
        got = dense(sp, h)
        assert np.array_equal(got, exp), h
        ref = oracle.process_histogram(exp, PS, precision=float(precision))
        assert int(red.counts[h]) == ref["total"]
        if ref["total"]:
            np.testing.assert_array_equal(red.pkeys[h], ref["pkeys"])
            np.testing.assert_array_equal(red.pvals[h], ref["pvals"])
            mags = magnitudes(precision) * exp.astype(np.float64)
            scale = float(np.sum(mags[np.isfinite(mags)]))
            if np.isfinite(ref["sum"]):
                assert abs(red.sums[h] - ref["sum"]) <= 1e-12 * scale, h
            else:
                assert np.array_equal(red.sums[h], ref["sum"], equal_nan=True), h


def exactness_inputs(torch, oracle):
    rng = np.random.default_rng(20261019)
    dev = "cuda:0"
    every16 = torch.arange(65536, dtype=torch.int32).to(torch.int16)
    f16 = every16.view(torch.float16).to(dev)
    bf16 = every16.view(torch.bfloat16).to(dev)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.17549435e-38, 1.1754942e-38,
                         3.4028235e38, -3.4028235e38, 1.0, -1.0, 0.5], np.float32)
    f32 = np.concatenate([specials, rng.integers(0, 1 << 32, 10 ** 6, dtype=np.uint64).astype(np.uint32).view(np.float32)])
    s64 = oracle.gen_stream(oracle.STREAM_S, 10 ** 6, 7)
    i32 = np.array([0, 1, -1, 2 ** 31 - 1, -2 ** 31, 123456789], np.int32)
    ties = [2 ** 53 + k for k in range(-3, 4)] + [2 ** 62 + 512 * k + d for k in range(4) for d in (-1, 0, 1)]
    i64 = np.array([0, -1, 2 ** 63 - 1, -2 ** 63] + ties + [-t for t in ties], np.int64)
    u64 = np.array([0, 1, 2 ** 64 - 1, 2 ** 63] + [2 ** 63 + 1024 * k + d for k in range(4) for d in (-1, 0, 1)] +
                   [2 ** 64 - 2048 + d for d in (-1, 0, 1)], np.uint64)
    return [f16, bf16, torch.from_numpy(f32).to(dev), torch.from_numpy(s64).to(dev), torch.from_numpy(i32).to(dev),
            torch.from_numpy(i64).to(dev), torch.from_numpy(u64.view(np.int64)).view(torch.uint64).to(dev)]


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_exactness_every_dtype(lh, torch, oracle, precision):
    """Every F16 and BF16 bit pattern, F32 specials and 10^6 random patterns, stream S as F64, and the integer extremes
    and round-to-nearest-even ties at 2^53 and 2^63: one snapshot, one row each, equal to the oracle."""
    arrays = exactness_inputs(torch, oracle)
    with lh.Engine(device=0, max_histograms=len(arrays), max_counters=1, precision=precision) as e:
        before = e.stats()
        red, sp = e.snapshot(PS, arrays=list(enumerate(arrays)))
        after = e.stats()
        total = sum(a.numel() for a in arrays)
        assert after["samples"] - before["samples"] == total
        check_rows(oracle, red, sp, [host_f64(torch, a) for a in arrays], precision)


def test_sizes_launches_and_layout(lh, torch, oracle):
    """n = 0, 1 and either side of BI_PIECE; a table that overflows the BlockRecorder table; 2 000 arrays over
    ceil(entries / 1024) launches; overlapping arrays and one array under two names."""
    rng = np.random.default_rng(5)
    with lh.Engine(device=0, max_histograms=2048, max_counters=1) as e:
        sizes = [0, 1, BI_PIECE - 1, BI_PIECE, BI_PIECE + 1, 3 * BI_PIECE + 7]
        base = torch.from_numpy(rng.standard_normal(4 * BI_PIECE) * 1e3).cuda()
        arrays = [(i, base[:n]) for i, n in enumerate(sizes)]
        wide = torch.from_numpy(rng.uniform(1e-6, 1e9, 1 << 20)).cuda()   # ~ 2 000 distinct keys per id over 16 ids
        arrays += [(16 + i, wide[i << 16:(i + 1) << 16]) for i in range(16)]
        arrays += [(40, base[100:900]), (41, base[500:1500]), (42, base[100:900])]   # overlaps, one range twice
        l0 = e.stats()["kernel_launches"]
        e.snapshot_begin()
        try:
            e.snapshot_ingest_arrays(arrays)
            assert e.stats()["kernel_launches"] == l0 + 1
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
        finally:
            e.snapshot_end()
        want = [np.zeros(0)] * 43
        for h, t in arrays:
            want[h] = host_f64(torch, t)
        check_rows(oracle, red, sp, want, 100)

        many = torch.from_numpy(rng.standard_normal(2000 * 37)).cuda()
        arrays = [(i, many[i * 37:(i + 1) * 37]) for i in range(2000)]
        l0 = e.stats()["kernel_launches"]
        e.snapshot_begin()
        try:
            e.snapshot_ingest_arrays(arrays + [(0, many[:0])] * 100)   # empty entries take no table slot
            assert e.stats()["kernel_launches"] == l0 + 2
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
        finally:
            e.snapshot_end()
        check_rows(oracle, red, sp, [host_f64(torch, t) for _, t in arrays], 100)


def test_2_to_28_elements(lh, torch, oracle):
    """One float32 array of 2^28 elements: every bucket equals the oracle's."""
    n = 1 << 28
    period = 65521
    x = ((torch.arange(n, device="cuda:0", dtype=torch.int64) % period).to(torch.float32) * 0.37 - 9000.0)
    uniq = ((np.arange(period) * np.float32(0.37)).astype(np.float32) - np.float32(9000.0)).astype(np.float64)
    mult = np.full(period, n // period, np.uint64)
    mult[:n % period] += 1
    exp = np.zeros(65536, np.uint64)
    np.add.at(exp, oracle.compress_many(uniq).astype(np.int64) & 0xFFFF, mult)
    assert np.array_equal(uniq, x[:period].cpu().numpy().astype(np.float64))
    with lh.Engine(device=0, max_histograms=1, max_counters=1) as e:
        red, sp = e.snapshot(PS, arrays=[(0, x)])
        assert np.array_equal(dense(sp, 0), exp)
        assert int(red.counts[0]) == n


def test_refusals_and_state(lh, torch):
    """Refusals come from validation before the state check (so outside a snapshot they are LH_ERR_INVALID /
    LH_ERR_RANGE, not LH_ERR_STATE) and launch nothing; valid arrays are refused with LH_ERR_STATE before
    lh_snapshot_begin and after the first read of the snapshot."""
    from loghisto_b200 import _lib
    from loghisto_b200.engine import LhError
    with lh.Engine(device=0, max_histograms=4, max_counters=1) as e:
        d = e.alloc(1000, np.float32)   # one allocation of exactly 4 000 bytes
        t = torch.zeros(64, dtype=torch.float64, device="cuda:0")
        host = np.zeros(16)
        pinned = e.pinned(16, np.float64)

        def call(*srcs):
            arr = (_lib.lh_array_src * max(len(srcs), 1))(*[_lib.lh_array_src(*s) for s in srcs])
            return e.lib.lh_snapshot_ingest_arrays(e.h, arr, len(srcs))

        bad = [((None, 1, F64, 0), LH_ERR_INVALID), ((d.ptr, 1, 7, 0), LH_ERR_INVALID),
               ((d.ptr, 0, 9, 0), LH_ERR_INVALID), ((d.ptr + 2, 1, F32, 0), LH_ERR_INVALID),
               ((d.ptr + 4, 1, F64, 0), LH_ERR_INVALID), ((d.ptr + 1, 1, F16, 0), LH_ERR_INVALID),
               ((d.ptr, 1001, F32, 0), LH_ERR_INVALID), ((d.ptr + 4, 1000, F32, 0), LH_ERR_INVALID),
               ((d.ptr, 501, F64, 0), LH_ERR_INVALID), ((d.ptr, 1 << 62, F32, 0), LH_ERR_INVALID),
               ((host.ctypes.data, 16, F64, 0), LH_ERR_INVALID), ((pinned.ptr, 16, F64, 0), LH_ERR_INVALID),
               ((d.ptr, 1, F32, 4), LH_ERR_RANGE)]
        l0 = e.stats()["kernel_launches"]
        for src, st in bad:
            assert call(src) == st, src
            assert call((d.ptr, 10, F32, 1), src) == st, src   # a good entry first changes nothing
        assert e.lib.lh_snapshot_ingest_arrays(e.h, None, 1) == LH_ERR_INVALID
        assert e.stats()["kernel_launches"] == l0
        # valid input outside a snapshot: only the state check refuses it
        assert call((d.ptr, 1000, F32, 0)) == LH_ERR_STATE
        assert call((d.ptr, 500, F64, 3), (t.data_ptr(), 64, F64, 2)) == LH_ERR_STATE
        assert call() == LH_ERR_STATE
        e.snapshot_begin()
        try:
            assert call() == LH_OK and call((d.ptr, 0, F32, 0)) == LH_OK
            assert e.stats()["kernel_launches"] == l0
            for src, st in bad:
                assert call(src) == st, src
            assert e.stats()["kernel_launches"] == l0
            assert call((d.ptr, 1000, F32, 0)) == LH_OK
            assert e.stats()["kernel_launches"] == l0 + 1
            assert call((t.data_ptr(), 64, F64, 1)) == LH_OK   # any number of calls before the first read
            e.snapshot_reduce(PS)
            assert call((t.data_ptr(), 64, F64, 1)) == LH_ERR_STATE
            l1 = e.stats()["kernel_launches"]
            assert call((d.ptr, 1, F32, 4)) == LH_ERR_RANGE
            assert e.stats()["kernel_launches"] == l1
        finally:
            e.snapshot_end()
        for reader in (lambda: e.snapshot_export(), lambda: e.snapshot_copy_histogram(0), lambda: e.snapshot_device(),
                       lambda: e.snapshot_reduce_async(PS)):
            e.snapshot_begin()
            try:
                reader()
                assert call((t.data_ptr(), 64, F64, 1)) == LH_ERR_STATE
            finally:
                e.snapshot_end()
        for bad_t in (torch.zeros(8, dtype=torch.int16, device="cuda:0"), torch.zeros(8), torch.zeros(8).pin_memory(),
                      torch.zeros(8, 8, device="cuda:0").t(), np.zeros(8)):
            with pytest.raises(TypeError):
                e.snapshot_ingest_arrays([(0, bad_t)])
        with pytest.raises(LhError):
            e.snapshot_ingest_arrays([(0, t)])   # no snapshot
        pinned.free()
        d.free()


def collect(ms):
    raw, metrics = ms.collect_and_process()
    return raw["Histograms"], metrics


def keys_of(oracle, vals):
    u, c = np.unique(oracle.compress_many(np.asarray(vals, np.float64)).astype(np.int64), return_counts=True)
    return {int(k): int(n) for k, n in zip(u, c)}


def test_metric_system_intervals(lh, torch, oracle, gwc):
    """Each interval equals the array's contents at its collection (rewritten with fill_, copy_ and lh::set_gauge),
    joined with Histogram, record-scope and graph-recorder samples of the name; replace and deregister; the Python
    argument checks; no extra launch per collection without distributions, ceil(entries / 1024) with them."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=16, max_counters=4)
    try:
        def launches():   # of a collection with one Histogram sample, so that every interval has an export
            ms.Histogram("h", 1.0)
            before = ms.stats()["kernel_launches"]
            ms.collect_and_process()
            return ms.stats()["kernel_launches"] - before
        launches()
        base = launches()
        x = torch.arange(10, dtype=torch.float32, device="cuda:0").reshape(2, 5)
        ms.RegisterDeviceDistribution("occ", x)
        assert launches() == base + 1
        x.fill_(3.5)
        torch.cuda.synchronize()
        h, m = collect(ms)
        assert h == {"occ": keys_of(oracle, [3.5] * 10)} and m["occ_count"] == 10.0
        assert m["occ_sum"] == oracle.process_histogram(oracle.ingest(np.full(10, 3.5)), PS)["sum"]
        x.copy_(torch.linspace(-4, 4, 10, device="cuda:0").reshape(2, 5))
        assert gwc.gwc_set(x.data_ptr() + 4, F32, int(np.float32(100.0).view(np.uint32)), None) == 0
        torch.cuda.synchronize()
        want = np.linspace(-4, 4, 10).astype(np.float32)
        want[1] = 100.0
        assert collect(ms)[0] == {"occ": keys_of(oracle, want.astype(np.float64))}
        # union with Histogram, a record scope and a graph recorder under the same name
        ms.Histogram("occ", 7.0)
        with ms.recording(histograms=["occ"]) as s:
            s.histograms({"occ": torch.tensor([1.0, 2.0], dtype=torch.float64, device="cuda:0")})
        with ms.graph_recorder(histograms=["occ"]) as g:
            g.histograms({"occ": torch.tensor([5.0], dtype=torch.float64, device="cuda:0")})
            torch.cuda.synchronize()
            h, m = collect(ms)
        assert h == {"occ": keys_of(oracle, list(want.astype(np.float64)) + [7.0, 1.0, 2.0, 5.0])}
        assert m["occ_count"] == 14.0
        # replace, two names on one tensor, deregister
        y = torch.tensor([[1, -2], [3, 2 ** 31 - 1]], dtype=torch.int32, device="cuda:0")
        ms.RegisterDeviceDistribution("occ", y)
        ms.RegisterDeviceDistribution("occ2", y)
        assert collect(ms)[0] == {"occ": keys_of(oracle, [1, -2, 3, 2 ** 31 - 1]),
                                  "occ2": keys_of(oracle, [1, -2, 3, 2 ** 31 - 1])}
        ms.RegisterDeviceDistribution("empty", torch.zeros(0, dtype=torch.bfloat16, device="cuda:0"))
        ms.DeregisterDeviceDistribution("occ")
        assert collect(ms)[0] == {"occ2": keys_of(oracle, [1, -2, 3, 2 ** 31 - 1])}
        ms.DeregisterDeviceDistribution("occ2")
        ms.DeregisterDeviceDistribution("empty")
        assert launches() == base and ms._device_dists == {}
        for bad in (torch.zeros(4, dtype=torch.int16, device="cuda:0"), torch.zeros(4), torch.zeros(4).pin_memory(),
                    torch.zeros(4, 4, device="cuda:0").t(), 3.0):
            with pytest.raises(TypeError):
                ms.RegisterDeviceDistribution("bad", bad)
        # 2 000 registered names of 3 elements: ceil(2000 / 1024) launches
        big = MetricSystem(60.0, False, max_histograms=2048, max_counters=4)
        try:
            z = torch.arange(3 * 2000, dtype=torch.float64, device="cuda:0")
            for i in range(2000):
                big.RegisterDeviceDistribution("d%d" % i, z[3 * i:3 * i + 3])
            big.collect_and_process()
            b0 = big.stats()["kernel_launches"]
            h = big.collect_and_process()[0]["Histograms"]
            assert len(h) == 2000 and h["d1999"] == keys_of(oracle, [5997.0, 5998.0, 5999.0])
            b1 = big.stats()["kernel_launches"]
            for i in range(977):
                big.DeregisterDeviceDistribution("d%d" % i)
            big.collect_and_process()
            assert (b1 - b0) - (big.stats()["kernel_launches"] - b1) == 1   # 1 023 entries: one launch fewer
        finally:
            big.close()
    finally:
        ms.close()


def test_no_free_id_drops_and_counts(lh, torch):
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=2, max_counters=4)
    try:
        ms.Histogram("a", 1.0)
        ms.Histogram("b", 1.0)
        x = torch.ones(5, dtype=torch.float32, device="cuda:0")
        ms.RegisterDeviceDistribution("d", x)
        d0 = ms.dropped()
        h, _ = collect(ms)
        assert set(h) == {"a", "b"} and ms.dropped() == d0 + 5
        for _ in range(3):
            h, _ = collect(ms)
            if "d" in h:
                break
        assert set(h) == {"d"} and sum(h["d"].values()) == 5
        for _ in range(3):   # a registered name keeps its id through intervals of other names
            ms.Histogram("a", 1.0)
            h, _ = collect(ms)
            assert sum(h["d"].values()) == 5
    finally:
        ms.close()


def test_collection_never_waits(lh, torch, oracle, spin):
    """A collection returns while a caller stream's write to the array waits behind a 200 ms spin, with the old
    contents; the next collection after the write has the new ones."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=4, max_counters=4)
    try:
        x = torch.full((1000,), 2.0, dtype=torch.float64, device="cuda:0")
        ms.RegisterDeviceDistribution("q", x)
        collect(ms)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            spin(200_000_000, s)
            x.fill_(9.0)
        t0 = time.perf_counter()
        h, _ = collect(ms)
        took = time.perf_counter() - t0
        assert not s.query(), "the spin ended before the collection returned"
        assert h == {"q": keys_of(oracle, [2.0] * 1000)} and took < 0.15
        s.synchronize()
        assert collect(ms)[0] == {"q": keys_of(oracle, [9.0] * 1000)}
    finally:
        ms.close()


def test_alternating_writer_never_tears(lh, torch, oracle, gwc):
    """While a kernel flips three uint64 elements between two patterns with strong stores, every recorded sample is
    one of the two patterns' values and every collection counts exactly three."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=4, max_counters=4)
    try:
        a = [0x0000000000000001, 0x7FFFFFFFFFFFFFFF, 0x00000000FFFFFFFF]
        b = [0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0xFFFFFFFF00000000]
        cells = torch.tensor([np.int64(np.uint64(v)) for v in a], dtype=torch.int64, device="cuda:0").view(torch.uint64)
        ms.RegisterDeviceDistribution("flip", cells)
        allowed = set(keys_of(oracle, [float(v) for v in a + b]))
        s = torch.cuda.Stream()
        ca, cb = (C.c_uint64 * 3)(*a), (C.c_uint64 * 3)(*b)
        assert gwc.gwc_flip(cells.data_ptr(), ca, cb, 1, 20_000_000, s.cuda_stream) == 0
        seen = 0
        while not s.query() and seen < 50:
            h, _ = collect(ms)
            assert sum(h["flip"].values()) == 3 and set(h["flip"]) <= allowed
            seen += 1
        s.synchronize()
        assert seen > 0
    finally:
        ms.close()


class Shifted:
    """What array_src sees of a tensor, at a byte offset and element count of the caller's choosing: a view that torch
    itself would not make (misaligned, or running past the tensor's allocation)."""

    def __init__(self, t, offset_bytes, numel):
        self.t, self.offset, self.n = t, offset_bytes, numel
        self.is_cuda, self.device, self.dtype = t.is_cuda, t.device, t.dtype

    def data_ptr(self):
        return self.t.data_ptr() + self.offset

    def numel(self):
        return self.n

    def is_contiguous(self):
        return True


def test_metric_system_refusals_launch_nothing(lh, torch, oracle, capfd):
    """Through the MetricSystem: a wrong dtype, CPU, pinned or non-contiguous tensor is a TypeError and a misaligned view
    a ValueError at registration; an array whose range runs past its allocation passes registration (its first element
    is readable), is refused at every collection (logged, the set delivered without it) and launches nothing."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=8, max_counters=4)
    try:
        def launches():
            ms.Histogram("h", 1.0)
            before = ms.stats()["kernel_launches"]
            raw = ms.collect_and_process()[0]
            return ms.stats()["kernel_launches"] - before, raw
        launches()
        base, _ = launches()
        x = torch.arange(64, dtype=torch.float32, device="cuda:0")
        for bad in (torch.zeros(4, dtype=torch.int16, device="cuda:0"), torch.zeros(4), torch.zeros(4).pin_memory(),
                    torch.zeros(4, 4, device="cuda:0").t()):
            with pytest.raises(TypeError):
                ms.RegisterDeviceDistribution("bad", bad)
        l0 = ms.stats()["kernel_launches"]
        for off in (1, 2, 3):
            with pytest.raises(ValueError):
                ms.RegisterDeviceDistribution("bad", Shifted(x, off, 8))
        assert ms.stats()["kernel_launches"] == l0   # lh_gauges_read refused before its launch
        assert launches()[0] == base
        ms.RegisterDeviceDistribution("past", Shifted(x, 0, 1 << 40))
        capfd.readouterr()
        n, raw = launches()
        assert n == base and raw["Histograms"] == {"h": keys_of(oracle, [1.0])}
        assert "lh_snapshot_ingest_arrays failed" in capfd.readouterr().err
        ms.RegisterDeviceDistribution("past", x)   # replaced by a good array: recorded again
        n, raw = launches()
        assert n == base + 1 and raw["Histograms"]["past"] == keys_of(oracle, np.arange(64.0))
    finally:
        ms.close()


def test_registry_calls_from_a_scope_holder_never_deadlock(lh, torch, oracle):
    """A collection that waits in lh_snapshot_begin for a record scope holds the registry; the scope's thread calling
    RegisterDeviceDistribution / DeregisterDeviceDistribution is refused (RuntimeError) instead of waiting for it, so the
    scope ends and the collection returns.  A thread without a scope waits for the collection and then succeeds."""
    import threading
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(60.0, False, max_histograms=8, max_counters=4)
    x = torch.full((16,), 4.0, dtype=torch.float64, device="cuda:0")
    y = torch.full((8,), 2.0, dtype=torch.float32, device="cuda:0")
    try:
        ms.RegisterDeviceDistribution("d", x)
        in_scope, done = threading.Event(), threading.Event()
        out = {}

        def holder():
            try:
                with ms.recording(histograms=["s"]):
                    in_scope.set()
                    time.sleep(0.3)   # the collector is waiting for this scope by now
                    for call in (lambda: ms.RegisterDeviceDistribution("e", y),
                                 lambda: ms.DeregisterDeviceDistribution("d")):
                        try:
                            call()
                            out.setdefault("accepted", 0)
                            out["accepted"] += 1
                        except RuntimeError:
                            out.setdefault("refused", 0)
                            out["refused"] += 1
            finally:
                done.set()

        def collector():
            in_scope.wait(30)
            out["raw"] = ms.collect_and_process()[0]

        def other():
            in_scope.wait(30)
            time.sleep(0.1)
            ms.RegisterDeviceDistribution("e", y)   # waits for the collection, then registers
            out["other"] = True

        ts = [threading.Thread(target=f, daemon=True) for f in (holder, collector, other)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(60)
        assert not any(t.is_alive() for t in ts), "a registry call from a scope holder deadlocked the collection"
        assert done.is_set() and out.get("refused") == 2 and "accepted" not in out and out.get("other")
        assert out["raw"]["Histograms"]["d"] == keys_of(oracle, [4.0] * 16)
        h = collect(ms)[0]
        assert h == {"d": keys_of(oracle, [4.0] * 16), "e": keys_of(oracle, [2.0] * 8)}
    finally:
        ms.close()


def test_reaper_delivers_distributions(lh, torch):
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(0.02, False, max_histograms=8, max_counters=4)
    sub = ms.SubscribeToProcessedMetrics(64)
    try:
        ms.RegisterDeviceDistribution("slots", torch.arange(100, dtype=torch.int32, device="cuda:0"))
        ms.Start()
        deadline, got = time.monotonic() + 10.0, None
        while got is None and time.monotonic() < deadline:
            m = sub.receive(0.5)
            if m and "slots_count" in m:
                got = m["slots_count"]
        assert got == 100.0
    finally:
        ms.Stop()
        sub.close()
        ms.close()


def test_boards_equal_collect_and_process(lh, torch, oracle):
    """With distributions registered beside Histogram samples, the processed board, the raw board and a raw board
    windowed over the last 3 collections answer what collect_and_process reports (for the window: processMetrics of
    the union of the last 3 raw sets), collection by collection, while the arrays are rewritten."""
    from loghisto_b200.metric_system import MetricSystem
    ps = {"%s_p50": 0.5, "%s_p99": 0.99}
    labels = sorted(ps.items())
    ms = MetricSystem(3600.0, False, max_histograms=16, max_counters=4)
    ms.SpecifyPercentiles(ps)
    names = ["occ", "tok", "mix", "never"]
    rng = np.random.default_rng(11)
    occ = torch.zeros(4096, dtype=torch.int32, device="cuda:0")
    tok = torch.zeros(256, dtype=torch.bfloat16, device="cuda:0")
    try:
        ms.RegisterDeviceDistribution("occ", occ)
        ms.RegisterDeviceDistribution("tok", tok)
        ms.RegisterDeviceDistribution("mix", tok[:17])
        ps_t = torch.tensor([p for _, p in labels], dtype=torch.float64, device="cuda:0")
        history = []
        with ms.device_subscription(histograms=names) as psub, ms.raw_device_subscription(histograms=names) as rsub, \
                ms.raw_device_subscription(histograms=names, window=3) as wsub:
            for j in range(5):
                occ.copy_(torch.from_numpy(rng.integers(0, 64 << j, 4096).astype(np.int32)))
                tok.copy_(torch.from_numpy(rng.lognormal(2, 3, 256)).to(torch.bfloat16))
                ms.HistogramMany("mix", rng.normal(0, 10, 50 + j))
                torch.cuda.synchronize()
                raw, want = ms.collect_and_process()
                history.append(raw["Histograms"])
                union = {}
                for hs in history[-3:]:
                    for nm, m in hs.items():
                        u = union.setdefault(nm, {})
                        for k, c in m.items():
                            u[k] = u.get(k, 0) + c
                want_w = ms.processMetrics({"Histograms": union})
                views = psub.read()
                _, vals, _ = rsub.percentiles(ps_t)
                _, wvals, _ = wsub.percentiles(ps_t)
                torch.cuda.synchronize()
                counts, sums = views["count"].cpu().numpy(), views["sum"].cpu().numpy()
                vals, wvals = vals.cpu().numpy(), wvals.cpu().numpy()
                for i, nm in enumerate(names):
                    if nm not in raw["Histograms"]:
                        assert counts[i] == 0 and nm == "never", (j, nm)
                        continue
                    assert counts[i] == want[nm + "_count"] and sums[i] == want[nm + "_sum"], (j, nm)
                    for c, (label, _) in enumerate(labels):
                        assert vals[i, c] == want[label % nm], (j, nm, label)
                        assert wvals[i, c] == want_w[label % nm], (j, nm, label)
    finally:
        ms.close()


@pytest.mark.parametrize("path", ["peer", "allreduce"])
@pytest.mark.parametrize("world", [2, 3])
def test_joined_ranks_equal_one_system_fed_every_array(path, world):
    """JoinRanks at world 2 and 3, over the peer all-reduce and over the caller's all-reduce: each rank registers a
    shared name (different contents per rank), a name of its own and one array under two names, beside Histogram
    samples; every rank's collection equals one unjoined system fed every rank's arrays as Histogram samples."""
    import torch
    import test_gpu_ranks as gr
    import test_gpu_ranks_allreduce as gra
    ndev = torch.cuda.device_count()
    join = gr.joined_systems if path == "peer" else gra.joined_allreduce
    systems, _ = join(world, ndev, 100, H=64, C=8)
    ref = gr.reference(100, 64, 8)
    rng = np.random.default_rng(100 * world + len(path))
    arrays = []
    try:
        for r, ms in enumerate(systems):
            dev = torch.device("cuda", r % ndev)
            a = torch.zeros(1000 + 100 * r, dtype=torch.float32, device=dev)
            b = torch.zeros(50, dtype=torch.int64, device=dev)
            ms.RegisterDeviceDistribution("shared", a)
            ms.RegisterDeviceDistribution("rank%d" % r, b)
            ms.RegisterDeviceDistribution("both", b)
            arrays.append((a, b))
        for interval in range(4):
            for r, (a, b) in enumerate(arrays):
                av = rng.lognormal(3, 2, a.numel()).astype(np.float32)
                bv = rng.integers(-(1 << 40), 1 << 40, b.numel())
                a.copy_(torch.from_numpy(av))
                b.copy_(torch.from_numpy(bv))
                ref.HistogramMany("shared", av.astype(np.float64))
                ref.HistogramMany("rank%d" % r, bv.astype(np.float64))
                ref.HistogramMany("both", bv.astype(np.float64))
                if (interval + r) % 2 == 0:
                    v = rng.normal(0, 5, 7)
                    systems[r].HistogramMany("shared", v)
                    ref.HistogramMany("shared", v)
            for d in range(ndev):
                torch.cuda.synchronize(d)
            got = gr.on_ranks(world, lambda r: systems[r].collect_and_process())
            want_raw, want = ref.collect_and_process()
            for r, (raw, metrics) in enumerate(got):
                assert raw["Histograms"] == want_raw["Histograms"], (interval, r)
                assert metrics == want, (interval, r)
                assert systems[r].ranks_info()["status"] == 0
    finally:
        for ms in systems:
            ms.close()
        ref.close()
