"""Device gauges (lh_gauges_read, MetricSystem::RegisterDeviceGauge): scalars in device memory read by every collection
in one sm_90a kernel on the snapshot stream, as Go's float64(x) of a gauge function's value.

The writing kernels live in tests/gauge_write_client.cu, a separate CUDA library built by build() that knows the engine
only through its public headers.  Bar: every conversion equals numpy / torch CPU astype(float64) bit for bit (NaN ->
NaN); every refusal launches nothing; values written by strong and by plain stores are never read torn; a read never
waits for a stream with a pending write; in a MetricSystem the values written by fill_ / copy_, lh::set_gauge and graph
replays appear bit for bit in Gauges and the processed metrics, and collections without device gauges issue the
launches they issued before."""
import ctypes as C
import math
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LH_OK, LH_ERR_INVALID = 0, -1
F64, F32, F16, BF16, I64, I32, U64 = range(7)
SRC = np.dtype([("d_value", "<u8"), ("dtype", "<u4"), ("reserved", "<u4")])


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def eng(lh):
    with lh.Engine(device=0, max_histograms=2, max_counters=2) as e:
        yield e


@pytest.fixture(scope="module")
def gwc():
    from loghisto_b200 import build
    lib = C.CDLL(build.GAUGE_CLIENT_LIB)
    lib.gwc_set.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p]
    lib.gwc_flip.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_int, C.c_uint64, C.c_void_p]
    lib.gwc_set.restype = lib.gwc_flip.restype = C.c_int
    return lib


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


def read_raw(eng, srcs, out=None):
    """lh_gauges_read of a SRC table: (status, values); values stay -1 where nothing was written."""
    from loghisto_b200 import _lib
    srcs = np.ascontiguousarray(srcs, dtype=SRC)
    if out is None:
        out = np.full(len(srcs), -1.0)
    p = srcs.ctypes.data_as(C.POINTER(_lib.lh_gauge_src)) if len(srcs) else None
    st = eng.lib.lh_gauges_read(eng.h, p, len(srcs), out.ctypes.data if out is not None else None)
    return st, out


def table(t, dtype):
    """One SRC entry per element of the contiguous CUDA tensor t."""
    n = t.numel()
    s = np.zeros(n, dtype=SRC)
    s["d_value"] = t.data_ptr() + np.arange(n, dtype=np.uint64) * t.element_size()
    s["dtype"] = dtype
    return s


def assert_same(got, want, what):
    want = np.asarray(want, dtype=np.float64)
    nan = np.isnan(want)
    assert (np.isnan(got) == nan).all(), what
    bad = np.flatnonzero(got[~nan].view(np.uint64) != want[~nan].view(np.uint64))
    assert bad.size == 0, (what, got[~nan][bad[:5]], want[~nan][bad[:5]])


def bits_f64(u):
    return np.asarray(u, dtype=np.uint64).view(np.float64)


def test_conversions_bit_exact(torch, eng):
    """Every F16 and BF16 bit pattern, F32 specials, subnormals, ±FLT_MAX and 10^6 random patterns, I32 / I64 / U64
    extremes and the round-to-nearest-even ties at and above 2^53 and 2^63, F64 specials: one call across many
    launches, each value equal to numpy / torch CPU astype(float64)."""
    rng = np.random.default_rng(20261017)
    u16 = np.arange(65536, dtype=np.uint16)
    fi = np.finfo(np.float32)
    f32 = np.concatenate([
        np.array([0.0, -0.0, np.inf, -np.inf, np.nan, fi.max, -fi.max, fi.tiny, -fi.tiny, 1.0, -1.0, 1 / 3], np.float32),
        np.array([1, 2, 0x7FFFFF, 0x400000, 0x80000001, 0x807FFFFF, 0x7FC00001, 0xFFFFFFFF, 0x7F800001],
                 np.uint32).view(np.float32),
        rng.integers(0, 1 << 32, 1_000_000, dtype=np.uint64).astype(np.uint32).view(np.float32)])
    i32 = np.concatenate([np.array([-(1 << 31), (1 << 31) - 1, 0, -1, 1, (1 << 24) + 1], np.int32),
                          rng.integers(-(1 << 31), 1 << 31, 10_000, dtype=np.int64).astype(np.int32)])
    t53, t62 = 1 << 53, 1 << 62
    i64 = np.concatenate([
        np.array([0, 1, -1, t53, t53 + 1, t53 + 2, t53 + 3, -(t53 + 1), -(t53 + 3), 2 * t53 + 2, 2 * t53 + 6,
                  t62 + 512, t62 + 3 * 512, t62 + 513, (1 << 63) - 1, (1 << 63) - 512, (1 << 63) - 513,
                  -(1 << 63), -(1 << 63) + 1, -(t62 + 512)], dtype=np.int64),
        rng.integers(-(1 << 63), (1 << 63) - 1, 100_000, dtype=np.int64, endpoint=True)])
    t63 = 1 << 63
    u64 = np.concatenate([
        np.array([0, 1, t53 + 1, t53 + 3, t63 - 1, t63 - 512, t63, t63 + 1, t63 + 1024, t63 + 1025, t63 + 3072,
                  t63 + 3071, (1 << 64) - 1, (1 << 64) - 1024, (1 << 64) - 1025, (1 << 64) - 3072, (1 << 64) - 2048],
                 dtype=np.uint64),
        rng.integers(0, (1 << 64) - 1, 100_000, dtype=np.uint64, endpoint=True)])
    f64 = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, -5e-324, 1.7976931348623157e308]),
                          rng.integers(0, (1 << 64) - 1, 10_000, dtype=np.uint64, endpoint=True).view(np.float64)])

    def dev(a, itype):
        return torch.from_numpy(np.ascontiguousarray(a).view(itype)).cuda()

    with np.errstate(invalid="ignore"):   # NaN patterns: the cast keeps them NaN
        want_f32 = f32.astype(np.float64)
    want_bf16 = torch.from_numpy(u16.view(np.int16)).view(torch.bfloat16).to(torch.float64).numpy()
    parts = [(dev(u16, np.int16), F16, u16.view(np.float16).astype(np.float64), "f16"),
             (dev(u16, np.int16), BF16, want_bf16, "bf16"),
             (dev(f32, np.int32), F32, want_f32, "f32"),
             (dev(i32, np.int32), I32, i32.astype(np.float64), "i32"),
             (dev(i64, np.int64), I64, i64.astype(np.float64), "i64"),
             (dev(u64, np.int64), U64, u64.astype(np.float64), "u64"),
             (dev(f64, np.int64), F64, f64, "f64")]
    srcs = np.concatenate([table(t, d) for t, d, _, _ in parts])
    torch.cuda.synchronize()
    before = eng.stats()
    st, out = read_raw(eng, srcs)
    after = eng.stats()
    assert st == LH_OK
    assert after["kernel_launches"] - before["kernel_launches"] == -(-len(srcs) // 1024)
    assert after["samples"] == before["samples"] and after["counter_ops"] == before["counter_ops"]
    o = 0
    for t, _, want, what in parts:
        assert_same(out[o:o + t.numel()], want, what)
        o += t.numel()
    assert o == len(srcs) > 1024
    # Engine.read_gauges on one-element views agrees with the table read
    assert_same(eng.read_gauges([parts[4][0][5], parts[5][0].view(torch.uint64)[10]]), [float(i64[5]), float(u64[10])],
                "read_gauges")


def test_validation_launches_nothing(torch, eng):
    """Every refusal is LH_ERR_INVALID with no launch and h_out untouched; one bad entry anywhere refuses the table."""
    cells = torch.zeros(4, dtype=torch.int64, device="cuda")
    base = cells.data_ptr()
    pinned = torch.zeros(2, dtype=torch.int64).pin_memory()
    pageable = np.zeros(2, dtype=np.int64)
    good = (base, F64, 0)
    cases = [[(base, 7, 0)], [(base, 0xFFFFFFFF, 0)], [(base, F64, 1)], [(0, F64, 0)], [(0, I32, 0)],
             [(base + 4, F64, 0)], [(base + 4, I64, 0)], [(base + 4, U64, 0)], [(base + 2, F32, 0)],
             [(base + 2, I32, 0)], [(base + 1, F16, 0)], [(base + 1, BF16, 0)],
             [(pinned.data_ptr(), F64, 0)], [(pageable.ctypes.data, F64, 0)],
             [good, good, (pageable.ctypes.data, I32, 0)], [good] * 2000 + [(base, F64, 2)]]
    others = []
    if torch.cuda.device_count() >= 2:
        others.append(torch.zeros(1, dtype=torch.float64, device="cuda:1"))
        cases.append([good, (others[0].data_ptr(), F64, 0)])
    before = eng.stats()["kernel_launches"]
    for c in cases:
        st, out = read_raw(eng, np.array(c, dtype=SRC))
        assert st == LH_ERR_INVALID and (out == -1.0).all(), c[-1]
    out = np.full(1, -1.0)
    assert eng.lib.lh_gauges_read(eng.h, None, 1, out.ctypes.data) == LH_ERR_INVALID
    from loghisto_b200 import _lib
    srcs = np.array([good], dtype=SRC)
    assert eng.lib.lh_gauges_read(eng.h, srcs.ctypes.data_as(C.POINTER(_lib.lh_gauge_src)), 1, None) == LH_ERR_INVALID
    assert read_raw(eng, np.zeros(0, dtype=SRC))[0] == LH_OK
    assert eng.stats()["kernel_launches"] == before
    # inside an allocation, at each natural alignment: accepted
    cells.copy_(torch.tensor([-3, 1 << 40, 7, 9], dtype=torch.int64))
    st, out = read_raw(eng, np.array([(base + 8, I64, 0), (base + 16, I32, 0), (base + 24, F16, 0)], dtype=SRC))
    assert st == LH_OK and list(out) == [float(1 << 40), 7.0, float(np.array([9], np.uint16).view(np.float16)[0])]
    assert eng.stats()["kernel_launches"] == before + 1
    for bad in (1.0, np.zeros(1), torch.zeros(1), torch.zeros(2, device="cuda"), torch.zeros(1, dtype=torch.int16, device="cuda")):
        with pytest.raises(TypeError):
            eng.read_gauges([bad])


@pytest.mark.parametrize("strong", [True, False], ids=["set_gauge", "plain_store"])
def test_no_torn_values(torch, eng, gwc, strong):
    """A bounded writer alternates two patterns in F64 / I64 / U64 cells (whose mixed halves convert to other values)
    while the host makes 1 000 reads: every value read is one of the two."""
    a = [0x3FF0000000000001, 1, 1]
    b = [0xC00FFFFFFFFFFFFE, 0xFFFFFFFFFFFFFFFE, 0xFFFFFFFFFFFFFFFE]
    allowed = [{bits_f64(a[0]).tobytes(), bits_f64(b[0]).tobytes()},
               {np.float64(1.0).tobytes(), np.float64(-2.0).tobytes()},
               {np.float64(1.0).tobytes(), np.uint64(b[2]).astype(np.float64).tobytes()}]
    cells = torch.tensor(np.array(a, dtype=np.uint64).view(np.int64), device="cuda")
    srcs = np.array([(cells.data_ptr(), F64, 0), (cells.data_ptr() + 8, I64, 0), (cells.data_ptr() + 16, U64, 0)], dtype=SRC)
    torch.cuda.synchronize()
    assert read_raw(eng, srcs)[0] == LH_OK
    s = torch.cuda.Stream()
    A, B = (C.c_uint64 * 3)(*a), (C.c_uint64 * 3)(*b)
    assert gwc.gwc_flip(cells.data_ptr(), A, B, 1 if strong else 0, 2_000_000, s.cuda_stream) == 0
    reads = np.empty((1000, 3))
    for i in range(1000):
        st, reads[i] = read_raw(eng, srcs)
        assert st == LH_OK
    s.synchronize()
    for col in range(3):
        got = {x.tobytes() for x in reads[:, col]}
        assert got <= allowed[col], (col, [np.frombuffer(x, np.float64)[0] for x in got - allowed[col]])
    assert len({x.tobytes() for x in reads[:, 0]}) == 2, "no read overlapped the writer"


def test_read_never_waits(torch, eng, spin):
    """Behind a 200 ms spin a stream holds a pending write of the gauge: the read returns the old value while the
    stream is still busy, and the new one after a synchronise."""
    g = torch.full((), 1.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    assert eng.read_gauges([g])[0] == 1.0
    s = torch.cuda.Stream()
    spin(200_000_000, s)
    with torch.cuda.stream(s):
        g.fill_(2.0)
    t0 = time.perf_counter()
    v = eng.read_gauges([g])
    dt = time.perf_counter() - t0
    pending = not s.query()
    assert v[0] == 1.0 and pending, dt
    s.synchronize()
    assert eng.read_gauges([g])[0] == 2.0


def expected(torch, x, code):
    """float64 of the value in the one-element tensor x (read back to the CPU)."""
    if code == U64:
        return float(x.view(torch.int64).cpu().numpy().reshape(-1).view(np.uint64).astype(np.float64)[0])
    if code in (I64, I32):
        return float(x.cpu().numpy().reshape(-1).astype(np.float64)[0])
    return float(x.cpu().to(torch.float64).reshape(-1)[0].item())


def bits(x):
    return np.float64(x).view(np.uint64)


def test_metric_system_values(torch, gwc):
    """Values written by fill_ / copy_, by lh::set_gauge in a kernel and by a torch.cuda.graph replay appear bit for bit
    in Gauges and in the processed metrics, in every collection while registered; a gauge function replaces a device
    gauge and back; deregistering removes it."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=8, max_counters=4)
    try:
        f32s = torch.zeros(4, dtype=torch.float32, device="cuda")
        cells = {"f64": (torch.zeros((), dtype=torch.float64, device="cuda"), F64),
                 "f32": (f32s[2], F32),
                 "f16": (torch.zeros((), dtype=torch.float16, device="cuda"), F16),
                 "bf16": (torch.zeros((), dtype=torch.bfloat16, device="cuda"), BF16),
                 "i64": (torch.zeros((), dtype=torch.int64, device="cuda"), I64),
                 "i32": (torch.zeros((), dtype=torch.int32, device="cuda"), I32),
                 "u64": (torch.zeros((), dtype=torch.int64, device="cuda").view(torch.uint64), U64)}
        for name, (x, _) in cells.items():
            ms.RegisterDeviceGauge(name, x)

        def check():
            torch.cuda.synchronize()
            want = {n: expected(torch, x, c) for n, (x, c) in cells.items()}
            for _ in range(2):
                raw, metrics = ms.collect_and_process()
                assert set(raw["Gauges"]) == set(want)
                for n, w in want.items():
                    assert bits(raw["Gauges"][n]) == bits(w) and bits(metrics[n]) == bits(w), (n, raw["Gauges"][n], w)
            return want

        # fill_ / copy_
        cells["f64"][0].fill_(math.pi)
        cells["f32"][0].copy_(torch.tensor(1 / 3, dtype=torch.float32))
        cells["f16"][0].fill_(-65504.0)
        cells["bf16"][0].fill_(3.14159)
        cells["i64"][0].fill_(-(1 << 63))
        cells["i32"][0].copy_(torch.tensor(-7, dtype=torch.int32))
        cells["u64"][0].view(torch.int64).fill_(-1)
        w = check()
        assert w["u64"] == 2.0 ** 64 and w["i64"] == -2.0 ** 63 and w["f16"] == -65504.0
        # lh::set_gauge in a kernel
        patterns = {"f64": 0x7FEFFFFFFFFFFFFF, "f32": 0x00000001, "f16": 0x8001, "bf16": 0x7F7F, "i64": (1 << 53) + 1,
                    "i32": 0x80000000, "u64": (1 << 63) + 1024}
        st = torch.cuda.current_stream().cuda_stream
        for n, (x, c) in cells.items():
            assert gwc.gwc_set(x.data_ptr(), c, patterns[n], st) == 0
        w = check()
        assert w["i64"] == 2.0 ** 53 and w["u64"] == 2.0 ** 63 and w["i32"] == -2.0 ** 31 and w["f32"] == 2.0 ** -149
        # a CUDA graph replay
        srcs = {n: torch.zeros_like(x.view(torch.int64) if c == U64 else x) for n, (x, c) in cells.items()}
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            for n, (x, c) in cells.items():
                (x.view(torch.int64) if c == U64 else x).copy_(srcs[n])
        for j in range(1, 3):
            srcs["f64"].fill_(-0.0 if j == 1 else 1e-310)
            srcs["f32"].fill_(float(j) / 7)
            srcs["f16"].fill_(6e-8 * j)
            srcs["bf16"].fill_(-1e38 * j)
            srcs["i64"].fill_((1 << 62) + 512 * j)
            srcs["i32"].fill_(123456789 * j)
            srcs["u64"].fill_(-1025 * j)
            torch.cuda.synchronize()
            g.replay()
            w = check()
            assert bits(w["f64"]) == bits(-0.0 if j == 1 else 1e-310)
        # a gauge function replaces a device gauge, and back; deregistering removes either
        ms.RegisterConstantGauge("f64", 42.0)
        assert ms.collect_and_process()[0]["Gauges"]["f64"] == 42.0
        ms.RegisterDeviceGauge("f64", cells["f64"][0])
        assert bits(ms.collect_and_process()[0]["Gauges"]["f64"]) == bits(w["f64"])
        ms.DeregisterGaugeFunc("f64")
        ms.DeregisterGaugeFunc("u64")
        assert set(ms.collect_and_process()[0]["Gauges"]) == set(cells) - {"f64", "u64"}
        with pytest.raises(TypeError):
            ms.RegisterDeviceGauge("bad", torch.zeros(2, device="cuda"))
        with pytest.raises(TypeError):
            ms.RegisterDeviceGauge("bad", torch.zeros(1, dtype=torch.uint8, device="cuda"))
        assert "bad" not in ms.collect_and_process()[0]["Gauges"]
    finally:
        ms.close()


def test_reaper_delivers_device_gauges(torch):
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(0.05, False, max_histograms=4, max_counters=4)
    sub = ms.SubscribeToProcessedMetrics(64)
    try:
        loss = torch.full((), 0.125, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        ms.RegisterDeviceGauge("loss", loss)
        ms.Start()
        deadline, got = time.monotonic() + 10.0, None
        while got is None and time.monotonic() < deadline:
            m = sub.receive(0.5)
            if m and "loss" in m:
                got = m["loss"]
        assert got == 0.125
    finally:
        ms.Stop()
        sub.close()
        ms.close()


def test_launches_per_collection(torch):
    """A collection with device gauges issues one launch more than one without (the read of every gauge, however
    many); without device gauges, before and after, it issues the same launches."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(1.0, False, max_histograms=4, max_counters=4)
    try:
        xs = torch.arange(64, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()

        def launches():
            ms.HistogramMany("lat", np.arange(1.0, 101.0))
            ms.Counter("req", 1)
            before = ms.stats()["kernel_launches"]
            ms.collect_and_process()
            return ms.stats()["kernel_launches"] - before

        plain = [launches() for _ in range(3)]
        for i in range(64):
            ms.RegisterDeviceGauge("g%d" % i, xs[i])
        with_gauges = [launches() for _ in range(3)]
        for i in range(64):
            ms.DeregisterGaugeFunc("g%d" % i)
        after = [launches() for _ in range(3)]
        assert len(set(plain)) == 1 and after == plain and with_gauges == [plain[0] + 1] * 3
    finally:
        ms.close()
