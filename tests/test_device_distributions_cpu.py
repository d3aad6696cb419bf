"""Distribution gauges bound to names (MetricSystem::RegisterDeviceDistribution, loghisto_b200/host/metric_system.cc) on
the CPU: the C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI, extended by
tests/stub_abi/lh_stub_distributions.c, whose "device" memory is host memory from lh_stub_gauge_alloc.  Covers the
registry and its name pinning, the call's place between lh_snapshot_begin and the first read, refusal at registration,
refusal of registry calls from a thread that holds a record scope, a call that fails at a collection (the set is still delivered), the C shim called from C, the Python argument checks,
the ctypes layout, and random sequences of registrations, rewrites, Histogram calls and collections against an exact
per-collection model.  tests/test_gpu_device_distributions.py runs the real library."""
import collections
import ctypes
import os
import random
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
LH_OK, LH_ERR_INVALID, LH_ERR_STATE = 0, -1, -5
F64, F32, F16, BF16, I64, I32, U64 = range(7)
NP_DTYPES = {F64: np.float64, F32: np.float32, F16: np.float16, I64: np.int64, I32: np.int32, U64: np.uint64}


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_distributions.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_distributions.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f)
                    for f in ("lh_stub_distributions.c", "lh_stub_gauges.c", "lh_stub_record.c")] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_distributions", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    s = ctypes.CDLL(stub)
    s.lh_stub_gauge_alloc.restype = ctypes.c_void_p
    s.lh_stub_gauge_alloc.argtypes = [ctypes.c_size_t]
    s.lh_stub_gauge_free.argtypes = [ctypes.c_void_p]
    s.lh_stub_dist_log.restype = ctypes.c_size_t
    s.lh_stub_dist_log.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    s.lh_stub_dist_last.restype = ctypes.c_uint32
    s.lho_compress.restype = ctypes.c_int16
    s.lho_compress.argtypes = [ctypes.c_double]
    return s, host


@pytest.fixture
def stub(stub_libs):
    s = stub_libs[0]
    log(s)   # start every test with an empty call log
    return s


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    made = []

    def make(max_histograms=8, interval=1.0):
        ms = m.MetricSystem(interval, False, max_histograms=max_histograms, max_counters=4)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


def log(stub) -> str:
    buf = ctypes.create_string_buffer(4096)
    n = stub.lh_stub_dist_log(buf, 4096)
    return buf.raw[:n].decode()


def last_ids(stub) -> list:
    from loghisto_b200 import _lib
    out = (_lib.lh_array_src * 256)()
    n = stub.lh_stub_dist_last(out, 256)
    return [(int(out[i].n), int(out[i].histogram_id)) for i in range(n)]


class Cells:
    """A "device" array from the stub's allocator, rewritten with numpy values of one dtype."""

    def __init__(self, stub, dtype, n):
        self.stub, self.dtype, self.n = stub, dtype, n
        self.ptr = stub.lh_stub_gauge_alloc(max(n, 1) * np.dtype(NP_DTYPES[dtype]).itemsize)

    def write(self, values):
        with np.errstate(over="ignore"):   # float16 overflows to infinity, as a store of the value would
            raw = np.ascontiguousarray(values, dtype=NP_DTYPES[self.dtype]).tobytes()
        ctypes.memmove(self.ptr, raw, len(raw))

    def free(self):
        if self.ptr:
            self.stub.lh_stub_gauge_free(self.ptr)
            self.ptr = None


def register(ms, name, ptr, n, dtype):
    return ms._lib.lhms_register_device_distribution(ms._h, name.encode(), ptr, n, dtype)


def buckets(stub, values) -> dict:
    """What Histogram(name, float64(x)) for every x of values records: {bucket key: count}."""
    return dict(collections.Counter(int(stub.lho_compress(float(v))) for v in values))


def test_registry_values_and_call_order(MS, stub):
    """Each collection records the array's current values under its name, in one call between lh_snapshot_begin and the
    reduction; without distributions a collection makes no such call."""
    ms = MS()
    a = Cells(stub, F32, 6)
    try:
        ms.HistogramMany("lat", [1.0, 2.0])
        assert ms.collect_and_process()[0]["Histograms"] == {"lat": buckets(stub, [1.0, 2.0])}
        assert log(stub) == "BREN"
        vals = [0.5, -3.25, 1e-40, 7.0, 7.0, 65504.0]
        a.write(vals)
        assert register(ms, "occ", a.ptr, a.n, F32) == LH_OK
        for j in range(3):
            raw, metrics = ms.collect_and_process()
            f32 = np.asarray(vals, np.float32).astype(np.float64)
            assert raw["Histograms"] == {"occ": buckets(stub, f32)}
            assert metrics["occ_count"] == 6.0
            assert log(stub) == "BAREN"
            vals = [v + j for v in vals]
            a.write(vals)
        ms.DeregisterDeviceDistribution("occ")
        assert ms.collect_and_process()[0]["Histograms"] == {}
        assert log(stub) == "BREN"
    finally:
        a.free()


def test_name_keeps_its_id_and_overflow_is_dropped(MS, stub):
    """A registered name is used in every interval, so it keeps its id while other names come and go around it; a name
    that gets no free id has its elements counted as dropped until an id frees up."""
    ms = MS(max_histograms=3)
    a = Cells(stub, I32, 4)
    a.write([1, 2, 3, 4])
    try:
        assert register(ms, "d", a.ptr, 4, I32) == LH_OK
        ms.collect_and_process()
        (n, hid), = last_ids(stub)
        assert n == 4
        for k in range(8):   # other names in turn, with idle intervals between them
            if k % 2:
                ms.Histogram("x%d" % k, 1.0)
                ms.Histogram("y%d" % k, 2.0)
            raw = ms.collect_and_process()[0]
            assert last_ids(stub) == [(4, hid)]
            assert sum(raw["Histograms"]["d"].values()) == 4
        ms.DeregisterDeviceDistribution("d")
        log(stub)
        ms2 = MS(max_histograms=2)
        ms2.Histogram("a", 1.0)
        ms2.Histogram("b", 1.0)
        assert register(ms2, "d", a.ptr, 4, I32) == LH_OK
        d0 = ms2.dropped()
        raw = ms2.collect_and_process()[0]
        assert "d" not in raw["Histograms"] and ms2.dropped() == d0 + 4
        assert log(stub) == "BREN"
        for _ in range(4):   # a and b go idle, retire, and free their ids
            raw = ms2.collect_and_process()[0]
            if "d" in raw["Histograms"]:
                break
        assert raw["Histograms"] == {"d": buckets(stub, [1, 2, 3, 4])}
        assert ms2.dropped() % 4 == d0 % 4
    finally:
        a.free()


def test_union_replace_and_two_names(MS, stub):
    """Samples of the array join the name's Histogram samples; registering again replaces the array; one array may
    stand under two names, and overlapping arrays each count their own elements."""
    ms = MS()
    a, b = Cells(stub, F64, 5), Cells(stub, U64, 3)
    a.write([1.0, 2.0, 3.0, 4.0, 5.0])
    b.write([0, 1 << 63, (1 << 64) - 1])
    try:
        assert register(ms, "m", a.ptr, 5, F64) == LH_OK
        assert register(ms, "m2", a.ptr, 5, F64) == LH_OK
        assert register(ms, "tail", a.ptr + 16, 3, F64) == LH_OK
        ms.Histogram("m", 3.0)
        ms.HistogramMany("m", [10.0, 11.0])
        raw = ms.collect_and_process()[0]["Histograms"]
        assert raw["m"] == buckets(stub, [1.0, 2.0, 3.0, 4.0, 5.0, 3.0, 10.0, 11.0])
        assert raw["m2"] == buckets(stub, [1.0, 2.0, 3.0, 4.0, 5.0])
        assert raw["tail"] == buckets(stub, [3.0, 4.0, 5.0])
        assert register(ms, "m", b.ptr, 3, U64) == LH_OK
        raw = ms.collect_and_process()[0]["Histograms"]
        assert raw["m"] == buckets(stub, [0.0, float(1 << 63), float((1 << 64) - 1)])
        assert register(ms, "m", a.ptr, 0, F64) == LH_OK   # empty: nothing recorded, the name absent
        raw = ms.collect_and_process()[0]["Histograms"]
        assert "m" not in raw and set(raw) == {"m2", "tail"}
    finally:
        a.free()
        b.free()


def test_registration_refused(MS, stub):
    """A refused dtype or first element registers nothing and leaves the array already under that name in place."""
    ms = MS()
    a = Cells(stub, F64, 4)
    a.write([1.0, 2.0, 3.0, 4.0])
    outside = ctypes.create_string_buffer(64)
    try:
        assert register(ms, "g", a.ptr, 4, F64) == LH_OK
        for ptr, n, dtype in ((None, 1, F64), (a.ptr + 4, 2, F64), (a.ptr + 2, 2, F32), (a.ptr + 1, 1, F16),
                              (a.ptr, 1, 7), (a.ptr, 0, 7), (a.ptr, 4, 0xFFFFFFFF), (ctypes.addressof(outside), 4, F64)):
            assert register(ms, "g", ptr, n, dtype) == LH_ERR_INVALID, (ptr, n, dtype)
            assert register(ms, "h", ptr, n, dtype) == LH_ERR_INVALID, (ptr, n, dtype)
        raw = ms.collect_and_process()[0]["Histograms"]
        assert raw == {"g": buckets(stub, [1.0, 2.0, 3.0, 4.0])}
        assert register(ms, "h", None, 0, BF16) == LH_OK   # no element to check
        assert ms._lib.lhms_register_device_distribution(None, b"x", a.ptr, 1, F64) == LH_ERR_INVALID
    finally:
        a.free()


def test_failed_call_delivers_the_set(MS, stub, capfd):
    """When lh_snapshot_ingest_arrays refuses a collection's arrays, the failure is logged and that set is delivered
    with everything else; the collection after the bad array is gone has the distributions again."""
    ms = MS()
    a, b = Cells(stub, I64, 2), Cells(stub, F32, 2)
    a.write([-5, 6])
    b.write([0.25, 0.5])
    try:
        assert register(ms, "a", a.ptr, 2, I64) == LH_OK and register(ms, "b", b.ptr, 2, F32) == LH_OK
        ms.HistogramMany("lat", np.arange(1.0, 11.0))
        ms.Counter("req", 3)
        a.free()   # "a" now points at memory the library refuses
        raw, metrics = ms.collect_and_process()
        assert set(raw["Histograms"]) == {"lat"} and raw["Rates"] == {"req": 3}
        assert metrics["lat_count"] == 10.0 and "b_count" not in metrics
        assert "lh_snapshot_ingest_arrays failed" in capfd.readouterr().err
        assert log(stub) == "BREN"
        ms.DeregisterDeviceDistribution("a")
        assert ms.collect_and_process()[0]["Histograms"] == {"b": buckets(stub, [0.25, 0.5])}
    finally:
        a.free()
        b.free()


def test_refused_from_a_thread_that_holds_a_record_scope(MS, stub):
    """Register and Deregister wait for a collection in progress, which may itself wait for the record scopes of its
    interval; from a thread that holds an open scope they are refused (LH_ERR_STATE, RuntimeError) instead, and the
    registry is unchanged."""
    ms = MS()
    a = Cells(stub, F64, 2)
    a.write([1.0, 2.0])
    try:
        assert register(ms, "d", a.ptr, 2, F64) == LH_OK
        with ms.recording(histograms=["x"]):
            assert register(ms, "e", a.ptr, 2, F64) == LH_ERR_STATE
            assert ms._lib.lhms_deregister_device_distribution(ms._h, b"d") == LH_ERR_STATE
            with pytest.raises(RuntimeError):
                ms.DeregisterDeviceDistribution("d")
        assert ms.collect_and_process()[0]["Histograms"] == {"d": buckets(stub, [1.0, 2.0])}
        assert ms._lib.lhms_deregister_device_distribution(ms._h, b"d") == LH_OK
        assert ms.collect_and_process()[0]["Histograms"] == {}
    finally:
        a.free()


def test_c_shim_from_c(tmp_path, stub_libs):
    """lhms_register_device_distribution / lhms_deregister_device_distribution called from C."""
    stub, host = stub_libs
    src = tmp_path / "client.c"
    src.write_text(r'''
#include <stdint.h>
#include <stdio.h>
#include <string.h>
void *lhms_new(int64_t, int, uint32_t, uint32_t, char *, int);
void lhms_free(void *);
int lhms_register_device_distribution(void *, const char *, const void *, uint64_t, uint32_t);
int lhms_deregister_device_distribution(void *, const char *);
int lhms_collect_and_process(void *, void (*)(void *, int, const char *, int, uint64_t, double), void *, char *, int);
void *lh_stub_gauge_alloc(size_t);
void lh_stub_gauge_free(void *);
static void emit(void *ctx, int kind, const char *name, int key, uint64_t u, double f) {
    (void)ctx;
    if (kind == 2) printf("H %s %d %llu\n", name, key, (unsigned long long)u);
    if (kind == 3 && strstr(name, "_count")) printf("M %s %g\n", name, f);
}
int main(void) {
    char err[256];
    void *ms = lhms_new(1000000000, 0, 4, 4, err, sizeof err);
    int32_t *v = (int32_t *)lh_stub_gauge_alloc(3 * sizeof(int32_t));
    v[0] = 7; v[1] = 7; v[2] = -1;
    printf("R %d %d\n", lhms_register_device_distribution(ms, "q", v, 3, 5),
           lhms_register_device_distribution(ms, "bad", v, 3, 9));
    if (lhms_collect_and_process(ms, emit, 0, err, sizeof err)) return 1;
    lhms_deregister_device_distribution(ms, "q");
    printf("--\n");
    if (lhms_collect_and_process(ms, emit, 0, err, sizeof err)) return 1;
    lh_stub_gauge_free(v);
    lhms_free(ms);
    return 0;
}
''')
    exe = tmp_path / "client"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src), host, os.path.join(BUILD, "liblh_stub_distributions.so"),
                    "-Wl,-rpath," + BUILD], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert out[0] == "R 0 -1"
    k7, km1 = int(stub.lho_compress(7.0)), int(stub.lho_compress(-1.0))
    rows = set(out[1:out.index("--")])
    assert rows == {"H q %d 2" % k7, "H q %d 1" % km1, "M q_count 3"}
    assert [x for x in out[out.index("--") + 1:] if x] == []


def test_python_argument_checks(MS):
    """RegisterDeviceDistribution takes contiguous CUDA tensors of the seven gauge dtypes only; anything else is a
    TypeError before the library sees it."""
    torch = pytest.importorskip("torch")
    ms = MS()
    for bad in (1.0, [1.0], np.zeros(4), torch.zeros(4), torch.zeros(4, dtype=torch.int16), torch.zeros(4, 4).t()):
        with pytest.raises(TypeError):
            ms.RegisterDeviceDistribution("x", bad)
    assert ms._device_dists == {}
    ms.DeregisterDeviceDistribution("never")


def test_layout_and_bindings(tmp_path, stub_libs):
    """lh_array_src as a C compiler sees it, the ctypes mirror, and the lhms_ shim."""
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    c = tmp_path / "layout.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "loghisto_b200.h"\nint main(void) {\n'
                 'printf("%zu %zu %zu %zu %zu\\n", sizeof(lh_array_src), offsetof(lh_array_src, d_values), '
                 'offsetof(lh_array_src, n), offsetof(lh_array_src, dtype), offsetof(lh_array_src, histogram_id));\n'
                 'return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", INC, "-o", str(exe), str(c)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    ct = _lib.lh_array_src
    assert out == [ctypes.sizeof(ct), ct.d_values.offset, ct.n.offset, ct.dtype.offset, ct.histogram_id.offset]
    assert out == [24, 0, 8, 16, 20]
    assert _lib.SIGNATURES["lh_snapshot_ingest_arrays"][1][1]._type_ is ct
    text = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    assert re.findall(r"LHMS_API [\w *]+?(lhms_\w*distribution\w*)\(", text) == \
        ["lhms_register_device_distribution", "lhms_deregister_device_distribution"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    assert L.lhms_register_device_distribution.argtypes is not None


@pytest.mark.parametrize("seed", range(6))
def test_random_sequences(MS, stub, seed):
    """Random interleavings of register, re-register, deregister, array rewrites, Histogram calls and collections:
    every collection's Histograms and _count metrics equal an exact model that records, per collection, each registered
    name's array contents at that time plus the Histogram samples since the previous collection."""
    rng = random.Random(seed)
    ms = MS(max_histograms=16)
    dtypes = [F64, F32, F16, I64, I32, U64]
    arrays = [Cells(stub, dtypes[i % len(dtypes)], rng.randint(0, 9)) for i in range(5)]
    contents = []

    def fresh(arr):
        if arr.dtype in (F64, F32, F16):
            v = [rng.choice([0.0, -1.5, 2.0 ** rng.randint(-30, 30), rng.uniform(-1e4, 1e4)]) for _ in range(arr.n)]
        elif arr.dtype == U64:
            v = [rng.choice([0, 1, (1 << 64) - 1, rng.getrandbits(64)]) for _ in range(arr.n)]
        else:
            bits = 31 if arr.dtype == I32 else 63
            v = [rng.randint(-(1 << bits), (1 << bits) - 1) for _ in range(arr.n)]
        arr.write(v)
        with np.errstate(over="ignore"):
            return [float(x) for x in np.asarray(v, NP_DTYPES[arr.dtype]).astype(np.float64)]

    try:
        contents = [fresh(a) for a in arrays]
        names = ["n%d" % i for i in range(6)]
        registered = {}    # name -> array index
        pending = collections.defaultdict(list)
        for step in range(120):
            op = rng.random()
            name = rng.choice(names)
            if op < 0.2:
                i = rng.randrange(len(arrays))
                assert register(ms, name, arrays[i].ptr, arrays[i].n, arrays[i].dtype) == LH_OK
                registered[name] = i
            elif op < 0.3:
                ms.DeregisterDeviceDistribution(name)
                registered.pop(name, None)
            elif op < 0.5:
                i = rng.randrange(len(arrays))
                contents[i] = fresh(arrays[i])
            elif op < 0.75:
                v = rng.uniform(-100, 100)
                ms.Histogram(name, v)
                pending[name].append(v)
            else:
                expect = collections.defaultdict(list)
                for nm, vals in pending.items():
                    expect[nm] += vals
                for nm, i in registered.items():
                    expect[nm] += contents[i]
                raw, metrics = ms.collect_and_process()
                want = {nm: buckets(stub, v) for nm, v in expect.items() if v}
                assert raw["Histograms"] == want, step
                for nm, v in expect.items():
                    if v:
                        assert metrics[nm + "_count"] == float(len(v))
                pending.clear()
        assert ms.dropped() == 0
    finally:
        for a in arrays:
            a.free()
