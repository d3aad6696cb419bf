"""Device gauges bound to names (MetricSystem::RegisterDeviceGauge, loghisto_b200/host/metric_system.cc) on the CPU: the
C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus tests/stub_abi/lh_stub_gauges.c, whose
"device" memory is host memory it hands out and whose lh_gauges_read refuses any other address.  Covers the name space
gauge functions and device gauges share, refusal at registration, a read that fails at a collection (only the device
gauges are dropped, the set is still delivered), one read per collection and none without device gauges, the reaper,
the Python argument checks, and the ctypes layout.  tests/test_gpu_device_gauges.py runs the real library."""
import ctypes
import os
import re
import struct
import subprocess
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
LH_OK, LH_ERR_INVALID = 0, -1
F64, F32, F16, BF16, I64, I32, U64 = range(7)


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_gauges.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_gauges.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in ("lh_stub.c", "lh_stub_gauges.c")] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_gauges", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    s = ctypes.CDLL(stub)
    s.lh_stub_gauge_alloc.restype = ctypes.c_void_p
    s.lh_stub_gauge_alloc.argtypes = [ctypes.c_size_t]
    s.lh_stub_gauge_free.argtypes = [ctypes.c_void_p]
    s.lh_stub_gauge_reads.restype = ctypes.c_uint64
    return s, host


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    made = []

    def make(interval=1.0):
        ms = m.MetricSystem(interval, False, max_histograms=4, max_counters=4)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


def cell(stub, fmt, value):
    """A "device" cell holding `value` packed with struct format `fmt`."""
    p = stub.lh_stub_gauge_alloc(8)
    raw = struct.pack("<" + fmt, value)
    ctypes.memmove(p, raw, len(raw))
    return p


def register(ms, name, ptr, dtype):
    return ms._lib.lhms_register_device_gauge(ms._h, name.encode(), ptr, dtype)


def test_shared_name_space(MS, stub):
    """A device gauge and a gauge function under one name replace each other; DeregisterGaugeFunc removes either; one
    read per collection while device gauges are registered, none otherwise."""
    ms = MS()
    p, q = cell(stub, "d", 2.5), cell(stub, "q", -(1 << 62) - 1)
    try:
        ms.RegisterConstantGauge("g", 1.5)
        r0 = stub.lh_stub_gauge_reads()
        assert ms.collect_and_process()[0]["Gauges"] == {"g": 1.5}
        assert stub.lh_stub_gauge_reads() == r0
        assert register(ms, "g", p, F64) == LH_OK
        assert register(ms, "i", q, I64) == LH_OK
        r1 = stub.lh_stub_gauge_reads()
        assert r1 == r0 + 2   # the validating read of each registration
        for j in range(3):
            raw, metrics = ms.collect_and_process()
            assert raw["Gauges"] == {"g": 2.5, "i": float(-(1 << 62) - 1)}
            assert metrics["g"] == 2.5 and metrics["i"] == float(-(1 << 62) - 1)
            assert stub.lh_stub_gauge_reads() == r1 + j + 1
        ctypes.memmove(p, struct.pack("<d", -7.0), 8)
        assert ms.collect_and_process()[0]["Gauges"]["g"] == -7.0
        ms.RegisterConstantGauge("g", 3.0)
        assert ms.collect_and_process()[0]["Gauges"] == {"g": 3.0, "i": float(-(1 << 62) - 1)}
        ms.DeregisterGaugeFunc("i")
        r2 = stub.lh_stub_gauge_reads()
        assert ms.collect_and_process()[0]["Gauges"] == {"g": 3.0}
        assert stub.lh_stub_gauge_reads() == r2
        assert register(ms, "g", p, F64) == LH_OK
        assert ms.collect_and_process()[0]["Gauges"] == {"g": -7.0}
        ms.DeregisterGaugeFunc("g")
        ms.DeregisterGaugeFunc("never")
        assert ms.collect_and_process()[0]["Gauges"] == {}
    finally:
        stub.lh_stub_gauge_free(p)
        stub.lh_stub_gauge_free(q)


def test_registration_refused(MS, stub):
    """A refused address or dtype registers nothing and leaves the gauge already under that name in place."""
    ms = MS()
    p = cell(stub, "f", 0.25)
    outside = ctypes.create_string_buffer(16)
    try:
        ms.RegisterConstantGauge("g", 1.0)
        for ptr, dtype in ((None, F64), (p + 4, F64), (p + 2, F32), (p + 1, F16), (p, 7), (p, 0xFFFFFFFF),
                           (ctypes.addressof(outside), F64)):
            assert register(ms, "g", ptr, dtype) == LH_ERR_INVALID, (ptr, dtype)
            assert register(ms, "h", ptr, dtype) == LH_ERR_INVALID, (ptr, dtype)
        assert ms.collect_and_process()[0]["Gauges"] == {"g": 1.0}
        assert register(ms, "h", p, F32) == LH_OK
        assert ms.collect_and_process()[0]["Gauges"] == {"g": 1.0, "h": 0.25}
        assert ms._lib.lhms_register_device_gauge(None, b"x", p, F32) == LH_ERR_INVALID
    finally:
        stub.lh_stub_gauge_free(p)


def test_failed_read_drops_only_device_gauges(MS, stub, capfd):
    """When the read at a collection fails, that set carries no device gauge but everything else, and the failure is
    logged; the next collection without the bad gauge has the device gauges again."""
    ms = MS()
    a, b = cell(stub, "i", -5), cell(stub, "Q", (1 << 64) - 1)
    try:
        ms.RegisterConstantGauge("f", 9.0)
        assert register(ms, "a", a, I32) == LH_OK and register(ms, "b", b, U64) == LH_OK
        ms.HistogramMany("lat", np.arange(1.0, 11.0))
        ms.Counter("req", 3)
        stub.lh_stub_gauge_free(a)   # "a" now points at memory the library refuses
        a = None
        raw, metrics = ms.collect_and_process()
        assert raw["Gauges"] == {"f": 9.0}
        assert sum(raw["Histograms"]["lat"].values()) == 10 and raw["Rates"] == {"req": 3}
        assert metrics["f"] == 9.0 and metrics["lat_count"] == 10.0 and "a" not in metrics and "b" not in metrics
        assert "lh_gauges_read failed" in capfd.readouterr().err
        ms.DeregisterGaugeFunc("a")
        assert ms.collect_and_process()[0]["Gauges"] == {"f": 9.0, "b": 18446744073709551616.0}
    finally:
        if a:
            stub.lh_stub_gauge_free(a)
        stub.lh_stub_gauge_free(b)


def test_reaper_delivers_device_gauges(MS, stub):
    ms = MS(interval=0.01)
    p = cell(stub, "e", 0.5)   # float16
    sub = ms.SubscribeToProcessedMetrics(64)
    try:
        assert register(ms, "h16", p, F16) == LH_OK
        ms.Start()
        deadline, got = time.monotonic() + 5.0, None
        while got is None and time.monotonic() < deadline:
            m = sub.receive(0.5)
            if m and "h16" in m:
                got = m["h16"]
        assert got == 0.5
    finally:
        ms.Stop()
        sub.close()
        stub.lh_stub_gauge_free(p)


def test_python_argument_checks(MS):
    """RegisterDeviceGauge takes one-element CUDA tensors of the seven gauge dtypes only; anything else is a TypeError
    before the library sees it."""
    torch = pytest.importorskip("torch")
    ms = MS()
    for bad in (1.0, np.zeros(1), torch.zeros(1), torch.zeros(1, dtype=torch.int16)):
        with pytest.raises(TypeError):
            ms.RegisterDeviceGauge("x", bad)
    from loghisto_b200.engine import _GAUGE_DTYPES
    assert sorted(_GAUGE_DTYPES.values()) == list(range(7))
    assert set(_GAUGE_DTYPES) == {"torch.float64", "torch.float32", "torch.float16", "torch.bfloat16", "torch.int64",
                                  "torch.int32", "torch.uint64"}


def test_layout_and_bindings(tmp_path, stub_libs):
    """lh_gauge_src and the LH_GAUGE_* values as a C compiler sees them, the ctypes mirror, and the lhms_ shim."""
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    names = ["LH_GAUGE_F64", "LH_GAUGE_F32", "LH_GAUGE_F16", "LH_GAUGE_BF16", "LH_GAUGE_I64", "LH_GAUGE_I32", "LH_GAUGE_U64"]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"', 'int main(void) {',
           'printf("%zu %zu %zu %zu\\n", sizeof(lh_gauge_src), offsetof(lh_gauge_src, d_value), '
           'offsetof(lh_gauge_src, dtype), offsetof(lh_gauge_src, reserved));']
    src += ['printf("%%d\\n", %s);' % n for n in names]
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", INC, "-o", str(exe), str(c)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    ct = _lib.lh_gauge_src
    assert [int(x) for x in out[0].split()] == [ctypes.sizeof(ct), ct.d_value.offset, ct.dtype.offset, ct.reserved.offset]
    assert ctypes.sizeof(ct) == 16
    assert [int(x) for x in out[1:8]] == [getattr(_lib, n) for n in names] == list(range(7))
    assert "lh_gauges_read" in _lib.SIGNATURES
    text = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    assert re.findall(r"LHMS_API [\w *]+?(lhms_\w*gauge\w*)\(", text) == \
        ["lhms_register_constant_gauge", "lhms_register_device_gauge", "lhms_deregister_gauge"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    assert L.lhms_register_device_gauge.argtypes is not None and L.lhms_deregister_gauge.argtypes is not None
