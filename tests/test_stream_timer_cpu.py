"""GPU timers of the MetricSystem mirror (MetricSystem::StartGpuTimer / GpuTimerToken, MetricSystem.StartGpuTimer /
gpu_timer in Python) on the CPU: the C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus
tests/stub_abi/lh_stub_stream_timer.c, whose timers read the host's monotonic clock.  Covers the host logic: names bound
at stop time, drop-and-count, the interval a stop lands in, the Python stream mapping and token consumption.
tests/test_gpu_stream_timer.py runs the real library."""
import ctypes
import os
import re
import subprocess
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUB = os.path.join(ROOT, "tests", "stub_abi")


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_stream_timer.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_stream_timer.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC,
                    os.path.join(STUB, "lh_stub.c"), os.path.join(STUB, "lh_stub_reduce_sparse.c"),
                    os.path.join(STUB, "lh_stub_record.c"), os.path.join(STUB, "lh_stub_stream_timer.c"),
                    os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_stream_timer", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    s = ctypes.CDLL(stub)
    s.lh_stub_gpu_timer_pool.argtypes = [ctypes.c_uint32]
    s.lh_stub_gpu_timer_stream.restype = ctypes.c_void_p
    s.lh_stub_gpu_timer_stops.restype = ctypes.c_uint64
    return s, host


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    stub, host = stub_libs
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
    made = []

    def make(max_histograms=4, pool=65536):
        stub.lh_stub_gpu_timer_pool(pool)
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=4)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


def one_sample(raw, name):
    """The bucket of the single sample of `name` in a raw set."""
    h = raw["Histograms"][name]
    assert sum(h.values()) == 1, h
    return next(iter(h))


def test_stop_records_the_span_under_its_name(MS, stub, oracle):
    import numpy as np
    ms = MS()
    out = np.zeros(1, dtype=np.int64)
    t = ms.StartGpuTimer("span")
    assert ms._lib.lhms_gpu_timer_stop(t._h, None, out.ctypes.data) == 0
    t._free()
    assert out[0] >= 0
    raw, m = ms.collect_and_process()
    assert one_sample(raw, "span") == oracle.compress(float(out[0]))
    assert m["span_count"] == 1
    assert ms.dropped() == 0


def test_unbound_name_drops_and_counts(MS, stub):
    """A full name table: the name binds to no id at stop time, so the sample is dropped and counted, not recorded."""
    ms = MS(max_histograms=2)
    for nm in ("a", "b"):
        ms.Histogram(nm, 1.0)
    t = ms.StartGpuTimer("new")
    t.Stop()
    assert ms.dropped() == 1
    assert stub.lh_stub_gpu_timer_stops() == 0
    raw, _ = ms.collect_and_process()
    assert set(raw["Histograms"]) == {"a", "b"}


def test_exhausted_pool_gives_a_token_that_drops_and_counts(MS, stub):
    """StartGpuTimer never fails: with every slot held it returns a token whose Stop drops and counts.  Releasing the
    slot (the first token's Stop consumes and frees it) makes the next start take it again."""
    ms = MS(pool=1)
    held = ms.StartGpuTimer("t")
    spare = ms.StartGpuTimer("t")
    spare.Stop()
    assert ms.dropped() == 1
    held.Stop()
    again = ms.StartGpuTimer("t")
    again.Stop()
    raw, m = ms.collect_and_process()
    assert m["t_count"] == 2
    assert ms.dropped() == 1


def test_stop_after_a_collection_lands_in_the_next_interval(MS, stub):
    """As Go's Stop calls Histogram at stop time: a timer started in interval k and stopped after its collection is a
    sample of interval k+1."""
    ms = MS()
    t = ms.StartGpuTimer("late")
    raw, _ = ms.collect_and_process()
    assert "late" not in raw["Histograms"]
    t.Stop()
    raw, m = ms.collect_and_process()
    assert m["late_count"] == 1


def test_name_recycled_while_held_still_records_under_it(MS, stub):
    """The name's id is recycled while the token is held (three collections without its use, and another name takes
    the id); the stop binds the name again and records under it."""
    ms = MS(max_histograms=3)
    ms.Histogram("x", 1.0)
    t = ms.StartGpuTimer("x")
    for _ in range(4):
        ms.Histogram("y", 1.0)
        ms.collect_and_process()
    ms.Histogram("z", 1.0)
    t.Stop()
    raw, m = ms.collect_and_process()
    assert set(raw["Histograms"]) == {"x", "z"}
    assert m["x_count"] == 1 and m["z_count"] == 1
    assert ms.dropped() == 0


def test_token_is_consumed_by_its_first_stop(MS, stub):
    ms = MS()
    t = ms.StartGpuTimer("once")
    t.Stop()
    t.Stop()
    assert stub.lh_stub_gpu_timer_stops() == 1
    with ms.gpu_timer("block"):
        pass
    raw, m = ms.collect_and_process()
    assert m["once_count"] == 1 and m["block_count"] == 1


def test_stream_mapping(MS, stub):
    """None and ints keep the ABI's meaning (0 = the ingest stream); a stream object whose handle is 0 (torch's default
    stream) is passed as cudaStreamLegacy (1), so it is timed as itself.  Stop(None) uses the start's stream."""
    from loghisto_b200.engine import _stream, _timer_stream
    default = types.SimpleNamespace(cuda_stream=0)
    other = types.SimpleNamespace(cuda_stream=0x5000)
    assert [_timer_stream(x) for x in (None, 0, 7, default, other)] == [0, 0, 7, 1, 0x5000]
    assert _stream(default) == 0    # the other entry points are unchanged
    ms = MS()
    t = ms.StartGpuTimer("s", default)
    assert stub.lh_stub_gpu_timer_stream() == 1
    t.Stop()
    assert stub.lh_stub_gpu_timer_stream() == 1
    t = ms.StartGpuTimer("s", other)
    t.Stop(default)
    assert stub.lh_stub_gpu_timer_stream() == 1
    with ms.gpu_timer("s", other):
        assert stub.lh_stub_gpu_timer_stream() == 0x5000
    assert stub.lh_stub_gpu_timer_stream() == 0x5000
    with ms.gpu_timer("s"):
        pass
    assert stub.lh_stub_gpu_timer_stream() is None


def test_gpu_timer_entry_points_are_bound(stub_libs):
    """Every lhms_gpu_timer_* entry point of the C shim is declared by metric_system._bind."""
    import loghisto_b200.metric_system as m
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    names = re.findall(r"LHMS_API [\w *]+?(lhms_gpu_timer_\w+)\(", src)
    assert sorted(names) == ["lhms_gpu_timer_free", "lhms_gpu_timer_start", "lhms_gpu_timer_stop"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm


def test_host_library_loads_over_a_stub_without_gpu_timers(tmp_path):
    """The timer symbols are weak in the mirror: over a C ABI without them it still links and loads, and a timer's
    Stop drops and counts."""
    stub = tmp_path / "liblh_stub_old.so"
    host = tmp_path / "libhost_old.so"
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-I", INC, os.path.join(STUB, "lh_stub.c"),
                    os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", str(stub), "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", str(host),
                    "-L", str(tmp_path), "-llh_stub_old", "-Wl,-rpath," + str(tmp_path), "-lpthread"], check=True)
    import loghisto_b200.metric_system as m
    L = m._bind(ctypes.CDLL(str(host)))
    err = ctypes.create_string_buffer(512)
    h = L.lhms_new(1000, 0, 4, 4, err, 512)
    assert h, err.value
    st = ctypes.c_int(-99)
    tok = L.lhms_gpu_timer_start(h, b"t", None, ctypes.byref(st))
    assert tok and st.value == 0
    assert L.lhms_gpu_timer_stop(tok, None, None) == 0
    L.lhms_gpu_timer_free(tok)
    assert L.lhms_dropped(h) == 1
    L.lhms_free(h)
