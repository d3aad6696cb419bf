"""Captured keyed samples, counter adds and GPU-timed spans of graph recorders (GraphRecorder.keyed / counters /
start_timer / stop_timer / timer) on the CPU: the Python layer and the C++ mirror over the TEST-ONLY oracle-backed stub of
the C ABI (tests/stub_abi/lh_stub_graph_calls.c over lh_stub_graph.c), whose recorders keep what these calls record
and drain it at each collection.  Covers name -> local id and dtype -> entry point mapping, that every error is raised before the ABI is
called, and a mirror loaded over a stub that lacks the calls.  tests/test_gpu_graph_recorder_calls.py runs the real
library."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUBS = ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c")
LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = -1, -5, -6


def build_pair(tag, graph_stub):
    """The stub (with `graph_stub` as its graph recorders) and the C++ mirror linked against it."""
    stub = os.path.join(BUILD, "liblh_stub_graph_calls%s.so" % tag)
    host = os.path.join(BUILD, "libloghisto_host_stub_graph_calls%s.so" % tag)
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in STUBS + (graph_stub,)] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_graph_calls%s" % tag, "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return ctypes.CDLL(stub), host


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    s, host = build_pair("", "lh_stub_graph_calls.c")
    s.lh_stub_graph_set_clock.argtypes = [ctypes.c_uint64]
    s.lh_stub_graph_calls.restype = ctypes.c_uint64
    s.lh_stub_graph_alive.restype = ctypes.c_uint32
    return s, host


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    stub, host = stub_libs
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    made = []

    def make(max_histograms=4, max_counters=4):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=max_counters)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()
    assert stub.lh_stub_graph_alive() == 0


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


class HostArray:
    """A host numpy array posing as a device array (the stub reads host pointers)."""

    def __init__(self, a, dtype=None):
        self.a = np.ascontiguousarray(a, dtype=dtype)
        self.__cuda_array_interface__ = {"shape": (self.a.size,), "typestr": self.a.dtype.str,
                                         "data": (self.a.ctypes.data, False), "version": 3}


def want_hist(oracle, vals):
    out = {}
    for v in vals:
        k = oracle.compress(float(v))
        out[k] = out.get(k, 0) + 1
    return out


@pytest.mark.parametrize("id_dtype", [np.uint16, np.int32, np.uint32])
@pytest.mark.parametrize("val_dtype", [np.float64, np.int64])
def test_keyed_samples_land_under_the_names_of_their_local_ids(MS, stub, oracle, id_dtype, val_dtype):
    """Local id i is histogram name i; ids past the names (a negative int32 among them) are dropped and counted.  The
    ids 65536 + 1 and 2^31 would read as other ids through the 16-bit entry point, so they pin the dtype mapping."""
    ms = MS()
    ids = [0, 1, 1, 2, 7, 0]
    if id_dtype is np.int32:
        ids += [-1]
    if id_dtype is np.uint32:
        ids += [65536 + 1, 2 ** 31]
    vals = np.arange(1, len(ids) + 1, dtype=val_dtype) * 3
    with ms.graph_recorder(histograms=["a", "b"]) as g:
        g.keyed(HostArray(ids, id_dtype), HostArray(vals))
        raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"a": want_hist(oracle, [vals[0], vals[5]]), "b": want_hist(oracle, vals[1:3])}
    assert ms.dropped() == len(ids) - 4


@pytest.mark.parametrize("id_dtype", [np.uint16, np.uint32])
@pytest.mark.parametrize("amt_dtype", [np.uint64, np.int64])
def test_counter_adds_wrap_and_drop(MS, oracle, id_dtype, amt_dtype):
    ms = MS()
    amounts = np.array([2 ** 64 - 5, 9, 3, 11, 4], dtype=np.uint64)
    ids = np.array([0, 0, 1, 2, 1], dtype=id_dtype)
    with ms.graph_recorder(counters=["x", "y"]) as g:
        g.counters(HostArray(ids), HostArray(amounts.view(amt_dtype)))
        raw, _ = ms.collect_and_process()
        assert raw["Rates"] == {"x": 4, "y": 7}
        g.counters(HostArray(ids[:1]), HostArray(amounts[1:2].view(amt_dtype)))
        raw, _ = ms.collect_and_process()
        assert raw["Rates"] == {"x": 9} and raw["Counters"]["x"] == 13
    assert ms.dropped() == 1


def test_timers_record_spans_under_their_names(MS, stub, oracle):
    ms = MS()
    out = HostArray(np.zeros(2, dtype=np.int64))
    with ms.graph_recorder(histograms=["layer", "step"]) as g:
        stub.lh_stub_graph_set_clock(100)
        g.start_timer("step")
        for i in range(3):
            with g.timer("layer"):
                stub.lh_stub_graph_set_clock(100 + 10 * (i + 1))
        stub.lh_stub_graph_set_clock(5000)
        g.stop_timer("step", out=out)
        assert out.a[0] == 4900
        g.stop_timer("step")                        # the mark stays: stopped again
        raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"layer": want_hist(oracle, [10, 10, 10]), "step": want_hist(oracle, [4900, 4900])}
    assert ms.dropped() == 0


def test_stop_without_start_is_dropped_and_counted(MS):
    ms = MS()
    with ms.graph_recorder(histograms=["never"]) as g:
        g.stop_timer("never")
        raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {} and ms.dropped() == 1


def test_every_error_is_raised_before_the_abi_is_called(MS, stub):
    import torch
    ms = MS()
    ids16, f64 = HostArray([0, 1], np.uint16), HostArray([1.0, 2.0])
    with ms.graph_recorder(histograms=["a", "b"], counters=["c"]) as g:
        before = stub.lh_stub_graph_calls()
        bad = [
            (TypeError, lambda: g.keyed(HostArray([0, 1], np.int64), f64)),                 # id dtypes
            (TypeError, lambda: g.keyed(HostArray([0, 1], np.uint8), f64)),
            (TypeError, lambda: g.keyed(ids16, HostArray([1.0, 2.0], np.float32))),          # value dtypes
            (TypeError, lambda: g.keyed(ids16, HostArray([1, 2], np.int32))),
            (TypeError, lambda: g.keyed(torch.zeros(2, dtype=torch.int32), f64)),            # CPU tensors
            (TypeError, lambda: g.keyed(ids16, torch.ones(2, dtype=torch.float64))),
            (TypeError, lambda: g.keyed(object(), f64)),
            (ValueError, lambda: g.keyed(ids16, HostArray([1.0]))),                          # lengths
            (TypeError, lambda: g.counters(ids16, HostArray([1.0, 2.0]))),                   # amount dtypes
            (TypeError, lambda: g.counters(ids16, HostArray([1, 2], np.uint32))),
            (TypeError, lambda: g.counters(HostArray([0, 1], np.float64), HostArray([1, 2], np.uint64))),
            (ValueError, lambda: g.counters(ids16, HostArray([1, 2, 3], np.uint64))),
            (KeyError, lambda: g.start_timer("c")),                                          # a counter's name
            (KeyError, lambda: g.stop_timer("nope")),
            (TypeError, lambda: g.stop_timer("a", out=HostArray([0.0]))),                    # out dtypes
            (TypeError, lambda: g.stop_timer("a", out=torch.zeros(1, dtype=torch.int64))),
        ]
        for exc, call in bad:
            with pytest.raises(exc):
                call()
        assert stub.lh_stub_graph_calls() == before
        # the C shim: a bad name index or id width throws in the mirror, before the library is called
        L, h = ms._lib, g._h
        assert L.lhms_graph_timer_start(h, 2, None) == LH_ERR_RANGE
        assert L.lhms_graph_timer_stop(h, 7, None, None) == LH_ERR_RANGE
        assert L.lhms_graph_keyed(h, 8, ids16.a.ctypes.data, f64.a.ctypes.data, 0, 2, None) == LH_ERR_STATE
        assert L.lhms_graph_counters(h, 1, ids16.a.ctypes.data, f64.a.ctypes.data, 2, None) == LH_ERR_STATE
        assert L.lhms_graph_keyed(None, 2, None, None, 0, 0, None) == LH_ERR_INVALID
        assert stub.lh_stub_graph_calls() == before
        # the library's own checks: the stub validates as the library does
        assert L.lhms_graph_keyed(h, 2, ids16.a.ctypes.data, f64.a.ctypes.data, 9, 2, None) == LH_ERR_STATE   # kind
        assert L.lhms_graph_keyed(h, 2, ids16.a.ctypes.data + 1, f64.a.ctypes.data, 0, 1, None) == LH_ERR_STATE
        assert L.lhms_graph_keyed(h, 2, ids16.a.ctypes.data, f64.a.ctypes.data, 0, 0, None) == 0             # n = 0
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {} and raw["Rates"] == {}
    with pytest.raises(RuntimeError, match="closed"):
        g.keyed(ids16, f64)
    with pytest.raises(RuntimeError, match="closed"):
        g.start_timer("a")
    assert ms.dropped() == 0


def test_mirror_over_a_library_without_the_calls(stub_libs, monkeypatch, oracle):
    """Bound weakly: over a C ABI that has graph recorders but not these calls, the mirror loads, the recorder works,
    and each new call reports an error instead of crashing."""
    import loghisto_b200.metric_system as m
    old, host = build_pair("_old", "lh_stub_graph.c")
    assert not hasattr(old, "lh_graph_recorder_timer_start")
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        with ms.graph_recorder(histograms=["a"], counters=["c"]) as g:
            ids, vals = HostArray([0], np.uint16), HostArray([1.0])
            for call in (lambda: g.keyed(ids, vals), lambda: g.keyed(HostArray([0], np.uint32), vals),
                         lambda: g.counters(ids, HostArray([1], np.uint64)), lambda: g.start_timer("a"),
                         lambda: g.stop_timer("a")):
                with pytest.raises(RuntimeError, match="status"):
                    call()
            g.histograms({"a": vals})
            raw, _ = ms.collect_and_process()
            assert raw["Histograms"] == {"a": {oracle.compress(1.0): 1}}
    finally:
        ms.close()


def test_new_entry_points_are_bound():
    """The six calls are in the header and in _lib.SIGNATURES, and the four lhms_graph_* wrappers in metric_system._bind."""
    import re
    from loghisto_b200 import _lib
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    calls = ["lh_graph_recorder_ingest_keyed_u16", "lh_graph_recorder_ingest_keyed_u32", "lh_graph_recorder_counter_add_u16",
             "lh_graph_recorder_counter_add_u32", "lh_graph_recorder_timer_start", "lh_graph_recorder_timer_stop"]
    for nm in calls:
        assert re.search(r"LH_API lh_status %s\(" % nm, hdr), nm
        assert nm in _lib.SIGNATURES, nm
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    assert sorted(re.findall(r"LHMS_API \w+ \*?(lhms_graph_(?!recorder_)\w+)\(", src)) == \
        ["lhms_graph_counters", "lhms_graph_keyed", "lhms_graph_timer_start", "lhms_graph_timer_stop"]
    for nm in calls:
        assert "#pragma weak " + nm in src, nm
