"""Graph recorders bound to names (MetricSystem::NewGraphRecorder, loghisto_b200/host/metric_system.cc) on the CPU: the
C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus tests/stub_abi/lh_stub_graph.c, whose
recorders drain the values recorded into them at every lh_graph_recorder_bind, the call the mirror makes for every open
recorder just before lh_snapshot_begin.  Covers the binding at each collection, the ids of a recorder's names while
names around it recycle, unbound names of a full table, the final drain of close(), and the Python argument checks.
tests/test_gpu_graph_recorder.py runs the real library."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
UNBOUND = 0xFFFFFFFF


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_graph.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_graph.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in
                    ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_graph.c")] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_graph", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    from loghisto_b200 import _lib
    s = ctypes.CDLL(stub)
    rp = ctypes.POINTER(_lib.lh_recorder)
    s.lh_stub_graph_record.argtypes = [rp, ctypes.c_uint32, ctypes.c_double]
    s.lh_stub_graph_record.restype = ctypes.c_int
    s.lh_stub_graph_count.argtypes = [rp, ctypes.c_uint32, ctypes.c_uint64]
    s.lh_stub_graph_count.restype = ctypes.c_int
    s.lh_stub_graph_alive.restype = ctypes.c_uint32
    s.lh_stub_graph_target.argtypes = [rp, ctypes.c_uint32, ctypes.c_int]
    s.lh_stub_graph_target.restype = ctypes.c_uint32
    return s, host


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    stub, host = stub_libs
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
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


def record(stub, g, name, v, reps=1):
    for _ in range(reps):
        assert stub.lh_stub_graph_record(ctypes.byref(g.recorder), g.histogram_ids[name], v) == 0


def count(stub, g, name, amount):
    assert stub.lh_stub_graph_count(ctypes.byref(g.recorder), g.counter_ids[name], amount) == 0


class HostArray:
    """n float64 / int64 values in host memory, posing as a device array (the stub reads host pointers)."""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a)
        self.__cuda_array_interface__ = {"shape": (self.a.size,), "typestr": self.a.dtype.str,
                                         "data": (self.a.ctypes.data, False), "version": 3}


def test_counts_are_labelled_with_the_recorders_names(MS, stub, oracle):
    ms = MS()
    with ms.graph_recorder(histograms=["lat", "size"], counters=["reqs"]) as g:
        assert g.histogram_ids == {"lat": 0, "size": 1} and g.counter_ids == {"reqs": 0}
        assert g.recorder.max_histograms == 2 and g.recorder.max_counters == 1
        record(stub, g, "lat", 7.0, 3)
        record(stub, g, "size", -2.5)
        count(stub, g, "reqs", 11)
        count(stub, g, "reqs", 4)
        ms.Histogram("host", 1.0)
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {"lat": {oracle.compress(7.0): 3}, "size": {oracle.compress(-2.5): 1},
                                     "host": {oracle.compress(1.0): 1}}
        assert raw["Rates"] == {"reqs": 15}
        raw, _ = ms.collect_and_process()           # nothing recorded since: nothing drained
        assert raw["Histograms"] == {} and raw["Rates"] == {}
        g.histograms({"size": HostArray([1.0, 2.0]), "lat": HostArray(np.array([5], dtype=np.int64))})
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {"size": {oracle.compress(1.0): 1, oracle.compress(2.0): 1},
                                     "lat": {oracle.compress(5.0): 1}}
    assert ms.dropped() == 0


def test_names_keep_their_ids_while_others_recycle(MS, stub, oracle):
    """A new host name every interval with one id to spare beyond the recorder's and the two intervals a name holds
    its id after its last use: ids recycle around the recorder, whose name keeps its id and its counts every interval."""
    ms = MS(max_histograms=4)
    with ms.graph_recorder(histograms=["g"]) as g:
        first = stub.lh_stub_graph_target(ctypes.byref(g.recorder), 0, 0)
        assert first != UNBOUND
        for it in range(12):
            ms.Histogram("churn%d" % it, 3.0)
            record(stub, g, "g", float(it + 1))
            raw, _ = ms.collect_and_process()
            assert raw["Histograms"] == {"g": {oracle.compress(float(it + 1)): 1},
                                         "churn%d" % it: {oracle.compress(3.0): 1}}, it
            assert stub.lh_stub_graph_target(ctypes.byref(g.recorder), 0, 0) == first
    assert ms.dropped() == 0


def test_full_table_drops_exactly_the_drained_samples(MS, stub, oracle):
    """No free id at creation and at the collection: the name is unbound there and its drained samples are dropped and
    counted, the other names unaffected.  Once an id is free, a later collection binds the name again."""
    ms = MS(max_histograms=2)
    ms.Histogram("a", 1.0)
    ms.Histogram("b", 1.0)
    with ms.graph_recorder(histograms=["late"]) as g:
        assert stub.lh_stub_graph_target(ctypes.byref(g.recorder), 0, 0) == UNBOUND
        record(stub, g, "late", 9.0, 5)
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {"a": {oracle.compress(1.0): 1}, "b": {oracle.compress(1.0): 1}}
        assert ms.dropped() == 5
        for _ in range(3):                          # a and b idle: their ids free up
            ms.collect_and_process()
        record(stub, g, "late", 9.0, 2)
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {"late": {oracle.compress(9.0): 2}}
        assert ms.dropped() == 5


def test_close_drains_leftovers_into_the_next_collection(MS, stub, oracle):
    ms = MS()
    with ms.graph_recorder(histograms=["x"], counters=["c"]) as g:
        record(stub, g, "x", 4.0, 2)
        count(stub, g, "c", 6)
    assert stub.lh_stub_graph_alive() == 0
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"x": {oracle.compress(4.0): 2}} and raw["Rates"] == {"c": 6}
    g.close()                                       # idempotent


def test_two_recorders_share_a_name(MS, stub, oracle):
    ms = MS()
    with ms.graph_recorder(histograms=["s", "t"]) as g1, ms.graph_recorder(histograms=["s"]) as g2:
        assert stub.lh_stub_graph_target(ctypes.byref(g1.recorder), 0, 0) == \
            stub.lh_stub_graph_target(ctypes.byref(g2.recorder), 0, 0)
        record(stub, g1, "s", 2.0, 2)
        record(stub, g2, "s", 2.0, 3)
        record(stub, g1, "t", 8.0)
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {"s": {oracle.compress(2.0): 5}, "t": {oracle.compress(8.0): 1}}


def test_python_argument_checks(MS, stub):
    """Unknown names, host tensors, other dtypes: refused before anything is issued; a closed recorder raises."""
    import torch
    ms = MS()
    with ms.graph_recorder(histograms=["x"]) as g:
        with pytest.raises(KeyError):
            g.histograms({"nope": HostArray([1.0])})
        with pytest.raises(TypeError):
            g.histograms({"x": torch.ones(3, dtype=torch.float64)})      # a CPU tensor
        with pytest.raises(TypeError):
            g.histograms({"x": HostArray(np.ones(3, dtype=np.float32))})
        with pytest.raises(TypeError):
            g.histograms({"x": object()})
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {}
    with pytest.raises(RuntimeError):
        g.histograms({"x": HostArray([1.0])})
    with pytest.raises(RuntimeError, match="status"):
        with ms.graph_recorder(histograms=["a", "b", "c", "d", "e"]):     # more names than max_histograms
            pass


def test_graph_recorder_entry_points_are_bound(stub_libs):
    """Every lhms_graph_recorder_* entry point of the C shim is declared by metric_system._bind, and every
    lh_graph_recorder_* call of the header by _lib.SIGNATURES."""
    import loghisto_b200.metric_system as m
    from loghisto_b200 import _lib
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    names = re.findall(r"LHMS_API \w+ \*?(lhms_graph_recorder_\w+)\(", src)
    assert sorted(names) == ["lhms_graph_recorder_close", "lhms_graph_recorder_free", "lhms_graph_recorder_histograms",
                             "lhms_graph_recorder_new"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    for nm in re.findall(r"LH_API lh_status (lh_graph_recorder_\w+)\(", hdr):
        assert nm in _lib.SIGNATURES, nm
    assert ctypes.sizeof(_lib.lh_graph_recorder) == 8 + ctypes.sizeof(_lib.lh_recorder)
