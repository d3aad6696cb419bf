"""Keyed samples and counter adds of record scopes (RecordScope.keyed / counters) on the CPU: the Python layer and the
C++ mirror over the TEST-ONLY oracle-backed stub of the C ABI (tests/stub_abi/lh_stub_scope_keyed.c, which applies the
scope's map on the host).  Covers local id -> name and dtype -> entry point mapping, drops under unbound names and ids
past the names, duplicate names, a scope without names, every error raised before the ABI is called, and a mirror
loaded over a stub that lacks the calls.  tests/test_gpu_scope_keyed.py runs the real library."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUBS = ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c")
CALLS = ["lh_ingest_keyed_mapped_u16", "lh_ingest_keyed_mapped_u32", "lh_counter_add_mapped_u16", "lh_counter_add_mapped_u32"]


def build_pair(tag, stub_src):
    stub = os.path.join(BUILD, "liblh_stub_scope_keyed%s.so" % tag)
    host = os.path.join(BUILD, "libloghisto_host_stub_scope_keyed%s.so" % tag)
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in STUBS + (stub_src,)] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_scope_keyed%s" % tag, "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return ctypes.CDLL(stub), host


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    s, host = build_pair("", "lh_stub_scope_keyed.c")
    s.lh_stub_mapped_calls.restype = ctypes.c_uint64
    return s, host


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    made = []

    def make(max_histograms=4, max_counters=4):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=max_counters)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


class HostArray:
    """A host numpy array posing as a device array (the stub reads host pointers)."""

    def __init__(self, a, dtype=None, offset_bytes=0):
        self.a = np.ascontiguousarray(a, dtype=dtype)
        n = self.a.size - (1 if offset_bytes else 0)          # a shifted view keeps inside the buffer
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": self.a.dtype.str,
                                         "data": (self.a.ctypes.data + offset_bytes, False), "version": 3}


def want_hist(oracle, vals):
    out = {}
    for v in vals:
        k = oracle.compress(float(v))
        out[k] = out.get(k, 0) + 1
    return out


@pytest.mark.parametrize("id_dtype", [np.uint16, np.int32, np.uint32])
@pytest.mark.parametrize("val_dtype", [np.float64, np.int64])
def test_keyed_samples_land_under_the_names_of_their_local_ids(MS, oracle, id_dtype, val_dtype):
    """Local id i is the scope's histogram name i; ids past the names (a negative int32 among them) are dropped and
    counted.  65536 + 1 and 2^31 would read as other ids through the 16-bit entry point, so they pin the mapping."""
    ms = MS()
    ids = [0, 1, 1, 2, 7, 0]
    if id_dtype is np.int32:
        ids += [-1]
    if id_dtype is np.uint32:
        ids += [65536 + 1, 2 ** 31]
    vals = np.arange(1, len(ids) + 1, dtype=val_dtype) * 3
    with ms.recording(histograms=["a", "b"]) as s:
        s.keyed(HostArray(ids, id_dtype), HostArray(vals))
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"a": want_hist(oracle, [vals[0], vals[5]]), "b": want_hist(oracle, vals[1:3])}
    assert ms.dropped() == len(ids) - 4


@pytest.mark.parametrize("id_dtype", [np.uint16, np.uint32])
@pytest.mark.parametrize("amt_dtype", [np.uint64, np.int64])
def test_counter_adds_wrap_and_drop(MS, id_dtype, amt_dtype):
    ms = MS()
    amounts = np.array([2 ** 64 - 5, 9, 3, 11, 4], dtype=np.uint64)
    ids = np.array([0, 0, 1, 2, 1], dtype=id_dtype)
    with ms.recording(counters=["x", "y"]) as s:
        s.counters(HostArray(ids), HostArray(amounts.view(amt_dtype)))
    raw, _ = ms.collect_and_process()
    assert raw["Counters"] == {"x": 4, "y": 7}
    assert ms.dropped() == 1


def test_unbound_names_and_duplicates(MS, oracle):
    """With two ids for three names, the third name is unbound: its samples and ops are dropped and counted one each.
    A repeated name maps two local ids to one row."""
    ms = MS(max_histograms=2, max_counters=2)
    with ms.recording(histograms=["a", "b", "c", "a"], counters=["x", "y", "z", "x"]) as s:
        assert s.histogram_ids["c"] == s.UNBOUND
        s.keyed(HostArray([0, 2, 2, 3, 1, 4], np.uint16), HostArray([1.0, 2.0, 3.0, 4.0, 5.0, 6.0]))
        s.counters(HostArray([0, 2, 3, 1, 9], np.uint32), HostArray([1, 2, 3, 4, 5], np.uint64))
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"a": want_hist(oracle, [1.0, 4.0]), "b": want_hist(oracle, [5.0])}
    assert raw["Counters"] == {"x": 4, "y": 4}
    assert ms.dropped() == 3 + 2


def test_scope_without_names_drops_everything(MS):
    ms = MS()
    with ms.recording() as s:
        s.keyed(HostArray([0, 1], np.uint16), HostArray([1.0, 2.0]))
        s.counters(HostArray([0], np.uint16), HostArray([5], np.uint64))
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {} and raw["Counters"] == {}
    assert ms.dropped() == 3


def test_errors_are_raised_before_anything_is_issued(MS, stub):
    ms = MS()
    ids, vals = HostArray([0, 1], np.uint16), HostArray([1.0, 2.0])
    before = stub.lh_stub_mapped_calls()
    with ms.recording(histograms=["a", "b"], counters=["x"]) as s:
        with pytest.raises(TypeError):
            s.keyed(HostArray([0, 1], np.int64), vals)                  # id dtype
        with pytest.raises(TypeError):
            s.keyed(ids, HostArray([1.0, 2.0], np.float32))             # value dtype
        with pytest.raises(ValueError):
            s.keyed(ids, HostArray([1.0]))                              # lengths
        with pytest.raises(TypeError):
            s.counters(ids, HostArray([1.0, 2.0]))                      # amount dtype
        with pytest.raises(RuntimeError):
            s.keyed(ids, HostArray(np.zeros(3), offset_bytes=4))        # misaligned values (library refuses)
        with pytest.raises(RuntimeError):
            s.keyed(HostArray([0, 1, 2], np.uint32, offset_bytes=2), vals)   # misaligned ids
        with pytest.raises(RuntimeError):
            s.counters(ids, HostArray(np.zeros(3, np.uint64), offset_bytes=4))
    with pytest.raises(RuntimeError):
        s.keyed(ids, vals)                                              # after end()
    with pytest.raises(RuntimeError):
        s.counters(ids, HostArray([1, 2], np.uint64))
    assert stub.lh_stub_mapped_calls() == before
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {} and ms.dropped() == 0


def test_abi_validation(stub):
    """The stub's validation, as the header states it: k > 4096 and a NULL map are invalid, an entry past the table
    other than LH_GRAPH_UNBOUND is out of range, an unknown kind is invalid."""
    stub.lh_create.restype = ctypes.c_int
    from loghisto_b200 import _lib
    cfg = _lib.lh_config()
    cfg.struct_size = ctypes.sizeof(cfg)
    cfg.max_histograms, cfg.max_counters = 4, 4
    ctx = ctypes.c_void_p()
    assert stub.lh_create(ctypes.byref(cfg), ctypes.byref(ctx)) == 0
    fn = stub.lh_ingest_keyed_mapped_u16
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32,
                   ctypes.c_size_t, ctypes.c_void_p]
    ids, vals = np.zeros(1, np.uint16), np.ones(1)
    m = (ctypes.c_uint32 * 4097)(*([0] * 4097))
    assert fn(ctx, m, 4097, ids.ctypes.data, vals.ctypes.data, 0, 1, None) == -1
    assert fn(ctx, None, 1, ids.ctypes.data, vals.ctypes.data, 0, 1, None) == -1
    assert fn(ctx, (ctypes.c_uint32 * 1)(4), 1, ids.ctypes.data, vals.ctypes.data, 0, 1, None) == -6
    assert fn(ctx, (ctypes.c_uint32 * 1)(0xFFFFFFFF), 1, ids.ctypes.data, vals.ctypes.data, 0, 1, None) == 0
    assert fn(ctx, (ctypes.c_uint32 * 1)(3), 1, ids.ctypes.data, vals.ctypes.data, 2, 1, None) == -1
    stub.lh_destroy(ctx)


def test_bindings_and_weak_symbols(stub_libs):
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    for nm in CALLS:
        assert re.search(r"LH_API lh_status %s\(" % nm, hdr), nm
        assert nm in _lib.SIGNATURES, nm
        assert "#pragma weak " + nm in src, nm
    names = re.findall(r"LHMS_API [\w *]+?(lhms_scoped_\w+)\(", src)
    assert names == ["lhms_scoped_keyed", "lhms_scoped_counters"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm


def test_mirror_over_a_stub_without_the_calls(monkeypatch):
    """The new symbols are weak: over a C ABI without them the mirror links and loads, and the calls refuse."""
    import loghisto_b200.metric_system as m
    _, host = build_pair("_old", "lh_stub_graph_calls.c")
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        with ms.recording(histograms=["a"], counters=["x"]) as s:
            with pytest.raises(RuntimeError):
                s.keyed(HostArray([0], np.uint16), HostArray([1.0]))
            with pytest.raises(RuntimeError):
                s.counters(HostArray([0], np.uint16), HostArray([1], np.uint64))
        raw, _ = ms.collect_and_process()
        assert raw["Histograms"] == {} and ms.dropped() == 0
    finally:
        ms.close()
