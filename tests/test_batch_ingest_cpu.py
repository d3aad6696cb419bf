"""Batch ingest (lh_ingest_batch) above the C ABI, on the CPU: Engine.ingest_batch, RecordScope::Histograms
(RecordScope.histograms in Python) and lhms_scope_histograms, over the TEST-ONLY oracle-backed stub of the C ABI plus
tests/stub_abi/lh_stub_batch.c.  Covers name binding and the drop-and-count of unbound names, the mapping from status
codes to exceptions, the Python dtype / device / contiguity checks and the marshalling of items.
tests/test_gpu_batch_ingest.py runs the real library."""
import ctypes
import os
import re
import subprocess
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUB = os.path.join(ROOT, "tests", "stub_abi")
HOST_SRCS = [os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
             os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc")]
F64, I64NS = 0, 1


def _build_pair(stub, host, with_batch=True):
    srcs = ["lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c"] + (["lh_stub_batch.c"] if with_batch else [])
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC]
                   + [os.path.join(STUB, s) for s in srcs]
                   + [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC]
                   + HOST_SRCS + ["-o", host, "-L", os.path.dirname(stub), "-l" + os.path.basename(stub)[3:-3],
                                  "-Wl,-rpath," + os.path.dirname(stub), "-lpthread"], check=True)


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_batch.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_batch.so")
    _build_pair(stub, host)
    s = ctypes.CDLL(stub)
    s.lh_stub_batch_calls.restype = ctypes.c_uint64
    s.lh_stub_batch_last.restype = ctypes.c_uint32
    return s, host


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


def last_call(stub):
    """(items as (address, n, id, kind) tuples, stream) of the latest lh_ingest_batch the stub saw."""
    from loghisto_b200 import _lib
    out = (_lib.lh_batch_item * 4096)()
    stream = ctypes.c_void_p()
    n = stub.lh_stub_batch_last(out, 4096, ctypes.byref(stream))
    return [(out[i].d_values or 0, out[i].n, out[i].histogram_id, out[i].kind) for i in range(n)], stream.value


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    made = []

    def make(max_histograms=4):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=4)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


@pytest.fixture
def engine(stub, monkeypatch):
    """An Engine over the stub: the ctypes binding of every entry point the stub has."""
    from loghisto_b200 import _lib, engine as E
    for name, (res, args) in _lib.SIGNATURES.items():
        if hasattr(stub, name):
            getattr(stub, name).restype = res
            getattr(stub, name).argtypes = args
    monkeypatch.setattr(_lib, "_lib", stub)
    e = E.Engine(max_histograms=5)
    yield e
    e.close()


class HostArray:
    """A host numpy array presented as device memory (__cuda_array_interface__): the stub reads host pointers."""

    def __init__(self, a, typestr=None, strides=None):
        self.a = a
        self.__cuda_array_interface__ = {"shape": a.shape, "typestr": typestr or a.dtype.str,
                                         "data": (a.ctypes.data, False), "version": 3, "strides": strides}


def dense_of(raw_hist):
    d = np.zeros(65536, np.uint64)
    for k, c in raw_hist.items():
        d[k & 0xFFFF] = c
    return d


def test_scope_histograms_bind_names_and_match_the_oracle(MS, stub, oracle):
    ms = MS()
    a = oracle.gen_stream(oracle.STREAM_S, 1000, 1)
    b = oracle.gen_stream(oracle.STREAM_L, 77, 2)
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, 300, 3).view(np.int64).copy()
    ns[::7] = np.resize(np.array([-5, 0, np.iinfo(np.int64).min, np.iinfo(np.int64).max, 12345], np.int64), ns[::7].size)
    calls = stub.lh_stub_batch_calls()
    with ms.recording(None, histograms=["a", "b", "ns"]) as s:
        ids = s.histogram_ids
        s.histograms({"a": HostArray(a), "b": HostArray(b), "ns": HostArray(ns)})
        items, stream = last_call(stub)
        assert items == [(a.ctypes.data, 1000, ids["a"], F64), (b.ctypes.data, 77, ids["b"], F64),
                         (ns.ctypes.data, 300, ids["ns"], I64NS)]
        assert stream is None
        s.histograms([("a", HostArray(a[:10])), ("a", HostArray(b))])       # a name may repeat
    assert stub.lh_stub_batch_calls() == calls + 2
    raw, m = ms.collect_and_process()
    assert (dense_of(raw["Histograms"]["a"]) == oracle.ingest(np.concatenate([a, a[:10], b]))).all()
    assert (dense_of(raw["Histograms"]["b"]) == oracle.ingest(b)).all()
    assert (dense_of(raw["Histograms"]["ns"]) == oracle.ingest(ns.astype(np.float64))).all()
    assert m["a_count"] == 1087 and m["ns_count"] == 300
    assert ms.dropped() == 0


def test_unbound_names_are_dropped_and_counted(MS, stub):
    ms = MS(max_histograms=2)
    for nm in ("x", "y"):
        ms.Histogram(nm, 1.0)
    v = np.arange(1, 40, dtype=np.float64)
    n = np.arange(5, dtype=np.int64)
    with ms.recording(None, histograms=["late", "x"]) as s:
        assert s.histogram_ids["late"] == s.UNBOUND
        s.histograms([("late", HostArray(v)), ("x", HostArray(v[:4])), ("late", HostArray(n))])
        items, _ = last_call(stub)
        assert items == [(v.ctypes.data, 4, s.histogram_ids["x"], F64)]
        s.histograms({"late": HostArray(v)})                                 # nothing bound: an empty call
        assert last_call(stub)[0] == []
    assert ms.dropped() == 39 + 5 + 39
    raw, m = ms.collect_and_process()
    assert "late" not in raw["Histograms"] and m["x_count"] == 5


def test_scope_errors(MS, stub):
    ms = MS()
    v = np.arange(1, 9, dtype=np.float64)
    calls = stub.lh_stub_batch_calls()
    with ms.recording(None, histograms=["a"]) as s:
        with pytest.raises(KeyError):
            s.histograms({"zz": HostArray(v)})
        with pytest.raises(TypeError):
            s.histograms({"a": HostArray(v.astype(np.float32))})
        with pytest.raises(TypeError):
            s.histograms({"a": v})                                            # host memory
        odd = types.SimpleNamespace(__cuda_array_interface__={"shape": (3,), "typestr": "<f8",
                                                              "data": (v.ctypes.data + 4, False), "version": 3})
        with pytest.raises(RuntimeError, match="status"):                    # refused by the library: misaligned
            s.histograms({"a": odd})
        assert ms._lib.lhms_scope_histograms(ms._h, ctypes.byref(s.recorder), (ctypes.c_uint32 * 1)(5),
                                                (ctypes.c_void_p * 1)(v.ctypes.data), (ctypes.c_uint64 * 1)(1),
                                                (ctypes.c_uint32 * 1)(F64), 1) == -6   # bad name index: LH_ERR_RANGE
    assert stub.lh_stub_batch_calls() == calls
    assert ms.dropped() == 0
    scope = s.recorder
    assert ms._lib.lhms_scope_histograms(ms._h, ctypes.byref(scope), None, None, None, None, 0) == -1   # ended


def test_engine_marshalling_and_status(engine, stub, oracle):
    e = engine
    a = oracle.gen_stream(oracle.STREAM_U, 500, 4)
    ns = np.array([3, -3, 0, 1 << 40], np.int64)
    e.ingest_batch([(0, HostArray(a)), (4, HostArray(ns)), (2, HostArray(a[:0])), (0, HostArray(a[7:9]))],
                   stream=types.SimpleNamespace(cuda_stream=0x7000))
    items, stream = last_call(stub)
    assert items == [(a.ctypes.data, 500, 0, F64), (ns.ctypes.data, 4, 4, I64NS), (a.ctypes.data, 0, 2, F64),
                     (a[7:].ctypes.data, 2, 0, F64)]
    assert stream == 0x7000
    red, sp = e.snapshot([0.5])
    assert sum(sp.histogram(0).values()) == 502 and sum(sp.histogram(4).values()) == 4
    assert int(red.counts[4]) == 4 and int(red.counts[0]) == 502
    from loghisto_b200 import LhError, _lib
    with pytest.raises(LhError) as ex:
        e.ingest_batch([(0, HostArray(a)), (5, HostArray(a))])
    assert ex.value.status == _lib.LH_ERR_RANGE
    odd = types.SimpleNamespace(__cuda_array_interface__={"shape": (3,), "typestr": "<f8",
                                                          "data": (a.ctypes.data + 4, False), "version": 3})
    with pytest.raises(LhError) as ex:
        e.ingest_batch([(1, odd)])
    assert ex.value.status == _lib.LH_ERR_INVALID
    with pytest.raises(ValueError):
        e.ingest_batch([(-1, HostArray(a))])
    e.ingest_batch([])
    assert last_call(stub)[0] == []
    assert e.snapshot([0.5])[0].counts.sum() == 0


def test_array_checks():
    from loghisto_b200.engine import DeviceArray, _batch_array

    def tensor(**kw):
        t = dict(is_cuda=True, data_ptr=lambda: 4096, is_contiguous=lambda: True, dtype="torch.float64",
                 numel=lambda: 6)
        t.update(kw)
        return types.SimpleNamespace(**t)
    assert _batch_array(tensor()) == (4096, 6, F64)
    assert _batch_array(tensor(dtype="torch.int64")) == (4096, 6, I64NS)
    for bad in (tensor(is_cuda=False), tensor(is_contiguous=lambda: False), tensor(dtype="torch.float32"),
                tensor(dtype="torch.int32"), tensor(dtype="torch.uint64")):
        with pytest.raises(TypeError):
            _batch_array(bad)
    a = np.zeros((3, 4), np.float64)
    assert _batch_array(HostArray(a)) == (a.ctypes.data, 12, F64)
    assert _batch_array(HostArray(a, strides=(32, 8))) == (a.ctypes.data, 12, F64)
    assert _batch_array(HostArray(a.astype(np.int64)))[2] == I64NS
    for bad in (HostArray(a, strides=(8, 24)), HostArray(a, typestr=">f8"), HostArray(a.astype(np.float32)),
                HostArray(a.astype(np.uint64)), a, 4096, None):
        with pytest.raises(TypeError):
            _batch_array(bad)
    d = DeviceArray.__new__(DeviceArray)
    d.dtype, d.ptr, d.n = np.dtype(np.int64), 8192, 9
    assert _batch_array(d) == (8192, 9, I64NS)
    d.dtype = np.dtype(np.uint16)
    with pytest.raises(TypeError):
        _batch_array(d)
    d.ptr = 0


def test_batch_item_layout_and_bindings(tmp_path, stub_libs):
    """lh_batch_item as a C compiler lays it out, the ctypes mirror, and the binding of lhms_scope_histograms."""
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    c = tmp_path / "layout.c"
    fields = [f for f, _ in _lib.lh_batch_item._fields_]
    c.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"',
                            'int main(void) { printf("%zu", sizeof(lh_batch_item));']
                           + ['printf(" %%zu", offsetof(lh_batch_item, %s));' % f for f in fields]
                           + ['printf(" %d %d\\n", LH_VALUES_F64, LH_VALUES_I64NS); return 0; }']))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", INC, "-o", str(exe), str(c)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[0] == ctypes.sizeof(_lib.lh_batch_item) == 24
    assert got[1:1 + len(fields)] == [getattr(_lib.lh_batch_item, f).offset for f in fields]
    assert got[-2:] == [_lib.LH_VALUES_F64, _lib.LH_VALUES_I64NS]
    src = open(HOST_SRCS[0]).read()
    names = re.findall(r"LHMS_API [\w *]+?(lhms_scope_\w+)\(", src)
    assert names == ["lhms_scope_histograms"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm


def test_host_library_loads_over_a_stub_without_batch_ingest(tmp_path, monkeypatch):
    """lh_ingest_batch is weak in the mirror: over a C ABI without it the host library still links and loads, and
    RecordScope::Histograms refuses (LH_ERR_STATE from the C shim) without dropping anything."""
    stub, host = str(tmp_path / "liblh_stub_nobatch.so"), str(tmp_path / "libhost_nobatch.so")
    _build_pair(stub, host, with_batch=False)
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        v = np.ones(3)
        with ms.recording(None, histograms=["a"]) as s:
            with pytest.raises(RuntimeError, match="status -5"):
                s.histograms({"a": HostArray(v)})
        assert ms.dropped() == 0
    finally:
        ms.close()
