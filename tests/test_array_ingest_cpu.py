"""Ingest of device arrays of any gauge dtype (lh_ingest_arrays) above the C ABI, on the CPU: RecordScope::Arrays
(RecordScope.arrays in Python), lhms_arrays_scope and Engine.ingest_arrays, over the TEST-ONLY oracle-backed stub of
the C ABI plus tests/stub_abi/lh_stub_ingest_arrays.c.  Covers name binding and the drop-and-count of unbound names,
status codes to exceptions, the TypeError / KeyError checks made before any call, a library without the call, and the
marshalling of items.  tests/test_gpu_array_ingest.py runs the real library."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUB = os.path.join(ROOT, "tests", "stub_abi")
HOST_SRCS = [os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
             os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc")]
F64, F32, F16, BF16, I64, I32, U64 = range(7)
NP = {F64: np.float64, F32: np.float32, F16: np.float16, BF16: np.uint16, I64: np.int64, I32: np.int32, U64: np.uint64}
TORCH_NAME = {F64: "torch.float64", F32: "torch.float32", F16: "torch.float16", BF16: "torch.bfloat16",
              I64: "torch.int64", I32: "torch.int32", U64: "torch.uint64"}


def _build_pair(tag, with_arrays):
    """The stub (with lh_stub_graph.c's graph recorders and, unless with_arrays is false, lh_stub_ingest_arrays.c) and the
    host mirror over it."""
    stub = os.path.join(BUILD, "liblh_stub_arrays%s.so" % tag)
    host = os.path.join(BUILD, "libloghisto_host_stub_arrays%s.so" % tag)
    srcs = ["lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_graph.c"] + \
        (["lh_stub_ingest_arrays.c"] if with_arrays else [])
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC]
                   + [os.path.join(STUB, s) for s in srcs]
                   + [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC]
                   + HOST_SRCS + ["-o", host, "-L", os.path.dirname(stub), "-l" + os.path.basename(stub)[3:-3],
                                  "-Wl,-rpath," + os.path.dirname(stub), "-lpthread"], check=True)
    return stub, host


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub, host = _build_pair("", True)
    s = ctypes.CDLL(stub)
    s.lh_stub_arrays_calls.restype = ctypes.c_uint64
    s.lh_stub_arrays_last.restype = ctypes.c_uint32
    return s, host


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


def last_call(stub):
    from loghisto_b200 import _lib
    out = (_lib.lh_array_src * 4096)()
    stream = ctypes.c_void_p()
    n = stub.lh_stub_arrays_last(out, 4096, ctypes.byref(stream))
    return [(out[i].d_values or 0, out[i].n, out[i].dtype, out[i].histogram_id) for i in range(n)], stream.value


def _ms_factory(host, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    made = []

    def make(max_histograms=4):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=4)
        made.append(ms)
        return ms
    return make, made


@pytest.fixture
def MS(stub_libs, monkeypatch):
    make, made = _ms_factory(stub_libs[1], monkeypatch)
    yield make
    for ms in made:
        ms.close()


class FakeCudaTensor:
    """A host numpy array presented as a contiguous CUDA tensor on device 0 (the stub reads host pointers)."""

    class _Dev:
        index = 0

    def __init__(self, a, dtype, contiguous=True, cuda=True, byte_offset=0):
        self.a, self.is_cuda, self._contig, self._off = a, cuda, contiguous, byte_offset
        self.device = self._Dev()
        self.dtype = TORCH_NAME.get(dtype, dtype)

    def is_contiguous(self):
        return self._contig

    def data_ptr(self):
        return self.a.ctypes.data + self._off

    def numel(self):
        return self.a.size


def values(oracle, dtype, n, seed):
    v = oracle.gen_stream(oracle.STREAM_S, n, seed)
    v[::3] *= -1
    if dtype in (F64, F32, F16):
        with np.errstate(over="ignore"):
            return v.astype(NP[dtype])
    if dtype == BF16:
        return np.arange(n, dtype=np.uint32).astype(np.uint16) * np.uint16(37)
    return np.resize(np.array([0, 1, -1, 2 ** 31 - 1, -2 ** 31, 12345], np.int64), n).astype(NP[dtype]) if dtype != U64 \
        else np.resize(np.array([0, 1, 2 ** 64 - 1, 2 ** 63 + 1025, 2 ** 53 + 1], np.uint64), n)


def as_f64(a, dtype):
    if dtype == BF16:
        return (a.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return a.astype(np.float64)


def dense_of(raw_hist):
    d = np.zeros(65536, np.uint64)
    for k, c in raw_hist.items():
        d[k & 0xFFFF] = c
    return d


def test_scope_arrays_bind_names_and_match_the_oracle(MS, stub, oracle):
    ms = MS(max_histograms=8)
    arrs = {dt: values(oracle, dt, 100 + dt, dt) for dt in range(7)}
    names = ["h%d" % dt for dt in range(7)]
    calls = stub.lh_stub_arrays_calls()
    with ms.recording(None, histograms=names) as s:
        ids = s.histogram_ids
        s.arrays({"h%d" % dt: FakeCudaTensor(a, dt) for dt, a in arrs.items()})
        items, stream = last_call(stub)
        assert items == [(a.ctypes.data, a.size, dt, ids["h%d" % dt]) for dt, a in arrs.items()]
        assert stream is None
        s.arrays([("h1", FakeCudaTensor(arrs[F32][:5], F32)), ("h1", FakeCudaTensor(arrs[F32], F32))])
    assert stub.lh_stub_arrays_calls() == calls + 2
    raw, _ = ms.collect_and_process()
    for dt, a in arrs.items():
        want = oracle.ingest(as_f64(a, dt))
        if dt == F32:
            want = want + oracle.ingest(as_f64(a[:5], dt)) + oracle.ingest(as_f64(a, dt))
        assert (dense_of(raw["Histograms"]["h%d" % dt]) == want).all(), dt


def test_refusals_before_any_call(MS, stub):
    ms = MS()
    a = np.ones(8, np.float32)
    calls = stub.lh_stub_arrays_calls()
    last = last_call(stub)
    with ms.recording(None, histograms=["x"]) as s:
        with pytest.raises(KeyError):
            s.arrays([("x", FakeCudaTensor(a, F32)), ("y", FakeCudaTensor(a, F32))])
        for bad in (FakeCudaTensor(a, F32, cuda=False), FakeCudaTensor(a, F32, contiguous=False),
                    FakeCudaTensor(a, "torch.int16"), a):
            with pytest.raises(TypeError):
                s.arrays([("x", FakeCudaTensor(a, F32)), ("x", bad)])
    assert stub.lh_stub_arrays_calls() == calls and last_call(stub) == last


def test_library_refusals_become_runtime_errors(MS, stub):
    ms = MS()
    a = np.ones(16, np.float32)
    with ms.recording(None, histograms=["x"]) as s:
        with pytest.raises(RuntimeError):   # LH_ERR_INVALID: not 4-byte aligned
            s.arrays({"x": FakeCudaTensor(a[:8], F32, byte_offset=2)})


def test_unbound_names_are_dropped_and_counted(MS, stub, oracle):
    ms = MS(max_histograms=2)
    a = np.arange(1, 11, dtype=np.int32)
    with ms.recording(None, histograms=["a", "b", "c"]) as s:
        unbound = [nm for nm, i in s.histogram_ids.items() if i == 0xFFFFFFFF]
        s.arrays([(nm, FakeCudaTensor(a, I32)) for nm in ("a", "b", "c")])
        items, _ = last_call(stub)
        assert len(items) == 3 - len(unbound)
    assert len(unbound) == 1 and ms.dropped() == 10


def test_shim_from_c(stub_libs, MS, oracle):
    """lhms_arrays_scope called as a C caller would: parallel arrays of name indices, pointers, lengths and dtypes."""
    ms = MS()
    host = ctypes.CDLL(stub_libs[1])
    a = np.array([1.5, -2.0, 3e9], np.float32)
    with ms.recording(None, histograms=["p", "q"]) as s:
        idx = (ctypes.c_uint32 * 1)(1)
        ptrs = (ctypes.c_void_p * 1)(a.ctypes.data)
        ns = (ctypes.c_uint64 * 1)(3)
        dts = (ctypes.c_uint32 * 1)(F32)
        fn = host.lhms_arrays_scope
        fn.restype = ctypes.c_int
        assert fn(ms._h, ctypes.byref(s.recorder), idx, ptrs, ns, dts, 1) == 0
        bad = (ctypes.c_uint32 * 1)(9)
        assert fn(ms._h, ctypes.byref(s.recorder), idx, ptrs, ns, bad, 1) != 0
        assert fn(ms._h, ctypes.byref(s.recorder), None, ptrs, ns, dts, 1) != 0
    raw, _ = ms.collect_and_process()
    assert (dense_of(raw["Histograms"]["q"]) == oracle.ingest(a.astype(np.float64))).all()


def test_library_without_the_call(monkeypatch):
    _, host = _build_pair("_without", False)
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        with ms.recording(None, histograms=["x"]) as s:
            with pytest.raises(RuntimeError):
                s.arrays({"x": FakeCudaTensor(np.ones(4, np.float32), F32)})
        with ms.graph_recorder(histograms=["g"]) as g:
            with pytest.raises(RuntimeError):
                g.arrays({"g": FakeCudaTensor(np.ones(4, np.float32), F32)})
    finally:
        ms.close()


def test_engine_ingest_arrays_marshals_items(stub, monkeypatch, oracle):
    from loghisto_b200 import _lib, engine as E
    for name, (res, args) in _lib.SIGNATURES.items():
        if hasattr(stub, name):
            getattr(stub, name).restype = res
            getattr(stub, name).argtypes = args
    monkeypatch.setattr(_lib, "_lib", stub)
    e = E.Engine(max_histograms=5)
    try:
        h = values(oracle, F16, 33, 1)
        b = values(oracle, BF16, 20, 2)
        e.ingest_arrays([(4, FakeCudaTensor(h, F16)), (0, FakeCudaTensor(b, BF16))])
        items, _ = last_call(stub)
        assert items == [(h.ctypes.data, 33, F16, 4), (b.ctypes.data, 20, BF16, 0)]
        with pytest.raises(ValueError):
            e.ingest_arrays([(-1, FakeCudaTensor(h, F16))])
        with pytest.raises(TypeError):
            e.ingest_arrays([(0, FakeCudaTensor(h, "torch.complex64"))])
        with pytest.raises(RuntimeError):
            e.ingest_arrays([(5, FakeCudaTensor(h, F16))])   # LH_ERR_RANGE from the library
    finally:
        e.close()


def test_shim_entry_points_are_bound(stub_libs):
    """The C shim's lhms_arrays_* entry points are exactly the two calls, each declared by metric_system._bind."""
    import re
    import loghisto_b200.metric_system as m
    src = open(HOST_SRCS[0]).read()
    names = re.findall(r"LHMS_API [\w *]+?(lhms_arrays_\w+)\(", src)
    assert names == ["lhms_arrays_scope", "lhms_arrays_graph_recorder"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm


def test_graph_recorder_arrays_match_the_oracle(MS, oracle):
    """GraphRecorder.arrays (GraphRecorder::Arrays, lhms_arrays_graph_recorder) under the recorder's names: the
    collection holds every element as float64(x); KeyError / TypeError and library refusals before anything is
    recorded."""
    ms = MS(max_histograms=4)
    h = values(oracle, F16, 300, 5)
    b = values(oracle, BF16, 70, 6)
    u = values(oracle, U64, 9, 7)
    with ms.graph_recorder(histograms=["g0", "g1"]) as g:
        g.arrays([("g1", FakeCudaTensor(h, F16)), ("g0", FakeCudaTensor(b, BF16)), ("g1", FakeCudaTensor(u, U64))])
        with pytest.raises(KeyError):
            g.arrays([("g0", FakeCudaTensor(b, BF16)), ("zz", FakeCudaTensor(b, BF16))])
        with pytest.raises(TypeError):
            g.arrays([("g0", FakeCudaTensor(b, BF16)), ("g0", FakeCudaTensor(b, "torch.int8"))])
        with pytest.raises(RuntimeError):   # misaligned: refused, so the first item is not recorded either
            g.arrays([("g0", FakeCudaTensor(b, BF16)), ("g0", FakeCudaTensor(h[:8], F16, byte_offset=1))])
        raw, _ = ms.collect_and_process()
    assert (dense_of(raw["Histograms"]["g0"]) == oracle.ingest(as_f64(b, BF16))).all()
    assert (dense_of(raw["Histograms"]["g1"]) == oracle.ingest(np.concatenate([as_f64(h, F16), as_f64(u, U64)]))).all()


def test_graph_shim_from_c(stub_libs, MS, oracle):
    """lhms_arrays_graph_recorder called as a C caller would, on the handle behind a Python graph recorder."""
    ms = MS()
    host = ctypes.CDLL(stub_libs[1])
    fn = host.lhms_arrays_graph_recorder
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_void_p),
                   ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32), ctypes.c_uint32, ctypes.c_void_p]
    a = np.array([7, -3, 7], np.int32)
    with ms.graph_recorder(histograms=["p", "q"]) as g:
        idx = (ctypes.c_uint32 * 1)(0)
        ptrs = (ctypes.c_void_p * 1)(a.ctypes.data)
        ns = (ctypes.c_uint64 * 1)(3)
        dts = (ctypes.c_uint32 * 1)(I32)
        assert fn(g._h, idx, ptrs, ns, dts, 1, None) == 0
        assert fn(g._h, (ctypes.c_uint32 * 1)(2), ptrs, ns, dts, 1, None) != 0      # no such name
        assert fn(g._h, idx, ptrs, ns, (ctypes.c_uint32 * 1)(7), 1, None) != 0      # unknown dtype
        assert fn(g._h, None, ptrs, ns, dts, 1, None) != 0
        raw, _ = ms.collect_and_process()
    assert (dense_of(raw["Histograms"]["p"]) == oracle.ingest(a.astype(np.float64))).all()
