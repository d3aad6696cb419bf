"""Raw device subscriptions bound to names (MetricSystem::NewRawDeviceSubscription, loghisto_b200/host/metric_system.cc)
on the CPU: the C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus
tests/stub_abi/lh_stub_raw_board.c, whose raw boards are host memory filled from the snapshot's export at every
lh_snapshot_publish_raw and queried on the CPU.  Covers the binding of every row at each collection, ids that recycle
under the subscribed names, closing while the reaper collects, the C shim, the Python layer's TypeErrors, the ctypes
layout of lh_raw_board, and the mirror over a library without the raw calls.  tests/test_gpu_raw_subscription.py runs
the real library."""
import ctypes
import os
import subprocess
import threading
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
UNBOUND = 0xFFFFFFFF
STUBS = ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_graph.c",
         "lh_stub_board.c")


def _build(tag, stubs):
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_%s.so" % tag)
    host = os.path.join(BUILD, "libloghisto_host_stub_%s.so" % tag)
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in stubs] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_%s" % tag, "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return stub, host


@pytest.fixture(scope="module")
def stub_libs():
    from loghisto_b200 import _lib
    stub, host = _build("raw_board", STUBS + ("lh_stub_raw_board.c",))
    s = ctypes.CDLL(stub)
    s.lh_stub_raw_alive.restype = ctypes.c_uint32
    s.lh_stub_raw_bound.argtypes = [ctypes.POINTER(_lib.lh_raw_board), ctypes.c_uint32]
    s.lh_stub_raw_bound.restype = ctypes.c_uint32
    return s, host


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    stub, host = stub_libs
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    made = []

    def make(max_histograms=4, max_counters=4, interval=1e-6):
        ms = m.MetricSystem(interval, False, max_histograms=max_histograms, max_counters=max_counters)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()
    assert stub.lh_stub_raw_alive() == 0


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


def query(sub, ps, values):
    """The shim's grid queries on host arrays (the stub's "device" memory): (keys, vals, pub) [k, m] for ps and
    (ranks, totals, pub) for values."""
    import loghisto_b200.metric_system as m
    k = sub.board.k
    ps = np.ascontiguousarray(ps, dtype=np.float64)
    values = np.ascontiguousarray(values, dtype=np.float64)
    keys, vals, pub = np.zeros((k, len(ps)), np.int32), np.zeros((k, len(ps))), np.zeros((k, len(ps)), np.uint64)
    assert m._lib.lhms_raw_subscription_percentiles(sub._h, ps.ctypes.data, len(ps), keys.ctypes.data, vals.ctypes.data,
                                                    pub.ctypes.data, None) == 0
    ranks, totals, rpub = np.zeros((k, len(values)), np.uint64), np.zeros(k, np.uint64), np.zeros((k, len(values)), np.uint64)
    assert m._lib.lhms_raw_subscription_ranks(sub._h, values.ctypes.data, len(values), ranks.ctypes.data,
                                              totals.ctypes.data, rpub.ctypes.data, None) == 0
    return keys, vals, pub, ranks, totals, rpub


def check(sub, raw, metrics, names, labels, values, publish):
    """Every row against the collection's RawMetricSet: labelled percentiles equal processMetrics', ranks equal the
    running sums of Histograms up to the oracle's compress(v)."""
    from oracle import oracle as o
    ps = [p for _, p in labels]
    keys, vals, pub, ranks, totals, rpub = query(sub, ps, values)
    assert (pub == publish).all() and (rpub == publish).all()
    for i, nm in enumerate(names):
        h = raw["Histograms"].get(nm)
        if h is None:
            assert (keys[i] == np.iinfo(np.int32).min).all() and np.isnan(vals[i]).all()
            assert (ranks[i] == 0).all() and totals[i] == 0
            continue
        assert int(totals[i]) == sum(h.values())
        for j, (label, p) in enumerate(labels):
            want = metrics.get(label % nm)
            if want is None:
                assert keys[i, j] == np.iinfo(np.int32).min
            else:
                assert vals[i, j] == want
        for j, v in enumerate(values):
            kv = int(o.compress(v))
            assert int(ranks[i, j]) == sum(c for key, c in h.items() if key <= kv)


LABELS = [("%s_p0", 0.0), ("%s_p50", 0.5), ("%s_p99", 0.99), ("%s_p100", 1.0)]


def test_binding_per_collection(MS, stub):
    """Each collection binds a row to the id its name carries in that collection, or leaves it unbound; answers equal
    the collection's RawMetricSet and the publish number advances by one per collection."""
    ms = MS(max_histograms=4)
    ms.SpecifyPercentiles(dict(LABELS))
    names = ["a", "b", "never"]
    sub = ms.raw_device_subscription(histograms=names)
    assert sub.rows == {"a": 0, "b": 1, "never": 2}
    values = [-1.0, 0.0, 1.0, 3.0, 7.0, 100.0, float("nan"), float("inf")]
    keys, vals, pub, ranks, totals, rpub = query(sub, [0.0, 0.5], values)   # before the first publish: empty rows
    assert (keys == np.iinfo(np.int32).min).all() and np.isnan(vals).all() and (ranks == 0).all() and (totals == 0).all()
    assert (pub == 0).all() and (rpub == 0).all()
    for j in range(5):
        ms.HistogramMany("a", np.arange(1.0, 2.0 + j))
        if j % 2:
            ms.Histogram("b", 7.0)
            ms.Histogram("b", -3.0)
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, names, LABELS, values, j + 1)
        bound = [stub.lh_stub_raw_bound(ctypes.byref(sub.board), r) for r in range(3)]
        assert bound[0] != UNBOUND and bound[2] == UNBOUND
        assert (bound[1] != UNBOUND) == bool(j % 2)
    sub.close()
    sub.close()


def test_recycling_under_subscribed_names(MS, stub):
    """A subscribed name idle long enough loses its id to other names: meanwhile its row is empty (other names'
    counts never show under it); when it comes back it is bound to its new id."""
    ms = MS(max_histograms=3)
    ms.SpecifyPercentiles({"%s_p50": 0.5})
    with ms.raw_device_subscription(histograms=["keep", "idle"]) as sub:
        ms.Histogram("idle", 1.0)
        ms.Histogram("keep", 1.0)
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, ["keep", "idle"], [("%s_p50", 0.5)], [1.0], 1)
        assert stub.lh_stub_raw_bound(ctypes.byref(sub.board), 1) != UNBOUND
        for j in range(6):
            ms.Histogram("keep", 2.0)
            ms.HistogramMany("other%d" % j, np.ones(j + 3))
            raw, metrics = ms.collect_and_process()
            check(sub, raw, metrics, ["keep", "idle"], [("%s_p50", 0.5)], [1.0, 5.0], j + 2)
            assert stub.lh_stub_raw_bound(ctypes.byref(sub.board), 1) == UNBOUND
        ms.HistogramMany("idle", np.ones(5))
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, ["keep", "idle"], [("%s_p50", 0.5)], [1.0, 5.0], 8)
        assert stub.lh_stub_raw_bound(ctypes.byref(sub.board), 1) != UNBOUND


def test_refusals_and_shim(MS):
    """Creation refuses more names than the table holds, or none; the shim refuses a NULL handle and a closed
    subscription."""
    import loghisto_b200.metric_system as m
    ms = MS(max_histograms=2)
    with pytest.raises(RuntimeError):
        ms.raw_device_subscription(histograms=["a", "b", "c"])
    with pytest.raises(RuntimeError):
        ms.raw_device_subscription()
    sub = ms.raw_device_subscription(histograms=["a", "b"])
    ps = np.array([0.5])
    out = np.zeros(8, np.uint64)
    assert m._lib.lhms_raw_subscription_percentiles(None, ps.ctypes.data, 1, out.ctypes.data, out.ctypes.data,
                                                    out.ctypes.data, None) != 0
    h = sub._h
    assert m._lib.lhms_raw_subscription_close(h) == 0
    assert m._lib.lhms_raw_subscription_percentiles(h, ps.ctypes.data, 1, out.ctypes.data, out.ctypes.data,
                                                    out.ctypes.data, None) != 0
    sub.close()
    with pytest.raises(RuntimeError):
        sub.percentiles(ps)


def test_close_during_collector_loop(MS, stub):
    """Raw subscriptions opened and closed while the reaper collects every millisecond: each publishes while open, the
    reaper keeps running, and every board is freed."""
    ms = MS(max_histograms=8, interval=1e-3)
    ms.Start()
    stop = threading.Event()

    def feed():
        while not stop.is_set():
            ms.Histogram("lat", 3.0)
            time.sleep(0.0002)
    t = threading.Thread(target=feed)
    t.start()
    try:
        for _ in range(20):
            with ms.raw_device_subscription(histograms=["lat", "other"]) as sub:
                deadline = time.monotonic() + 2.0
                while query(sub, [0.5], [3.0])[2][0, 0] < 2 and time.monotonic() < deadline:
                    time.sleep(0.001)
                assert query(sub, [0.5], [3.0])[2][0, 0] >= 2
            assert sub._h is None
    finally:
        stop.set()
        t.join()
        ms.Stop()
    assert stub.lh_stub_raw_alive() == 0


def test_python_type_errors(MS):
    """percentiles() / ranks() take a contiguous 1-D float64 CUDA tensor; anything else is a TypeError raised before
    the library is called."""
    import torch
    ms = MS(max_histograms=2)
    with ms.raw_device_subscription(histograms=["a"]) as sub:
        for bad in (np.array([0.5]), [0.5], torch.tensor([0.5], dtype=torch.float64), torch.tensor([0.5], dtype=torch.float32),
                    torch.zeros((2, 2), dtype=torch.float64), None):
            with pytest.raises(TypeError):
                sub.percentiles(bad)
            with pytest.raises(TypeError):
                sub.ranks(bad)


def test_mirror_without_raw_calls(tmp_path):
    """Over a library without the raw calls (the stub without lh_stub_raw_board.c), NewRawDeviceSubscription reports an
    error instead of crashing, and the rest of the mirror still works."""
    import loghisto_b200.metric_system as m
    _, host = _build("no_raw", STUBS)
    L = m._bind(ctypes.CDLL(host))
    saved = m._lib
    m._lib = L
    try:
        ms = m.MetricSystem(1e-6, False, max_histograms=2, max_counters=2)
        try:
            with pytest.raises(RuntimeError):
                ms.raw_device_subscription(histograms=["a"])
            ms.Histogram("a", 1.0)
            raw, _ = ms.collect_and_process()
            assert sum(raw["Histograms"]["a"].values()) == 1
        finally:
            ms.close()
    finally:
        m._lib = saved


def test_raw_board_layout_and_bindings(tmp_path, stub_libs):
    """lh_raw_row_header and lh_raw_board as a C compiler lays them out, the ctypes mirrors, LH_RAW_CELLS_OFFSET, the
    ctypes signatures of the new calls, and the binding of the lhms_raw_subscription_* shim."""
    import re
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    structs = ("lh_raw_row_header", "lh_raw_board")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"', 'int main(void) {']
    for s in structs:
        fields = [f for f, _ in getattr(_lib, s)._fields_]
        lines.append('printf("%%zu", sizeof(%s));' % s)
        lines += ['printf(" %%zu", offsetof(%s, %s));' % (s, f) for f in fields]
        lines.append('printf("\\n");')
    lines.append('for (unsigned k = 1; k < 300; k += 37) printf("%llu ", (unsigned long long)LH_RAW_CELLS_OFFSET(k));')
    lines.append('printf("\\n"); return 0; }')
    c = tmp_path / "layout.c"
    c.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", INC, "-o", str(exe), str(c)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()
    for line, s in zip(out, structs):
        got = [int(x) for x in line.split()]
        ct = getattr(_lib, s)
        assert got[0] == ctypes.sizeof(ct), s
        assert got[1:] == [getattr(ct, f).offset for f, _ in ct._fields_], s
    assert [int(x) for x in out[2].split()] == [_lib.LH_RAW_CELLS_OFFSET(k) for k in range(1, 300, 37)]
    assert (ctypes.sizeof(_lib.lh_raw_row_header), ctypes.sizeof(_lib.lh_raw_board)) == (32, 80)
    for nm in ("lh_raw_board_create", "lh_snapshot_publish_raw", "lh_raw_percentiles", "lh_raw_ranks",
               "lh_raw_percentiles_grid", "lh_raw_ranks_grid", "lh_raw_board_destroy"):
        assert nm in _lib.SIGNATURES
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    names = re.findall(r"LHMS_API [\w *]+?(lhms_raw_subscription_\w+)\(", src)
    assert names == ["lhms_raw_subscription_new", "lhms_raw_subscription_percentiles", "lhms_raw_subscription_ranks",
                     "lhms_raw_subscription_close", "lhms_raw_subscription_free"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm
