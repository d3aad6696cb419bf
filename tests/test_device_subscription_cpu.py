"""Device subscriptions bound to names (MetricSystem::NewDeviceSubscription, loghisto_b200/host/metric_system.cc) on the
CPU: the C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus tests/stub_abi/lh_stub_board.c,
whose boards are host memory filled from the snapshot's export at every lh_snapshot_publish.  Covers the binding of
every row at each collection (present exactly when the name is in Histograms / Rates, counts and rates of that
collection, totals equal Counters), ids that recycle under the subscribed names, label changes, unbound rows, the
C shim, and closing subscriptions while the reaper collects.  tests/test_gpu_device_subscription.py runs the real
library."""
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
P = 32
HDR = np.dtype([("seq", "<u8"), ("publishes", "<u8"), ("np", "<u4"), ("reserved", "<u4", (3,)), ("percentiles", "<f8", (P,))])
HIST_ROW = np.dtype([("count", "<u8"), ("sum", "<f8"), ("avg", "<f8"), ("present", "<u4"), ("reserved", "<u4"),
                     ("pvals", "<f8", (P,)), ("pkeys", "<i4", (P,))])
CTR_ROW = np.dtype([("rate", "<u8"), ("total", "<u8"), ("present", "<u4"), ("reserved", "<u4")])


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_board.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_board.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in
                    ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_graph.c",
                     "lh_stub_board.c")] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_board", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    from loghisto_b200 import _lib
    s = ctypes.CDLL(stub)
    s.lh_stub_board_alive.restype = ctypes.c_uint32
    s.lh_stub_board_bound.argtypes = [ctypes.POINTER(_lib.lh_board), ctypes.c_uint32]
    s.lh_stub_board_bound.restype = ctypes.c_uint32
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
    assert stub.lh_stub_board_alive() == 0


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


def image(sub):
    """The board of a subscription, as the stub holds it in host memory: (header, histogram rows, counter rows)."""
    b = sub.board
    buf = (ctypes.c_char * b.bytes).from_address(b.d_board)
    raw = np.frombuffer(bytes(buf), dtype=np.uint8)
    h = raw[:HDR.itemsize].view(HDR)[0]
    rows = raw[HDR.itemsize:HDR.itemsize + b.k * HIST_ROW.itemsize].view(HIST_ROW)
    crows = raw[HDR.itemsize + b.k * HIST_ROW.itemsize:].view(CTR_ROW)
    return h, rows, crows


def check(sub, raw, metrics, hnames, cnames):
    h, rows, crows = image(sub)
    assert h["seq"] % 2 == 0
    for i, nm in enumerate(hnames):
        if nm in raw["Histograms"]:
            assert rows[i]["present"] == 1 and float(rows[i]["count"]) == metrics[nm + "_count"]
        else:
            assert rows[i]["present"] == 0 and rows[i]["count"] == 0
    for i, nm in enumerate(cnames):
        assert crows[i]["present"] == (nm in raw["Rates"])
        assert int(crows[i]["rate"]) == raw["Rates"].get(nm, 0)
        assert int(crows[i]["total"]) == raw["Counters"].get(nm, 0)
    return h


def test_binding_per_collection(MS, stub):
    """Each collection binds a row to the id its name carries in that collection, or leaves it unbound; label
    changes between collections change nothing in the binding."""
    ms = MS(max_histograms=4, max_counters=4)
    hnames, cnames = ["a", "b", "never"], ["x", "y"]
    sub = ms.device_subscription(histograms=hnames, counters=cnames)
    assert sub.histogram_rows == {"a": 0, "b": 1, "never": 2} and sub.counter_rows == {"x": 0, "y": 1}
    for j in range(6):
        ms.SpecifyPercentiles([{}, {"%s_p50": 0.5}, {"%s_p50": 0.5, "%s_p99": 0.99, "%s_bad": 2.0}][j % 3])
        ms.HistogramMany("a", np.arange(1.0, 2.0 + j))
        if j % 2:
            ms.Histogram("b", 7.0)
            ms.Counter("y", 0)
        ms.Counter("x", j + 1)
        raw, metrics = ms.collect_and_process()
        h = check(sub, raw, metrics, hnames, cnames)
        assert h["publishes"] == j + 1
        bound = [stub.lh_stub_board_bound(ctypes.byref(sub.board), r) for r in range(5)]
        assert bound[0] != UNBOUND and bound[2] == UNBOUND and bound[3] != UNBOUND
        assert (bound[1] != UNBOUND) == bool(j % 2) and (bound[4] != UNBOUND) == bool(j % 2)
    sub.close()
    sub.close()


def test_recycling_under_subscribed_names(MS, stub):
    """A subscribed name idle long enough loses its id to other names: meanwhile its row is unbound (other names'
    counts never show under it); when it comes back it is bound to its new id."""
    ms = MS(max_histograms=3, max_counters=2)
    with ms.device_subscription(histograms=["keep", "idle"], counters=["c"]) as sub:
        ms.Histogram("idle", 1.0)
        ms.Histogram("keep", 1.0)
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, ["keep", "idle"], ["c"])
        first = stub.lh_stub_board_bound(ctypes.byref(sub.board), 1)
        assert first != UNBOUND
        for j in range(6):
            ms.Histogram("keep", 2.0)
            ms.HistogramMany("other%d" % j, np.ones(j + 3))
            raw, metrics = ms.collect_and_process()
            check(sub, raw, metrics, ["keep", "idle"], ["c"])
            assert stub.lh_stub_board_bound(ctypes.byref(sub.board), 1) == UNBOUND
        ms.HistogramMany("idle", np.ones(5))
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, ["keep", "idle"], ["c"])
        again = stub.lh_stub_board_bound(ctypes.byref(sub.board), 1)
        assert again != UNBOUND and image(sub)[1][1]["count"] == 5


def test_counter_totals_and_shim(MS, stub_libs):
    """Totals are Counters values (names counted once keep their total while absent from Rates); lhms_subscription_read
    copies the board; creation refuses more names than the tables hold, or none."""
    import loghisto_b200.metric_system as m
    ms = MS(max_histograms=2, max_counters=2)
    with pytest.raises(RuntimeError):
        ms.device_subscription(histograms=["a", "b", "c"])
    with pytest.raises(RuntimeError):
        ms.device_subscription()
    sub = ms.device_subscription(counters=["c0", "c1"])
    for j, (a0, a1) in enumerate([(3, None), (None, 4), (5, 6)]):
        if a0 is not None:
            ms.Counter("c0", a0)
        if a1 is not None:
            ms.Counter("c1", a1)
        raw, metrics = ms.collect_and_process()
        check(sub, raw, metrics, [], ["c0", "c1"])
    _, _, crows = image(sub)
    assert list(crows["total"]) == [8, 10] and list(crows["rate"]) == [5, 6]
    out = np.zeros(sub.board.bytes, dtype=np.uint8)
    assert m._lib.lhms_subscription_read(sub._h, out.ctypes.data, None) == 0
    assert out.view(np.uint64)[1] == 3   # publishes
    sub.close()
    assert m._lib.lhms_subscription_read(None, out.ctypes.data, None) != 0


def test_close_during_collector_loop(MS, stub):
    """Subscriptions opened and closed while the reaper collects every millisecond: each publishes while open, the
    reaper keeps running, and every board is freed."""
    ms = MS(max_histograms=8, max_counters=4, interval=1e-3)
    ms.Start()
    stop = threading.Event()

    def feed():
        while not stop.is_set():
            ms.Histogram("lat", 3.0)
            ms.Counter("req", 1)
            time.sleep(0.0002)
    t = threading.Thread(target=feed)
    t.start()
    try:
        for _ in range(20):
            with ms.device_subscription(histograms=["lat"], counters=["req"]) as sub:
                deadline = time.monotonic() + 2.0
                while image(sub)[0]["publishes"] < 2 and time.monotonic() < deadline:
                    time.sleep(0.001)
                assert image(sub)[0]["publishes"] >= 2
            assert sub._h is None
    finally:
        stop.set()
        t.join()
        ms.Stop()
    assert stub.lh_stub_board_alive() == 0


def test_board_layout_and_bindings(tmp_path, stub_libs):
    """The board structs as a C compiler lays them out, the ctypes mirrors, the numpy layouts the tests read images
    with, and the binding of the lhms_subscription_* shim."""
    import re
    from loghisto_b200 import _lib, engine
    import loghisto_b200.metric_system as m
    structs = {"lh_board_header": HDR, "lh_board_hist_row": HIST_ROW, "lh_board_counter_row": CTR_ROW, "lh_board": None}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"', 'int main(void) {']
    for s in structs:
        fields = [f for f, _ in getattr(_lib, s)._fields_]
        lines.append('printf("%%zu", sizeof(%s));' % s)
        lines += ['printf(" %%zu", offsetof(%s, %s));' % (s, f) for f in fields]
        lines.append('printf("\\n");')
    lines.append('return 0; }')
    c = tmp_path / "layout.c"
    c.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", INC, "-o", str(exe), str(c)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()
    for line, (s, dt) in zip(out, structs.items()):
        got = [int(x) for x in line.split()]
        ct = getattr(_lib, s)
        assert got[0] == ctypes.sizeof(ct), s
        assert got[1:] == [getattr(ct, f).offset for f, _ in ct._fields_], s
        if dt is not None:
            assert dt.itemsize == got[0] and [dt.fields[f][1] for f in dt.names if f in dict(ct._fields_)] == \
                [getattr(ct, f).offset for f in dt.names if f in dict(ct._fields_)], s
    assert (ctypes.sizeof(_lib.lh_board_header), ctypes.sizeof(_lib.lh_board_hist_row),
            ctypes.sizeof(_lib.lh_board_counter_row), ctypes.sizeof(_lib.lh_board)) == (288, 416, 24, 32)
    assert (engine._BOARD_HDR_WORDS, engine._BOARD_ROW_WORDS, engine._BOARD_CTR_WORDS) == (36, 52, 3)
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    names = re.findall(r"LHMS_API [\w *]+?(lhms_subscription_\w+)\(", src)
    assert names == ["lhms_subscription_new", "lhms_subscription_read", "lhms_subscription_close", "lhms_subscription_free"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm
