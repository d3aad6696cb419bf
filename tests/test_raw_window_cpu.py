"""Window raw device subscriptions bound to names (MetricSystem::NewRawDeviceSubscription(names, window),
loghisto_b200/host/metric_system.cc) on the CPU: the C++ mirror compiled against the TEST-ONLY oracle-backed stub of
the C ABI with tests/stub_abi/lh_stub_raw_window.c, whose window boards sum each row's last `window` intervals in host
memory.  Covers names bound at every collection (absent and recycled names enter the window as empty intervals), the
Python layer's checks of `window`, the mirror over a library without lh_raw_board_create_window, and the C shim from a
plain C client.  tests/test_gpu_raw_window.py runs the real library."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUBS = ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_graph.c",
         "lh_stub_board.c")
INT32_MIN = -(1 << 31)


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
    stub, host = _build("raw_window", STUBS + ("lh_stub_raw_window.c",))
    s = ctypes.CDLL(stub)
    s.lh_stub_raw_alive.restype = ctypes.c_uint32
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
    assert stub.lh_stub_raw_alive() == 0


def query(sub, ps, values):
    """The shim's grid queries on host arrays (the stub's "device" memory)."""
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
    return keys, pub, ranks, totals


def check_window(sub, history, names, ps, values):
    """Every row against the sum of its name's Histograms over the last `window` collections of `history`: totals,
    ranks at the oracle's compress(v), percentile keys by the reference's rule, and the publish number."""
    from oracle import oracle as o
    keys, pub, ranks, totals = query(sub, ps, values)
    assert (pub == len(history)).all()
    for i, nm in enumerate(names):
        d = {}
        for raw in history[-sub.window:]:
            for key, c in raw["Histograms"].get(nm, {}).items():
                d[key] = d.get(key, 0) + c
        total = sum(d.values())
        assert int(totals[i]) == total, (nm, len(history))
        for j, v in enumerate(values):
            kv = int(o.compress(v))
            assert int(ranks[i, j]) == sum(c for key, c in d.items() if key <= kv), (nm, v)
        for j, p in enumerate(ps):
            run, want = 0, INT32_MIN
            for key in sorted(d):
                run += d[key]
                if d[key] and run / total >= p:
                    want = key
                    break
            assert keys[i, j] == want, (nm, p, len(history))


def test_names_bound_per_collection(MS):
    """Windows of 1, 2 and 4 collections follow names: "a" in every collection, "b" in every other one, "c" idle long
    enough to lose its id to other names and back, "never" never seen.  Each collection enters once, the name's
    buckets or nothing."""
    ms = MS(max_histograms=4)
    names = ["a", "b", "c", "never"]
    subs = [ms.raw_device_subscription(histograms=names, window=w) for w in (1, 2, 4)]
    assert [s.window for s in subs] == [1, 2, 4]
    ps, values = [0.0, 0.5, 0.99, 1.0], [-1.0, 1.0, 3.0, 7.0, 100.0]
    history = []
    for j in range(12):
        ms.HistogramMany("a", np.arange(1.0, 2.0 + j))
        if j % 2:
            ms.Histogram("b", 7.0)
            ms.Histogram("b", -3.0)
        if j in (0, 1, 10):
            ms.HistogramMany("c", np.full(3 + j, 50.0))
        if 3 <= j <= 8:                       # fill the table so that "c" loses its id meanwhile
            for i in range(3):
                ms.Histogram("x%d.%d" % (j, i), 2.0)
        raw, _ = ms.collect_and_process()
        history.append(raw)
        for s in subs:
            check_window(s, history, names, ps, values)
    assert "c" in history[1]["Histograms"] and "c" not in history[9]["Histograms"] and "c" in history[10]["Histograms"]
    for s in subs:
        s.close()


def test_window_argument_checks(MS, stub_libs):
    """window must be an int >= 1: anything else raises TypeError / ValueError before the library is called.  Above
    LH_RAW_MAX_WINDOW the library refuses it."""
    from loghisto_b200 import _lib as L
    from loghisto_b200.engine import RawBoard
    stub = stub_libs[0]
    ms = MS(max_histograms=2)
    for bad, err in ((0, ValueError), (-3, ValueError), (2.5, TypeError), ("2", TypeError), (True, TypeError),
                     (None, TypeError), (np.float64(2.0), TypeError)):
        with pytest.raises(err):
            ms.raw_device_subscription(histograms=["a"], window=bad)
        with pytest.raises(err):
            RawBoard(object(), 1, window=bad)   # checked before the engine is touched
        assert stub.lh_stub_raw_alive() == 0
    with pytest.raises(RuntimeError):
        ms.raw_device_subscription(histograms=["a"], window=L.LH_RAW_MAX_WINDOW + 1)
    with ms.raw_device_subscription(histograms=["a"], window=np.int64(3)) as sub:
        assert sub.window == 3 and isinstance(sub.window, int)
    assert stub.lh_stub_raw_alive() == 0


def test_mirror_without_window_boards():
    """Over a library with raw boards but without lh_raw_board_create_window (the stub with lh_stub_raw_board.c), a
    window above 1 reports an error, window 1 still works, and nothing is left allocated."""
    import loghisto_b200.metric_system as m
    stub, host = _build("raw_no_window", STUBS + ("lh_stub_raw_board.c",))
    s = ctypes.CDLL(stub)
    s.lh_stub_raw_alive.restype = ctypes.c_uint32
    saved = m._lib
    m._lib = m._bind(ctypes.CDLL(host))
    try:
        ms = m.MetricSystem(1e-6, False, max_histograms=2, max_counters=2)
        try:
            with pytest.raises(RuntimeError):
                ms.raw_device_subscription(histograms=["a"], window=2)
            assert s.lh_stub_raw_alive() == 0
            with ms.raw_device_subscription(histograms=["a"]) as sub:
                assert sub.window == 1
                ms.Histogram("a", 1.0)
                ms.collect_and_process()
                _, pub, _, totals = query(sub, [0.5], [1.0])
                assert totals[0] == 1 and pub[0, 0] == 1
        finally:
            ms.close()
        assert s.lh_stub_raw_alive() == 0
    finally:
        m._lib = saved


C_CLIENT = r"""
#include <stdio.h>
#include <stdint.h>
#include "loghisto_b200.h"
typedef void (*emit_fn)(void *, int, const char *, int, uint64_t, double);
void *lhms_new(int64_t interval_ns, int device, uint32_t max_histograms, uint32_t max_counters, char *err, int errlen);
void lhms_free(void *ms);
void lhms_histogram(void *ms, const char *name, double v);
int lhms_collect_and_process(void *ms, emit_fn emit, void *ctx, char *err, int errlen);
void *lhms_raw_window_subscription_new(void *ms, uint32_t n_h, const char *const *h_names, uint32_t window,
                                       lh_raw_board *out, int *status);
int lhms_raw_subscription_ranks(void *d, const double *d_values, uint32_t m, uint64_t *d_ranks, uint64_t *d_totals,
                                uint64_t *d_publish, void *stream);
int lhms_raw_subscription_close(void *d);
void lhms_raw_subscription_free(void *d);
static void ignore(void *c, int k, const char *n, int key, uint64_t u, double f) { (void)c; (void)k; (void)n; (void)key; (void)u; (void)f; }

int main(void) {
    char err[256];
    void *ms = lhms_new(1000, 0, 4, 4, err, sizeof err);
    if (!ms) { printf("lhms_new: %s\n", err); return 2; }
    const char *names[2] = {"lat", "never"};
    lh_raw_board b;
    int st = 0;
    if (lhms_raw_window_subscription_new(ms, 2, names, 0, &b, &st) || st == 0) return 3;       /* window 0 */
    void *sub = lhms_raw_window_subscription_new(ms, 2, names, 3, &b, &st);
    if (!sub || st != 0 || b.k != 2) return 4;
    uint64_t want[6] = {1, 3, 6, 9, 12, 15};   /* collection j adds j + 1 samples: sums over the last 3 */
    for (int j = 0; j < 6; j++) {
        for (int i = 0; i <= j; i++) lhms_histogram(ms, "lat", 2.0);
        if (lhms_collect_and_process(ms, ignore, NULL, err, sizeof err) != 0) return 5;
        double v = 2.0;
        uint64_t ranks[2], totals[2], pub[2];
        if (lhms_raw_subscription_ranks(sub, &v, 1, ranks, totals, pub, NULL) != 0) return 6;
        if (totals[0] != want[j] || ranks[0] != want[j] || totals[1] != 0 || pub[0] != (uint64_t)j + 1) {
            printf("collection %d: total %llu rank %llu\n", j, (unsigned long long)totals[0], (unsigned long long)ranks[0]);
            return 7;
        }
    }
    if (lhms_raw_subscription_close(sub) != 0) return 8;
    lhms_raw_subscription_free(sub);
    lhms_free(ms);
    printf("ok\n");
    return 0;
}
"""


def test_c_shim_from_plain_c(stub_libs, tmp_path):
    """lhms_raw_window_subscription_new from a C11 program: window 0 is refused, a window of 3 answers for the last
    three collections."""
    _, host = stub_libs
    src = tmp_path / "client.c"
    src.write_text(C_CLIENT)
    exe = tmp_path / "client"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I", INC, str(src), "-o", str(exe), host,
                    "-Wl,-rpath," + BUILD], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", (out.returncode, out.stdout, out.stderr)


def test_bindings(stub_libs):
    """The ctypes signatures of the new ABI call and shim entry, and LH_RAW_MAX_WINDOW as the header defines it."""
    import re
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    assert "lh_raw_board_create_window" in _lib.SIGNATURES
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    assert int(re.search(r"#define LH_RAW_MAX_WINDOW (\d+)", hdr).group(1)) == _lib.LH_RAW_MAX_WINDOW == 4096
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    assert L.lhms_raw_window_subscription_new.argtypes is not None
