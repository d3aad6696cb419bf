"""Recording from CUDA kernels under MetricSystem names (MetricSystem.recording / MetricSystem::BeginRecording) and
device-side timers (lh::start_timer / lh::stop), on the real library.  The kernels live in tests/named_record_client.cu,
built by build().  References: the CPU oracle (bucket arithmetic and processHistograms) and its port of metrics.go
(oracle.OracleMetricSystem), which has no name limit."""
import ctypes as C
import importlib.util
import os
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNBOUND = 0xFFFFFFFF
LABELS = {"_min": 0.0, "_50": .5, "_75": .75, "_90": .9, "_95": .95, "_99": .99, "_99.9": .999, "_99.99": .9999,
          "_max": 1.0}


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def client():
    from loghisto_b200 import _lib, build
    assert os.path.exists(build.NAMED_CLIENT_LIB), "build() did not produce " + build.NAMED_CLIENT_LIB
    lib = C.CDLL(build.NAMED_CLIENT_LIB)
    rp, vp, sz, u32 = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t, C.c_uint32
    lib.nrc_set_device.argtypes = [C.c_int]
    lib.nrc_record_one.argtypes = [rp, u32, vp, sz, vp]
    lib.nrc_count_one.argtypes = [rp, u32, C.c_uint64, sz, vp]
    lib.nrc_timer_pair.argtypes = [rp, u32, vp, sz, vp]
    lib.nrc_timer_start.argtypes = [vp, u32, sz, vp]
    lib.nrc_timer_stop.argtypes = [rp, vp, vp, sz, vp]
    for f in ("nrc_set_device", "nrc_record_one", "nrc_count_one", "nrc_timer_pair", "nrc_timer_start", "nrc_timer_stop"):
        getattr(lib, f).restype = C.c_int
    assert lib.nrc_set_device(0) == 0
    return lib


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, monkeypatch):
    from loghisto_b200.metric_system import MetricSystem
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
    made = []

    def make(max_histograms=16, max_counters=16, precision=0):
        m = MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=max_counters, precision=precision)
        made.append(m)
        return m
    yield make
    for m in made:
        m.close()


def _cases():
    spec = importlib.util.spec_from_file_location("name_recycling_cases",
                                                  os.path.join(ROOT, "tests", "_name_recycling_cases.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def dense(hist):
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in hist.items():
        out[int(k) & 0xFFFF] = c
    return out


def record(client, s, stream, name, d_vals):
    assert client.nrc_record_one(C.byref(s.recorder), s.histogram_ids[name], d_vals.data_ptr(), d_vals.numel(),
                                 stream.cuda_stream) == 0


def count(client, s, stream, name, amount, n):
    assert client.nrc_count_one(C.byref(s.recorder), s.counter_ids[name], amount, n, stream.cuda_stream) == 0


@pytest.mark.parametrize("precision", [100, 37])
def test_host_and_device_samples_of_the_same_names(MS, client, oracle, torch, precision):
    """Host Histogram() calls and device records of the same names in one interval: raw buckets equal the oracle over
    the union, the processed statistics equal processHistograms of that union, and device counter deltas appear in
    Rates and in the cumulative Counters."""
    rng = np.random.default_rng(precision)
    ms = MS(precision=precision)
    st = torch.cuda.Stream()
    host = {"lat": np.exp(rng.uniform(-3, 18, 3000)), "size": rng.normal(0, 1e4, 2000)}
    dev = {"lat": np.exp(rng.uniform(-3, 18, 50_000)), "size": rng.normal(0, 1e4, 70_000)}
    d_dev = {nm: torch.from_numpy(v).cuda() for nm, v in dev.items()}
    torch.cuda.synchronize()
    cum = 0
    for interval in range(2):
        for nm, v in host.items():
            ms.HistogramMany(nm, v)
        ms.Counter("req", 3)
        with ms.recording(st, histograms=["lat", "size"], counters=["req", "dev_only"]) as s:
            for nm in ("lat", "size"):
                record(client, s, st, nm, d_dev[nm])
            count(client, s, st, "req", 7, 1000)
            count(client, s, st, "dev_only", 2 ** 40 + 1, 300)
        raw, m = ms.collect_and_process()
        assert set(raw["Histograms"]) == {"lat", "size"}
        for nm in ("lat", "size"):
            want = oracle.ingest(np.concatenate([host[nm], dev[nm]]), precision=precision)
            assert (dense(raw["Histograms"][nm]) == want).all(), (precision, nm)
            ref = oracle.process_histogram(want, list(LABELS.values()), precision)
            assert m[nm + "_count"] == ref["total"] == host[nm].size + dev[nm].size
            for stat in ("sum", "avg"):
                assert abs(m[nm + "_" + stat] - ref[stat]) <= 1e-12 * abs(ref[stat]), (nm, stat)
            for j, lab in enumerate(LABELS):
                assert m[nm + lab] == ref["pvals"][j], (nm, lab)
        assert raw["Rates"] == {"req": 3 + 7 * 1000, "dev_only": (2 ** 40 + 1) * 300}
        cum += 1
        assert raw["Counters"] == {"req": cum * (3 + 7000), "dev_only": cum * (2 ** 40 + 1) * 300}
    assert ms.dropped() == 0


def test_churn_matches_the_port(MS, client, oracle, torch):
    """14 intervals, a table of 8, a window of 3 names sliding one name per interval plus names that come back after
    1 and 3 idle intervals.  Names are recorded only from scopes, only from the host, or from both (by their index).
    Every interval's raw set and processed metrics equal the port's, which drops nothing."""
    rng = np.random.default_rng(5)
    ms = MS(max_histograms=8, max_counters=8)
    ref = oracle.OracleMetricSystem()
    st = torch.cuda.Stream()
    cases = _cases()
    try:
        for k in range(14):
            names = ["w%d" % (k + j) for j in range(3)] + ["gap%d" % g for g in (1, 3) if k % (g + 1) == 0]
            scoped, dev_vals, dev_amounts = [], {}, {}
            for i, nm in enumerate(names):
                mode = (int(nm[1:]) if nm[0] == "w" else int(nm[3:])) % 3   # 0: scope only, 1: host only, 2: both
                if mode != 1:
                    scoped.append(nm)
                    dev_vals[nm] = np.exp(rng.uniform(-4, 20, int(rng.integers(1, 400))))
                    dev_amounts[nm] = int(rng.integers(1, 2 ** 40))
                    for v in dev_vals[nm]:
                        ref.Histogram("h_" + nm, float(v))
                    ref.Counter("c_" + nm, dev_amounts[nm] * 32)
                if mode != 0:
                    for v in np.exp(rng.uniform(-4, 20, int(rng.integers(1, 6)))):
                        ms.Histogram("h_" + nm, float(v))
                        ref.Histogram("h_" + nm, float(v))
                    amt = int(rng.integers(1, 2 ** 40))
                    ms.Counter("c_" + nm, amt)
                    ref.Counter("c_" + nm, amt)
            d_vals = {nm: torch.from_numpy(v).cuda() for nm, v in dev_vals.items()}
            torch.cuda.synchronize()
            with ms.recording(st, histograms=["h_" + nm for nm in scoped], counters=["c_" + nm for nm in scoped]) as s:
                for nm in scoped:
                    assert client.nrc_record_one(C.byref(s.recorder), s.histogram_ids["h_" + nm], d_vals[nm].data_ptr(),
                                                 d_vals[nm].numel(), st.cuda_stream) == 0
                    assert client.nrc_count_one(C.byref(s.recorder), s.counter_ids["c_" + nm], dev_amounts[nm], 32,
                                                st.cuda_stream) == 0
            raw, m = ms.collect_and_process()
            rraw, rm = ref.collect_and_process()
            cases._compare_interval(raw, m, rraw, rm)
        assert ms.dropped() == 0
    finally:
        ref.close()


def test_race_scopes_against_a_collector(MS, client, oracle, torch):
    """A collector collects about every millisecond while 8 threads open scopes over overlapping name sets, launch,
    record and end.  Name i records 1000 * 1.07^i only (a bucket no other name uses) and counter amount p_i (a prime),
    so a sample filed under the wrong name shows; per-name totals over all intervals equal what was launched."""
    nnames, threads, rounds = 12, 8, 40
    values = [1000.0 * 1.07 ** i for i in range(nnames)]
    keys = [oracle.compress(v) for v in values]
    assert len(set(keys)) == nnames
    primes = _cases()._primes(nnames)
    ms = MS(max_histograms=nnames + 4, max_counters=nnames + 4)
    d_vals = [torch.full((4096,), v, dtype=torch.float64, device="cuda") for v in values]
    torch.cuda.synchronize()
    launched_h = np.zeros(nnames, dtype=np.int64)
    launched_c = np.zeros(nnames, dtype=np.int64)
    got_h = np.zeros(nnames, dtype=np.int64)
    got_c = np.zeros(nnames, dtype=np.int64)
    lock = threading.Lock()
    errors = []
    done = threading.Event()

    def absorb(raw):
        for nm, hist in raw["Histograms"].items():
            i = int(nm[1:])
            assert set(hist) == {keys[i]}, (nm, hist)
            got_h[i] += hist[keys[i]]
        for nm, r in raw["Rates"].items():
            i = int(nm[1:])
            assert r % primes[i] == 0, (nm, r)
            got_c[i] += r // primes[i]

    def worker(t):
        try:
            rng = np.random.default_rng(t)
            st = torch.cuda.Stream()
            for r in range(rounds):
                idx = [(t + j) % nnames for j in range(4)]
                with ms.recording(st, histograms=["h%d" % i for i in idx], counters=["c%d" % i for i in idx]) as s:
                    for i in idx:
                        n = int(rng.integers(1, 4096))
                        c = int(rng.integers(1, 64))
                        assert client.nrc_record_one(C.byref(s.recorder), s.histogram_ids["h%d" % i],
                                                     d_vals[i].data_ptr(), n, st.cuda_stream) == 0
                        assert client.nrc_count_one(C.byref(s.recorder), s.counter_ids["c%d" % i], primes[i], c,
                                                    st.cuda_stream) == 0
                        with lock:
                            launched_h[i] += n
                            launched_c[i] += c
        except BaseException as e:      # reported by the main thread
            errors.append(e)

    def collector():
        try:
            while not done.is_set():
                raw, _ = ms.collect_and_process()
                absorb(raw)
                time.sleep(0.001)
        except BaseException as e:
            errors.append(e)

    col = threading.Thread(target=collector)
    col.start()
    ws = [threading.Thread(target=worker, args=(t,)) for t in range(threads)]
    for w in ws:
        w.start()
    for w in ws:
        w.join()
    done.set()
    col.join()
    assert not errors, errors
    raw, _ = ms.collect_and_process()
    absorb(raw)
    assert ms.dropped() == 0
    assert (got_h == launched_h).all(), (got_h, launched_h)
    assert (got_c == launched_c).all(), (got_c, launched_c)


@pytest.mark.parametrize("split", [False, True], ids=["one_kernel", "token_across_kernels"])
def test_device_timer(MS, client, oracle, torch, split):
    """start_timer / stop in one kernel, or a token written to memory by one kernel and stopped by a later kernel on
    the same stream.  Recorded buckets equal the oracle over the returned durations, each of which lies between 0 and
    the host's wall time around the launches."""
    n = 20_000
    ms = MS()
    st = torch.cuda.Stream()
    out = torch.zeros(n, dtype=torch.int64, device="cuda")
    tokens = torch.zeros(2 * n, dtype=torch.int64, device="cuda")     # 16 bytes per token
    torch.cuda.synchronize()
    t0 = time.perf_counter_ns()
    with ms.recording(st, histograms=["kernel_ns"]) as s:
        hid = s.histogram_ids["kernel_ns"]
        if split:
            assert client.nrc_timer_start(tokens.data_ptr(), hid, n, st.cuda_stream) == 0
            assert client.nrc_timer_stop(C.byref(s.recorder), tokens.data_ptr(), out.data_ptr(), n, st.cuda_stream) == 0
        else:
            assert client.nrc_timer_pair(C.byref(s.recorder), hid, out.data_ptr(), n, st.cuda_stream) == 0
    st.synchronize()
    wall = time.perf_counter_ns() - t0
    ns = out.cpu().numpy()
    assert (ns >= 0).all() and (ns <= wall).all(), (ns.min(), ns.max(), wall)
    if not split:
        assert ns.max() >= 16 * 250      # the longest spin is measured
    raw, _ = ms.collect_and_process()
    assert (dense(raw["Histograms"]["kernel_ns"]) == oracle.ingest(ns.astype(np.float64))).all()
    assert ms.dropped() == 0


def test_scope_histogram_equals_bare_ingest(MS, torch):
    """s.histogram(name, tensor) equals lh_ingest_f64 of the same tensor on a bare engine, bucket for bucket."""
    import loghisto_b200 as lh
    from oracle import oracle as o
    rng = np.random.default_rng(3)
    vals = np.concatenate([np.exp(rng.uniform(-5, 40, 1_500_000)) * rng.choice([-1, 1], 1_500_000),
                           [0.0, -0.0, np.inf, -np.inf, np.nan, 1e308]])
    t = torch.from_numpy(vals).cuda()
    torch.cuda.synchronize()
    ms = MS()
    st = torch.cuda.Stream()
    with ms.recording(st, histograms=["payload"]) as s:
        s.histogram("payload", t)
        with pytest.raises(TypeError):
            s.histogram("payload", t.float())
    raw, _ = ms.collect_and_process()
    with lh.Engine(device=0, max_histograms=1, max_counters=1) as eng:
        eng.ingest_f64(0, t, t.numel())
        _, sp = eng.snapshot(list(o.DEFAULT_PERCENTILES.values()))
        want = dense(sp.histogram(0))
    assert (dense(raw["Histograms"]["payload"]) == want).all()
    assert int(want.sum()) == vals.size


def test_collect_while_holding_a_scope_and_unbound_names(MS, client, oracle, torch):
    """Collecting from the thread that holds a scope raises; after the scope ends nothing is lost and the system keeps
    working.  A name with no free id is bound to 0xFFFFFFFF and its records are dropped and counted.  lh::count of 0
    leaves the delta at 0, so (unlike the host's Counter(name, 0)) the name does not appear in Rates."""
    ms = MS(max_histograms=3, max_counters=3)
    st = torch.cuda.Stream()
    d = torch.full((5000,), 42.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    ms.Counter("zero", 0)
    ms.Histogram("h", 2.0)
    with ms.recording(st, histograms=["h"], counters=["dev_zero"]) as s:
        record(client, s, st, "h", d)
        count(client, s, st, "dev_zero", 0, 100)
        with pytest.raises(RuntimeError, match="record scope"):
            ms.collect_and_process()
    raw, _ = ms.collect_and_process()
    assert raw["Rates"] == {"zero": 0}
    assert raw["Histograms"] == {"h": {oracle.compress(2.0): 1, oracle.compress(42.0): 5000}}
    for nm in ("a", "b"):
        ms.Histogram(nm, 1.0)
    before = ms.dropped()
    with ms.recording(st, histograms=["h", "new"], counters=["c"]) as s:
        assert s.histogram_ids["new"] == UNBOUND and s.histogram_ids["h"] != UNBOUND
        assert ms.dropped() == before
        record(client, s, st, "new", d)
        record(client, s, st, "h", d)
        s.histogram("new", d[:10])
    raw, _ = ms.collect_and_process()
    assert ms.dropped() - before == 5000 + 10
    assert raw["Histograms"] == {"h": {oracle.compress(42.0): 5000}, "a": {oracle.compress(1.0): 1},
                                 "b": {oracle.compress(1.0): 1}}
