"""GPU timers driven from host code (lh_gpu_timer_start / _stop / _release, Engine.gpu_timer_*, MetricSystem.StartGpuTimer
and gpu_timer) on the real library.  Spans of known length come from tests/gpu_timer_client.cu, built by build(): one
thread spinning on %globaltimer, the clock the timers read.  References: the CPU oracle's bucket arithmetic and
processHistograms."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LABELS = {"_min": 0.0, "_50": .5, "_75": .75, "_90": .9, "_95": .95, "_99": .99, "_99.9": .999, "_99.99": .9999,
          "_max": 1.0}
SPANS = [0, 1_000, 10_000, 100_000, 1_000_000, 10_000_000]
MS50 = 50_000_000


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def spin():
    """spin(ns, stream): enqueue at least `ns` of GPU time on a torch stream or a raw handle (0 = the legacy default)."""
    from loghisto_b200 import build
    lib = C.CDLL(build.TIMER_CLIENT_LIB)
    lib.gtc_set_device.argtypes = [C.c_int]
    lib.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    lib.gtc_set_device.restype = lib.gtc_spin.restype = C.c_int
    assert lib.gtc_set_device(0) == 0

    def run(ns, stream):
        h = stream if isinstance(stream, int) else stream.cuda_stream
        assert lib.gtc_spin(int(ns), h) == 0
    return run


@pytest.fixture
def MS():
    from loghisto_b200.metric_system import MetricSystem
    made = []

    def make(max_histograms=16, precision=0):
        m = MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=4, precision=precision)
        made.append(m)
        return m
    yield make
    for m in made:
        m.close()


@pytest.fixture
def engines(lh):
    made = []

    def make(**kw):
        e = lh.Engine(device=0, **kw)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


def dense(hist):
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in hist.items():
        out[int(k) & 0xFFFF] = c
    return out


def status(lh, fn):
    with pytest.raises(lh.LhError) as e:
        fn()
    return e.value.status


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_known_spans_match_the_oracle(MS, spin, oracle, torch, precision):
    """Spans of 0 ns to 10 ms, each stopped with `out`: every duration covers its span, the raw buckets equal the
    oracle's compress of the returned durations, and the processed percentiles equal processHistograms of them."""
    ms = MS(precision=precision)
    st = torch.cuda.Stream()
    out = torch.zeros(len(SPANS), dtype=torch.int64, device="cuda")
    for i, ns in enumerate(SPANS):
        t = ms.StartGpuTimer("span", st)
        if ns:
            spin(ns, st)
        t.Stop(out=out[i:i + 1])
    torch.cuda.synchronize()
    durs = out.cpu().numpy()
    assert (durs >= np.array(SPANS)).all() and (durs < 1_000_000_000).all(), durs
    raw, m = ms.collect_and_process()
    want = oracle.ingest(durs.astype(np.float64), precision=precision)
    assert (dense(raw["Histograms"]["span"]) == want).all()
    ref = oracle.process_histogram(want, list(LABELS.values()), precision)
    assert m["span_count"] == ref["total"] == len(SPANS)
    for j, lab in enumerate(LABELS):
        assert m["span" + lab] == ref["pvals"][j], lab
    assert ms.dropped() == 0


def test_repeated_stop_adds_one_sample_each(engines, spin, oracle, torch, lh):
    """Go's Stop may be called repeatedly: three stops of one token after growing spins give three samples, each one
    sequence number and one lh_stats.samples, with non-decreasing durations from the same start."""
    e = engines(max_histograms=2)
    st = torch.cuda.Stream()
    out = torch.zeros(3, dtype=torch.int64, device="cuda")
    seq0, samples0 = e.ingest_seq(), e.stats()["samples"]
    t = e.gpu_timer_start(st)
    for i, ns in enumerate([10_000, 100_000, 1_000_000]):
        spin(ns, st)
        e.gpu_timer_stop(t, 1, st, out[i:i + 1])
    torch.cuda.synchronize()
    d = out.cpu().numpy()
    assert d[0] >= 10_000 and d[1] >= 110_000 and d[2] >= 1_110_000 and (np.diff(d) >= 0).all(), d
    assert e.ingest_seq() - seq0 == 3 and e.stats()["samples"] - samples0 == 3
    red, sp = e.snapshot([0.5])
    assert int(red.counts[1]) == 3 and int(red.counts[0]) == 0
    assert (dense(sp.histogram(1)) == oracle.ingest(d.astype(np.float64))).all()
    e.gpu_timer_release(t)


def test_stop_on_another_stream_waits_for_the_start(engines, spin, torch):
    """Stream A spins 50 ms, then starts; stream B stops at once with no ordering from the caller.  The library makes B
    wait for the start's mark, so the stop reads a written slot: a duration >= 0 and below the 50 ms spin."""
    e = engines(max_histograms=1)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    out = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    spin(MS50, a)
    t = e.gpu_timer_start(a)
    e.gpu_timer_stop(t, 0, b, out)
    torch.cuda.synchronize()
    assert 0 <= int(out.item()) < MS50
    e.gpu_timer_release(t)


def test_released_slot_is_reused_only_after_its_kernels(engines, spin, torch, lh):
    """Pool of one slot: a token started and stopped on A around a 50 ms spin is released at once.  Starting on idle B
    is refused (LH_ERR_RANGE, never a wait) until A's kernels have run, and then takes the slot without touching A's
    duration; a further start while B's token holds the slot is refused."""
    from loghisto_b200 import _lib
    e = engines(max_histograms=1)
    e.tune("gpu_timer_slots", 1)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    t = e.gpu_timer_start(a)
    spin(MS50, a)
    e.gpu_timer_stop(t, 0, a, out)
    e.gpu_timer_release(t)
    refused, deadline = 0, time.monotonic() + 10.0
    while True:
        try:
            t2 = e.gpu_timer_start(b)
            break
        except lh.LhError as x:
            assert x.status == _lib.LH_ERR_RANGE
            refused += 1
            assert time.monotonic() < deadline
            time.sleep(0.001)
    assert refused >= 1
    torch.cuda.synchronize()
    assert int(out.item()) >= MS50
    assert status(lh, lambda: e.gpu_timer_start(b)) == _lib.LH_ERR_RANGE
    assert status(lh, lambda: e.tune("gpu_timer_slots", 4)) == _lib.LH_ERR_STATE
    e.gpu_timer_stop(t2, 0, b)
    e.gpu_timer_release(t2)


def test_stale_and_foreign_handles_are_refused(engines, lh):
    from loghisto_b200 import _lib
    e1, e2 = engines(max_histograms=2), engines(max_histograms=2)
    t = e1.gpu_timer_start()
    e1.gpu_timer_release(t)
    assert status(lh, lambda: e1.gpu_timer_stop(t, 0)) == _lib.LH_ERR_INVALID
    assert status(lh, lambda: e1.gpu_timer_release(t)) == _lib.LH_ERR_INVALID
    t1 = e1.gpu_timer_start()
    t2 = e2.gpu_timer_start()
    assert status(lh, lambda: e2.gpu_timer_stop(t1, 0)) == _lib.LH_ERR_INVALID
    assert status(lh, lambda: e2.gpu_timer_release(t1)) == _lib.LH_ERR_INVALID
    forged = _lib.lh_gpu_timer(t1.handle ^ (1 << 20))   # another generation of the same slot
    assert status(lh, lambda: e1.gpu_timer_stop(forged, 0)) == _lib.LH_ERR_INVALID
    assert status(lh, lambda: e1.gpu_timer_stop(t1, 2)) == _lib.LH_ERR_RANGE
    e1.gpu_timer_stop(t1, 1)
    e2.gpu_timer_stop(t2, 0)
    # destroy with tokens outstanding
    for e in (e1, e2):
        assert e.lib.lh_destroy(e.h) == 0
        e.h = None


def test_capture_is_refused_and_records_nothing(engines, torch, lh):
    from loghisto_b200 import _lib
    e = engines(max_histograms=1)
    pre = e.gpu_timer_start()
    e.sync()
    seq0, samples0 = e.ingest_seq(), e.stats()["samples"]
    s = torch.cuda.Stream()
    x = torch.zeros(1, device="cuda")
    g = torch.cuda.CUDAGraph()
    got = []
    with torch.cuda.graph(g, stream=s):
        x.add_(1)
        got.append(status(lh, lambda: e.gpu_timer_start(s)))
        got.append(status(lh, lambda: e.gpu_timer_stop(pre, 0, s)))
    assert got == [_lib.LH_ERR_STATE, _lib.LH_ERR_STATE]
    g.replay()
    torch.cuda.synchronize()
    assert float(x.item()) == 1.0
    assert e.ingest_seq() == seq0 and e.stats()["samples"] == samples0
    red, _ = e.snapshot([0.5])
    assert int(red.counts[0]) == 0
    e.gpu_timer_release(pre)


def test_stop_after_a_snapshot_lands_in_the_next_interval(engines, lh):
    e = engines(max_histograms=1)
    t = e.gpu_timer_start()
    red, _ = e.snapshot([0.5])
    assert int(red.counts[0]) == 0
    e.gpu_timer_stop(t, 0)
    red, _ = e.snapshot([0.5])
    assert int(red.counts[0]) == 1
    e.gpu_timer_release(t)


def test_threads_on_their_own_streams_beside_a_collector(MS, spin, oracle, torch):
    """16 host threads, each on its own stream, start and stop timers while a collector loops.  Over all intervals the
    count equals the stops, and every bucket of every name equals the oracle's compress of the written durations."""
    ms = MS()
    n_threads, per = 16, 40
    streams = [torch.cuda.Stream() for _ in range(n_threads)]
    outs = torch.zeros((n_threads, per), dtype=torch.int64, device="cuda")
    done, errors, seen = threading.Event(), [], []

    def collector():
        try:
            while not done.is_set():
                seen.append(ms.collect_and_process()[0]["Histograms"])
        except Exception as x:   # noqa: BLE001 -- reported below
            errors.append(x)

    def worker(i):
        try:
            for k in range(per):
                t = ms.StartGpuTimer("w%d" % (i % 4), streams[i])
                spin((k % 5) * 2_000, streams[i])
                t.Stop(out=outs[i, k:k + 1])
        except Exception as x:   # noqa: BLE001
            errors.append(x)
    col = threading.Thread(target=collector)
    col.start()
    workers = [threading.Thread(target=worker, args=(i,)) for i in range(n_threads)]
    for w in workers:
        w.start()
    for w in workers:
        w.join()
    done.set()
    col.join()
    assert not errors, errors
    torch.cuda.synchronize()
    seen.append(ms.collect_and_process()[0]["Histograms"])
    d = outs.cpu().numpy()
    total = {}
    for hs in seen:
        for nm, h in hs.items():
            total[nm] = total.get(nm, np.zeros(65536, dtype=np.uint64)) + dense(h)
    assert sum(int(v.sum()) for v in total.values()) == n_threads * per
    for j in range(4):
        want = oracle.ingest(d[j::4].reshape(-1).astype(np.float64))
        assert (total["w%d" % j] == want).all(), j
    assert ms.dropped() == 0


def test_names_bind_at_stop_time(MS, torch):
    """A name idle long enough for its id to be recycled (and taken by another name) between start and stop still
    records under its name; a name that finds no free id is dropped and counted."""
    ms = MS(max_histograms=3)
    ms.Histogram("x", 1.0)
    t = ms.StartGpuTimer("x")
    for _ in range(4):
        ms.Histogram("y", 1.0)
        ms.collect_and_process()
    ms.Histogram("z", 1.0)
    t.Stop()
    raw, m = ms.collect_and_process()
    assert set(raw["Histograms"]) == {"x", "z"} and m["x_count"] == 1
    assert ms.dropped() == 0
    for nm in ("a", "b", "c"):      # x and z are live: at least two of these find no id, and the table is full
        ms.Histogram(nm, 1.0)
    before = ms.dropped()
    ms.StartGpuTimer("full").Stop()
    assert ms.dropped() - before == 1
    raw, _ = ms.collect_and_process()
    assert "full" not in raw["Histograms"]


def test_torch_default_stream_is_timed_as_itself(MS, spin, oracle, torch):
    """torch's default stream has handle 0, which the C ABI reads as the ingest stream.  A timer given that stream
    object must time the default stream: the span covers a 20 ms spin enqueued there."""
    ms = MS()
    cur = torch.cuda.current_stream()
    assert cur.cuda_stream == 0
    torch.cuda.synchronize()
    with ms.gpu_timer("dflt", cur):
        spin(20_000_000, 0)
    torch.cuda.synchronize()
    raw, _ = ms.collect_and_process()
    h = raw["Histograms"]["dflt"]
    assert sum(h.values()) == 1
    assert next(iter(h)) >= oracle.compress(20_000_000.0)
