"""The reference's own tests (metrics_test.go), replayed against the C++ MetricSystem mirror over the CUDA path,
plus a randomized comparison with the oracle's structure-faithful port."""
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture()
def MS():
    from loghisto_b200.metric_system import MetricSystem
    made = []

    def make(interval_s=1e-6, **kw):
        m = MetricSystem(interval_s, False, max_histograms=kw.get("max_histograms", 64), max_counters=kw.get("max_counters", 64))
        made.append(m)
        return m
    yield make
    for m in made:
        m.close()


def test_example_metric_system_keys(MS):
    # metrics_test.go:28-109: the key-naming contract of one counter, one histogram, one timer
    ms = MS()
    t = ms.StartTimer("submit_metrics")
    ms.Counter("range_splits", 1)
    ms.Histogram("some_ipc_latency", 123)
    t.Stop()
    ms.RegisterConstantGauge("sys.NumGoroutine", 7)
    sub = ms.SubscribeToProcessedMetrics(2)
    ms.Start()
    m = sub.receive(2.0)
    ms.Stop()
    assert m is not None
    for k in ("some_ipc_latency_99.9", "some_ipc_latency_max", "some_ipc_latency_count", "some_ipc_latency_agg_count",
              "some_ipc_latency_sum", "some_ipc_latency_avg", "some_ipc_latency_agg_avg", "range_splits",
              "range_splits_rate", "submit_metrics_sum", "sys.NumGoroutine"):
        assert k in m and m[k] != 0, k
    assert abs(m["some_ipc_latency_max"] - 122.965) < 1e-3      # bucket 482


def test_timer(MS):
    # metrics_test.go:183-200
    ms = MS()
    t1, t2 = ms.StartTimer("timer1"), ms.StartTimer("timer1")
    t1.Stop()
    time.sleep(5e-6)
    d2 = t2.Stop()
    t3 = ms.StartTimer("timer1")
    time.sleep(1e-5)
    t3.Stop()
    _, result = ms.collect_and_process()
    assert result["timer1_min"] <= result["timer1_50"] <= result["timer1_max"]
    assert result["timer1_count"] == 3 and d2 > 0


def test_rate(MS):
    # metrics_test.go:202-223
    ms = MS()
    ms.Counter("rate1", 777)
    _, m = ms.collect_and_process()
    assert m["rate1_rate"] == 777
    ms.Counter("rate1", 1223)
    _, m = ms.collect_and_process()
    assert m["rate1_rate"] == 1223
    ms.Counter("rate1", 1223)
    ms.Counter("rate1", 1223)
    _, m = ms.collect_and_process()
    assert m["rate1_rate"] == 2446


def test_counter(MS):
    # metrics_test.go:225-240
    ms = MS()
    ms.Counter("counter1", 3290)
    _, m = ms.collect_and_process()
    assert m["counter1"] == 3290
    ms.Counter("counter1", 10000)
    _, m = ms.collect_and_process()
    assert m["counter1"] == 13290
    _, m = ms.collect_and_process()
    assert m["counter1"] == 13290 and "counter1_rate" not in m


def test_processed_broadcast(MS):
    # metrics_test.go:289-319
    ms = MS()
    sub = ms.SubscribeToProcessedMetrics(128)
    ms.Histogram("histogram1", 33)
    ms.Histogram("histogram1", 59)
    ms.Histogram("histogram1", 330000)
    ms.Start()
    m = sub.receive(2.0)
    assert m is not None
    assert int(m["histogram1_sum"]) == 331132
    assert int(m["histogram1_agg_avg"]) == 110377
    assert int(m["histogram1_count"]) == 3
    sub.unsubscribe()
    ms.Stop()


def test_raw_broadcast(MS):
    # metrics_test.go:321-346
    ms = MS()
    sub = ms.SubscribeToRawMetrics(128)
    ms.Counter("counter2", 10)
    ms.Counter("counter2", 111)
    ms.Start()
    raw = sub.receive(2.0)
    assert raw["Counters"]["counter2"] == 121 and raw["Rates"]["counter2"] == 121
    sub.unsubscribe()
    ms.Stop()


def test_slow_subscriber_is_closed_not_blocked_on(MS):
    # metrics.go:570-580: a subscriber that misses twice is closed; the reaper never blocks
    ms = MS()
    sub = ms.SubscribeToProcessedMetrics(1)
    ms.Start()
    # long enough for the reaper to send once and miss twice even where one collection takes a few hundred ms
    # (a host whose CPU quota throttles the process); receiving earlier would drain the channel between its passes
    time.sleep(2.0)
    got = sub.receive(0.5)           # the one buffered set
    assert got is not None
    with pytest.raises(EOFError):
        for _ in range(5):
            sub.receive(0.2)
    ms.Stop()


def test_stop_is_idempotent_and_leaves_no_thread(MS):
    import threading
    before = threading.active_count()
    ms = MS()
    ms.Start()
    ms.Stop()
    ms.Stop()
    assert threading.active_count() == before


def test_mixed_ops_match_oracle_port(MS, oracle):
    """Random Histogram/Counter/Timer-like traffic over 40 names and three intervals: every raw bucket, counter,
    rate and processed metric equals the oracle's port of metrics.go (sums to 1e-12, the rest exactly)."""
    rng = np.random.default_rng(3)
    ms = MS(max_histograms=64, max_counters=64)
    ref = oracle.OracleMetricSystem()
    custom = {"%s_p10": 0.1, "%s_median": 0.5, "%s_p100": 1.0, "%s_bogus": 1.5}
    ms.SpecifyPercentiles(custom)
    ref.SpecifyPercentiles(custom)
    for interval in range(3):
        n = 20000
        names = ["h%d" % i for i in rng.integers(0, 40, n)]
        vals = np.where(rng.random(n) < 0.02, -1.0, 1.0) * np.exp(rng.uniform(-8, 44, n))
        for nm, v in zip(names, vals):
            ms.Histogram(nm, float(v))
            ref.Histogram(nm, float(v))
        for i in rng.integers(0, 20, 3000):
            amt = int(rng.integers(0, 2 ** 40))
            ms.Counter("c%d" % i, amt)
            ref.Counter("c%d" % i, amt)
        raw, m = ms.collect_and_process()
        rraw, rm = ref.collect_and_process()
        assert raw["Histograms"] == rraw["Histograms"]
        assert raw["Counters"] == rraw["Counters"] and raw["Rates"] == rraw["Rates"]
        got_keys = {k for k in m if not k.endswith(("_agg_avg", "_agg_count", "_agg_sum"))}
        ref_keys = {k for k in rm if not k.endswith(("_agg_avg", "_agg_count", "_agg_sum"))}
        assert got_keys == ref_keys
        assert not any(k.endswith("_bogus") for k in m)          # p = 1.5: percentile() errors, key omitted
        for k in got_keys:
            if k.endswith(("_sum", "_avg")):
                assert abs(m[k] - rm[k]) <= 1e-12 * abs(rm[k]), k
            else:
                assert m[k] == rm[k], k
    assert ms.dropped() == 0


def test_names_beyond_capacity_are_dropped_and_counted(MS):
    ms = MS(max_histograms=4, max_counters=4)
    for i in range(6):
        ms.Histogram("h%d" % i, 1.0)
        ms.Counter("c%d" % i, 1)
    raw, _ = ms.collect_and_process()
    assert len(raw["Histograms"]) == 4 and len(raw["Counters"]) == 4
    assert ms.dropped() == 4



def test_per_call_api_parity_and_rate(MS):
    """The per-call path an instrumented service uses -- Histogram(name, value) once per sample from many threads
    (thread-local name cache, one staging shard per thread) -- must land every sample in exactly the bucket the
    oracle's structure-faithful port puts it in (lho_ms_histogram: metrics.go:273-295)."""
    import os
    import numpy as np
    from oracle import oracle as o
    o.build()
    H, n, threads = 64, 20_000_000, min(32, os.cpu_count() or 1)
    names = ["histogram%d" % i for i in range(H)]
    ms = MS(interval_s=3600.0, max_histograms=H)
    dt = ms.histogram_stream(names, o.STREAM_L, o.DEFAULT_SEED, 12345, n, threads)
    raw, metrics = ms.collect_and_process()
    want = o.stream_ingest_keyed(o.STREAM_L, n, H, o.DEFAULT_SEED, val_start=12345, ids_start=12345)
    # a few samples through the oracle's own MetricSystem port as well: same name -> same bucket
    oms = o.OracleMetricSystem()
    vals = o.gen_stream(o.STREAM_L, 1000, o.DEFAULT_SEED, start=12345)
    ids = o.gen_ids(0, 1000, H, o.DEFAULT_SEED, start=12345)
    for i in range(1000):
        oms.Histogram(names[ids[i]], float(vals[i]))
    oraw, _ = oms.collect_and_process()
    oms.close()
    for name, buckets in oraw["Histograms"].items():
        for k, c in buckets.items():
            assert raw["Histograms"][name].get(k, 0) >= c
    assert ms.dropped() == 0
    for h in range(H):
        got = np.zeros(65536, dtype=np.uint64)
        for k, c in raw["Histograms"].get(names[h], {}).items():
            got[k & 0xFFFF] = c
        assert (got == want[h]).all(), h
        assert metrics[names[h] + "_count"] == float(want[h].sum())
    print("per-call Histogram(): %d calls from %d threads in %.3f s = %.1f M calls/s" % (n, threads, dt, n / dt / 1e6))


def test_counter_zero_amount_appears_in_rates(MS):
    """metrics.go:430-433: a counter touched this interval is in Rates even when only Counter(name, 0) was called."""
    ms = MS()
    ms.Counter("quiet", 0)
    ms.Counter("busy", 5)
    raw, metrics = ms.collect_and_process()
    assert raw["Rates"] == {"quiet": 0, "busy": 5}
    assert metrics["quiet_rate"] == 0.0 and metrics["quiet"] == 0.0
    raw, _ = ms.collect_and_process()
    assert raw["Rates"] == {} and raw["Counters"] == {"quiet": 0, "busy": 5}


@pytest.mark.parametrize("shard_lock", ["0", "1"])
def test_collects_race_with_per_call_ingest(MS, monkeypatch, shard_lock):
    """The same race as tests/test_host_logic_cpu.py, against the real library: 24 threads call Histogram() while the
    main thread collects in a loop; 8 exclusive shards (membarrier handshake; shard_lock=1: spin-locked fallback) plus
    the shared overflow shards.  The union of all intervals must be the oracle's histogram, nothing dropped."""
    import threading
    import numpy as np
    from oracle import oracle as o
    o.build()
    monkeypatch.setenv("LOGHISTO_B200_SHARDS", "8")
    monkeypatch.setenv("LOGHISTO_B200_STAGING_BYTES", "262144")
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", shard_lock)
    H, n = 16, 12_000_000
    names = ["name%d" % i for i in range(H)]
    ms = MS(interval_s=3600.0, max_histograms=H)
    total = np.zeros((H, 65536), dtype=np.uint64)

    def add(raw):
        for h in range(H):
            for k, c in raw["Histograms"].get(names[h], {}).items():
                total[h, k & 0xFFFF] += c

    collects = 0
    for rnd in range(2):
        t = threading.Thread(target=ms.histogram_stream, args=(names, o.STREAM_U, o.DEFAULT_SEED, rnd * n, n, 24))
        t.start()
        while t.is_alive():
            raw, _ = ms.collect_and_process()
            add(raw)
            collects += 1
        t.join()
        raw, _ = ms.collect_and_process()
        add(raw)
    want = o.stream_ingest_keyed(o.STREAM_U, 2 * n, H, o.DEFAULT_SEED)
    assert collects >= 2 and ms.dropped() == 0
    assert int(total.sum()) == 2 * n
    assert (total == want).all()
