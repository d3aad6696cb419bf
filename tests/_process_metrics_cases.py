"""processMetrics on RawMetricSets the system did not collect, driven through the Python face of the C++ MetricSystem
mirror.  Shared by tests/test_reduce_sparse_cpu.py (mirror over the oracle-backed stub of the C ABI) and
tests/test_gpu_reduce_sparse.py (mirror over the CUDA library).  `MS(**kw)` makes a MetricSystem."""
import math


def same(a: dict, b: dict) -> bool:
    """Equal metric dicts, NaN equal to NaN."""
    if a.keys() != b.keys():
        return False
    return all(x == y or (math.isnan(x) and math.isnan(y)) for x, y in ((a[k], b[k]) for k in a))


def histogram_metrics(m: dict, name: str) -> dict:
    """The metrics processHistograms produced for `name`: _count / _sum / _avg and the percentile labels, no aggregates."""
    return {k: v for k, v in m.items() if k.startswith(name + "_") and not k.startswith(name + "_agg_")
            and not k.endswith("_rate")}


def check_kat1_bare_keys(MS):
    """metrics_test.go:289-319 (33, 59, 330000 -> buckets 353, 409, 1271) as a hand-built set: no samples, just keys."""
    ms = MS()
    m = ms.processMetrics({"Histograms": {"histogram1": {353: 1, 409: 1, 1271: 1}}}, aggregates=True)
    assert int(m["histogram1_sum"]) == 331132
    assert m["histogram1_count"] == 3
    assert int(m["histogram1_agg_avg"]) == 110377
    assert m["histogram1_max"] > m["histogram1_min"]


def check_union_of_two_systems(MS):
    """The histogram maps of two systems' raw sets, summed key by key, reduce to what one system that saw every sample
    reports."""
    a, b, both = MS(), MS(), MS()
    va = [0.5 * i for i in range(1, 400)]
    vb = [float(i) ** 1.5 for i in range(1, 700)] + [-3.0, 0.0]
    for v in va:
        a.Histogram("lat", v)
        both.Histogram("lat", v)
    for v in vb:
        b.Histogram("lat", v)
        b.Histogram("only_b", -v)
        both.Histogram("lat", v)
        both.Histogram("only_b", -v)
    ra, _ = a.collect_and_process()
    rb, _ = b.collect_and_process()
    _, want = both.collect_and_process()
    union = {}
    for raw in (ra, rb):
        for name, hist in raw["Histograms"].items():
            u = union.setdefault(name, {})
            for k, c in hist.items():
                u[k] = u.get(k, 0) + c
    got = a.processMetrics({"Histograms": union})
    for name in ("lat", "only_b"):
        assert same(histogram_metrics(got, name), histogram_metrics(want, name)), name


def check_empty_map(MS):
    """A name with an empty map: processHistograms gives count 0, sum 0, avg 0/0 and no percentile."""
    ms = MS()
    m = ms.processMetrics({"Histograms": {"empty": {}}, "Counters": {"c": 5}, "Gauges": {"g": 1.5}})
    assert m["empty_count"] == 0 and m["empty_sum"] == 0 and math.isnan(m["empty_avg"])
    assert set(histogram_metrics(m, "empty")) == {"empty_count", "empty_sum", "empty_avg"}
    assert m["c"] == 5 and m["g"] == 1.5


def check_collected_set_fed_back(MS):
    """A collected raw dict, processed again through processMetrics, gives the metrics collect_and_process gave."""
    ms = MS()
    for i in range(1, 300):
        ms.Histogram("h1", i * 1.25)
        ms.Histogram("h2", -float(i) ** 2)
    ms.Counter("c1", 12)
    ms.RegisterConstantGauge("g1", 2.5)
    raw, want = ms.collect_and_process()
    assert same(ms.processMetrics(raw), want)
