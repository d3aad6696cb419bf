"""Pin the CPU oracle against every known-answer vector the reference holds for
the ingest + reduction path (SURVEY.md section 8c, KAT-1..KAT-6).

All citations are <file>:<line> in the reference repository; nothing here reads it.
"""
import math

import numpy as np
import pytest

# KAT-5: full-precision decompress() outputs printed by real Go runs.
# readme.md:35-43 and print_benchmark.go:34-39.  Go prints %v = shortest
# round-trip repr, so each literal identifies exactly one float64.
GO_PRINTED = [
    (1702, 2.4642914167480484e+07), (850, 4913.768840299134), (691, 1001.2472422902518),
    (428, 71.24044000732538), (422, 67.03348428941965), (420, 65.68633104092515),
    (416, 63.07152259993664), (409, 58.739891704145194), (-649, -657.5233632152207),
    (1750, 3.982478339757623e+07), (1747, 3.864778314316012e+07), (1505, 3.4366224772310276e+06),
    (1452, 2.0228126576114902e+06), (1306, 469769.7083161708), (1177, 129313.15075081984),
]


def test_kat5_decompress_bit_exact(oracle):
    L = oracle.lib()
    for k, v in GO_PRINTED:
        assert L.lho_decompress(k) == v, k
        # the pure-Go exp restatement reproduces them too (documented in DESIGN.md)
        assert L.lho_decompress_purego(k) == v, k
        # and compress() maps every printed value back to its bucket
        assert oracle.compress(v) == k


def test_kat5_glibc_would_fail():
    # evidence that the KAT discriminates: glibc's exp misses readme.md:39 (bucket 422)
    assert math.exp(4.22) - 1.0 != 67.03348428941965


def test_kat1_processed_broadcast(oracle):
    # metrics_test.go:289-319
    ms = oracle.OracleMetricSystem()
    for v in (33, 59, 330000):
        ms.Histogram("histogram1", v)
    raw, m = ms.collect_and_process()
    assert raw["Histograms"]["histogram1"] == {353: 1, 409: 1, 1271: 1}
    assert int(m["histogram1_sum"]) == 331132
    assert int(m["histogram1_agg_avg"]) == 110377
    assert int(m["histogram1_count"]) == 3


def test_kat2_percentile(oracle):
    # metrics_test.go:111-149
    metrics = {10: 9000, 25: 900, 33: 90, 47: 9, 500: 1}
    expected = {0: 10, .99: 25, .999: 33, .9991: 47, .9999: 47, 1: 500}
    total = sum(metrics.values())
    for p, e in expected.items():
        r = oracle.percentile(total, list(metrics.keys()), list(metrics.values()), p)
        assert r == e  # the rule is exact selection; the reference only asks for 1%
    with pytest.raises(ValueError):
        oracle.percentile(total, list(metrics.keys()), list(metrics.values()), 1.5)
    with pytest.raises(ValueError):
        oracle.percentile(total, list(metrics.keys()), list(metrics.values()), float("nan"))


def test_kat3_compress_roundtrip(oracle):
    # metrics_test.go:151-172
    expect = {-421408208120481: -3367, -1: -69, 0: 0, 1: 69, 214141241241241: 3300}
    for f, k in expect.items():
        assert oracle.compress(f) == k
        result = oracle.decompress(oracle.compress(f))
        diff = abs(f - result) if result == 0 else abs(f / result - 1)
        assert diff <= .01


def test_kat4_example(oracle):
    # metrics_test.go:34-37: Histogram(..., 123) -> bucket 482
    assert oracle.compress(123) == 482
    assert abs(oracle.decompress(482) - 122.965) < 1e-3


def test_kat6_counters_and_rates(oracle):
    # metrics_test.go:202-240, 321-346
    ms = oracle.OracleMetricSystem()
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
    assert m["rate1"] == 777 + 1223 + 2446

    ms = oracle.OracleMetricSystem()
    ms.Counter("counter1", 3290)
    _, m = ms.collect_and_process()
    assert m["counter1"] == 3290
    ms.Counter("counter1", 10000)
    _, m = ms.collect_and_process()
    assert m["counter1"] == 13290

    ms = oracle.OracleMetricSystem()
    ms.Counter("counter2", 10)
    ms.Counter("counter2", 111)
    raw, _ = ms.collect_and_process()
    assert raw["Counters"]["counter2"] == 121 and raw["Rates"]["counter2"] == 121
    # untouched counter: still exported cumulatively, no rate (metrics.go:430-457)
    raw, m = ms.collect_and_process()
    assert raw["Counters"]["counter2"] == 121 and "counter2" not in raw["Rates"]
    assert "counter2_rate" not in m


def test_compress_edge_semantics(oracle):
    # amd64 float->int16 (CVTTSD2SL, low 16 bits): SURVEY.md section 8a row a1
    c = oracle.compress
    assert c(float("nan")) == 0 and c(float("inf")) == 0 and c(float("-inf")) == 0
    assert c(-0.0) == 0 and c(0.0) == 0
    assert c(0.005012520859401071) == 1 and c(0.00501) == 0
    assert c(-0.005012520859401071) == -1
    assert c(0.9837718355371597) == 69
    assert c(9.193239032374088e18) == 4367
    assert c(1e142) == 32697
    assert c(2.03e142) == -32768       # wraps through int16 (metrics.go:312-315 "fails")
    assert c(-2.03e142) == -32768      # -1 * -32768 wraps back to -32768
    assert c(1.7976931348623157e308) == 70978 - 65536


def test_go_log_matches_libm_to_1ulp(oracle):
    L = oracle.lib()
    rng = np.random.default_rng(7)
    xs = np.exp(rng.uniform(0, 700, 20000))
    bad = 0
    for x in xs:
        a, b = L.lho_go_log(float(x)), math.log(float(x))
        assert abs(a - b) <= abs(b) * 2.3e-16
        bad += a != b
    assert bad < 0.05 * xs.size


def test_histogram_absent_when_untouched_and_interval_delta(oracle):
    # metrics.go:460-463: histogram cache is swapped, so a second collection is empty
    ms = oracle.OracleMetricSystem()
    ms.Histogram("h", 5.0)
    raw, m = ms.collect_and_process()
    assert "h" in raw["Histograms"] and m["h_count"] == 1
    raw, m = ms.collect_and_process()
    assert raw["Histograms"] == {} and "h_count" not in m and "h_agg_count" not in m
    ms.Histogram("h", 7.0)
    raw, m = ms.collect_and_process()
    assert m["h_count"] == 1 and m["h_agg_count"] == 2


def test_dense_ingest_equals_map_port(oracle):
    vals = oracle.gen_stream(oracle.STREAM_S, 200000)
    dense = oracle.ingest(vals)
    ms = oracle.OracleMetricSystem()
    L = oracle.lib()
    for v in vals[:20000]:
        L.lho_ms_histogram(ms._h, b"x", float(v))
    raw, _ = ms.collect_and_process()
    dense2 = oracle.ingest(vals[:20000])
    got = np.zeros(65536, dtype=np.uint64)
    for k, c in raw["Histograms"]["x"].items():
        got[k & 0xFFFF] = c
    assert (got == dense2).all()
    assert dense.sum() == vals.size
    mt = oracle.ingest(vals, threads=4)
    assert (mt == dense).all()


def test_streams_shape(oracle):
    u = oracle.gen_stream(oracle.STREAM_U, 100000)
    assert u.min() >= 1.0 and u.max() < 2.0 ** 63
    keys = oracle.compress_many(u)
    assert keys.min() >= 69 and keys.max() <= 4367
    l = oracle.gen_stream(oracle.STREAM_L, 100000)
    kl = oracle.compress_many(l)
    assert 300 < np.unique(kl).size < 700
    # generator is index-addressable: shards concatenate to the whole
    a = oracle.gen_stream(oracle.STREAM_U, 1000, start=0)
    b = oracle.gen_stream(oracle.STREAM_U, 500, start=500)
    assert (a[500:] == b).all()
