"""lh_reduce_sparse_host (`k_scatter_segments` + K3 `k_reduce` + `k_sparse_epilogue` + `k_clear_touched` on the call's
own scratch rows) against the Go-map reference of tests/_go_map_reference.py, against the snapshot path
(round trip of an export, aggregation of many exports), beside a live snapshot, and through the C++ mirror.

Bar as tests/test_gpu_reduce.py: percentile keys exact, values bit-exact against the decompress table, counts exact,
sums within the rounding bound of the summation (rc.sum_ok), averages bit-exact as sum / float64(count)."""
import ctypes
import math
import random
import threading

import numpy as np
import pytest

import _process_metrics_cases as pmc
import _reduce_cases as rc
from _go_map_reference import GoMapReference
from test_gpu_reduce import check_reduced

pytestmark = pytest.mark.gpu

SEED = 0x5BA25E
PS = [0.0, -0.0, -math.inf, 1e-9, 0.25, 0.5, 0.9, 0.99, 0.999, 1.0, 1.5, math.nan]
BATCH = 256                      # K6_BATCH scratch rows of the library


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


def zero_count_cases(precision: int) -> list:
    """Maps with keys whose merged count is 0 (both rules of k_sparse_epilogue)."""
    w = rc.window(precision)
    return [
        ("zero_below", {-5: 0, 0: 3, 7: 2}),
        ("zero_inside", {0: 3, 4: 0, 7: 2}),
        ("zero_outside_window", {-w - 3: 0, 0: 3, w - 1: 1}),
        ("zero_min_key", {-32768: 0, 5: 4}),                   # -Inf at precision 46: NaN sum, p <= 0 -> -32768
        ("zero_plus_inf", {32767: 0, 5: 4, -3: 2}),            # +Inf at precision 46: NaN sum
        ("zero_both_ends", {-32768: 0, -32767: 0, 32767: 0, 1: 1}),
        ("all_zero", {1: 0, -2: 0}),
        ("empty", {}),
    ]


def split_entries(hist: dict, rng: random.Random) -> list:
    """(key, count) entries whose counts sum, mod 2^64, to each bucket's count: 1 to 3 per bucket, some wrapping."""
    out = []
    for k, c in hist.items():
        parts = rng.randrange(1, 4)
        if parts == 1:
            out.append((k, c))
            continue
        wrap = rng.random() < 0.5
        cuts = [rng.randrange(2 ** 64) if wrap else rng.randrange(c + 1) for _ in range(parts - 1)]
        if not wrap:
            cuts = sorted(cuts)
            bounds = [0] + cuts + [c]
            out += [(k, b - a) for a, b in zip(bounds, bounds[1:])]
        else:
            out += [(k, x) for x in cuts] + [(k, (c - sum(cuts)) % 2 ** 64)]
    rng.shuffle(out)
    return out


def csr(hists: list, rng: random.Random):
    offsets, keys, counts = [0], [], []
    for hist in hists:
        for k, c in split_entries(hist, rng):
            keys.append(k)
            counts.append(c)
        offsets.append(len(keys))
    return np.array(offsets, np.uint32), np.array(keys, np.int16), np.array(counts, np.uint64)


def wrapped_zero_count_cases(precision: int) -> list:
    """Wrapped maps with zero-count keys: with a total of 0 a key before the first non-empty one has ratio 0/0.0 = NaN,
    so p <= 0 answers the first non-empty key; with a wrapped total above 0 it answers the smallest key present."""
    w, H = rc.window(precision), 2 ** 63
    return [
        ("wrap0_zero_keys", {-9: 0, -7: H, 9: H, 20: 0}),
        ("wrap0_zero_keys_outside", {-w - 3: 0, -7: H, 5: 0, 9: H}),
        ("wrap5_zero_keys", {-9: 0, -7: H, -3: H, 9: 5}),
    ]


@pytest.mark.parametrize("precision", rc.PRECISIONS)
def test_constructed_cases_as_split_shuffled_segments(lh, oracle, precision):
    table = oracle.decompress_table(precision)
    cases = [(c["name"], c["hist"]) for c in rc.make_cases(precision, table, SEED)] + zero_count_cases(precision)
    wrapped = [(c["name"], c["hist"]) for c in rc.make_wrapped_cases(precision, table, SEED)]
    wrapped += wrapped_zero_count_cases(precision)
    pool = rc.percentile_pool([{"hist": h} for _, h in cases], table, SEED)
    pool += rc.wrapped_percentile_pool([{"hist": h} for _, h in wrapped if all(h.values())], table, SEED)
    cases += wrapped
    refs = [GoMapReference(h, table, name) for name, h in cases]
    assert refs[-3].percentile(0.0) == -7 and refs[-1].percentile(0.0) == -9
    batches = rc.percentile_batches(pool)
    rng = random.Random(SEED + precision)
    with lh.Engine(device=0, max_histograms=1, max_counters=1, precision=precision) as eng:
        for r, ps in enumerate(batches):
            offsets, keys, counts = csr([h for _, h in cases], rng)     # a new split and order every time
            red = eng.reduce_sparse(offsets, keys, counts, ps)
            check_reduced(red, refs, ps, table, (precision, r))
        st = eng.stats()
        assert st["samples"] == 0 and st["snapshots"] == 0


def bits(a) -> np.ndarray:
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def assert_identical(got, want, what):
    for f in ("counts", "sums", "avgs", "pkeys", "pvals"):
        assert np.array_equal(bits(getattr(got, f)), bits(getattr(want, f))), (what, f)


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_export_round_trip_is_bit_identical(lh, precision):
    H, n = 64, 1 << 20
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng:
        for i, kind in enumerate((lh.STREAM_U, lh.STREAM_L, lh.STREAM_S)):
            d_v = eng.gen_stream(kind, n, SEED + i)
            d_i = eng.gen_ids_u16(0, n, H, SEED + i)
            eng.ingest_keyed_f64_u16(d_i, d_v, n)
        eng.sync()
        red, sp = eng.snapshot(PS)
        assert int(red.counts.sum()) == 3 * n
        assert_identical(eng.reduce_sparse(sp, PS), red, precision)


def exports(lh, n_exports: int, H: int, n: int) -> list:
    """n_exports snapshots of H histograms of stream U, one seed each (the exports of as many hosts)."""
    out = []
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        for e in range(n_exports):
            d_v = eng.gen_stream(lh.STREAM_U, n, SEED + 17 * e)
            d_i = eng.gen_ids_u16(0, n, H, SEED + 17 * e)
            eng.ingest_keyed_f64_u16(d_i, d_v, n)
            _, sp = eng.snapshot([], export=True)
            out.append(sp)
    return out


def concatenate(sps: list, H: int):
    """Segment h = histogram h of every export, one after the other."""
    offsets, keys, counts = [0], [], []
    for h in range(H):
        for sp in sps:
            a, b = int(sp.offsets[h]), int(sp.offsets[h + 1])
            keys.append(sp.keys[a:b])
            counts.append(sp.counts[a:b])
        offsets.append(offsets[-1] + sum(int(sp.offsets[h + 1]) - int(sp.offsets[h]) for sp in sps))
    return np.array(offsets, np.uint32), np.concatenate(keys), np.concatenate(counts)


def test_aggregation_of_many_exports(lh):
    """16 exports of 1024 histograms, concatenated per name, against merging the same triples into a fresh engine and
    reducing its snapshot: bit-identical.  1024 segments are four scratch batches; the engine with max_histograms = 1
    shows the call is not bounded by it."""
    H, n_exports = 1024, 16
    sps = exports(lh, n_exports, H, 1 << 22)
    offsets, keys, counts = concatenate(sps, H)
    assert H > BATCH
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as ref:
        ids = np.repeat(np.arange(H, dtype=np.uint32), np.diff(offsets.astype(np.int64)))
        ref.merge_counts_host(ids, keys, counts)
        want, _ = ref.snapshot(PS, export=False)
        assert_identical(ref.reduce_sparse(offsets, keys, counts, PS), want, "H=1024 engine")
    with lh.Engine(device=0, max_histograms=1, max_counters=1) as small:
        assert_identical(small.reduce_sparse(offsets, keys, counts, PS), want, "H=1 engine")
        # a subset of the segments, on both sides of the scratch batch boundaries
        sel = np.array([0, 1, 255, 256, 257, 511, 1023], np.int64)
        sub_off = np.concatenate([[0], np.cumsum(np.diff(offsets.astype(np.int64))[sel])]).astype(np.uint32)
        sub_keys = np.concatenate([keys[offsets[h]:offsets[h + 1]] for h in sel])
        sub_counts = np.concatenate([counts[offsets[h]:offsets[h + 1]] for h in sel])
        got = small.reduce_sparse(sub_off, sub_keys, sub_counts, PS)
        assert np.array_equal(got.counts, want.counts[sel]) and np.array_equal(bits(got.pvals), bits(want.pvals[sel]))


def test_isolation_from_a_live_snapshot(lh, oracle):
    """Between the reduction and the export of an open snapshot, while another thread ingests the next interval, the call
    runs several times: the snapshot's reduction and export, and the next interval's counts, are the oracle's."""
    H, n = 64, 1 << 21
    ps = [0.0, 0.5, 0.99, 1.0]
    want1 = oracle.stream_ingest_keyed(lh.STREAM_U, n, H, lh.DEFAULT_SEED)
    want2 = oracle.stream_ingest_keyed(lh.STREAM_U, n, H, lh.DEFAULT_SEED, val_start=n, ids_start=n)
    rng = random.Random(SEED)
    foreign = [{rng.randrange(-3000, 3000): rng.randrange(1, 2 ** 30) for _ in range(rng.randrange(1, 900))}
               for _ in range(300)]
    offsets, keys, counts = csr(foreign, rng)
    table = oracle.decompress_table(100)
    refs = [GoMapReference(h, table, "foreign %d" % i) for i, h in enumerate(foreign)]
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        d_v = eng.gen_stream(lh.STREAM_U, n, lh.DEFAULT_SEED)
        d_i = eng.gen_ids_u16(0, n, H, lh.DEFAULT_SEED)
        eng.ingest_keyed_f64_u16(d_i, d_v, n)
        d_v2 = eng.gen_stream(lh.STREAM_U, n, lh.DEFAULT_SEED, start=n)
        d_i2 = eng.gen_ids_u16(0, n, H, lh.DEFAULT_SEED, start=n)
        eng.sync()
        eng.snapshot_begin()
        try:
            red = eng.snapshot_reduce(ps)
            t = threading.Thread(target=lambda: (eng.ingest_keyed_f64_u16(d_i2, d_v2, n), eng.sync()))
            t.start()
            for _ in range(3):
                check_reduced(eng.reduce_sparse(offsets, keys, counts, ps), refs, ps, table, "foreign")
            t.join()
            sp = eng.snapshot_export()
        finally:
            eng.snapshot_end()
        red2, sp2 = eng.snapshot(ps)
    for want, r, s, what in ((want1, red, sp, "open snapshot"), (want2, red2, sp2, "next interval")):
        got = np.zeros((H, 65536), dtype=np.uint64)
        got[np.repeat(np.arange(H), np.diff(s.offsets.astype(np.int64))), s.keys.view(np.uint16)] = s.counts
        assert np.array_equal(got, want), what
        for h in range(H):
            o = oracle.process_histogram(want[h], ps)
            assert int(r.counts[h]) == o["total"] and np.array_equal(r.pkeys[h], o["pkeys"]), (what, h)


def test_invalid_arguments(lh):
    with lh.Engine(device=0, max_histograms=4, max_counters=1) as eng:
        offsets, keys, counts = np.array([0, 2, 3], np.uint32), np.array([1, 2, 3], np.int16), np.ones(3, np.uint64)
        ps = np.zeros(33)
        out = [np.zeros(2, np.uint64), np.zeros(2), np.zeros(2), np.zeros(66, np.int32), np.zeros(66)]
        outp = [a.ctypes.data for a in out]
        f = eng.lib.lh_reduce_sparse_host
        bad = np.array([0, 3, 2], np.uint32)
        assert f(eng.h, 2, bad.ctypes.data, keys.ctypes.data, counts.ctypes.data, ps.ctypes.data, 1, *outp) == -1
        assert f(eng.h, 2, offsets.ctypes.data, keys.ctypes.data, counts.ctypes.data, ps.ctypes.data, 33, *outp) == -1
        assert f(eng.h, 2, offsets.ctypes.data, None, counts.ctypes.data, ps.ctypes.data, 1, *outp) == -1
        assert f(eng.h, 2, offsets.ctypes.data, keys.ctypes.data, None, ps.ctypes.data, 1, *outp) == -1
        assert f(eng.h, 2, None, keys.ctypes.data, counts.ctypes.data, ps.ctypes.data, 1, *outp) == -1
        assert f(eng.h, 0, None, None, None, None, 0, None, None, None, None, None) == 0
        assert not out[0].any()
        red = eng.reduce_sparse(offsets, keys, counts, [0.5, 1.0])
        assert list(red.counts) == [2, 1] and list(red.pkeys[:, 1]) == [2, 3]
        eng.merge_counts_host(np.zeros(1, np.uint32), np.array([7], np.int16), np.array([5], np.uint64))
        r, _ = eng.snapshot([0.5], export=False)
        assert int(r.counts[0]) == 5 and int(r.pkeys[0, 0]) == 7


@pytest.fixture()
def MS():
    from loghisto_b200.metric_system import MetricSystem
    made = []

    def make(interval_s=3600.0, **kw):
        m = MetricSystem(interval_s, False, max_histograms=kw.get("max_histograms", 64), max_counters=kw.get("max_counters", 64))
        made.append(m)
        return m
    yield make
    for m in made:
        m.close()


def test_mirror_kat1_bare_keys(MS):
    pmc.check_kat1_bare_keys(MS)


def test_mirror_union_of_two_systems(MS):
    pmc.check_union_of_two_systems(MS)


def test_mirror_empty_map(MS):
    pmc.check_empty_map(MS)


def test_mirror_collected_set_fed_back(MS):
    pmc.check_collected_set_fed_back(MS)


def test_mirror_wrapped_count(MS, oracle):
    """processMetrics of a hand-built set whose counts sum past 2^64: _count is the uint64 total (wrapped), _avg is
    sum / float64(count), a percentile above 1 is emitted where Go's ratio reaches it, and the aggregate count store
    adds the wrapped count."""
    table = oracle.decompress_table(100)
    hist = {-1800: 2 ** 63, -10: 2 ** 63, 3000: 5}
    ms = MS()
    ms.SpecifyPercentiles({"%s_p50": 0.5, "%s_p150": 1.5, "%s_pbig": 1e18})
    ref = GoMapReference(hist, table)
    assert ref.count == 5 and ref.percentile(1.5) == -1800 and ref.percentile(1e18) == -1800
    m = ms.processMetrics({"Histograms": {"lat": hist}}, aggregates=True)
    assert m["lat_count"] == 5.0
    assert rc.sum_ok(m["lat_sum"], ref) and rc.same_bits(m["lat_avg"], rc.avg_of(m["lat_sum"], ref))
    for label in ("p50", "p150", "pbig"):
        assert m["lat_" + label] == float(table[-1800 & 0xFFFF]), label
    assert m["lat_agg_count"] == 5.0
    # a total of 0: no _agg_ metrics (the store holds 0), every percentile but NaN answers the first bucket
    m = ms.processMetrics({"Histograms": {"zero": {-7: 2 ** 63, 9: 2 ** 63}}}, aggregates=True)
    assert m["zero_count"] == 0.0 and math.isinf(m["zero_avg"])
    assert m["zero_p50"] == m["zero_p150"] == float(table[-7 & 0xFFFF])
    assert "zero_agg_count" not in m
    m = ms.processMetrics({"Histograms": {"lat": hist}}, aggregates=True)
    assert m["lat_agg_count"] == 10.0
