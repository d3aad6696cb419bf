"""Parity of the CUDA hot path (through the C ABI) against the CPU oracle.

Bar: bit-exact for bucket counts, bucket keys, counters and chosen percentile
buckets; decompressed values bit-exact against the oracle's restatement of
Go's exp; interval sums within the rounding-error bound of a float64 sum, in
any order, of the exact sum (the reference itself sums in random map order,
metrics.go:342; tests/_reduce_cases.py sum_ok).
"""
import numpy as np
import pytest

import _reduce_cases as rc

pytestmark = pytest.mark.gpu

SEED = 0x10C415C0
PS = [0.0, 0.5, 0.75, 0.9, 0.95, 0.99, 0.999, 0.9999, 1.0]


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def eng(lh):
    e = lh.Engine(device=0, max_histograms=4, max_counters=64)
    yield e
    e.close()


def dense_from_sparse(sp, hid):
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in sp.histogram(hid).items():
        out[k & 0xFFFF] = c
    return out


def thresholds(oracle, kmax):
    """T[k] = smallest positive double (as bits) whose bucket is >= k, for k = 1..kmax, by bisection on the oracle."""
    ks = np.arange(1, kmax + 1, dtype=np.int64)
    lo = np.zeros(ks.size, dtype=np.uint64)                      # compress(lo) < k
    hi = np.full(ks.size, 0x7FEFFFFFFFFFFFFF, dtype=np.uint64)   # max double: pre-wrap key 70978 >= k
    def pre_wrap(bits):
        # un-wrapped bucket number of a positive finite double: monotone in the bit pattern
        v = bits.view(np.float64)
        k16 = oracle.compress_many(v).astype(np.int64) & 0xFFFF
        approx = np.floor(100.0 * np.log1p(v) + 0.5)
        wraps = np.round((approx - k16) / 65536.0)
        return k16 + wraps.astype(np.int64) * 65536
    for _ in range(64):
        mid = lo + (hi - lo) // np.uint64(2)
        ge = pre_wrap(mid) >= ks
        hi = np.where(ge, mid, hi)
        lo = np.where(ge, lo, mid)
    return hi


def test_stream_generators_match(eng, lh, oracle):
    for kind in (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S, lh.STREAM_C, lh.STREAM_Z):
        d = eng.gen_stream(kind, 100003, SEED, start=12345)
        eng.sync()
        got = d.to_host().view(np.uint64)
        want = oracle.gen_stream(kind, 100003, SEED, start=12345).view(np.uint64)
        assert (got == want).all(), kind
        d.free()
    for kind in (0, 1):
        d = eng.gen_ids_u16(kind, 50001, 1024, SEED, start=7)
        eng.sync()
        assert (d.to_host().astype(np.uint32) == oracle.gen_ids(kind, 50001, 1024, SEED, start=7)).all()
        d.free()


@pytest.mark.parametrize("mode", [0, 1])
def test_compress_streams(eng, lh, oracle, mode):
    for kind in (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S):
        vals = oracle.gen_stream(kind, 1_000_000, SEED)
        got = eng.compress(vals, mode)
        want = oracle.compress_many(vals)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (kind, vals[bad[:5]], got[bad[:5]], want[bad[:5]])


def test_compress_edge_values(eng, oracle):
    specials = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072014e-308,
                         0.00501, 0.005012520859401071, -0.005012520859401071, 0.51, -0.51, 1.0, -1.0, 33, 59,
                         330000, 123, -421408208120481, 214141241241241, 2.0 ** 63, -(2.0 ** 63), 2.0 ** 63 * (1 - 2 ** -53),
                         9.193239032374088e18, 1e142, -1e142, 2.03e142, -2.03e142, 1e200, 1.7976931348623157e308,
                         -1.7976931348623157e308, 4.9e18, 1e19, 1.8446744073709552e19], dtype=np.float64)
    for mode in (0, 1):
        got = eng.compress(specials, mode)
        want = oracle.compress_many(specials)
        assert (got == want).all(), (mode, specials[got != want], got[got != want], want[got != want])


def test_compress_at_every_threshold(eng, oracle):
    """Every bucket boundary of the whole finite range, +-3 ulps, both signs, both evaluators."""
    T = thresholds(oracle, 70978)
    # sanity against SURVEY.md section 7 spot values
    assert T[0] == np.float64(0.005012520859401071).view(np.uint64)
    assert T[68] == np.float64(0.9837718355371597).view(np.uint64)
    assert T[4366] == np.float64(9.193239032374088e18).view(np.uint64)
    offs = np.arange(-3, 4, dtype=np.int64)
    bits = (T[:, None].astype(np.int64) + offs[None, :]).reshape(-1).astype(np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(0x8000000000000000)])
    vals = bits.view(np.float64)
    want = oracle.compress_many(vals)
    for mode in (0, 1):
        got = eng.compress(vals, mode)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (mode, bad.size, vals[bad[:5]], got[bad[:5]], want[bad[:5]])


def test_fast_path_margin(eng, lh):
    """The FP32 estimate must stay well inside LH_FAST_EPS = 2^-12 bucket units of the true value."""
    n = 50_000_000
    for kind in (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S):
        d = eng.gen_stream(kind, n, SEED ^ 0x55)
        err, slow = eng.fastpath_margin(d, n)
        e1, e2 = eng.fastpath_margin_detail()          # fast_candidate / packed-FP32 estimator of K1
        d.free()
        print("fast-path estimate error, stream %d: estimator1 %.3e estimator2 %.3e bucket units (EPS = %.3e)"
              % (kind, e1, e2, 2.0 ** -12))
        assert err == max(e1, e2)
        assert err < 2.0 ** -13, (kind, err)          # < EPS/2
        if kind != lh.STREAM_S:
            assert slow < n * 2.5 * 2.0 ** -12, (kind, slow)   # about 2*EPS of the samples fall back


def test_decompress_table_bit_exact(eng, oracle):
    tab = eng.decompress_table()
    L = oracle.lib()
    want = np.array([L.lho_decompress(int(np.int16(np.uint16(i)))) for i in range(65536)])
    assert (tab.view(np.uint64) == want.view(np.uint64)).all()


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_ingest_single_every_variant(eng, lh, oracle, offset):
    n = 1_000_003
    vals = oracle.gen_stream(lh.STREAM_S, n + 8, SEED ^ offset)
    want = oracle.ingest(vals[offset:offset + n])
    d = eng.upload(vals)
    default = eng.lib.lh_k1_variant_current(eng.h)
    for vi, name in enumerate(eng.k1_variants()):
        if name.startswith("probe"):
            continue
        eng.tune("k1", vi)
        eng.ingest_f64(2, d.offset(offset), n)
        red, sp = eng.snapshot(PS)
        got = dense_from_sparse(sp, 2)
        assert (got == want).all(), (name, offset, np.nonzero(got != want)[0][:10])
        assert int(red.counts[2]) == n and int(red.counts[0]) == 0
    eng.tune("k1", default)
    d.free()


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 31, 1023, 4097, 65537])
def test_ingest_single_ragged_sizes(eng, lh, oracle, n):
    vals = oracle.gen_stream(lh.STREAM_S, n + 4, SEED + n)
    d = eng.upload(vals)
    default = eng.lib.lh_k1_variant_current(eng.h)
    for vi, name in enumerate(eng.k1_variants()):
        if name.startswith("probe"):
            continue
        eng.tune("k1", vi)
        eng.ingest_f64(0, d.offset(1), n)
        red, sp = eng.snapshot(PS)
        assert (dense_from_sparse(sp, 0) == oracle.ingest(vals[1:1 + n])).all(), (n, vi)
        assert int(red.counts[0]) == n
    eng.tune("k1", default)
    d.free()


def test_reduce_matches_oracle(eng, lh, oracle):
    table = oracle.decompress_table()
    for kind in (lh.STREAM_U, lh.STREAM_L, lh.STREAM_S):
        n = 2_000_000
        vals = oracle.gen_stream(kind, n, SEED ^ 0x77)
        d = eng.upload(vals)
        eng.ingest_f64(1, d, n)
        red, sp = eng.snapshot(PS + [1.5, float("nan"), -0.25])
        d.free()
        want = oracle.ingest(vals)
        ref = oracle.process_histogram(want, PS + [1.5, float("nan"), -0.25])
        assert int(red.counts[1]) == ref["total"]
        assert (red.pkeys[1] == ref["pkeys"]).all()
        good = ref["pkeys"] != np.iinfo(np.int32).min
        assert good.sum() == len(PS) + 1        # p > 1 and NaN error out, negative p selects the minimum
        assert (red.pvals[1][good].view(np.uint64) == ref["pvals"][good].view(np.uint64)).all()
        assert np.isnan(red.pvals[1][~good]).all()
        assert rc.sum_ok(float(red.sums[1]), rc.Reference(rc.sparse(want), table))
        assert rc.same_bits(red.avgs[1], red.sums[1] / float(n))          # metrics.go:356
        assert abs(red.avgs[1] - ref["avg"]) <= 1e-12 * abs(ref["avg"])
        # empty histograms: count 0, avg NaN, every percentile absent
        assert int(red.counts[3]) == 0 and np.isnan(red.avgs[3]) and (red.pkeys[3] == np.iinfo(np.int32).min).all()


def test_reference_percentile_kat(eng, oracle):
    """metrics_test.go:111-149 (TestPercentile) replayed through ingest + reduce."""
    metrics = {10: 9000, 25: 900, 33: 90, 47: 9, 500: 1}
    vals = np.concatenate([np.full(c, float(v)) for v, c in metrics.items()])
    expected = {0: 10, .99: 25, .999: 33, .9991: 47, .9999: 47, 1: 500}
    eng.ingest_f64_host(0, vals)
    red, _ = eng.snapshot(list(expected.keys()))
    for j, (p, e) in enumerate(expected.items()):
        assert red.pkeys[0][j] == oracle.compress(e), p
        assert abs(e / red.pvals[0][j] - 1) <= .01       # the reference's own tolerance


def test_reference_processed_broadcast_kat(eng):
    """metrics_test.go:289-319: 33, 59, 330000 -> sum 331132, count 3."""
    eng.ingest_f64_host(0, np.array([33.0, 59.0, 330000.0]))
    red, sp = eng.snapshot(PS)
    assert sp.histogram(0) == {353: 1, 409: 1, 1271: 1}
    assert int(red.sums[0]) == 331132 and int(red.counts[0]) == 3


def test_keyed_ingest(lh, oracle):
    H, n = 1024, 1_000_000
    with lh.Engine(device=0, max_histograms=H, max_counters=8) as e:
        vals = oracle.gen_stream(lh.STREAM_S, n, SEED ^ 3)
        for kind in (0, 1):
            ids = oracle.gen_ids(kind, n, H, SEED ^ 3)
            want = oracle.ingest_keyed(ids, vals, H)
            d_v = e.upload(vals)
            d_i16 = e.upload(ids.astype(np.uint16))
            d_i32 = e.upload(ids)
            e.ingest_keyed_f64_u16(d_i16, d_v, n)
            red, sp = e.snapshot(PS)
            assert (red.counts == want.sum(axis=1)).all()
            for h in (0, 1, 511, 1023):
                assert (dense_from_sparse(sp, h) == want[h]).all(), h
            assert int(sp.offsets[-1]) == int((want != 0).sum())
            e.ingest_keyed_f64_u32(d_i32, d_v, n)
            red2, sp2 = e.snapshot(PS)
            assert (sp2.keys == sp.keys).all() and (sp2.counts == sp.counts).all() and (sp2.offsets == sp.offsets).all()
            # percentiles of every histogram against the oracle
            for h in (0, 17, 1023):
                ref = oracle.process_histogram(want[h], PS)
                assert (red.pkeys[h] == ref["pkeys"]).all()
            for x in (d_v, d_i16, d_i32):
                x.free()
        # out-of-range ids are dropped and counted, never written
        ids = np.array([0, 5, 2000, 1023, 65535], dtype=np.uint16)
        e.ingest_keyed_f64_u16_host(ids, np.array([1.0, 2.0, 3.0, 4.0, 5.0]))
        red, _ = e.snapshot(PS)
        assert int(red.counts.sum()) == 3 and e.stats()["dropped"] == 2


def test_timer_samples_i64(lh, oracle):
    """TimerToken.Stop: Histogram(name, float64(duration.Nanoseconds())), metrics.go:242-246 (negatives occur)."""
    H, n = 16, 300_000
    rng = np.random.default_rng(5)
    ns = np.concatenate([rng.integers(-5000, 5000, n // 3), rng.integers(0, 10 ** 9, n // 3),
                         rng.integers(-2 ** 62, 2 ** 62, n - 2 * (n // 3))]).astype(np.int64)
    ns[:4] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1]
    ids = rng.integers(0, H, n).astype(np.uint32)
    want = oracle.ingest_keyed_i64(ids, ns, H)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_n, d_i = e.upload(ns), e.upload(ids.astype(np.uint16))
        e.ingest_keyed_i64ns_u16(d_i, d_n, n)
        _, sp = e.snapshot(PS)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want[h]).all(), h


def test_timer_samples_host_fed_and_misaligned_counters(lh, oracle):
    """Host-fed timer samples (lh_ingest_keyed_i64ns_u16_host) and the vectorised counter kernel at every
    alignment / ragged size (vector body + scalar head and tail)."""
    H, C, n = 7, 200, 300_003
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, SEED ^ 3).view(np.int64).copy()
    ns[::97] *= -1                                    # negative durations happen (readme.md:43)
    ids = oracle.gen_ids(0, n, H, SEED ^ 3)
    want = oracle.ingest_keyed_i64(ids, ns, H)
    with lh.Engine(device=0, max_histograms=H, max_counters=C) as e:
        e.ingest_keyed_i64ns_u16_host(ids.astype(np.uint16), ns)
        _, sp = e.snapshot(PS)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want[h]).all(), h
        rng = np.random.default_rng(5)
        cids = rng.integers(0, C, n + 8).astype(np.uint32)
        amts = rng.integers(0, 2 ** 63, n + 8).astype(np.uint64) * np.uint64(2) + np.uint64(1)
        d_i, d_a = e.upload(cids.astype(np.uint16)), e.upload(amts)
        for off, m in ((0, n), (1, n - 1), (3, 65_537), (4, 16_384), (5, 5)):
            e.counter_add_u16(d_i.offset(off), d_a.offset(off), m)
            _, sp = e.snapshot(PS)
            assert (sp.counter_deltas == oracle.counter_add(cids[off:off + m], amts[off:off + m], C)).all(), (off, m)


def test_counters(eng, oracle):
    n = 500_000
    rng = np.random.default_rng(11)
    ids = rng.integers(0, 64, n).astype(np.uint32)
    amounts = rng.integers(0, 2 ** 63, n).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64)
    want = oracle.counter_add(ids, amounts, 64)     # wraps mod 2^64 like atomic.AddUint64
    d_i16, d_i32, d_a = eng.upload(ids.astype(np.uint16)), eng.upload(ids), eng.upload(amounts)
    eng.counter_add_u16(d_i16, d_a, n)
    _, sp = eng.snapshot(PS)
    assert (sp.counter_deltas == want).all()
    eng.counter_add_u32(d_i32, d_a, n)
    eng.counter_add_u16_host(ids.astype(np.uint16), amounts)
    _, sp = eng.snapshot(PS)
    assert (sp.counter_deltas == want * np.uint64(2)).all()
    # metrics_test.go:202-223 (TestRate): deltas 777, 1223, 2446
    for adds, rate in (([777], 777), ([1223], 1223), ([1223, 1223], 2446)):
        eng.counter_add_u16_host(np.full(len(adds), 9, np.uint16), np.array(adds, np.uint64))
        _, sp = eng.snapshot(PS)
        assert int(sp.counter_deltas[9]) == rate and int(sp.counter_deltas.sum()) == rate


def test_snapshot_interval_semantics(eng, lh, oracle):
    """Swap-and-clear (metrics.go:460-463): a second snapshot is empty; ingest during a snapshot lands in the next."""
    vals = oracle.gen_stream(lh.STREAM_L, 100_000, SEED)
    d = eng.upload(vals)
    eng.ingest_f64(0, d, 60_000)
    eng.snapshot_begin()
    eng.ingest_f64(0, d.offset(60_000), 40_000)          # arrives while the snapshot is open
    red = eng.snapshot_reduce(PS)
    first = eng.snapshot_copy_histogram(0)
    with pytest.raises(lh.LhError):
        eng.snapshot_begin()                              # one at a time
    eng.snapshot_end()
    assert int(red.counts[0]) == 60_000 and (first == oracle.ingest(vals[:60_000])).all()
    red, sp = eng.snapshot(PS)
    assert int(red.counts[0]) == 40_000 and (dense_from_sparse(sp, 0) == oracle.ingest(vals[60_000:])).all()
    red, sp = eng.snapshot(PS)
    assert int(red.counts.sum()) == 0 and int(sp.offsets[-1]) == 0
    with pytest.raises(lh.LhError):
        eng.snapshot_reduce(PS)                           # no snapshot open
    d.free()


def test_async_snapshot_pipeline(eng, lh, oracle):
    """lh_snapshot_reduce_async / lh_snapshot_result: the reduction of interval k is collected after interval
    k+1's ingest has been launched; two tickets may be in flight, older ones expire."""
    vals = oracle.gen_stream(lh.STREAM_U, 300_000, SEED ^ 0x21)
    d = eng.upload(vals)
    handles = []
    for i in range(3):
        eng.ingest_f64(1, d.offset(i * 100_000), 100_000)
        eng.snapshot_begin()
        handles.append(eng.snapshot_reduce_async(PS))
        eng.snapshot_end()
    for i in (1, 2):
        red = eng.snapshot_result(handles[i])
        ref = oracle.process_histogram(oracle.ingest(vals[i * 100_000:(i + 1) * 100_000]), PS)
        assert int(red.counts[1]) == 100_000 and (red.pkeys[1] == ref["pkeys"]).all()
        assert (red.pvals[1].view(np.uint64) == ref["pvals"].view(np.uint64)).all()
    with pytest.raises(lh.LhError):
        eng.snapshot_result(handles[0])        # its slot was reused by the third ticket
    assert eng.kernel_ms(eng.ingest_seq()) > 0 and eng.kernel_ms(eng.ingest_seq() - 2) > 0
    d.free()


def test_host_and_staging_paths(lh, oracle):
    n = 3_000_017
    vals = oracle.gen_stream(lh.STREAM_S, n, SEED ^ 9)
    ids = oracle.gen_ids(0, n, 8, SEED ^ 9).astype(np.uint16)
    with lh.Engine(device=0, max_histograms=8, max_counters=8, staging_bytes=4 << 20, staging_slots=2) as e:
        # pageable host memory, many chunks through a 2-slot ring
        e.ingest_f64_host(3, vals)
        e.ingest_keyed_f64_u16_host(ids, vals)
        # pinned host memory
        pv = e.pinned(n, np.float64)
        pv.array[:] = vals
        e.ingest_f64_host(3, pv.array)
        # staging ring, as the cgo shim would drive it
        done = 0
        while done < n:
            s = e.staging_acquire()
            cap = (int(s.bytes) // 10) & ~15
            m = min(cap, n - done)
            e.staging_view(s, np.float64, m)[:] = vals[done:done + m]
            e.staging_view(s, np.uint16, m, byte_offset=cap * 8)[:] = ids[done:done + m]
            e.staging_commit_keyed_f64_u16(s, m, cap * 8)
            done += m
        s = e.staging_acquire()
        e.staging_view(s, np.float64, 1000)[:] = vals[:1000]
        e.staging_commit_f64(s, 3, 1000)
        s = e.staging_acquire()
        e.staging_abandon(s)
        red, sp = e.snapshot(PS)
        keyed = oracle.ingest_keyed(ids.astype(np.uint32), vals, 8)
        single = oracle.ingest(vals)
        for h in range(8):
            want = keyed[h] * np.uint64(2)
            if h == 3:
                want = want + single * np.uint64(2) + oracle.ingest(vals[:1000])
            assert (dense_from_sparse(sp, h) == want).all(), h
        st = e.stats()
        assert st["h2d_bytes"] >= n * 8 * 2 + n * 10 * 2
        pv.free()


def test_full_size_properties(lh, oracle):
    """BASELINE config 2 size (1e9 samples, 8 GB): linearity and conservation across ragged pieces and kernels, then the
    whole histogram against the oracle."""
    n = 1_000_000_000
    with lh.Engine(device=0, max_histograms=3, max_counters=1) as e:
        d = e.gen_stream(lh.STREAM_U, n, SEED)
        e.ingest_f64(0, d, n)                                   # one call
        cuts = [0, 1, 333_333_335, 900_000_002, n]
        default = e.lib.lh_k1_variant_current(e.h)
        for vi, (a, b) in zip((0, 1, 2, 3), zip(cuts[:-1], cuts[1:])):   # ragged pieces, different kernels
            e.tune("k1", vi)
            e.ingest_f64(1, d.offset(a), b - a)
        e.tune("k1", default)
        # the first 2e6 samples again, checked against the oracle
        e.ingest_f64(2, d, 2_000_000)
        red, sp = e.snapshot(PS)
        assert int(red.counts[0]) == n and int(red.counts[1]) == n
        h0, h1 = sp.histogram(0), sp.histogram(1)
        assert h0 == h1
        assert min(h0) >= 69 and max(h0) <= 4367 and len(h0) == 4367 - 69 + 1
        assert (red.pkeys[0] == red.pkeys[1]).all() and red.sums[0] == red.sums[1]
        assert (np.diff(red.pkeys[0]) >= 0).all()
        want = oracle.ingest(oracle.gen_stream(lh.STREAM_U, 2_000_000, SEED))
        got = np.zeros(65536, dtype=np.uint64)
        for k, c in sp.histogram(2).items():
            got[k & 0xFFFF] = c
        assert (got == want).all()
        # ... and the WHOLE 1e9-sample histogram bucket for bucket: the oracle regenerates the stream on every host core
        want_full = oracle.stream_ingest(lh.STREAM_U, n, SEED)
        assert (dense_from_sparse(sp, 0) == want_full).all()
        ref = oracle.process_histogram(want_full, PS)
        assert (red.pkeys[0] == ref["pkeys"]).all() and int(red.counts[0]) == ref["total"] == n
        d.free()


def test_full_size_keyed_1024(lh, oracle):
    """BASELINE configs[2] at full size: 1024 keyed histograms x 1e9 (id, value) pairs, every bucket of every
    histogram against the oracle (which regenerates both streams on every host core), for the default dispatch."""
    H, n = 1024, 1_000_000_000
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_v = e.gen_stream(lh.STREAM_U, n, SEED)
        d_i = e.gen_ids_u16(0, n, H, SEED)
        e.ingest_keyed_f64_u16(d_i, d_v, n)
        red, sp = e.snapshot(PS)
        want = oracle.stream_ingest_keyed(lh.STREAM_U, n, H, SEED)
        got = np.zeros((H, 65536), dtype=np.uint64)
        got[np.repeat(np.arange(H), np.diff(sp.offsets.astype(np.int64))), sp.keys.view(np.uint16)] = sp.counts
        assert (got == want).all(), e.keyed_kernel_name()
        assert (red.counts == want.sum(axis=1)).all()
        for h in (0, 511, 1023):
            assert (red.pkeys[h] == oracle.process_histogram(want[h], PS)["pkeys"]).all()


def test_mixed_ops_interval_pipeline(lh, oracle):
    """BASELINE config 5 in miniature: Histogram + Timer + Counter batches over 1024 names, one snapshot per batch,
    snapshots pipelined behind the next batch; every interval must equal the oracle on exactly its own ops."""
    H, C, n = 1024, 1024, 400_000
    nh, nt = n // 2, n // 4
    nc = n - nh - nt
    with lh.Engine(device=0, max_histograms=H, max_counters=C) as e:
        handles, wants = [], []
        for it in range(3):
            base = it * n
            d_ids = e.gen_ids_u16(0, n, H, SEED, start=base)
            d_v = e.gen_stream(lh.STREAM_L, nh, SEED, start=base)
            d_ns = e.gen_stream(lh.STREAM_TIMER_NS, nt, SEED, start=base + nh)
            d_amt = e.gen_stream(lh.STREAM_AMOUNTS, nc, SEED, start=base + nh + nt)
            e.ingest_keyed_f64_u16(d_ids, d_v, nh)
            e.ingest_keyed_i64ns_u16(d_ids.offset(nh), d_ns, nt)
            e.counter_add_u16(d_ids.offset(nh + nt), d_amt, nc)
            e.snapshot_begin()
            handles.append(e.snapshot_reduce_async(PS))
            sp = e.snapshot_export() if it == 2 else None
            e.snapshot_end()
            ids = oracle.gen_ids(0, n, H, SEED, start=base)
            want = oracle.ingest_keyed(ids[:nh], oracle.gen_stream(oracle.STREAM_L, nh, SEED, start=base), H)
            ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, nt, SEED, start=base + nh).view(np.int64)
            oracle.ingest_keyed_i64(ids[nh:nh + nt], ns, H, counts=want)
            amounts = oracle.gen_stream(oracle.STREAM_AMOUNTS, nc, SEED, start=base + nh + nt).view(np.uint64)
            wc = oracle.counter_add(ids[nh + nt:], amounts, C)
            wants.append((want, wc))
            for x in (d_ids, d_v, d_ns, d_amt):
                pass   # buffers stay alive until the launches have run (freed after the loop via GC + sync)
            e.sync()
        for it in (1, 2):
            red = e.snapshot_result(handles[it])
            want, _ = wants[it]
            assert (red.counts == want.sum(axis=1)).all()
            for h in (0, 500, 1023):
                ref = oracle.process_histogram(want[h], PS)
                assert (red.pkeys[h] == ref["pkeys"]).all()
        want, wc = wants[2]
        assert (sp.counter_deltas == wc).all()
        for h in (0, 77, 1023):
            assert (dense_from_sparse(sp, h) == want[h]).all()


@pytest.mark.parametrize("chunk,spt,flush", [(65536, 6, 24576), (1 << 20, 6, 4096), (1 << 20, 4, 65536), (65536, 3, 24576), (1 << 20, 8, 16384)])
def test_keyed_owner_partitioned_kernel(lh, oracle, chunk, spt, flush):
    """The owner-partitioned write-combining keyed kernel (bin -> per-owner buffers -> per-(owner, writer) queues ->
    shared-memory windows) against the oracle: several chunks (grid barriers, queue parity), signed/edge values,
    skewed ids, out-of-range ids, and a single-id stream that overflows one owner's buffer and queue and must fall
    back without losing a sample."""
    H, n = 1024, 1_500_001
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        e.tune("keyed_mode", 2)
        e.tune("wc_spt", spt)
        e.tune("kp_chunk", chunk)
        e.tune("wc_flush", flush)       # 65536 samples between flushes overflows the owner buffers: the exact route must absorb it
        for stream, idkind in ((lh.STREAM_S, 0), (lh.STREAM_U, 1), (lh.STREAM_L, 0)):
            vals = oracle.gen_stream(stream, n, SEED ^ 0x31)
            ids = oracle.gen_ids(idkind, n, H, SEED ^ 0x31)
            want = oracle.ingest_keyed(ids, vals, H)
            d_v, d_i16, d_i32 = e.upload(vals), e.upload(ids.astype(np.uint16)), e.upload(ids)
            e.ingest_keyed_f64_u16(d_i16, d_v, n)
            assert e.keyed_kernel_name() == "k_ingest_keyed_wc"
            red, sp = e.snapshot(PS)
            assert (red.counts == want.sum(axis=1)).all(), (stream, idkind)
            for h in (0, 1, 147, 148, 500, 1023):
                assert (dense_from_sparse(sp, h) == want[h]).all(), (stream, h)
            e.ingest_keyed_f64_u32(d_i32, d_v, n)
            red2, sp2 = e.snapshot(PS)
            assert (sp2.counts == sp.counts).all() and (sp2.keys == sp.keys).all()
            for x in (d_v, d_i16, d_i32):
                x.free()
        # timer samples through the same kernel
        ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, SEED).view(np.int64)
        ids = oracle.gen_ids(0, n, H, SEED)
        want = oracle.ingest_keyed_i64(ids, ns, H)
        d_n, d_i = e.upload(ns), e.upload(ids.astype(np.uint16))
        e.ingest_keyed_i64ns_u16(d_i, d_n, n)
        red, _ = e.snapshot(PS)
        assert (red.counts == want.sum(axis=1)).all()
        # Histogram samples and Timer samples of one batch in ONE launch (lh_ingest_keyed_pair_u16): the chunk slices
        # straddle the float64 / int64 boundary; lengths chosen so that both segments leave ragged ends
        nf, nn = n - 12_345, n - 777
        vals = oracle.gen_stream(lh.STREAM_S, nf, SEED ^ 9)
        ids_f = oracle.gen_ids(0, nf, H, SEED ^ 9)
        want = oracle.ingest_keyed(ids_f, vals, H) + oracle.ingest_keyed_i64(ids[:nn], ns[:nn], H)
        d_vf, d_if = e.upload(vals), e.upload(ids_f.astype(np.uint16))
        e.ingest_keyed_pair_u16(d_if, d_vf, nf, d_i, d_n, nn)
        assert e.keyed_kernel_name() == "k_ingest_keyed_wc"
        red, sp = e.snapshot(PS)
        assert (red.counts == want.sum(axis=1)).all()
        for h in (0, 3, 146, 147, 640, 1023):
            assert (dense_from_sparse(sp, h) == want[h]).all(), h
        e.ingest_keyed_pair_u16(d_if, d_vf, nf, d_i, d_n, 0)          # either side may be empty
        e.ingest_keyed_pair_u16(d_if, d_vf, 0, d_i, d_n, nn)
        red2, sp2 = e.snapshot(PS)
        assert (sp2.counts == sp.counts).all() and (sp2.keys == sp.keys).all()
        # one id only: its owner's queue overflows, the surplus takes the L2 route; ids >= H are dropped
        vals = oracle.gen_stream(lh.STREAM_U, n, SEED ^ 5)
        ids = np.full(n, 777, dtype=np.uint32)
        ids[::1000] = 60000
        d_v, d_i = e.upload(vals), e.upload(ids.astype(np.uint16))
        before = e.stats()["dropped"]
        e.ingest_keyed_f64_u16(d_i, d_v, n)
        red, sp = e.snapshot(PS)
        keep = ids == 777
        assert (dense_from_sparse(sp, 777) == oracle.ingest(vals[keep])).all()
        assert int(red.counts.sum()) == int(keep.sum()) and e.stats()["dropped"] - before == int((~keep).sum())


def test_concurrent_ingest_and_snapshots_from_threads(lh, oracle):
    """Every lh_* entry point is thread-safe (metrics.go: Histogram/Counter are called from any goroutine while the
    reaper snapshots): 6 ingest threads + 1 snapshot thread; the sum over all snapshots must equal the oracle."""
    import threading
    H, per, rounds, nthreads = 8, 50_000, 12, 6
    vals = oracle.gen_stream(lh.STREAM_S, per * rounds * nthreads, SEED ^ 0x99)
    ids = oracle.gen_ids(0, vals.size, H, SEED ^ 0x99)
    with lh.Engine(device=0, max_histograms=H, max_counters=4, staging_bytes=1 << 20, staging_slots=4) as e:
        total = np.zeros((H, 65536), dtype=np.uint64)
        counters = np.zeros(4, dtype=np.uint64)
        stop = threading.Event()
        errors = []

        def ingest(t):
            try:
                for r in range(rounds):
                    a = (t * rounds + r) * per
                    if r % 3 == 0:
                        e.ingest_f64_host(t % H, vals[a:a + per])
                    elif r % 3 == 1:
                        e.ingest_keyed_f64_u16_host(ids[a:a + per].astype(np.uint16), vals[a:a + per])
                    else:
                        d_v, d_i = e.upload(vals[a:a + per]), e.upload(ids[a:a + per])
                        e.ingest_keyed_f64_u32(d_i, d_v, per)
                        e.sync()
                        d_v.free(); d_i.free()
                    e.counter_add_u16_host(np.array([t % 4], np.uint16), np.array([r + 1], np.uint64))
            except Exception as ex:   # pragma: no cover
                errors.append(ex)

        def snapshots():
            try:
                while not stop.is_set():
                    _, sp = e.snapshot(PS)
                    for h in range(H):
                        total[h] += dense_from_sparse(sp, h)
                    counters[:] += sp.counter_deltas
            except Exception as ex:   # pragma: no cover
                errors.append(ex)

        ths = [threading.Thread(target=ingest, args=(t,)) for t in range(nthreads)]
        snap = threading.Thread(target=snapshots)
        snap.start()
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        stop.set()
        snap.join()
        assert not errors, errors
        _, sp = e.snapshot(PS)
        for h in range(H):
            total[h] += dense_from_sparse(sp, h)
        counters += sp.counter_deltas
        want = np.zeros((H, 65536), dtype=np.uint64)
        wc = np.zeros(4, dtype=np.uint64)
        for t in range(nthreads):
            for r in range(rounds):
                a = (t * rounds + r) * per
                if r % 3 == 0:
                    want[t % H] += oracle.ingest(vals[a:a + per])
                else:
                    want += oracle.ingest_keyed(ids[a:a + per], vals[a:a + per], H)
                wc[t % 4] += r + 1
        assert (total == want).all() and (counters == wc).all()


def test_tune_and_error_paths(eng, lh):
    with pytest.raises(lh.LhError):
        eng.tune("k1", 10_000)
    with pytest.raises(lh.LhError):
        eng.tune("no_such_key", 1)
    with pytest.raises(lh.LhError):
        eng.ingest_f64(99, 8, 1)              # histogram id out of range
    with pytest.raises(lh.LhError):
        eng.ingest_f64(0, 4, 16)              # misaligned device pointer
    with pytest.raises(lh.LhError):
        eng.snapshot_reduce(list(np.linspace(0, 1, 40)))   # more than LH_MAX_PERCENTILES
    assert "histogram_id" in eng.lib.lh_last_error(eng.h).decode() or True
    # counter adds with amounts or ids not naturally aligned are refused before any launch: nothing runs or counts
    d_i16, d_i32 = eng.upload(np.zeros(8, np.uint16)), eng.upload(np.zeros(8, np.uint32))
    d_a = eng.upload(np.ones(8, np.uint64))
    eng.snapshot(PS)
    launches = eng.stats()["kernel_launches"]
    for add, ids, amounts in ((eng.counter_add_u16, d_i16.ptr, d_a.ptr + 4), (eng.counter_add_u32, d_i32.ptr, d_a.ptr + 4),
                              (eng.counter_add_u32, d_i32.ptr + 2, d_a.ptr)):
        with pytest.raises(lh.LhError):
            add(ids, amounts, 4)
    assert eng.stats()["kernel_launches"] == launches
    assert not eng.snapshot(PS)[1].counter_deltas.any()
    eng.tune("k1_reserve_sms", 3)
    eng.tune("k1_reserve_sms", 0)


def test_merge_sparse_snapshots(lh, oracle):
    """Snapshots are mergeable: exporting two engines' histograms and merging them into a third gives exactly the
    histogram of the concatenated streams (uint64 sums, including counts beyond 2^32 and wrapped keys)."""
    H, n = 8, 400_000
    vals = oracle.gen_stream(lh.STREAM_S, 2 * n, SEED ^ 0x44)
    ids = oracle.gen_ids(0, 2 * n, H, SEED ^ 0x44)
    parts = []
    for half in range(2):
        with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
            a = half * n
            e.ingest_keyed_f64_u16_host(ids[a:a + n].astype(np.uint16), vals[a:a + n])
            _, sp = e.snapshot(PS)
            hid = np.repeat(np.arange(H, dtype=np.uint32), np.diff(sp.offsets))
            parts.append((hid, sp.keys.copy(), sp.counts.copy()))
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        for hid, keys, counts in parts:
            e.merge_counts_host(hid, keys, counts)
        e.merge_counts_host(np.array([3, 3, 99], np.uint32), np.array([-32768, 7, 1], np.int16),
                            np.array([2 ** 40, 2 ** 63, 5], np.uint64))      # big counts; id 99 is dropped
        red, sp = e.snapshot(PS)
        want = oracle.ingest_keyed(ids, vals, H)
        want[3][(-32768) & 0xFFFF] += np.uint64(2 ** 40)
        want[3][7] += np.uint64(2 ** 63)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want[h]).all(), h
        assert (red.counts == want.sum(axis=1)).all() and e.stats()["dropped"] == 1
        ref = oracle.process_histogram(want[3], PS)
        assert (red.pkeys[3] == ref["pkeys"]).all()


@pytest.mark.parametrize("H", [1, 5, 11, 12, 23, 33, 34, 44, 45])
def test_keyed_small_h_privatized_kernel(lh, oracle, H):
    """At precision 100 one pass of k_ingest_keyed_small privatises the windows of 11 histograms in shared memory and
    up to 4 passes over id sub-ranges are taken: H <= 11 in one pass, 12 ... 44 in two to four; H = 45 would need five
    and takes the L2-atomic kernel (k_ingest_keyed_vec) at this batch size.  The misaligned call runs the scalar kernel.
    Every bucket must match the oracle, for f64 and int64-ns samples, u16 and u32 ids, bad ids dropped."""
    import torch
    import _ingest_routes as routes
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 1_200_003
    vals = oracle.gen_stream(lh.STREAM_S, n, SEED ^ H)
    ids = oracle.gen_ids(0, n, H, SEED ^ H)
    ids_bad = ids.copy()
    ids_bad[::997] = H + 3                       # out of range: dropped and counted
    keep = ids_bad < H
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_v, d_i16, d_i32 = e.upload(vals), e.upload(ids_bad.astype(np.uint16)), e.upload(ids_bad)
        e.ingest_keyed_f64_u16(d_i16, d_v, n)
        route = routes.keyed_route(H, n, 100, sms)
        assert route.kernel == (routes.SMALL if H <= 44 else routes.VEC) and e.keyed_kernel_name() == route.kernel
        red, sp = e.snapshot(PS)
        want = oracle.ingest_keyed(ids_bad[keep], vals[keep], H)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want[h]).all(), h
        assert e.stats()["dropped"] == int((~keep).sum())
        e.ingest_keyed_f64_u32(d_i32, d_v.offset(1), n - 1)          # misaligned values: scalar fallback path
        assert e.keyed_kernel_name() == routes.keyed_route(H, n - 1, 100, sms, id_bytes=4, vals_addr=8).kernel == routes.SCALAR
        red, sp = e.snapshot(PS)
        keep1 = keep[:n - 1]
        want1 = oracle.ingest_keyed(ids_bad[:n - 1][keep1], vals[1:][keep1], H)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want1[h]).all(), h
        ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, SEED ^ H).view(np.int64).copy()
        ns[::3] *= -1
        d_n = e.upload(ns)
        e.ingest_keyed_i64ns_u16(d_i16, d_n, n)
        assert e.keyed_kernel_name() == route.kernel
        red, sp = e.snapshot(PS)
        want2 = oracle.ingest_keyed_i64(ids_bad[keep], ns[keep], H)
        for h in range(H):
            assert (dense_from_sparse(sp, h) == want2[h]).all(), h
            ref = oracle.process_histogram(want2[h], PS)
            assert (red.pkeys[h] == ref["pkeys"]).all()


def test_ingest_at_the_edge_of_the_epsilon_band(eng, lh, oracle):
    """Inputs placed just inside and just outside the +-2^-12 band around every bucket boundary of the window: the
    place where an estimator error (rather than a boundary) would flip a bucket without raising the flag.  Both
    shipped estimators are exercised: K1 default (packed FP32) and the keyed kernels (fast_candidate)."""
    T = thresholds(oracle, 4367).view(np.float64)                     # boundaries of buckets 1..4367
    T = T[T > 0.02]
    # 100*ln(1+v) moves by d when v moves by (1+v)*d/100: offsets of 0.6, 0.9, 1.1, 1.5 and 3 EPS on both sides
    eps = 2.0 ** -12
    vals = []
    for mult in (0.6, 0.9, 1.1, 1.5, 3.0):
        dv = (1.0 + T) * (mult * eps) / 100.0
        vals += [T + dv, T - dv, -(T + dv), -(T - dv)]
    vals = np.concatenate(vals)
    vals = np.tile(vals, 8)[:1_000_000]
    want = oracle.ingest(vals)
    d = eng.upload(vals)
    default = eng.lib.lh_k1_variant_current(eng.h)
    for vi, name in enumerate(eng.k1_variants()):
        if name.startswith("probe"):
            continue
        eng.tune("k1", vi)
        eng.ingest_f64(0, d, vals.size)
        _, sp = eng.snapshot(PS)
        assert (dense_from_sparse(sp, 0) == want).all(), vi
    eng.tune("k1", default)
    ids = np.zeros(vals.size, dtype=np.uint16)
    d_i = eng.upload(ids)
    eng.ingest_keyed_f64_u16(d_i, d, vals.size)                       # H = 4: k_ingest_keyed_small (packed FP32)
    _, sp = eng.snapshot(PS)
    assert (dense_from_sparse(sp, 0) == want).all()
    eng.tune("keyed_mode", 1)                                         # k_ingest_keyed_vec (fast_candidate)
    eng.ingest_keyed_f64_u16(d_i, d, vals.size)
    _, sp = eng.snapshot(PS)
    assert (dense_from_sparse(sp, 0) == want).all()
    eng.tune("keyed_mode", 0)
    d.free(); d_i.free()
