"""Configurable `precision` (reference metrics.go:40-43: `precision = 100`; compress/decompress :316-332 use it):
every kernel family against the oracle across the supported range 1 ... 250.  Bar: bit-exact keys, counts, percentile buckets and
decompressed values."""
import numpy as np
import pytest

import _ingest_routes as routes
import _reduce_cases as rc

pytestmark = pytest.mark.gpu

SEED = 0x10C415C0
PS = [0.0, 0.5, 0.75, 0.9, 0.95, 0.99, 0.999, 0.9999, 1.0]
# 1 and 2: a_int = floor(precision * ln 2) is 0 and 1; 146 / 147 and 249 / 250: the top of the range; and the last
# precision before / the first at which lh_create runs another K1 variant's code under a variant's name (its ring and
# the sub-histogram no longer fit shared memory; tests/_ingest_routes.py k1_variants has the table)
_K1_SUBSTITUTED = set(routes.k1_substitution_precisions().values())
PRECISIONS = sorted({1, 2, 50, 100, 146, 147, 200, 249, 250} | _K1_SUBSTITUTED | {p - 1 for p in _K1_SUBSTITUTED})


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


def dense_from_sparse(sp, hid):
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in sp.histogram(hid).items():
        out[k & 0xFFFF] = c
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
def test_compress_at_every_threshold(lh, oracle, precision):
    """Every bucket boundary of the whole finite range, +-3 ulps, both signs, both evaluators, at this precision."""
    kmax = int(np.floor(precision * np.log1p(1.7976931348623157e308) + 0.5))
    T = routes.thresholds(oracle, precision, kmax)
    offs = np.arange(-3, 4, dtype=np.int64)
    bits = (T[:, None].astype(np.int64) + offs[None, :]).reshape(-1).astype(np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(0x8000000000000000)])
    vals = bits.view(np.float64)
    want = oracle.compress_many(vals, precision)
    with lh.Engine(device=0, precision=precision) as eng:
        for mode in (0, 1):
            got = eng.compress(vals, mode)
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, (precision, mode, bad.size, vals[bad[:5]], got[bad[:5]], want[bad[:5]])
        tab = eng.decompress_table()
        assert (tab.view(np.uint64) == oracle.decompress_table(precision).view(np.uint64)).all()
        # the FP32 estimate stays inside its epsilon at this precision
        d = eng.gen_stream(lh.STREAM_U, 20_000_000, SEED ^ 0x77)
        err, slow = eng.fastpath_margin(d, 20_000_000)
        eps = 2.0 ** -12 * max(1.0, precision / 100.0)
        assert err < eps / 2, (precision, err)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_every_ingest_kernel(lh, oracle, precision):
    n = 2_000_003
    table = oracle.decompress_table(precision)
    for stream in (lh.STREAM_S, lh.STREAM_U, lh.STREAM_N):
        vals = oracle.gen_stream(stream, n, SEED ^ precision)
        want = oracle.ingest(vals, precision=precision)
        ref = oracle.process_histogram(want, PS, precision)
        exact = rc.Reference(rc.sparse(want), table)
        # K1, every variant
        with lh.Engine(device=0, max_histograms=2, precision=precision) as eng:
            d = eng.upload(vals)
            for vi, name in enumerate(eng.k1_variants()):
                if name.startswith("probe"):
                    continue
                eng.tune("k1", vi)
                eng.ingest_f64(1, d, n)
                red, sp = eng.snapshot(PS)
                assert (dense_from_sparse(sp, 1) == want).all(), (precision, stream, name)
                assert int(red.counts[1]) == n and (red.pkeys[1] == ref["pkeys"]).all()
                assert (red.pvals[1].view(np.uint64) == ref["pvals"].view(np.uint64)).all()
                assert rc.sum_ok(float(red.sums[1]), exact), (precision, stream, name)
        # keyed kernels: few ids (shared-memory windows), many ids (L2 atomics), many ids (owner-partitioned)
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        for H, mode in ((3, 0), (300, 1), (300, 2)):
            ids = oracle.gen_ids(0, n, H, SEED ^ precision)
            wantk = np.zeros((H, 65536), dtype=np.uint64)
            keys = oracle.compress_many(vals, precision).view(np.uint16)
            np.add.at(wantk, (ids, keys), 1)
            with lh.Engine(device=0, max_histograms=H, precision=precision) as eng:
                eng.tune("keyed_mode", mode)
                d, di = eng.upload(vals), eng.upload(ids.astype(np.uint16))
                eng.ingest_keyed_f64_u16(di, d, n)
                assert eng.keyed_kernel_name() == routes.keyed_route(H, n, precision, sms, keyed_mode=mode).kernel == \
                    (routes.SMALL, routes.VEC, routes.WC)[mode], (precision, H, mode)
                red, sp = eng.snapshot(PS)
                assert (red.counts == wantk.sum(axis=1)).all(), (precision, stream, H, mode, eng.keyed_kernel_name())
                for h in (0, 1, H - 1):
                    assert (dense_from_sparse(sp, h) == wantk[h]).all(), (precision, stream, H, mode, h)


def test_precision_range_is_checked(lh):
    with pytest.raises(lh.LhError):
        lh.Engine(device=0, precision=251)
    with lh.Engine(device=0, precision=250) as e:     # the largest supported (test_every_ingest_kernel runs full streams there)
        vals = np.array([1.0, -1.0, 1e18, 0.0, 3.5], dtype=np.float64)
        d = e.upload(vals)
        e.ingest_f64(0, d, vals.size)
        red, _ = e.snapshot(PS)
        assert int(red.counts[0]) == vals.size
