"""Keyed samples and counter adds under local ids (lh_ingest_keyed_mapped_*, lh_counter_add_mapped_*, and
RecordScope.keyed / counters above them) on the GPU.

Bar: every bucket of every row equal to what the raw keyed call gives for the same samples under their global ids
(itself checked against the oracle on every route by test_gpu_ingest_routes.py), and to the oracle directly on the
smaller cases; lh_keyed_kernel_name naming the planned route on both sides of each plan boundary; drops under ids >= k
and under unbound rows counted exactly once; counter totals equal to numpy's wrapping sums."""
import threading

import numpy as np
import pytest

from test_gpu_device_record import PS, SEED, want_keyed

pytestmark = pytest.mark.gpu

UNBOUND = 0xFFFFFFFF


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def dev_at(torch, a, off):
    """`a` on the device, starting `off` elements past the start of its allocation."""
    t = torch.empty(a.size + off, dtype=getattr(torch, a.dtype.name), device="cuda")
    t[off:] = torch.from_numpy(a).cuda()
    return t[off:]


def sparse(eng):
    _, sp = eng.snapshot(PS)
    eng.sync()
    return sp, eng.stats()["dropped"]


def make_map(rng, k, H):
    """k rows out of H: distinct where possible, one duplicate and one unbound entry when k >= 4."""
    m = rng.permutation(H)[:k].astype(np.int64)
    if k >= 4:
        m[1] = m[0]
        m[2] = UNBOUND
    return [int(x) for x in m]


def global_ids(local, m, H):
    mm = np.array(m + [UNBOUND], dtype=np.int64)
    g = mm[np.minimum(local.astype(np.int64), len(m))]
    return np.where(g == UNBOUND, H, g)


# (H, k, n, id offset, precision, expected route) -- each plan boundary from both sides
CASES = [
    (1024, 8, 4096 * 4, 0, 100, "k_ingest_keyed_small"),          # n4 = 4096: the small kernel
    (1024, 8, 4096 * 4 - 4, 0, 100, "k_ingest_keyed_vec"),        # n4 = 4095
    (1024, 44, 1 << 20, 0, 100, "k_ingest_keyed_small"),          # 4 passes of 11 ids at precision 100
    (1024, 45, 1 << 20, 0, 100, "k_ingest_keyed_vec"),            # 5 passes: not the small kernel
    (1024, 16, 1 << 20, 0, 250, "k_ingest_keyed_small"),          # 4 passes of 4 ids at precision 250
    (1024, 17, 1 << 20, 0, 250, "k_ingest_keyed_vec"),
    (1024, 1024, 1 << 22, 0, 100, "k_ingest_keyed_wc"),           # 2^22 pairs: the write-combining kernel
    (1024, 1024, (1 << 22) - 4, 0, 100, "k_ingest_keyed_vec"),
    (2048, 1000, (1 << 22) + 12345, 0, 100, "k_ingest_keyed_wc"),  # ragged tail after whole tiles
    (2048, 1000, (1 << 22) + 12345, 0, 250, "k_ingest_keyed_vec"),  # 8 ids per owner x 10 916 cells: not 16-bit records
    (1024, 8, 100003, 1, 100, "k_ingest_keyed"),                  # misaligned ids: the scalar kernel only
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "H%d_k%d_n%d_off%d_p%d" % c[:5])
@pytest.mark.parametrize("id_bytes", [2, 4])
@pytest.mark.parametrize("kind", ["f64", "i64"])
@pytest.mark.parametrize("stream_kind", ["U", "L"])
def test_mapped_keyed_equals_raw_keyed_on_every_route(lh, torch, case, id_bytes, kind, stream_kind):
    H, k, n, off, precision, route = case
    rng = np.random.default_rng(SEED + k + n)
    m = make_map(rng, k, H)
    local = rng.integers(0, k + 2, n).astype(np.uint16 if id_bytes == 2 else np.uint32)     # ~2/(k+2) past the names
    with lh.Engine(max_histograms=H, max_counters=4, precision=precision) as ea, \
         lh.Engine(max_histograms=H, max_counters=4, precision=precision) as eb:
        vals = ea.gen_stream(lh.STREAM_U if stream_kind == "U" else lh.STREAM_L, n, SEED).to_host()
        if kind == "i64":
            vals = np.clip(np.abs(vals) * 1e6, 0, 2.0 ** 62).astype(np.int64)
        d_vals = dev_at(torch, vals, 0)
        d_local = dev_at(torch, local, off)
        ea.ingest_keyed_mapped_u16(m, d_local, d_vals, int(kind == "i64"), n) if id_bytes == 2 else \
            ea.ingest_keyed_mapped_u32(m, d_local, d_vals, int(kind == "i64"), n)
        assert ea.keyed_kernel_name() == route
        g = global_ids(local, m, H)
        if kind == "f64" and id_bytes == 4:
            eb.ingest_keyed_f64_u32(dev_at(torch, g.astype(np.uint32), off), d_vals, n)
        elif kind == "f64":
            eb.ingest_keyed_f64_u16(dev_at(torch, g.astype(np.uint16), off), d_vals, n)
        else:                                   # the raw int64 call takes uint16 ids only
            eb.ingest_keyed_i64ns_u16(dev_at(torch, g.astype(np.uint16), off), d_vals, n)
        torch.cuda.synchronize()
        spa, da = sparse(ea)
        spb, db = sparse(eb)
    assert np.array_equal(spa.offsets, spb.offsets)
    assert np.array_equal(spa.keys, spb.keys) and np.array_equal(spa.counts, spb.counts)
    assert da == db == int((g >= H).sum())


@pytest.mark.parametrize("k", [8, 1024])
def test_mapped_keyed_against_the_oracle(lh, torch, oracle, k):
    H, n = 1024, (1 << 22) + 4
    rng = np.random.default_rng(SEED + k)
    m = make_map(rng, k, H)
    local = rng.integers(0, k + 1, n).astype(np.uint16)
    vals = rng.lognormal(0.0, 4.0, n) * rng.choice([-1.0, 1.0], n)
    with lh.Engine(max_histograms=H, max_counters=4) as e:
        e.ingest_keyed_mapped_u16(m, dev_at(torch, local, 0), dev_at(torch, vals, 0), 0, n)
        torch.cuda.synchronize()
        sp, dropped = sparse(e)
    g = global_ids(local, m, H)
    want = want_keyed(oracle, g, vals, H, 100)
    hid = np.repeat(np.arange(H), np.diff(sp.offsets.astype(np.int64)))
    got = np.zeros((H, 65536), dtype=np.uint64)
    got[hid, sp.keys.view(np.uint16)] = sp.counts
    assert np.array_equal(got, want)
    assert dropped == int((g >= H).sum())


@pytest.mark.parametrize("kc,n", [(16, 1 << 20), (1024, 1 << 20), (4096, (1 << 20) + 3), (8, 1001)])
@pytest.mark.parametrize("id_bytes", [2, 4])
@pytest.mark.parametrize("unbound", [True, False])
def test_mapped_counters_wrap_like_numpy(lh, torch, kc, n, id_bytes, unbound):
    C = 8192
    rng = np.random.default_rng(SEED + kc)
    m = make_map(rng, kc, C)
    if not unbound:                      # no unbound row: the kernels check only the bound per op
        m = [C - 1 - i if x == UNBOUND else x for i, x in enumerate(m)]
    local = rng.integers(0, kc + 1, n).astype(np.uint16 if id_bytes == 2 else np.uint32)
    amounts = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(3)
    with lh.Engine(max_histograms=1, max_counters=C) as e:
        f = e.counter_add_mapped_u16 if id_bytes == 2 else e.counter_add_mapped_u32
        f(m, dev_at(torch, local, 0), dev_at(torch, amounts, 1 if n % 2 else 0), n)
        torch.cuda.synchronize()
        sp, dropped = sparse(e)
    g = global_ids(local, m, C)
    want = np.zeros(C + 1, dtype=np.uint64)
    np.add.at(want, g, amounts)
    assert np.array_equal(sp.counter_deltas, want[:C])
    assert dropped == int((g >= C).sum())


def test_mapped_call_errors(lh, torch):
    with lh.Engine(max_histograms=4, max_counters=4) as e:
        ids, vals = dev_at(torch, np.zeros(8, np.uint16), 0), dev_at(torch, np.ones(8), 0)
        for bad, st in (([0] * 4097, -1), ([4], -6), ([0], None)):
            if st is None:
                e.ingest_keyed_mapped_u16(bad, ids, vals, 0, 8)
                continue
            with pytest.raises(lh.LhError) as ex:
                e.ingest_keyed_mapped_u16(bad, ids, vals, 0, 8)
            assert ex.value.status == st
        with pytest.raises(lh.LhError):
            e.counter_add_mapped_u16([5], ids, dev_at(torch, np.ones(8, np.uint64), 0), 8)
        e.ingest_keyed_mapped_u16([], ids, vals, 0, 8)            # k = 0: everything dropped
        torch.cuda.synchronize()
        sp, dropped = sparse(e)
    assert int(sp.counts.sum()) == 8 and dropped == 8


def test_scope_keyed_metric_system(lh, torch, oracle):
    """A scope on a side stream lands in its interval; processMetrics equals per-name arrays through histograms();
    per-call Histogram() from 16 threads on the same names loses nothing."""
    from loghisto_b200.metric_system import MetricSystem
    names = ["r%d" % i for i in range(12)]
    rng = np.random.default_rng(SEED)
    n = 1 << 20
    local = rng.integers(0, len(names), n).astype(np.int32)
    vals = rng.lognormal(2.0, 2.0, n)
    amts = rng.integers(1, 1000, n, dtype=np.int64)
    side = torch.cuda.Stream()
    ms_a, ms_b = MetricSystem(1e-6, False), MetricSystem(1e-6, False)
    try:
        with ms_a.recording(stream=side, histograms=names, counters=names[:3]) as s:
            s.keyed(dev_at(torch, local, 0), dev_at(torch, vals, 0))
            s.counters(dev_at(torch, local % 4, 0), dev_at(torch, amts, 0))      # local id 3 is past the counters
        per_thread = 1000

        def hammer(t):
            for i in range(per_thread):
                ms_a.Histogram(names[(t + i) % len(names)], 1.0)
        ts = [threading.Thread(target=hammer, args=(t,)) for t in range(16)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        torch.cuda.synchronize()
        raw_a, _ = ms_a.collect_and_process()
        with ms_b.recording(histograms=names, counters=names[:3]) as s:
            s.histograms([(nm, dev_at(torch, vals[local == i], 0)) for i, nm in enumerate(names)])
        for t in range(16):
            for i in range(per_thread):
                ms_b.Histogram(names[(t + i) % len(names)], 1.0)
        for i, nm in enumerate(names[:3]):
            ms_b.Counter(nm, int(amts[(local % 4) == i].sum()))
        torch.cuda.synchronize()
        raw_b, _ = ms_b.collect_and_process()
        assert raw_a["Histograms"] == raw_b["Histograms"] and raw_a["Counters"] == raw_b["Counters"]
        part = lambda r: {"Histograms": r["Histograms"], "Counters": r["Counters"]}   # noqa: E731
        assert ms_a.processMetrics(part(raw_a)) == ms_b.processMetrics(part(raw_b))
        assert ms_a.dropped() == int(((local % 4) == 3).sum())
    finally:
        ms_a.close()
        ms_b.close()
