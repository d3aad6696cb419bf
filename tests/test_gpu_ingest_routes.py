"""Every keyed and counter ingest route against the oracle at its dispatch and capacity boundaries.

Each case first asks tests/_ingest_routes.py which kernel the host should pick (and, for the write-combining kernel,
with which owner-buffer size), asserts that this kernel ran, and only then compares the result: every bucket of every
histogram, every counter and the dropped tally exact."""
import numpy as np
import pytest

import _ingest_routes as R

pytestmark = pytest.mark.gpu

SEED = 0x10C415C0
PS = [0.5, 0.99]
N = (1 << 22) + 4099          # past the write-combining kernel's 2^22-sample minimum, with a ragged tail


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_cache = {}


def samples(oracle, precision):
    """(float64 values, int64 ns, their uint16 keys at this precision), shared by every case of one precision."""
    if precision not in _cache:
        vals = oracle.gen_stream(oracle.STREAM_S, N, SEED ^ precision)
        vals[::7] = oracle.gen_stream(oracle.STREAM_N, N, SEED + 1)[::7]          # negatives: the exact route
        specials = np.array([np.inf, -np.inf, np.nan, 2.0 ** 63, -(2.0 ** 64), 0.0, -0.0, 5e-324, 1e300], np.float64)
        vals[3::1009] = specials[np.arange(vals[3::1009].size) % specials.size]
        ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, N, SEED ^ precision).view(np.int64).copy()
        ns[::5] *= -1
        _cache[precision] = (vals, ns, oracle.compress_many(vals, precision).view(np.uint16),
                             oracle.compress_many(ns.astype(np.float64), precision).view(np.uint16))
    return _cache[precision]


def reference(H, ids, keys):
    """Exact sparse histograms of (ids, keys): (sorted flat index id * 65536 + key, uint64 counts, dropped samples)."""
    ok = ids < H
    u, c = np.unique(ids[ok].astype(np.int64) * 65536 + keys[ok], return_counts=True)
    return u, c.astype(np.uint64), int((~ok).sum())


def merged(*refs):
    """The sum of several references."""
    u, inv = np.unique(np.concatenate([r[0] for r in refs]), return_inverse=True)
    c = np.zeros(u.size, np.uint64)
    np.add.at(c, inv, np.concatenate([r[1] for r in refs]))
    return u, c, sum(r[2] for r in refs)


def check(e, H, ref, dropped_before, what):
    """The interval's snapshot equals `ref` bucket for bucket, and exactly ref's samples were dropped."""
    red, sp = e.snapshot(PS)
    u, c, dropped = ref
    flat = np.repeat(np.arange(H, dtype=np.int64), np.diff(sp.offsets.astype(np.int64))) * 65536 + sp.keys.view(np.uint16)
    order = np.argsort(flat, kind="stable")
    assert flat.size == u.size and (flat[order] == u).all(), (what, flat.size, u.size)
    assert (sp.counts[order] == c).all(), (what, np.nonzero(sp.counts[order] != c)[0][:5])
    totals = np.zeros(H, np.uint64)
    np.add.at(totals, u >> 16, c)
    assert (red.counts == totals).all(), what
    assert e.stats()["dropped"] - dropped_before == dropped, what


def run_keyed_variants(e, lh, oracle, H, precision, sms, tune, label):
    """u16 ids / float64, u32 ids (with ids >= 65536) / float64, u16 / int64 ns, and the fused pair: route, then buckets."""
    vals, ns, keys, nskeys = samples(oracle, precision)
    ids = oracle.gen_ids(0, N, H, SEED ^ H).astype(np.uint32)
    # the same samples are dropped from both id widths: u16 ids H and 65535, u32 ids 65536 + (H - 1), 2^31, 2^32 - 1
    ids16 = R.with_bad_ids(ids, np.array([H, 65535], np.uint32), 997)
    ids32 = R.with_bad_ids(ids, R.high_ids(H, H - 1), 997)
    ref_f, ref_ns = reference(H, ids16, keys), reference(H, ids16, nskeys)
    d_v, d_n = e.upload(vals), e.upload(ns)
    d_i16, d_i32 = e.upload(ids16.astype(np.uint16)), e.upload(ids32)
    for name, call, id_bytes, ref in (
            ("f64_u16", lambda: e.ingest_keyed_f64_u16(d_i16, d_v, N), 2, ref_f),
            ("f64_u32", lambda: e.ingest_keyed_f64_u32(d_i32, d_v, N), 4, ref_f),
            ("i64ns_u16", lambda: e.ingest_keyed_i64ns_u16(d_i16, d_n, N), 2, ref_ns)):
        want = R.keyed_route(H, N, precision, sms, id_bytes=id_bytes, **tune)
        before = e.stats()["dropped"]
        call()
        assert e.keyed_kernel_name() == want.kernel, (label, name, want)
        check(e, H, ref, before, (label, name))
    # both segments of one fused launch (N is not a whole number of tiles, so both leave a ragged end)
    want = R.pair_route(H, N, N, precision, sms, **tune)
    before = e.stats()["dropped"]
    e.ingest_keyed_pair_u16(d_i16, d_v, N, d_i16, d_n, N)
    assert e.keyed_kernel_name() == want.kernel, (label, "pair", want)
    check(e, H, merged(ref_f, ref_ns), before, (label, "pair"))
    for x in (d_v, d_n, d_i16, d_i32):
        x.free()
    return want


def boundary_cases(precision, sms, reserve):
    """[(label, H)] of the keyed route boundaries at this precision and P = sm_count - reserve."""
    P = sms - reserve
    caps, hmax = R.wc_h_by_row_cap(precision, sms, reserve, lo=1, hi=8192)
    cases = []
    if reserve == 0:
        edge = R.small_edge(precision)
        cases += [("small_edge", edge), ("past_small_edge", edge + 1)]
    if R.small_edge(precision) + 1 < P:
        cases.append(("idle_owners", (R.small_edge(precision) + P) // 2))
    for cap in sorted(caps, reverse=True):
        hs = [h for h in caps[cap] if h > R.small_edge(precision) and h % P]
        cases.append(("row_cap_%d" % cap, hs[len(hs) // 2]))
    cases += [("wc_max", hmax), ("past_wc_max", hmax + 1)]
    return cases


@pytest.mark.parametrize("precision", [50, 100, 200])
@pytest.mark.parametrize("reserve", ["0", "1", "sm-8"])
def test_keyed_route_boundaries(lh, oracle, sms, precision, reserve):
    """At every route boundary: the kernel the predictor names runs, and all its buckets are exact.  reserve "1" is
    the benchmark's setting (one SM left to the snapshot stream); "sm-8" is the smallest P the write-combining kernel
    takes.  The write-combining cases use H that P does not divide."""
    k1_reserve = {"0": 0, "1": 1, "sm-8": sms - 8}[reserve]
    tune = {"k1_reserve_sms": k1_reserve}
    seen = set()
    for label, H in boundary_cases(precision, sms, k1_reserve):
        want = R.keyed_route(H, N, precision, sms, k1_reserve_sms=k1_reserve)
        expect = {"small_edge": R.SMALL, "past_small_edge": R.WC, "idle_owners": R.WC, "past_wc_max": R.VEC}.get(label, R.WC)
        assert want.kernel == expect, (label, H, want)
        if label.startswith("row_cap_"):
            assert want.wc.row_cap == int(label[8:]), (label, H, want)
        if label == "idle_owners":
            assert H < want.wc.P
        with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as e:
            e.tune("k1_reserve_sms", k1_reserve)
            run_keyed_variants(e, lh, oracle, H, precision, sms, tune, (precision, reserve, label, H))
        seen.add(want.kernel)
    assert R.WC in seen and R.VEC in seen


def test_every_row_cap_is_reached(sms):
    """The boundary cases above reach each owner-buffer size the host can pick, at P = sm_count and P = sm_count - 1."""
    for reserve in (0, 1):
        caps = set()
        for precision in (50, 100, 200):
            for label, H in boundary_cases(precision, sms, reserve):
                r = R.keyed_route(H, N, precision, sms, k1_reserve_sms=reserve)
                if r.wc:
                    caps.add(r.wc.row_cap)
        assert caps == set(R.CONST["WC_ROW_CAPS"]), (reserve, caps)


@pytest.mark.parametrize("reserve", [0, 1])
def test_wc_rare_queue_overflow(lh, oracle, sms, reserve):
    """A batch whose every sample needs the exact route, at the default chunk size: each CTA sets aside more than
    WC_RARE_CAP samples in one chunk, so the surplus takes the on-the-spot exact path."""
    H, precision = 300, 100
    n = (1 << 22) + 3
    vals = R.exact_route_values(oracle, n, SEED)
    ids = oracle.gen_ids(0, n, H, SEED ^ 0x5A).astype(np.uint32)
    ids = R.with_bad_ids(ids, R.high_ids(H, 7), 1013)
    want = R.keyed_route(H, n, precision, sms, id_bytes=4, k1_reserve_sms=reserve)
    assert want.kernel == R.WC
    rare = R.definitely_exact(vals) | (ids >= H)
    assert R.wc_slice_counts(rare, want.wc).max() > R.CONST["WC_RARE_CAP"]
    keys = oracle.compress_many(vals, precision).view(np.uint16)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        e.tune("k1_reserve_sms", reserve)
        d_v, d_i = e.upload(vals), e.upload(ids)
        before = e.stats()["dropped"]
        e.ingest_keyed_f64_u32(d_i, d_v, n)
        assert e.keyed_kernel_name() == R.WC
        check(e, H, reference(H, ids, keys), before, "rare overflow")


def one_owner_case(sms, H, reserve):
    """(tuning, predicted route, ids) of a one-owner case.  At P = sm_count and sm_count - 1 the chunks are two tiles
    per writer and every tile flushes, so each writer offers its sub-queue of the owner 2 x row_cap records per chunk,
    more than the queue's `cap`.  At P = 8 an owner's expected share of a tile (TILE / 8) already exceeds row_cap, so its
    sub-queues are sized past anything one buffer can deliver: only the buffer overflows there."""
    reserve = sms - 8 if reserve == "sm-8" else reserve
    tune = {"k1_reserve_sms": reserve}
    P = sms - reserve
    if P > 8:
        threads, per = R.CONST["WC_SHAPES"][R.DEFAULTS["wc_spt"]]
        tune.update(kp_chunk=2 * P * threads * per, wc_flush=4096)
    want = R.keyed_route(H, N, 100, sms, **tune)
    return tune, want, R.same_residue_ids(N, H, P, 3, SEED)


@pytest.mark.parametrize("H,reserve", [(1024, 0), (1000, 1), (100, "sm-8")])
def test_wc_one_owner_takes_every_record(lh, oracle, sms, H, reserve):
    """Distinct ids that are all congruent modulo P: every record goes to one owner, whose shared-memory buffer
    overflows in every writer, and (at P = sm_count and sm_count - 1) whose per-(owner, writer) sub-queues overflow in
    every chunk.  The surplus must take the exact route without losing or doubling a sample."""
    precision = 100
    vals, _, keys, _ = samples(oracle, precision)
    tune, want, ids = one_owner_case(sms, H, reserve)
    assert want.kernel == R.WC
    P = want.wc.P
    _, spilled = R.wc_owner_queue(~R.definitely_exact(vals[:want.wc.taken]), want.wc)
    assert (spilled.sum() > 0) == (P > 8), (H, P, want.wc)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        for k, v in tune.items():
            e.tune(k, v)
        d_v, d_i = e.upload(vals), e.upload(ids.astype(np.uint16))
        before = e.stats()["dropped"]
        e.ingest_keyed_f64_u16(d_i, d_v, N)
        assert e.keyed_kernel_name() == R.WC
        check(e, H, reference(H, ids, keys), before, ("one owner", H, P))


def test_high_u32_ids_are_dropped_on_every_route(lh, oracle, sms):
    """u32 ids 65536 + k, 2^31 and 2^32 - 1 (k a valid id) through the small, vector, write-combining and scalar keyed
    kernels and the sparse merge: dropped and counted, never added to k.  (test_counter_routes sends them through both
    counter kernels.)"""
    precision = 100
    vals, _, keys, _ = samples(oracle, precision)
    for H, tune in ((5, {}), (300, {"keyed_mode": 1}), (300, {})):
        ids = oracle.gen_ids(0, N, H, SEED ^ H).astype(np.uint32)
        ids = R.with_bad_ids(ids, R.high_ids(H, H // 2), 101)
        with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
            for k, v in tune.items():
                e.tune(k, v)
            d_v, d_i = e.upload(vals), e.upload(ids)
            for off, n in ((0, N), (1, 100_003)):     # off 1: ids not 16-byte aligned, scalar kernel only
                want = R.keyed_route(H, n, precision, sms, id_bytes=4, ids_addr=4 * off, **tune)
                assert (want.kernel == R.SCALAR) == (off == 1), want
                before = e.stats()["dropped"]
                e.ingest_keyed_f64_u32(d_i.offset(off), d_v, n)
                assert e.keyed_kernel_name() == want.kernel, (H, tune, off)
                check(e, H, reference(H, ids[off:off + n], keys[:n]), before, (H, tune, off))
    # the sparse merge
    with lh.Engine(device=0, max_histograms=8, max_counters=1) as e:
        before = e.stats()["dropped"]
        e.merge_counts_host(np.concatenate([R.high_ids(8, 5), [5]]).astype(np.uint32),
                            np.array([10, 11, 12, 13], np.int16), np.array([1, 2, 3, 4], np.uint64))
        _, sp = e.snapshot(PS)
        assert sp.histogram(5) == {13: 4} and int(sp.offsets[-1]) == 1
        assert e.stats()["dropped"] - before == 3


@pytest.mark.parametrize("C", [8192, 8193, 70000])
def test_counter_routes(lh, oracle, C):
    """Both sides of K2_SMEM_COUNTERS: the privatised kernel (vector body + scalar head and tail) and the global one.
    Amounts that carry out of every half (2^32 - 1, 2^32, 2^64 - 1, 2^63), u16 and u32 ids, u32 ids >= 65536,
    misaligned heads.  The number of launches is the predicted route's."""
    n = 300_007
    rng = np.random.default_rng(C)
    ids = rng.integers(0, min(C, 65536), n + 8).astype(np.uint32)
    ids[::3] = 5                                                   # one hot counter: carries pile up in it
    amounts = rng.integers(0, 2 ** 64, n + 8, dtype=np.uint64)
    special = np.array([2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, 1 << 63], np.uint64)
    amounts[::2] = special[np.arange(amounts[::2].size) % 4]
    ids32 = R.with_bad_ids(ids, R.high_ids(min(C, 65536), 5), 89)
    if C > 65536:
        ids32[1::97] = rng.integers(65536, C, ids32[1::97].size)   # valid ids past 16 bits
    with lh.Engine(device=0, max_histograms=1, max_counters=C) as e:
        d_i16, d_i32, d_a = e.upload(ids.astype(np.uint16)), e.upload(ids32), e.upload(amounts)
        for name, d_i, host_ids, id_bytes in (("u16", d_i16, ids, 2), ("u32", d_i32, ids32, 4)):
            for off, m in ((0, n), (1, n - 1), (3, 65_541), (2, 20_000)):
                route = R.counter_route(C, m, id_bytes=id_bytes, amounts_addr=8 * off, ids_addr=id_bytes * off)
                st0 = e.stats()
                (e.counter_add_u16 if id_bytes == 2 else e.counter_add_u32)(d_i.offset(off), d_a.offset(off), m)
                assert e.stats()["kernel_launches"] - st0["kernel_launches"] == route.extra["launches"], (name, off, route)
                _, sp = e.snapshot(PS)              # the dropped tally is read after the snapshot has waited for the kernels
                sel = host_ids[off:off + m]
                ok = sel < C
                want = oracle.counter_add(sel[ok], amounts[off:off + m][ok], C)
                assert (sp.counter_deltas == want).all(), (C, name, off, np.nonzero(sp.counter_deltas != want)[0][:5])
                assert e.stats()["dropped"] - st0["dropped"] == int((~ok).sum()), (C, name, off)


@pytest.mark.parametrize("keyed_mode", [0, 1])
def test_hot_window_past_2_32(lh, oracle, sms, keyed_mode):
    """One interval of constant-value batches, almost all into histogram 0: more than 2^32 samples land in one cell of
    the uint32 hot window, so the fold guard must drain it between two calls and in the middle of one."""
    H, cap = 2, 1_500_000_000
    calls = [cap, cap, 300_000_000, cap, cap, cap]
    plan = R.hot_window_plan(calls)
    assert any(ev[0] == "fold" for ev in plan) and any("fold" in ev[1:] for ev in plan)
    sentinels = np.array([0, 12_345, 299_999_999, 1_294_967_294, 1_294_967_295, cap - 1], np.int64)
    import torch
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        e.tune("keyed_mode", keyed_mode)
        d_v, d_i = None, None
        try:
            d_v = e.gen_stream(lh.STREAM_C, cap, SEED)
            d_i = torch.zeros(cap, dtype=torch.int16, device="cuda:0")     # every id 0 ...
            d_i[torch.as_tensor(sentinels, device="cuda:0")] = 1             # ... but a few in histogram 1
            torch.cuda.synchronize()
            for m in calls:
                e.ingest_keyed_f64_u16(d_i, d_v, m)
                assert e.keyed_kernel_name() == R.keyed_route(H, m, 100, sms, keyed_mode=keyed_mode).kernel
            red, sp = e.snapshot(PS)
        finally:                                                              # 15 GB: give it back even on a failure
            if d_v is not None:
                e.sync()
                d_v.free()
            del d_i
            torch.cuda.empty_cache()
        key = int(oracle.compress(float(oracle.gen_stream(oracle.STREAM_C, 1, SEED)[0])))
        total = sum(calls)
        in1 = sum(int((sentinels < m).sum()) for m in calls)
        assert total > 1 << 32
        assert sp.histogram(0) == {key: total - in1}
        assert sp.histogram(1) == {key: in1}
        assert int(red.counts[0]) == total - in1 and int(red.counts[1]) == in1
