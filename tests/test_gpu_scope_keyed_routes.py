"""Record-scope keyed samples and counter adds (lh_ingest_keyed_mapped_*, lh_counter_add_mapped_*) against the oracle on
global ids, at every dispatch and capacity boundary of the mapped kernels.

The mapped forms are separate instantiations of the keyed and counter kernels.  They plan on the scope's k local ids,
not on max_histograms, and read the map wherever a row address is formed: the scalar and vector lookups, the small
kernel's flush, and in the write-combining kernel the spills, the rare path and the final flush.  Each case first asks
tests/_ingest_routes.py (with H := k) which kernel, or how many counter launches, the host should pick and asserts that
it ran, with the prediction showing the case is on the intended side of its boundary (row_cap, several chunks, spilled
records, rare-list overflow).  Only then does it compare every bucket of every row, every counter and the dropped tally
exactly with the oracle on global ids: local id l < k is row map[l], and l >= k or an unbound entry drops the sample.
Every engine has more rows than k and every map is a scattered permutation with unbound and shared entries, so a kernel
that takes the local id, or max_histograms, for a row fails."""
import numpy as np
import pytest

import _ingest_routes as R

gpu = pytest.mark.gpu

SEED = 0x5C09E
PS = [0.5, 0.99]
N = (1 << 22) + 4099            # past the write-combining kernel's 2^22-sample minimum, with a ragged tail
UNBOUND = 0xFFFFFFFF
MAP_MAX = R._int_expr(R._src("lh_kernels.cuh"), r"constexpr uint32_t LH_MAP_MAX = ([^;]+);", {})
H_BIG = 2 * MAP_MAX             # rows of the boundary engines: more than any k
PRECISIONS = [31, 50, 100, 200, 250]
SPECIALS = np.array([np.inf, -np.inf, np.nan, 2.0 ** 63, -(2.0 ** 64), 0.0, -0.0, 5e-324, 1e300], np.float64)
# int64 nanoseconds converted like TimerToken.Stop: the extremes, and 2^53 +- 1 and the ties above 2^53 that round to even
I64_EDGES = np.array([0, 1, -1, -(1 << 63), (1 << 63) - 1, -(1 << 63) + 1, (1 << 53) - 1, 1 << 53, (1 << 53) + 1,
                      (1 << 53) + 3, (1 << 54) + 2, (1 << 54) + 6, -((1 << 53) + 1), -((1 << 54) + 6), (1 << 62) + (1 << 9),
                      (1 << 62) + 3 * (1 << 9)], dtype=np.int64)


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------ references
def scatter_map(k, H, seed, unbound=(), dup=()):
    """k distinct rows of [0, H) in random order; then every local id in `unbound` is unbound and, for every (a, b) in
    `dup`, local id b shares local id a's row."""
    m = np.random.default_rng(seed).permutation(H)[:k].astype(np.int64)
    for a, b in dup:
        m[b] = m[a]
    for l in unbound:
        m[l] = UNBOUND
    return [int(x) for x in m]


def awkward_map(k, H, seed):
    """A scattered map with unbound entries at k/2 and k - 1 and shared rows between 0 and k - 2 and between 1 and k/3:
    later passes of the small kernel, owners other than 1 and 2 of the write-combining kernel (k >= 8)."""
    return scatter_map(k, H, seed, unbound=(k // 2, k - 1), dup=((0, k - 2), (1, k // 3)))


def fold(lrow, lkey, lc, m, dropped=0):
    """Local-id counts (local row, key, count) through map m: (sorted flat row * 65536 + key, uint64 counts, dropped)."""
    mm = np.array(list(m) + [UNBOUND], dtype=np.int64)
    rows = mm[np.minimum(lrow.astype(np.int64), len(m))]
    ok = rows != UNBOUND
    u, inv = np.unique(rows[ok] * 65536 + lkey[ok].astype(np.int64), return_inverse=True)
    c = np.zeros(u.size, np.uint64)
    np.add.at(c, inv, lc[ok].astype(np.uint64))
    return u, c, int(dropped) + int(lc[~ok].astype(np.uint64).sum())


def reference(local, keys, m):
    """The exact sparse histograms of samples with these local ids and uint16 keys, under map m."""
    ok = local < len(m)
    lu, lc = np.unique((local[ok].astype(np.uint32) << np.uint32(16)) | keys[ok].astype(np.uint32), return_counts=True)
    return fold(lu >> np.uint32(16), lu & np.uint32(0xFFFF), lc, m, int((~ok).sum()))


def fold_dense(counts, m, dropped=0):
    """A dense [k][65536] local-id histogram through map m."""
    lrow, lkey = np.nonzero(counts)
    return fold(lrow, lkey, counts[lrow, lkey], m, dropped)


def global_rows(local, m):
    """Each local id's row (int64), -1 where the op is dropped."""
    mm = np.array(list(m) + [UNBOUND], dtype=np.int64)
    g = mm[np.minimum(local.astype(np.int64), len(m))]
    return np.where(g == UNBOUND, -1, g)


def check(e, H, ref, dropped_before, what):
    """The interval's snapshot equals `ref` bucket for bucket and exactly ref's samples were dropped; returns it."""
    red, sp = e.snapshot(PS)
    u, c, dropped = ref
    flat = np.repeat(np.arange(H, dtype=np.int64), np.diff(sp.offsets.astype(np.int64))) * 65536 + sp.keys.view(np.uint16)
    order = np.argsort(flat, kind="stable")
    assert flat.size == u.size and (flat[order] == u).all(), (what, flat.size, u.size)
    assert (sp.counts[order] == c).all(), (what, np.nonzero(sp.counts[order] != c)[0][:5])
    totals = np.zeros(H, np.uint64)
    np.add.at(totals, u >> 16, c)
    assert (red.counts == totals).all(), what
    assert e.stats()["dropped"] - dropped_before == dropped, (what, e.stats()["dropped"] - dropped_before, dropped)
    return red, sp


_values = {}


def values(oracle, precision):
    """(float64 values, int64 ns, their uint16 keys at this precision) of N samples, shared per precision: stream S with
    every 7th value negative, the specials, and at every 17th sample the inputs just inside and outside the +-2^-12
    band around this precision's bucket boundaries; timer ns with every 5th negated and the int64 edges."""
    if precision not in _values:
        vals = oracle.gen_stream(oracle.STREAM_S, N, SEED ^ precision)
        vals[::7] = oracle.gen_stream(oracle.STREAM_N, N, SEED + 1)[::7]
        vals[3::1009] = SPECIALS[np.arange(vals[3::1009].size) % SPECIALS.size]
        band = R.epsilon_band_values(oracle, precision)
        at = np.arange(5, N, 17)[:band.size]
        vals[at] = band[:at.size]
        ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, N, SEED ^ precision).view(np.int64).copy()
        ns[::5] *= -1
        ns[2::97] = I64_EDGES[np.arange(ns[2::97].size) % I64_EDGES.size]
        _values[precision] = (vals, ns, oracle.compress_many(vals, precision).view(np.uint16),
                              oracle.compress_many(ns.astype(np.float64), precision).view(np.uint16))
    return _values[precision]


def mapped_call(e, id_bytes, m, d_ids, d_vals, kind, n):
    (e.ingest_keyed_mapped_u16 if id_bytes == 2 else e.ingest_keyed_mapped_u32)(m, d_ids, d_vals, kind, n)


def poke(e, d, positions, new):
    """d[positions] = new, element by element, from the host."""
    for p, v in zip(positions, new):
        a = np.array([v], dtype=d.dtype)
        e._check(e.lib.lh_memcpy_h2d(e.h, d.offset(int(p)), a.ctypes.data, a.nbytes))


# ------------------------------------------------------------------------------------------------------ full size
@gpu
@pytest.mark.parametrize("stream", ["U", "L"])
@pytest.mark.parametrize("n_log", [27, 30])
def test_mapped_full_size_against_the_oracle(lh, oracle, sms, n_log, stream):
    """k = 1024 at 2^27 and 2^30 samples generated on the device (2^30 is several chunks of the write-combining kernel):
    the identity map on a 1024-row engine, then, in its own interval, the raw call on the same arrays, which must give a
    bit-identical snapshot; and a scattered map into 4096 rows with a shared and an unbound entry on other owners.
    A strided handful of ids is overwritten with k, k + 1 and 65535."""
    k, n = 1024, 1 << n_log
    kind = oracle.STREAM_U if stream == "U" else oracle.STREAM_L
    want = R.keyed_route(k, n, 100, sms)
    assert want.kernel == R.WC and (want.wc.nchunks > 1) == (n_log == 30), want.wc
    P = want.wc.P
    ident = list(range(k))
    perm = scatter_map(k, 4 * k, SEED ^ n_log, unbound=(5 * P + 7,), dup=((P + 11, 3 * P + 20),))
    pos = np.arange(777, n, n // 48)
    bad = np.array([k, k + 1, 65535])[np.arange(pos.size) % 3]
    local = oracle.stream_ingest_keyed(kind, n, k, SEED)
    orig = np.array([oracle.gen_ids(0, 1, k, SEED, start=int(p))[0] for p in pos], np.int64)
    pkeys = oracle.compress_many(np.array([oracle.gen_stream(kind, 1, SEED, start=int(p))[0] for p in pos])).view(np.uint16)
    np.subtract.at(local, (orig, pkeys.astype(np.int64)), np.uint64(1))
    ref_ident, ref_perm = fold_dense(local, ident, pos.size), fold_dense(local, perm, pos.size)
    del local
    with lh.Engine(device=0, max_histograms=k, max_counters=1) as ea, \
         lh.Engine(device=0, max_histograms=4 * k, max_counters=1) as eb:
        d_v, d_i = ea.gen_stream(kind, n, SEED), ea.gen_ids_u16(0, n, k, SEED)
        ea.sync()
        poke(ea, d_i, pos, bad)
        before = ea.stats()["dropped"]
        ea.ingest_keyed_mapped_u16(ident, d_i, d_v, 0, n)
        assert ea.keyed_kernel_name() == R.WC
        red_m, sp_m = check(ea, k, ref_ident, before, ("identity", n_log, stream))
        ea.ingest_keyed_f64_u16(d_i, d_v, n)
        assert ea.keyed_kernel_name() == R.WC
        red_r, sp_r = ea.snapshot(PS)
        for a, b in ((sp_m.offsets, sp_r.offsets), (sp_m.keys, sp_r.keys), (sp_m.counts, sp_r.counts),
                     (red_m.counts, red_r.counts), (red_m.pkeys, red_r.pkeys)):
            assert np.array_equal(a, b)
        before = eb.stats()["dropped"]
        eb.ingest_keyed_mapped_u16(perm, d_i, d_v, 0, n)
        assert eb.keyed_kernel_name() == R.WC
        check(eb, 4 * k, ref_perm, before, ("scattered", n_log, stream))
        ea.sync()
        d_v.free()
        d_i.free()


@gpu
@pytest.mark.parametrize("kc", [16, 1024])
def test_mapped_counters_full_size_against_the_oracle(lh, oracle, kc):
    """2^27 counter adds generated on the device under kc local ids, through a scattered map into 8192 counters with a
    shared and an unbound entry."""
    C, n = 8192, 1 << 27
    m = scatter_map(kc, C, SEED ^ kc, unbound=(kc // 2,), dup=((1, kc - 1),))
    want_route = R.counter_route(kc, n)
    local = oracle.stream_counter(n, kc, SEED)
    ops_unbound = int((oracle.gen_ids(0, n, kc, SEED) == kc // 2).sum())
    g = np.array(m, np.int64)
    want = np.zeros(C, np.uint64)
    np.add.at(want, g[g != UNBOUND], local[g != UNBOUND])
    with lh.Engine(device=0, max_histograms=1, max_counters=C) as e:
        d_a, d_i = e.gen_stream(lh.STREAM_AMOUNTS, n, SEED), e.gen_ids_u16(0, n, kc, SEED)
        st0 = e.stats()
        e.counter_add_mapped_u16(m, d_i, d_a, n)
        assert e.stats()["kernel_launches"] - st0["kernel_launches"] == want_route.extra["launches"], want_route
        _, sp = e.snapshot(PS)
        assert (sp.counter_deltas == want).all(), np.nonzero(sp.counter_deltas != want)[0][:5]
        assert e.stats()["dropped"] - st0["dropped"] == ops_unbound
        d_a.free()
        d_i.free()


# ------------------------------------------------------------------------------------------------- route boundaries
def scope_cases(precision, sms, reserve):
    """[(label, k)] of the mapped keyed route boundaries at this precision and P = sm_count - reserve, k <= LH_MAP_MAX:
    the small kernel's edge from both sides, idle owners (k < P), each owner-buffer size the host can pick, and the
    write-combining kernel's largest k and the one past it (or the full map where it takes every k)."""
    P = sms - reserve
    caps, kmax = R.wc_h_by_row_cap(precision, sms, reserve, lo=1, hi=MAP_MAX + 1)
    edge = R.small_edge(precision)
    cases = []
    if reserve == 0:
        cases += [("small_edge", edge), ("past_small_edge", edge + 1)]
    if edge + 1 < P:
        cases.append(("idle_owners", (edge + P) // 2))
    for cap in sorted(caps, reverse=True):
        ks = [h for h in caps[cap] if h > edge and h % P]
        if ks:
            cases.append(("row_cap_%d" % cap, ks[len(ks) // 2]))
    cases.append(("full_map", kmax) if kmax == MAP_MAX else ("wc_max", kmax))
    if kmax < MAP_MAX:
        cases.append(("past_wc_max", kmax + 1))
    return cases


RESERVES = {"0": lambda sms: 0, "1": lambda sms: 1, "sm-8": lambda sms: sms - 8}


@gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("reserve", list(RESERVES))
def test_mapped_route_boundaries(lh, oracle, sms, precision, reserve):
    """At every route boundary in local-id space: the predicted kernel runs, and every bucket is exact, for u16 and u32
    ids (u16: ids k and 65535; u32: 65536 + j, 2^31, 2^32 - 1 with j bound) and float64 and int64 values."""
    k1_reserve = RESERVES[reserve](sms)
    vals, ns, keys, nskeys = values(oracle, precision)
    with lh.Engine(device=0, max_histograms=H_BIG, max_counters=1, precision=precision) as e:
        e.tune("k1_reserve_sms", k1_reserve)
        d_v, d_n = e.upload(vals), e.upload(ns)
        for label, k in scope_cases(precision, sms, k1_reserve):
            want = R.keyed_route(k, N, precision, sms, k1_reserve_sms=k1_reserve)
            expect = {"small_edge": R.SMALL, "past_wc_max": R.VEC}.get(label, R.WC)
            assert want.kernel == expect, (label, k, want)
            if label.startswith("row_cap_"):
                assert want.wc.row_cap == int(label[8:]), (label, k, want)
            if label == "idle_owners":
                assert k < want.wc.P
            if label == "small_edge":
                assert want.passes == R.CONST["KS_MAX_PASSES"]
            m = awkward_map(k, H_BIG, SEED ^ k ^ precision)
            local = oracle.gen_ids(0, N, k + 2, SEED ^ k)                   # ~2/(k+2) of them past the names
            assert m[2] != UNBOUND
            l16 = R.with_bad_ids(local, np.array([k, 65535], np.uint32), 997)
            l32 = R.with_bad_ids(local, R.high_ids(k, 2), 997)              # 65538 must not be counted into local id 2
            ref_f, ref_n = reference(l16, keys, m), reference(l16, nskeys, m)
            d16, d32 = e.upload(l16.astype(np.uint16)), e.upload(l32)
            for name, d_i, id_bytes, d_x, kind, ref in (("u16_f64", d16, 2, d_v, 0, ref_f), ("u32_f64", d32, 4, d_v, 0, ref_f),
                                                        ("u16_i64", d16, 2, d_n, 1, ref_n), ("u32_i64", d32, 4, d_n, 1, ref_n)):
                route = R.keyed_route(k, N, precision, sms, id_bytes=id_bytes, k1_reserve_sms=k1_reserve)
                assert route.kernel == want.kernel
                before = e.stats()["dropped"]
                mapped_call(e, id_bytes, m, d_i, d_x, kind, N)
                assert e.keyed_kernel_name() == route.kernel, (precision, reserve, label, k, name)
                check(e, H_BIG, ref, before, (precision, reserve, label, k, name))
            d16.free()
            d32.free()


# misaligned values / ids: (k, n, value offset, id offset) in elements, and the route each must take
def misaligned_cases():
    out = []
    for off in range(4):                      # the scalar head before a vector body (write-combining, small kernel)
        out += [(300, N - 3, off, off), (R.small_edge(100), 1 << 20, off, off)]
    out += [(300, 100_003, 0, 1), (300, 100_003, 2, 1), (300, 100_003, 1, 3)]   # ids misaligned: the scalar kernel only
    return out


@gpu
@pytest.mark.parametrize("id_bytes", [2, 4])
def test_mapped_misaligned(lh, oracle, sms, id_bytes):
    """The scalar head before the vector body and the scalar-only route, at element offsets 0 - 3."""
    precision, H = 100, 2048
    vals, _, keys, _ = values(oracle, precision)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_v = e.upload(vals)
        for k, n, voff, ioff in misaligned_cases():
            m = awkward_map(k, H, SEED ^ k)
            local = oracle.gen_ids(0, n + 3, k + 1, SEED ^ k ^ voff)
            if id_bytes == 4:
                local = R.with_bad_ids(local, R.high_ids(k, 2), 101)
            d_i = e.upload(local.astype(np.uint16 if id_bytes == 2 else np.uint32))
            want = R.keyed_route(k, n, precision, sms, id_bytes=id_bytes, vals_addr=8 * voff, ids_addr=id_bytes * ioff)
            assert (want.kernel == R.SCALAR) == (voff != ioff), want
            assert (want.head > 0) == (voff == ioff and voff > 0), want
            before = e.stats()["dropped"]
            mapped_call(e, id_bytes, m, d_i.offset(ioff), d_v.offset(voff), 0, n)
            assert e.keyed_kernel_name() == want.kernel, (k, n, voff, ioff)
            check(e, H, reference(local[ioff:ioff + n], keys[voff:voff + n], m), before, (k, n, voff, ioff))
            d_i.free()


# --------------------------------------------------------------------------------------------------- capacity paths
@gpu
@pytest.mark.parametrize("chunk,spt,flush", [(65536, 6, 24576), (1 << 20, 6, 4096), (1 << 20, 4, 65536), (65536, 3, 24576),
                                             (1 << 20, 8, 16384)])
def test_mapped_wc_many_chunks(lh, oracle, sms, chunk, spt, flush):
    """Several chunks of the mapped write-combining kernel (grid barriers, sub-queue parity) with every tile shape,
    skewed ids (the owners of low ids overflow their buffers at wc_flush 65536)."""
    k, H, precision = 1000, 2048, 100
    tune = dict(kp_chunk=chunk, wc_spt=spt, wc_flush=flush)
    vals, ns, keys, nskeys = values(oracle, precision)
    m = awkward_map(k, H, SEED ^ chunk ^ spt)
    local = R.with_bad_ids(oracle.gen_ids(1, N, k + 2, SEED ^ spt), R.high_ids(k, 2), 1001)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        for key, v in tune.items():
            e.tune(key, v)
        d_v, d_n = e.upload(vals), e.upload(ns)
        d16, d32 = e.upload(np.minimum(local, 65535).astype(np.uint16)), e.upload(local)
        for name, d_i, id_bytes, d_x, kind, kk in (("u16_f64", d16, 2, d_v, 0, keys), ("u32_i64", d32, 4, d_n, 1, nskeys)):
            want = R.keyed_route(k, N, precision, sms, id_bytes=id_bytes, **tune)
            assert want.kernel == R.WC and want.wc.nchunks > 1, want
            before = e.stats()["dropped"]
            mapped_call(e, id_bytes, m, d_i, d_x, kind, N)
            assert e.keyed_kernel_name() == R.WC
            check(e, H, reference(local, kk, m), before, (chunk, spt, flush, name))


@gpu
@pytest.mark.parametrize("k,reserve", [(1024, 0), (1000, 1)])
def test_mapped_wc_one_owner_takes_every_record(lh, oracle, sms, k, reserve):
    """Distinct local ids all congruent modulo P, mapped to scattered rows (one unbound, two sharing a row): one owner
    receives every record, its buffer overflows in every writer and its sub-queues in every chunk, so the surplus goes
    through wc_spill, which must resolve the row through the map."""
    H, precision = 2048, 100
    P = sms - reserve
    tune = {"k1_reserve_sms": reserve}
    threads, per = R.CONST["WC_SHAPES"][R.DEFAULTS["wc_spt"]]
    tune.update(kp_chunk=2 * P * threads * per, wc_flush=4096)
    vals = oracle.gen_stream(oracle.STREAM_S, N, SEED ^ 0x0E)
    vals[::7] = -vals[::7]
    keys = oracle.compress_many(vals, precision).view(np.uint16)
    local = R.same_residue_ids(N, k, P, 3, SEED)
    pool = np.arange(3, k, P)
    m = scatter_map(k, H, SEED ^ k, unbound=(int(pool[1]),), dup=((int(pool[2]), int(pool[4])),))
    want = R.keyed_route(k, N, precision, sms, **tune)
    assert want.kernel == R.WC and want.wc.P == P
    _, spilled = R.wc_owner_queue(~R.definitely_exact(vals[:want.wc.taken]), want.wc)
    assert spilled.sum() > 0, want.wc
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        for key, v in tune.items():
            e.tune(key, v)
        d_v, d_i = e.upload(vals), e.upload(local.astype(np.uint16))
        before = e.stats()["dropped"]
        e.ingest_keyed_mapped_u16(m, d_i, d_v, 0, N)
        assert e.keyed_kernel_name() == R.WC
        check(e, H, reference(local, keys, m), before, ("one owner", k, P))


@gpu
@pytest.mark.parametrize("reserve", [0, 1])
def test_mapped_wc_rare_queue_overflow(lh, oracle, sms, reserve):
    """Every sample needs the exact route: each CTA sets aside more than WC_RARE_CAP samples per chunk and resolves the
    rest on the spot through the mapped keyed_one_slow_v, with unbound entries, ids >= k and high u32 ids mixed in."""
    k, H, precision, n = 300, 2048, 100, (1 << 22) + 3
    vals = R.exact_route_values(oracle, n, SEED)
    local = R.with_bad_ids(oracle.gen_ids(0, n, k + 3, SEED ^ 0x5A), R.high_ids(k, 7), 1013)
    m = awkward_map(k, H, SEED ^ 0x5A)
    assert m[7] != UNBOUND
    want = R.keyed_route(k, n, precision, sms, id_bytes=4, k1_reserve_sms=reserve)
    assert want.kernel == R.WC
    rare = R.definitely_exact(vals) | (local >= k)
    assert R.wc_slice_counts(rare, want.wc).max() > R.CONST["WC_RARE_CAP"]
    keys = oracle.compress_many(vals, precision).view(np.uint16)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        e.tune("k1_reserve_sms", reserve)
        d_v, d_i = e.upload(vals), e.upload(local)
        before = e.stats()["dropped"]
        e.ingest_keyed_mapped_u32(m, d_i, d_v, 0, n)
        assert e.keyed_kernel_name() == R.WC
        check(e, H, reference(local, keys, m), before, "rare overflow")


@gpu
def test_mapped_small_kernel_later_passes(lh, oracle, sms):
    """A 4-pass launch of the small kernel whose unbound and shared entries sit in passes 1 - 3 only."""
    precision, H = 100, 2048
    per = R.ks_ids_per_pass(precision)
    k = R.small_edge(precision)
    want = R.keyed_route(k, N, precision, sms)
    assert want.kernel == R.SMALL and want.passes == 4
    m = scatter_map(k, H, SEED ^ 0x44, unbound=(per + 3, 3 * per + 5), dup=((per + 7, 2 * per + 1), (2 * per, 3 * per)))
    vals, ns, keys, nskeys = values(oracle, precision)
    local = oracle.gen_ids(0, N, k + 2, SEED ^ 0x44)
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_v, d_n, d_i = e.upload(vals), e.upload(ns), e.upload(local.astype(np.uint16))
        for d_x, kind, kk in ((d_v, 0, keys), (d_n, 1, nskeys)):
            before = e.stats()["dropped"]
            e.ingest_keyed_mapped_u16(m, d_i, d_x, kind, N)
            assert e.keyed_kernel_name() == R.SMALL
            check(e, H, reference(local, kk, m), before, ("small passes", kind))


# ----------------------------------------------------------------------------------------------------------- values
@gpu
@pytest.mark.parametrize("k,tune,off", [(44, {}, 0), (300, {"keyed_mode": 1}, 0), (1000, {}, 0), (300, {}, 1)])
def test_mapped_i64_edges_against_the_oracle(lh, oracle, sms, k, tune, off):
    """int64 nanoseconds on every mapped route (small, vector, write-combining, scalar): negatives, 0, INT64_MIN,
    INT64_MAX, 2^53 +- 1 and the ties above 2^53, against oracle.ingest_keyed_i64 on the local ids, folded through the
    map."""
    H = 2048
    n = N if off == 0 else 100_003
    _, ns, _, _ = values(oracle, 100)
    ns = ns[:n].copy()
    ns[1::13] = I64_EDGES[np.arange(ns[1::13].size) % I64_EDGES.size]
    m = awkward_map(k, H, SEED ^ k ^ 0x64)
    local = oracle.gen_ids(0, n + off, k + 1, SEED ^ 0x64)
    sel = local[off:off + n]
    ok = sel < k
    dense = oracle.ingest_keyed_i64(sel[ok], ns[ok], k)
    ref = fold_dense(dense, m, int((~ok).sum()))
    del dense
    want = R.keyed_route(k, n, 100, sms, ids_addr=2 * off, **tune)
    assert want.kernel == {44: R.SMALL, 1000: R.WC}.get(k, R.SCALAR if off else R.VEC), want
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        for key, v in tune.items():
            e.tune(key, v)
        d_n, d_i = e.upload(ns), e.upload(local.astype(np.uint16))
        before = e.stats()["dropped"]
        e.ingest_keyed_mapped_u16(m, d_i.offset(off), d_n, 1, n)
        assert e.keyed_kernel_name() == want.kernel
        check(e, H, ref, before, (k, tune, off))


@gpu
def test_mapped_high_u32_ids_are_dropped_on_every_route(lh, oracle, sms):
    """u32 local ids 65536 + j, 2^31 and 2^32 - 1 (map[j] a bound row) through the small, vector, write-combining and
    scalar mapped kernels: dropped and counted, never added to row map[j]."""
    precision, H = 100, 2048
    vals, _, keys, _ = values(oracle, precision)
    for k, tune in ((5, {}), (300, {"keyed_mode": 1}), (300, {})):
        m = scatter_map(k, H, SEED ^ k, unbound=(3,), dup=((0, 4),)) if k < 8 else awkward_map(k, H, SEED ^ k)
        j = 2
        assert m[j] != UNBOUND
        local = R.with_bad_ids(oracle.gen_ids(0, N, k, SEED ^ k), R.high_ids(k, j), 101)
        with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
            for key, v in tune.items():
                e.tune(key, v)
            d_v, d_i = e.upload(vals), e.upload(local)
            for off, n in ((0, N), (1, 100_003)):     # off 1: ids not 16-byte aligned, the scalar kernel only
                want = R.keyed_route(k, n, precision, sms, id_bytes=4, ids_addr=4 * off, **tune)
                assert (want.kernel == R.SCALAR) == (off == 1), want
                before = e.stats()["dropped"]
                e.ingest_keyed_mapped_u32(m, d_i.offset(off), d_v, 0, n)
                assert e.keyed_kernel_name() == want.kernel, (k, tune, off)
                check(e, H, reference(local[off:off + n], keys[:n], m), before, (k, tune, off))


# ---------------------------------------------------------------------------------------------------------- counters
@gpu
@pytest.mark.parametrize("kc", [16, 1024, MAP_MAX])
@pytest.mark.parametrize("unbound", [True, False])
def test_mapped_counter_routes(lh, oracle, kc, unbound):
    """The mapped shared-memory counter kernels (vector body, scalar head and tail; kc = LH_MAP_MAX is 48 KiB of shared
    memory for the counters and the map), with and without an unbound entry: amounts that carry out of every half
    (2^32 - 1, 2^32, 2^64 - 1, 2^63) piled on one hot local id, u16 and u32 ids (u32 also >= 65536), ids >= kc.  The
    number of launches is the predicted route's."""
    C, n = 8192, 300_007
    rng = np.random.default_rng(kc)
    local = rng.integers(0, kc + 2, n + 8).astype(np.uint32)
    local[::3] = 5                                                 # one hot counter: carries pile up in it
    amounts = rng.integers(0, 2 ** 64, n + 8, dtype=np.uint64)
    special = np.array([2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, 1 << 63], np.uint64)
    amounts[::2] = special[np.arange(amounts[::2].size) % 4]
    l32 = R.with_bad_ids(local, R.high_ids(kc, 5), 89)
    m = scatter_map(kc, C, SEED ^ kc, unbound=(kc // 2, kc - 1) if unbound else (), dup=((0, kc - 2), (1, kc // 3)))
    assert m[5] != UNBOUND and m[5] != m[kc - 1]
    with lh.Engine(device=0, max_histograms=1, max_counters=C) as e:
        d_i16, d_i32, d_a = e.upload(local.astype(np.uint16)), e.upload(l32), e.upload(amounts)
        for name, d_i, host_ids, id_bytes in (("u16", d_i16, local, 2), ("u32", d_i32, l32, 4)):
            f = e.counter_add_mapped_u16 if id_bytes == 2 else e.counter_add_mapped_u32
            for off, cnt in ((0, n), (1, n - 1), (3, 65_541), (2, 20_000)):
                route = R.counter_route(kc, cnt, id_bytes=id_bytes, amounts_addr=8 * off, ids_addr=id_bytes * off)
                assert route.kernel == R.COUNTER_SMEM
                st0 = e.stats()
                f(m, d_i.offset(off), d_a.offset(off), cnt)
                assert e.stats()["kernel_launches"] - st0["kernel_launches"] == route.extra["launches"], (name, off, route)
                _, sp = e.snapshot(PS)
                g = global_rows(host_ids[off:off + cnt], m)
                ok = g >= 0
                want = oracle.counter_add(g[ok], amounts[off:off + cnt][ok], C)
                assert (sp.counter_deltas == want).all(), (kc, name, off, np.nonzero(sp.counter_deltas != want)[0][:5])
                assert e.stats()["dropped"] - st0["dropped"] == int((~ok).sum()), (kc, name, off)


# -------------------------------------------------------------------------------------------------------- scope limit
@gpu
def test_scope_keyed_name_limit(lh, torch, oracle):
    """A MetricSystem record scope over LH_MAP_MAX + 1 histogram names: keyed() raises before anything is enqueued and
    counts nothing as dropped, and the scope still takes histograms() and ends.  Exactly LH_MAP_MAX names work."""
    from loghisto_b200.metric_system import MetricSystem
    names = ["s%d" % i for i in range(MAP_MAX + 1)]
    n = 1 << 20
    rng = np.random.default_rng(SEED)
    vals = rng.lognormal(2.0, 3.0, n)
    local = rng.integers(0, MAP_MAX + 1, n).astype(np.int32)      # local id MAP_MAX is past the names of the second scope
    d_vals, d_local = torch.from_numpy(vals).cuda(), torch.from_numpy(local).cuda()

    def dense(h):
        out = np.zeros(65536, np.uint64)
        for key, c in h.items():
            out[int(key) & 0xFFFF] += c
        return out
    ms = MetricSystem(1e-6, False, max_histograms=2 * MAP_MAX)
    try:
        with ms.recording(histograms=names) as s:
            with pytest.raises(RuntimeError):
                s.keyed(d_local, d_vals)
            s.histograms([(names[-1], d_vals[:1000])])
        torch.cuda.synchronize()
        assert ms.dropped() == 0
        raw, _ = ms.collect_and_process()
        got = {nm: h for nm, h in raw["Histograms"].items() if sum(h.values())}
        assert list(got) == [names[-1]] and (dense(got[names[-1]]) == oracle.ingest(vals[:1000])).all()

        with ms.recording(histograms=names[:MAP_MAX]) as s:
            s.keyed(d_local, d_vals)
        torch.cuda.synchronize()
        assert ms.dropped() == int((local == MAP_MAX).sum())
        raw, _ = ms.collect_and_process()
        for i in range(MAP_MAX):
            assert sum(raw["Histograms"].get(names[i], {}).values()) == int((local == i).sum()), names[i]
        for i in (0, 1, MAP_MAX // 2, MAP_MAX - 1):
            assert (dense(raw["Histograms"][names[i]]) == oracle.ingest(vals[local == i])).all(), names[i]
    finally:
        ms.close()


# ----------------------------------------------------------------------------------------------------- without a GPU
def test_scope_cases_reach_every_route_and_row_cap():
    """On a 132-SM H100 the cases above reach every keyed route, each owner-buffer size at P = sm_count and
    sm_count - 1, k = LH_MAP_MAX on the write-combining kernel with the smallest buffer, several chunks at 2^30, and
    the scalar head and scalar-only routes."""
    sms = 132
    for reserve in (0, 1):
        caps, kernels, full = set(), set(), []
        for precision in PRECISIONS:
            for label, k in scope_cases(precision, sms, reserve):
                r = R.keyed_route(k, N, precision, sms, k1_reserve_sms=reserve)
                kernels.add(r.kernel)
                if r.wc:
                    caps.add(r.wc.row_cap)
                if k == MAP_MAX:
                    full.append((precision, r.kernel, r.wc and r.wc.row_cap))
        assert caps == set(R.CONST["WC_ROW_CAPS"]), (reserve, caps)
        assert kernels == ({R.SMALL} if reserve == 0 else set()) | {R.WC, R.VEC}, (reserve, kernels)
        assert (31, R.WC, min(R.CONST["WC_ROW_CAPS"])) in full, (reserve, full)
    assert R.keyed_route(1024, 1 << 30, 100, sms).wc.nchunks > 1
    assert R.keyed_route(1024, 1 << 27, 100, sms).wc.nchunks == 1
    for id_bytes in (2, 4):
        routes = [R.keyed_route(k, n, 100, sms, id_bytes=id_bytes, vals_addr=8 * v, ids_addr=id_bytes * i)
                  for k, n, v, i in misaligned_cases()]
        assert {r.kernel for r in routes} == {R.SMALL, R.WC, R.SCALAR}
        assert any(r.head for r in routes if r.kernel == R.WC) and any(r.head for r in routes if r.kernel == R.SMALL)
