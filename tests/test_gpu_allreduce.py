"""K5 (`k_peer_allreduce`, behind lh_snapshot_allreduce) against the exact reduction reference of
tests/_reduce_cases.py.

The constructed histograms of every precision (totals up to 2^64 - 2, keys at +-(win-1), +-win, 0, -1, -32768 and
32767) are split over 2, 3 and 4 ranks -- more where the box has more GPUs; rank r runs on device r % device_count(),
so on a single GPU every rank shares it.  A histogram is untouched everywhere, on one rank only, dense on one rank
and window-only on another (a third untouched), or spread over every rank in parts that sum exactly (some 0).  Each
rank is fed its share with merge_counts_host; after the all-reduce every rank must give the merged histogram: counts,
percentile keys and values exact, sums within rc.sum_ok, averages bit-exact as sum / float64(count), the export, the
dense rows of lh_snapshot_copy_histogram, and every bit of the results of one context given the union of the shares.

H sits on either side of the payload switch between the one-shot and the two-shot form (H * (2 win - 1) * 8 bytes
against 1 MiB), computed from the window, and the form is asserted through last_bytes_from_peers.  One rank is held
back by a bounded spin on its ingest stream before its last write, so the others' K5 waits for its arrival.

Only the parity case injects a failure (one extra local snapshot on one rank), and it returns at once: no test leaves
a rank without its collective.  No write-combining keyed launch is queued behind a waiting K5."""
import contextlib
import ctypes as C
import math
import random

import numpy as np
import pytest

import _ingest_routes as R
import _reduce_cases as rc

pytestmark = pytest.mark.gpu

SEED = 0xA11ED0CE
PRECISIONS = (1, 46, 100, 146, 147, 250)
FORMS = ("one-shot", "two-shot")
PAYLOAD_SWITCH = 1 << 20          # lh_snapshot_allreduce: the two-shot form from this many window bytes on
NC = 3000                         # counters: more than one pass of K5's 1024-thread counter loop
MS = 1_000_000                    # one millisecond of spin, in ns
PS = [0.0, 0.25, 0.5, 0.9, 0.99, 1.0]
U64 = 2 ** 64
LH_ERR_INVALID, LH_ERR_STATE = -1, -5


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def ndev():
    import torch
    n = torch.cuda.device_count()
    assert n >= 1
    return n


@pytest.fixture(scope="module")
def spin(ndev):
    """spin(engine, ns): one bounded spin of at least `ns` on the engine's ingest stream (tests/gpu_timer_client.cu),
    so that the engine's next write, and with it its K5, starts that much later.  The spin kernel is launched once on
    every device first (see warm_up)."""
    import torch
    from loghisto_b200 import build
    lib = C.CDLL(build.TIMER_CLIENT_LIB)
    lib.gtc_set_device.argtypes = [C.c_int]
    lib.gtc_spin.argtypes = [C.c_uint64, C.c_void_p]
    lib.gtc_set_device.restype = lib.gtc_spin.restype = C.c_int
    for d in range(ndev):
        assert lib.gtc_set_device(d) == 0 and lib.gtc_spin(1000, None) == 0
        torch.cuda.synchronize(d)

    def run(eng, ns):
        assert 5 * MS <= ns <= 30 * MS
        assert lib.gtc_set_device(eng.device) == 0
        assert lib.gtc_spin(int(ns), eng.ingest_stream) == 0
    return run


# ------------------------------------------------------------------------------------------------ shapes
def wcells(precision: int) -> int:
    return 2 * rc.window(precision) - 1


def form_H(precision: int, form: str) -> int:
    """The largest H of the one-shot form, or the smallest of the two-shot form, at this precision."""
    two = -(-PAYLOAD_SWITCH // (8 * wcells(precision)))        # smallest H with H * wcells * 8 >= 1 MiB
    return two if form == "two-shot" else two - 1


def expected_bytes(flags, precision: int, world: int, form: str) -> int:
    """last_bytes_from_peers: every dense histogram counts 65536 cells, every window-only one 2 win - 1."""
    cells = sum(65536 if f & 2 else wcells(precision) for f in flags if f)
    return cells * 8 * (world - 1) // world if form == "two-shot" else cells * 8 * (world - 1)


def test_form_edges():
    """The H on either side of the switch: 15 / 16 at precision 100, 6 / 7 at 250, 1472 / 1473 at 1."""
    assert [form_H(p, f) for p in (1, 100, 250) for f in FORMS] == [1472, 1473, 15, 16, 6, 7]
    for p in PRECISIONS:
        for f in FORMS:
            H = form_H(p, f)
            assert (H * wcells(p) * 8 >= PAYLOAD_SWITCH) == (f == "two-shot")
            assert ((H + (1 if f == "one-shot" else -1)) * wcells(p) * 8 >= PAYLOAD_SWITCH) == (f == "one-shot")


def warm_up(engs, ingest=None):
    """Every kernel a rank may launch while a peer's K5 waits for it, launched once beforehand, outside any collective.
    With CUDA's lazy module loading the first launch of a kernel may synchronise the context; on a device shared with
    a waiting K5 it would wait for that K5, which waits for this rank: the peers would give up after 10 s.  `ingest(r,
    e)` issues a rank's writes; by default one merge and one counter add.  Each rank then takes one local snapshot
    (reduction, export, copy), so the ranks stay in lock-step."""
    for r, e in enumerate(engs):
        if ingest is not None:
            ingest(r, e)
        else:
            e.merge_counts_host(np.zeros(1, np.uint32), np.zeros(1, np.int16), np.ones(1, np.uint64))
            e.counter_add_u16_host(np.zeros(1, np.uint16), np.ones(1, np.uint64))
        e.snapshot_begin()
        try:
            e.snapshot_result(e.snapshot_reduce_async(PS))
            e.snapshot_export()
            e.snapshot_copy_histogram(0)
        finally:
            e.snapshot_end()
        e.sync()


@contextlib.contextmanager
def contexts(lh, ndev, world, H, C, precision):
    """`world` mapped contexts (rank r on device r % ndev), warmed up, and one unmapped reference context on device 0."""
    engs = []
    try:
        for r in range(world):
            engs.append(lh.Engine(device=r % ndev, max_histograms=H, max_counters=C, precision=precision))
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, world, handles)
        warm_up(engs)
        engs.append(lh.Engine(device=0, max_histograms=H, max_counters=C, precision=precision))
        yield engs[:world], engs[world]
    finally:
        for e in engs:
            e.close()


def collective(engs, counters, hold=None, skewed=None, before=None):
    """snapshot_begin + snapshot_allreduce on every rank, the skewed rank last, with `hold()` (its spin and last write)
    just before it and `before(r, e)` after each rank's snapshot_begin.  Every rank issues its all-reduce even when a
    call before it raised, so no rank's K5 is left waiting for a peer; the first error is raised afterwards."""
    order = [r for r in range(len(engs)) if r != skewed] + ([skewed] if skewed is not None else [])
    seqs, err = [0] * len(engs), None
    for r in order:
        if r == skewed and hold is not None:
            try:
                hold()
            except BaseException as ex:         # pragma: no cover - reported below
                err = err or ex
        engs[r].snapshot_begin()
        if before is not None:
            try:
                before(r, engs[r])
            except BaseException as ex:         # pragma: no cover - reported below
                err = err or ex
        seqs[r] = engs[r].snapshot_allreduce(counters)
    if err is not None:
        raise err
    return seqs


# ------------------------------------------------------------------------------------------------ splitting
def split_hist(hist: dict, layout: str, world: int, precision: int, rng: random.Random) -> list:
    """[(key, count)] per rank for one histogram.  "one": every triple on one rank.  "mixed": out-of-window keys on one
    rank, window keys on a second (both on two ranks, alternating, when there are only window keys), the others
    untouched.  "all": every key on every rank, the count cut at random points, so that parts of 0 occur and the
    parts sum to the count exactly.  "spread": every key on every rank with a world-th of its count (the remainder on
    random ranks), so that a histogram whose counts sum to 2^64 or more reaches each rank as a share below 2^64."""
    w = rc.window(precision)
    pick = rng.sample(range(world), 2)
    parts = [[] for _ in range(world)]
    if layout == "one":
        parts[pick[0]] = list(hist.items())
    elif layout == "mixed":
        window_only = all(-w < k < w for k in hist)
        for i, (k, c) in enumerate(sorted(hist.items())):
            inside = -w < k < w
            parts[pick[i % 2] if window_only else pick[1 if inside else 0]].append((k, c))
    elif layout == "spread":
        for k, c in hist.items():
            amounts = [c // world] * world
            for r in rng.sample(range(world), c % world):
                amounts[r] += 1
            for r in range(world):
                parts[r].append((k, amounts[r]))
    else:
        for k, c in hist.items():
            cuts = sorted(rng.randrange(c + 1) for _ in range(world - 1))
            amounts = [b - a for a, b in zip([0] + cuts, cuts + [c])]
            if world > 2:                         # one rank merges an explicit 0 count
                z, to = rng.sample(range(world), 2)
                amounts[to] += amounts[z]
                amounts[z] = 0
            for r in range(world):
                parts[r].append((k, amounts[r]))
    return parts


def triples(rows: list) -> tuple:
    """(ids, keys, counts) arrays of [(hid, key, count)]."""
    if not rows:
        return np.zeros(0, np.uint32), np.zeros(0, np.int16), np.zeros(0, np.uint64)
    h, k, c = zip(*rows)
    return np.array(h, np.uint32), np.array(k, np.int16), np.array(c, np.uint64)


def counter_shares(world: int, seed: int) -> list:
    """Per rank (u16 ids, amounts): amounts near 2^64 so the sums wrap, every id up to NC - 1, one hot id."""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(world):
        n = 4000 + 17 * r
        ids = rng.integers(0, NC, n).astype(np.uint16)
        ids[:3] = (0, NC - 1, 1024)
        ids[::5] = 7
        amounts = (U64 - 1 - rng.integers(0, 1 << 20, n, dtype=np.uint64)).astype(np.uint64)
        out.append((ids, amounts))
    return out


def counter_sum(oracle, shares) -> np.ndarray:
    want = np.zeros(NC, np.uint64)
    for ids, amounts in shares:
        oracle.counter_add(ids.astype(np.uint32), amounts, NC, want)
    return want


# ------------------------------------------------------------------------------------------------ expectations
class Expect:
    """What a reduction of `refs` (one rc.Reference per histogram id) with percentiles `ps` must give."""

    def __init__(self, refs: list, ps: list):
        H, n = len(refs), len(ps)
        self.refs, self.ps = refs, ps
        self.counts = np.array([r.count for r in refs], np.uint64)
        self.pkeys = np.full((H, n), rc.INT32_MIN, np.int32)
        self.pvals = np.full((H, n), math.nan)
        self.live = [h for h, r in enumerate(refs) if r.nnz]        # a count that wrapped to 0 is live
        for h in self.live:
            res = refs[h].results(ps)
            self.pkeys[h] = [rc.INT32_MIN if k is None else k for k in res["keys"]]
            self.pvals[h] = res["values"]
        nnz = np.array([r.nnz for r in refs], np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(nnz)])
        self.keys = np.concatenate([r.keys for r in refs] + [np.zeros(0, np.int16)])
        self.xcounts = np.concatenate([r.counts for r in refs] + [np.zeros(0, np.uint64)])

    def check(self, red, sp, what):
        assert (red.counts == self.counts).all(), (what, np.flatnonzero(red.counts != self.counts)[:5])
        bad = np.flatnonzero((red.pkeys != self.pkeys).any(axis=1))
        assert bad.size == 0, (what, [(int(h), self.refs[h].name) for h in bad[:5]])
        assert rc.same_bits(red.pvals, self.pvals).all(), (what, np.flatnonzero(~rc.same_bits(red.pvals, self.pvals).all(axis=1))[:5])
        dead = [h for h, r in enumerate(self.refs) if not r.nnz]
        assert (red.sums[dead] == 0).all() and np.isnan(red.avgs[dead]).all(), what
        for h in self.live:
            s = float(red.sums[h])
            assert rc.sum_ok(s, self.refs[h]), (what, h, self.refs[h].name, s, float(self.refs[h].sum))
            assert rc.same_bits(red.avgs[h], rc.avg_of(s, self.refs[h])), (what, h, self.refs[h].name)
        if sp is not None:
            assert (sp.offsets.astype(np.int64) == self.offsets).all(), what
            assert (sp.keys == self.keys).all() and (sp.counts == self.xcounts).all(), what


def same_results(a, b) -> bool:
    """Every bit of two reductions (sums, averages and NaN payloads included)."""
    return ((a.counts == b.counts).all() and (a.pkeys == b.pkeys).all()
            and (a.sums.view(np.uint64) == b.sums.view(np.uint64)).all()
            and (a.avgs.view(np.uint64) == b.avgs.view(np.uint64)).all()
            and (a.pvals.view(np.uint64) == b.pvals.view(np.uint64)).all())


def same_export(a, b) -> bool:
    return ((a.offsets == b.offsets).all() and (a.keys == b.keys).all() and (a.counts == b.counts).all())


_CASES = {}


def cases_for(oracle, precision):
    """(table, cases, {case index: Reference}, percentile batches, number of make_cases cases, batches of the wrapped
    cases), built once per precision.  The cases of make_wrapped_cases (precisions of tests/_reduce_cases.py) follow
    those of make_cases."""
    if precision not in _CASES:
        table = oracle.decompress_table(precision)
        cases = rc.make_cases(precision, table, SEED)
        batches = rc.percentile_batches(rc.percentile_pool(cases, table, SEED))
        n_plain = len(cases)
        wbatches = []
        if precision in rc.PRECISIONS:
            wrapped = rc.make_wrapped_cases(precision, table, SEED)
            cases = cases + wrapped
            wbatches = rc.percentile_batches(rc.wrapped_percentile_pool(wrapped, table, SEED))
        refs = [rc.Reference(c["hist"], table, c["name"]) for c in cases]
        _CASES[precision] = (table, cases, refs, batches, n_plain, wbatches)
    return _CASES[precision]


# ------------------------------------------------------------------------------------------------ the matrix
@pytest.mark.parametrize("world", [2, 3, 4, "all"])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_allreduce_constructed_cases(lh, oracle, ndev, spin, precision, form, world):
    """Every constructed case of the precision, packed into intervals of H - 1 histograms at random ids (at least one
    id untouched), each split over the ranks by a layout that rotates over the cases; one rank held back per
    interval; counters included in every other interval; then an empty interval.  Then the cases whose counts sum to
    2^64 or more, each spread so that every rank's share stays below 2^64 (those that need more ranks are left out)."""
    if world == "all":
        world = min(8, ndev)
        if world <= 4:
            pytest.skip("needs more than 4 GPUs")
    H = form_H(precision, form)
    table, cases, case_refs, batches, n_plain, wbatches = cases_for(oracle, precision)
    empty = rc.Reference({}, table, "untouched")
    rng = random.Random(SEED ^ (precision * 1009 + world * 7 + H))
    per = H - 1
    order = list(range(n_plain))
    rng.shuffle(order)
    intervals = [order[i:i + per] for i in range(0, len(order), per)]
    wrapped = [ci for ci in range(n_plain, len(cases)) if cases[ci]["total"] // world + len(cases[ci]["hist"]) < 2 ** 64]
    assert not wbatches or len(wrapped) >= len(cases) - n_plain - 2         # only two_wraps (both forms) needs three ranks
    rng.shuffle(wrapped)
    n_wrapped_intervals = -(-len(wrapped) // per)
    intervals += [wrapped[i:i + per] for i in range(0, len(wrapped), per)] + [[]]
    with contexts(lh, ndev, world, H, NC, precision) as (engs, ref):
        for i, chosen in enumerate(intervals):
            ids = rng.sample(range(H), len(chosen))
            refs = [empty] * H
            flags = [0] * H
            hists = {}
            parts = [[] for _ in range(world)]
            for h, ci in zip(ids, chosen):
                refs[h] = case_refs[ci]
                hists[h] = cases[ci]["hist"]
                flags[h] = rc.expected_flag(cases[ci]["hist"], precision)
                wraps = cases[ci]["total"] >= 2 ** 64
                layout = "spread" if wraps else ("one", "mixed", "all")[(ci + i) % 3]
                split = split_hist(cases[ci]["hist"], layout, world, precision, rng)
                if wraps:
                    assert all(sum(c for _, c in share) < 2 ** 64 for share in split), (cases[ci]["name"], world)
                for r, share in enumerate(split):
                    parts[r] += [(h, k, c) for k, c in share]
            shares = [triples(p) for p in parts]
            counters = counter_shares(world, SEED + i)
            with_counters = i % 2 == 0
            skewed = i % world
            first_wrapped = len(intervals) - 1 - n_wrapped_intervals
            if first_wrapped <= i < len(intervals) - 1:
                ps = wbatches[(i - first_wrapped) % len(wbatches)]
            else:
                ps = batches[i % len(batches)]
            what = (precision, form, world, i)

            for r, e in enumerate(engs):
                e.counter_add_u16_host(*counters[r])
                if r != skewed:
                    e.merge_counts_host(*shares[r])

            def hold():
                spin(engs[skewed], (5 + 5 * (i % 6)) * MS)
                engs[skewed].merge_counts_host(*shares[skewed])
            seqs = collective(engs, with_counters, hold, skewed)

            ref.merge_counts_host(*(np.concatenate(a) for a in zip(*shares)))
            for r in range(world):
                ref.counter_add_u16_host(*counters[r])
            want = Expect(refs, ps)
            rows = [h for h in ids if flags[h]][:6] + [h for h in range(H) if not flags[h]][:1]
            ref.snapshot_begin()
            try:
                ref_red, ref_sp = ref.snapshot_reduce(ps), ref.snapshot_export()
            finally:
                ref.snapshot_end()
            want.check(ref_red, ref_sp, what + ("reference context",))
            total_counters = counter_sum(oracle, counters)
            assert (ref_sp.counter_deltas == total_counters).all(), what

            for r, e in enumerate(engs):
                try:
                    red = e.snapshot_reduce(ps)
                    sp = e.snapshot_export()
                    got_rows = {h: e.snapshot_copy_histogram(h) for h in rows}
                finally:
                    e.snapshot_end()
                info = e.comm_info()
                tag = what + (r,)
                assert info["status"] == 0 and info["allreduces"] == i + 1, (tag, info)
                assert info["last_bytes_from_peers"] == expected_bytes(flags, precision, world, form), (tag, info)
                assert e.comm_allreduce_ms(seqs[r]) > 0, tag
                want.check(red, sp, tag)
                assert same_results(red, ref_red), tag
                assert same_export(sp, ref_sp), tag
                for h in rows:
                    assert (got_rows[h] == rc.dense(hists.get(h, {}))).all(), (tag, h)
                own = counter_sum(oracle, [counters[r]])
                assert (sp.counter_deltas == (total_counters if with_counters else own)).all(), (tag, with_counters)


# ------------------------------------------------------------------------------------------------ intervals and call order
@pytest.mark.parametrize("form", FORMS)
def test_intervals_and_call_order(lh, oracle, ndev, spin, form):
    """World 3 at precision 100.  Dense intervals followed by window-only ones on the same ids, in both halves of the
    double buffer: the reduced arrays must not keep a cell of an earlier interval (the whole dense row of every id is
    compared).  In every snapshot a reduction is enqueued before the all-reduce (its ticket gives this rank's own
    counts), then the all-reduce, a reduction, the export and copy_histogram (global); a second all-reduce in the same
    snapshot is refused with LH_ERR_STATE."""
    world, precision = 3, 100
    H = form_H(precision, form)
    w = rc.window(precision)
    K = w - 1
    table = oracle.decompress_table(precision)
    rng = random.Random(SEED ^ H)
    used = [0, 4, H - 2, H - 1]

    def window_hist():
        return {k: rng.randrange(1, 2 ** 40) for k in rng.sample(range(-K, K + 1), 40) + [-K, K, -1, 0]}

    def dense_hist():
        d = window_hist()
        d.update({-32768: rng.randrange(1, 2 ** 50), 32767: 3, w: 5, -w: 2 ** 33, -w - 1: 1, w + 7: 9})
        return d

    intervals = ["dense", "window", "window", "dense", "window", "window", "empty"]
    with contexts(lh, ndev, world, H, 1, precision) as (engs, _):
        for i, kind in enumerate(intervals):
            hists = {} if kind == "empty" else {h: (dense_hist() if kind == "dense" and h != H - 2 else window_hist()) for h in used}
            parts = [[] for _ in range(world)]
            for j, (h, hist) in enumerate(hists.items()):
                for r, share in enumerate(split_hist(hist, ("mixed", "all", "one", "all")[(j + i) % 4], world, precision, rng)):
                    parts[r] += [(h, k, c) for k, c in share]
            shares = [triples(p) for p in parts]
            own_refs = [[rc.Reference({k: c for hh, k, c in parts[r] if hh == h}, table) for h in range(H)] for r in range(world)]
            refs = [rc.Reference(hists.get(h, {}), table, "interval %d" % i) for h in range(H)]
            skewed = (i + 1) % world
            for r, e in enumerate(engs):
                if r != skewed:
                    e.merge_counts_host(*shares[r])
            tickets = {}

            def hold():
                spin(engs[skewed], (30 - 4 * i) * MS)
                engs[skewed].merge_counts_host(*shares[skewed])

            def early(r, e):
                tickets[r] = e.snapshot_reduce_async(PS)
            seqs = collective(engs, False, hold, skewed, before=early)
            want = Expect(refs, PS)
            for r, e in enumerate(engs):
                tag = (form, i, kind, r)
                try:
                    with pytest.raises(lh.LhError) as ex:
                        e.snapshot_allreduce()
                    assert ex.value.status == LH_ERR_STATE, tag
                    local = e.snapshot_result(tickets[r])
                    red = e.snapshot_reduce(PS)
                    sp = e.snapshot_export()
                    rows = {h: e.snapshot_copy_histogram(h) for h in range(H)}
                finally:
                    e.snapshot_end()
                Expect(own_refs[r], PS).check(local, None, tag + ("issued before the all-reduce",))
                want.check(red, sp, tag)
                for h in range(H):
                    assert (rows[h] == rc.dense(hists.get(h, {}))).all(), (tag, h)
                assert e.comm_allreduce_ms(seqs[r]) > 0, tag
                info = e.comm_info()
                assert info["status"] == 0, (tag, info)
                flags = [rc.expected_flag(hists.get(h, {}), precision) for h in range(H)]
                assert info["last_bytes_from_peers"] == expected_bytes(flags, precision, world, form), (tag, info)


# ------------------------------------------------------------------------------------------------ ingest legs
def leg_values(oracle, n, seed):
    """Stream S with every 5th sample from stream L: window keys and some beyond the window at every precision."""
    v = oracle.gen_stream(oracle.STREAM_S, n, seed)
    v[3::5] = oracle.gen_stream(oracle.STREAM_L, n, seed + 2)[3::5]
    return v


FAR = np.array([1e300, -1e300, np.inf, -np.inf, 2.0 ** 70, -(2.0 ** -70), 5e-324, 0.0], np.float64)


@pytest.mark.parametrize("precision", [50, 100, 200])
def test_every_writer_raises_the_flags_k5_reads(lh, oracle, ndev, spin, precision):
    """World 3: rank 0 writes through K1 (ingest_f64), rank 1 through the keyed L2-atomic kernel (keyed_mode 1), float64
    and int64 nanoseconds, rank 2 through ingest_batch.  Histogram r also gets values far outside the window from rank
    r alone, and histogram H - 1 stays untouched; every rank must hold the oracle's histograms of the concatenated
    stream.  One rank is held back before its last ingest call."""
    world, H, n = 3, 6, 200_003
    skewed = {50: 0, 100: 1, 200: 2}[precision]
    vals = [leg_values(oracle, n, SEED + 31 * r + precision) for r in range(world)]
    ids = oracle.gen_ids(0, n, H - 1, SEED + precision).astype(np.uint16)
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, SEED + precision).view(np.int64).copy()
    want = np.zeros((H, 65536), np.uint64)

    def add(hids, values):
        keys = oracle.compress_many(np.asarray(values, np.float64), precision).view(np.uint16)
        np.add.at(want, (np.asarray(hids, np.int64), keys.astype(np.int64)), np.uint64(1))

    with contexts(lh, ndev, world, H, 1, precision) as (engs, _):
        e0, e1, e2 = engs
        e1.tune("keyed_mode", 1)
        bufs = []

        def up(e, a):
            bufs.append(e.upload(a))
            return bufs[-1]
        # rank 0: K1 into every live histogram, the far values into histogram 0
        calls = {0: [], 1: [], 2: []}
        for h in range(H - 1):
            a = (h * n) // (H - 1)
            d = up(e0, vals[0][a:a + n // 7])
            calls[0].append(lambda d=d, h=h, m=n // 7: e0.ingest_f64(h, d, m))
            add(np.full(n // 7, h), vals[0][a:a + n // 7])
        d = up(e0, FAR)
        calls[0].append(lambda d=d: e0.ingest_f64(0, d, FAR.size))
        add(np.zeros(FAR.size), FAR)
        # rank 1: keyed, float64 and int64 nanoseconds; the far values in histogram 1
        v1 = vals[1].copy()
        v1[ids == 1] = FAR[np.arange(int((ids == 1).sum())) % FAR.size]
        d_i, d_v, d_n = up(e1, ids), up(e1, v1), up(e1, ns)
        calls[1].append(lambda: e1.ingest_keyed_f64_u16(d_i, d_v, n))
        calls[1].append(lambda: e1.ingest_keyed_i64ns_u16(d_i, d_n, n))
        add(ids, v1)
        add(ids, ns.astype(np.float64))
        # rank 2: one batch, float64 and int64 items; the far values in histogram 2
        items = []
        for h in range(H - 1):
            part = vals[2][h * 1000:h * 1000 + 20_000 + h]
            items.append((h, up(e2, part)))
            add(np.full(part.size, h), part)
        items.append((2, up(e2, FAR)))
        add(np.full(FAR.size, 2), FAR)
        items.append((3, up(e2, ns[:5000])))
        add(np.full(5000, 3), ns[:5000].astype(np.float64))
        calls[2].append(lambda: e2.ingest_batch(items))

        warm_up(engs, lambda r, e: [call() for call in calls[r]])
        for r in range(world):
            if r != skewed:
                for call in calls[r]:
                    call()
        assert e1.keyed_kernel_name() == R.VEC or skewed == 1

        def hold():
            for call in calls[skewed][:-1]:
                call()
            spin(engs[skewed], 20 * MS)
            calls[skewed][-1]()
        seqs = collective(engs, False, hold, skewed)
        assert e1.keyed_kernel_name() == R.VEC
        for r, e in enumerate(engs):
            try:
                red = e.snapshot_reduce(PS)
                sp = e.snapshot_export()
            finally:
                e.snapshot_end()
            assert e.comm_info()["status"] == 0 and e.comm_allreduce_ms(seqs[r]) > 0
            for h in range(H):
                got = np.zeros(65536, np.uint64)
                for k, c in sp.histogram(h).items():
                    got[k & 0xFFFF] = c
                assert (got == want[h]).all(), (precision, r, h)
                o = oracle.process_histogram(want[h], PS, precision)
                assert int(red.counts[h]) == o["total"], (precision, r, h)
                if o["total"]:
                    assert (red.pkeys[h] == o["pkeys"]).all(), (precision, r, h)
                    assert (red.pvals[h].view(np.uint64) == o["pvals"].view(np.uint64)).all(), (precision, r, h)
            assert int(red.counts[H - 1]) == 0
        for b in bufs:
            b.free()


# ------------------------------------------------------------------------------------------------ validation
def test_import_validation(lh):
    """lh_comm_import refuses handles of another shape, a handles[rank] that is not the context's own, rank >= world,
    world > 16 (LH_ERR_INVALID), and any import during a snapshot (LH_ERR_STATE)."""
    def status(call):
        with pytest.raises(lh.LhError) as ex:
            call()
        return ex.value.status

    shapes = [dict(max_histograms=3, max_counters=4, precision=100), dict(max_histograms=4, max_counters=4, precision=100),
              dict(max_histograms=3, max_counters=5, precision=100), dict(max_histograms=3, max_counters=4, precision=99),
              dict(max_histograms=3, max_counters=4, precision=100)]
    engs = [lh.Engine(device=0, **s) for s in shapes]
    try:
        h = [e.comm_export() for e in engs]
        a = engs[0]
        for other in (1, 2, 3):
            assert status(lambda: a.comm_import(0, 2, h[0] + h[other])) == LH_ERR_INVALID, other
        assert status(lambda: a.comm_import(0, 2, h[4] + h[0])) == LH_ERR_INVALID       # handles[0] is rank 4's
        assert status(lambda: a.comm_import(2, 2, h[0] + h[4])) == LH_ERR_INVALID       # rank >= world
        assert status(lambda: a.comm_import(0, 17, h[0] + h[4] * 16)) == LH_ERR_INVALID
        a.comm_import(0, 2, h[0] + h[4])                                                   # a valid import still works
        a.snapshot_begin()
        try:
            assert status(lambda: a.comm_import(0, 2, h[0] + h[4])) == LH_ERR_STATE
        finally:
            a.snapshot_end()
    finally:
        for e in engs:
            e.close()


# ------------------------------------------------------------------------------------------------ failed all-reduce
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("form", FORMS)
def test_parity_slip_keeps_own_counts(lh, oracle, ndev, form, world):
    """Rank 0 takes one extra local snapshot, so at the next all-reduce the ranks froze different halves of their
    double buffers: every rank must report status 2 and keep exactly its own frozen counts, flags and counters (no
    peer writes into its reduced arrays, and last_bytes_from_peers is 0).  Once the other ranks have taken one local
    snapshot each, the next all-reduce must report status 0 and the global sums again."""
    precision = 100
    H = form_H(precision, form)
    w = rc.window(precision)
    table = oracle.decompress_table(precision)
    rng = random.Random(SEED ^ (world * 31 + H))

    def interval_parts():
        hists = {}
        for h in rng.sample(range(H), H - 2):
            hist = {k: rng.randrange(1, 2 ** 58) for k in rng.sample(range(-w + 1, w), 30)}
            if h % 3 == 0:
                hist[rng.choice((w, -w, -32768, 32767))] = rng.randrange(1, 2 ** 40)
            hists[h] = hist
        parts = [[] for _ in range(world)]
        for j, (h, hist) in enumerate(sorted(hists.items())):
            for r, share in enumerate(split_hist(hist, ("one", "mixed", "all")[j % 3], world, precision, rng)):
                parts[r] += [(h, k, c) for k, c in share]
        return hists, parts

    def run(engs, seed):
        hists, parts = interval_parts()
        counters = counter_shares(world, seed)
        for r, e in enumerate(engs):
            e.merge_counts_host(*triples(parts[r]))
            e.counter_add_u16_host(*counters[r])
        collective(engs, True)
        out = []
        for e in engs:
            try:
                out.append((e.snapshot_reduce(PS), e.snapshot_export(), [e.snapshot_copy_histogram(h) for h in range(H)]))
            finally:
                e.snapshot_end()
            out[-1] += (e.comm_info(),)
        return hists, parts, counters, out

    with contexts(lh, ndev, world, H, NC, precision) as (engs, _):
        # lock-step: the global histogram
        hists, _, counters, out = run(engs, 1)
        want = Expect([rc.Reference(hists.get(h, {}), table) for h in range(H)], PS)
        for r, (red, sp, rows, info) in enumerate(out):
            assert info["status"] == 0, (r, info)
            want.check(red, sp, ("before", r))
        # rank 0 slips one snapshot: every rank keeps its own counts
        engs[0].merge_counts_host(*triples([(0, 5, 1000)]))
        engs[0].snapshot_begin()
        engs[0].snapshot_end()
        hists, parts, counters, out = run(engs, 2)
        for r, (red, sp, rows, info) in enumerate(out):
            own = {}
            for h, k, c in parts[r]:
                own.setdefault(h, {})[k] = c
            tag = ("parity slip", form, world, r)
            assert info["status"] == 2, (tag, info)
            Expect([rc.Reference(own.get(h, {}), table) for h in range(H)], PS).check(red, sp, tag)
            for h in range(H):
                assert (rows[h] == rc.dense(own.get(h, {}))).all(), (tag, h)
            assert (sp.counter_deltas == counter_sum(oracle, [counters[r]])).all(), tag
            assert info["last_bytes_from_peers"] == 0, (tag, info)
        # the other ranks slip one snapshot each: lock-step again, and the status of this all-reduce is 0
        for e in engs[1:]:
            e.snapshot_begin()
            e.snapshot_end()
        hists, _, counters, out = run(engs, 3)
        want = Expect([rc.Reference(hists.get(h, {}), table) for h in range(H)], PS)
        flags = [rc.expected_flag(hists.get(h, {}), precision) for h in range(H)]
        for r, (red, sp, rows, info) in enumerate(out):
            tag = ("parity restored", form, world, r)
            assert info["status"] == 0, (tag, info)
            assert info["last_bytes_from_peers"] == expected_bytes(flags, precision, world, form), (tag, info)
            want.check(red, sp, tag)
            for h in range(H):
                assert (rows[h] == rc.dense(hists.get(h, {}))).all(), (tag, h)
            assert (sp.counter_deltas == counter_sum(oracle, counters)).all(), tag
