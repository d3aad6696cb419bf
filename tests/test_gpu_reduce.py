"""K3 (`k_reduce`: window path and dense path), K4 (`k_scan_nnz` + `k_export`), `k_clear_touched` and
`k_merge_sparse` against the exact reference of tests/_reduce_cases.py on constructed histograms: totals from 1 to
just below 2^64, percentiles on and one ulp beside every sampled crossing, keys on both sides of the window edge,
precisions 46 (+-Inf buckets), 100, 146 (largest window-path precision), 147 (always dense) and 250.

Bar: percentile keys exact, values bit-exact against the decompress table, counts exact, sums within the rounding
bound of the summation (rc.sum_ok), averages bit-exact as sum / float64(count) (metrics.go:356), exports exact."""
import math
import random

import numpy as np
import pytest

import _reduce_cases as rc

pytestmark = pytest.mark.gpu

SEED = 0x10C415C0
H = 64


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def frozen_flags(eng) -> np.ndarray:
    """Per-histogram flags of the open snapshot's frozen buffer."""
    v = eng.snapshot_device()
    out = np.zeros(eng.H, dtype=np.uint32)
    eng._check(eng.lib.lh_memcpy_d2h(eng.h, out.ctypes.data, v.d_flags, out.nbytes))
    return out


def check_reduced(red, refs, ps, table, what):
    for h, ref in enumerate(refs):
        tag = (what, h, ref.name)
        assert int(red.counts[h]) == ref.count, tag
        want = ref.results(ps)
        keys = np.array([rc.INT32_MIN if k is None else k for k in want["keys"]], dtype=np.int32)
        bad = np.flatnonzero(red.pkeys[h] != keys)
        assert bad.size == 0, (tag, [(ps[j], int(red.pkeys[h][j]), int(keys[j])) for j in bad[:5]])
        assert rc.same_bits(red.pvals[h], want["values"]).all(), tag
        s = float(red.sums[h])
        assert rc.sum_ok(s, ref), (tag, s, float(ref.sum), float(ref.abs_sum))
        assert rc.same_bits(red.avgs[h], rc.avg_of(s, ref)), (tag, red.avgs[h], s)


def check_export(sp, refs, what):
    nnz = np.array([ref.nnz for ref in refs], dtype=np.int64)
    assert (sp.offsets.astype(np.int64) == np.concatenate([[0], np.cumsum(nnz)])).all(), what
    for h, ref in enumerate(refs):
        a, b = int(sp.offsets[h]), int(sp.offsets[h + 1])
        assert (sp.keys[a:b] == ref.keys).all() and (sp.counts[a:b] == ref.counts).all(), (what, h, ref.name)


def case_sets(precision, table):
    """(kind, cases, percentile pool): the constructed cases of make_cases, then those whose counts wrap at 2^64."""
    cases = rc.make_cases(precision, table, SEED)
    wrapped = rc.make_wrapped_cases(precision, table, SEED)
    return [("plain", cases, rc.percentile_pool(cases, table, SEED)),
            ("wrapped", wrapped, rc.wrapped_percentile_pool(wrapped, table, SEED))]


@pytest.mark.parametrize("precision", rc.PRECISIONS)
def test_reduce_and_export_constructed_cases(lh, oracle, precision):
    """Every case in its own histogram id, merged again before each reduction (a snapshot clears): every p batch
    against every case, one reduction through lh_snapshot_reduce_async, one with the export first, one with no
    percentiles.  Merging the same counts into the two halves of the double buffer in turn also checks that each
    snapshot cleared what it froze.  The cases of make_cases, then the wrapped ones, in an engine each."""
    table = oracle.decompress_table(precision)
    for kind, cases, pool in case_sets(precision, table):
        reduce_and_export(lh, table, precision, cases, pool, kind)


def reduce_and_export(lh, table, precision, cases, pool, kind):
    refs = [rc.Reference(c["hist"], table, c["name"]) for c in cases]
    refs += [rc.Reference({}, table, "untouched")] * (H - len(cases))
    batches = rc.percentile_batches(pool)
    ids, keys, counts = rc.merge_triples(cases)
    flags = np.array([rc.expected_flag(c["hist"], precision) for c in cases] + [0] * (H - len(cases)), np.uint32)
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng:
        assert (eng.decompress_table().view(np.uint64) == table.view(np.uint64)).all()
        for r, ps in enumerate(batches):
            eng.merge_counts_host(ids, keys, counts)
            eng.snapshot_begin()
            try:
                if r == 0:
                    assert (frozen_flags(eng) == flags).all(), (frozen_flags(eng), flags)
                if r == 1:
                    red = eng.snapshot_result(eng.snapshot_reduce_async(ps))
                    sp = eng.snapshot_export()
                elif r == 2:
                    sp = eng.snapshot_export()
                    red = eng.snapshot_reduce(ps)
                else:
                    red = eng.snapshot_reduce(ps)
                    sp = eng.snapshot_export()
            finally:
                eng.snapshot_end()
            check_reduced(red, refs, ps, table, (precision, kind, r))
            check_export(sp, refs, (precision, kind, r))
        for _ in range(2):                    # both halves of the double buffer are empty again
            red, sp = eng.snapshot(rc.SPECIAL_PS)
            empty = [rc.Reference({}, table, "empty")] * H
            check_reduced(red, empty, rc.SPECIAL_PS, table, (precision, "empty"))
            check_export(sp, empty, (precision, "empty"))


@pytest.mark.parametrize("precision", [100, 147])
def test_intervals_after_out_of_window_counts(lh, oracle, precision):
    """A histogram with out-of-window counts (flag 3) followed by intervals that write only window keys to the same
    id: each interval must reduce and export exactly its own counts, in both halves of the double buffer.  The keys
    just outside the window share K3 / K4 warps with the window, so a stale cell there would show."""
    w = rc.window(precision)
    K = w - 1
    table = oracle.decompress_table(precision)
    rng = random.Random(SEED + precision)
    ps = [0.0, 0.25, 0.5, 0.9, 1.0]

    def window_hist():
        return {k: rng.randrange(1, 2 ** 34) for k in rng.sample(range(-K, K + 1), 50) + [-K, K]}

    outside = {-32768: 2 ** 40 + 3, -w: 5, w: 2 ** 33 + 1, 32767: 7, 0: 11, K: 13}
    intervals = [
        {1: outside, 2: window_hist()},
        {1: window_hist(), 2: window_hist()},
        {1: window_hist(), 3: {5: 0}},
        {1: window_hist()},
        {1: window_hist(), 2: {-w - 1: 3, w + 1: 4}},
        {1: window_hist()},
        {},
    ]
    with lh.Engine(device=0, max_histograms=4, max_counters=1, precision=precision) as eng:
        for i, hists in enumerate(intervals):
            trip = [(h, k, c) for h, hist in hists.items() for k, c in hist.items()]
            if trip:
                hs, ks, cs = zip(*trip)
                eng.merge_counts_host(np.array(hs, np.uint32), np.array(ks, np.int16), np.array(cs, np.uint64))
            red, sp = eng.snapshot(ps)
            refs = [rc.Reference(hists.get(h, {}), table, "interval %d" % i) for h in range(4)]
            check_reduced(red, refs, ps, table, (precision, i))
            check_export(sp, refs, (precision, i))


@pytest.mark.parametrize("precision", [100, 250])
def test_board_rows_of_wrapped_histograms(lh, oracle, torch, precision):
    """lh_snapshot_publish of wrapped histograms: each row is present, including those whose count wrapped to 0, and
    holds the reduction's count, sum, average and percentiles; an untouched id and an unbound row are absent."""
    table = oracle.decompress_table(precision)
    cases = rc.make_wrapped_cases(precision, table, SEED)
    ps = [0.0, 0.5, 1.0, 1.5, math.inf, math.nan]
    refs = [rc.Reference(c["hist"], table, c["name"]) for c in cases]
    k = len(cases) + 2
    hid = np.array(list(range(len(cases))) + [len(cases), 0xFFFFFFFF], np.uint32)    # an untouched id, an unbound row
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng, eng.board(k, 0) as b:
        eng.merge_counts_host(*rc.merge_triples(cases))
        eng.snapshot_begin()
        try:
            red = eng.snapshot_reduce(ps)
            b.publish(hid)
        finally:
            eng.snapshot_end()
        check_reduced(red, refs + [rc.Reference({}, table, "untouched")] * (H - len(cases)), ps, table, precision)
        v = {name: a.cpu().numpy() for name, a in b.read().items()}
    n = len(cases)
    assert (v["present"][:n] == 1).all() and (v["present"][n:] == 0).all()
    assert any(r.count == 0 for r in refs)
    assert (v["count"].view(np.uint64)[:n] == red.counts[:n]).all() and (v["count"][n:] == 0).all()
    assert (v["sum"][:n].view(np.uint64) == red.sums[:n].view(np.uint64)).all()
    assert (v["avg"][:n].view(np.uint64) == red.avgs[:n].view(np.uint64)).all()
    assert (v["pkeys"][:n, :len(ps)] == red.pkeys[:n]).all()
    assert (v["pvals"][:n, :len(ps)].view(np.uint64) == red.pvals[:n].view(np.uint64)).all()
