"""The exact reference of tests/_reduce_cases.py against the oracle's key-ordered processHistograms, and the promises
of its case generator.  Runs without a GPU: both restatements must agree before either judges the engine
(tests/test_gpu_reduce.py)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import _reduce_cases as rc

SEED = 0x10C415C0


@pytest.fixture(scope="module", params=rc.PRECISIONS)
def generated(request, oracle):
    p = request.param
    table = oracle.decompress_table(p)
    cases = rc.make_cases(p, table, SEED)
    return p, table, cases, rc.percentile_pool(cases, table, SEED)


@pytest.fixture(scope="module", params=rc.PRECISIONS)
def wrapped(request, oracle):
    p = request.param
    table = oracle.decompress_table(p)
    cases = rc.make_wrapped_cases(p, table, SEED)
    return p, table, cases, rc.wrapped_percentile_pool(cases, table, SEED)


def check_against_oracle(precision, table, cases, ps, oracle):
    for c in cases:
        ref = rc.Reference(c["hist"], table)
        got = oracle.process_histogram(rc.dense(c["hist"]), ps, precision)
        want = ref.results(ps)
        keys = np.array([rc.INT32_MIN if k is None else k for k in want["keys"]], dtype=np.int32)
        bad = np.flatnonzero(got["pkeys"] != keys)
        assert bad.size == 0, (c["name"], [(ps[j], got["pkeys"][j], keys[j]) for j in bad[:5]])
        assert rc.same_bits(got["pvals"], want["values"]).all(), c["name"]
        assert got["total"] == ref.count == c["total"] % 2 ** 64
        # the oracle's sequential sum obeys the bound the engine is held to, and avg = sum / float64(count)
        assert rc.sum_ok(got["sum"], ref), (c["name"], got["sum"], float(ref.sum))
        assert rc.same_bits(got["avg"], rc.avg_of(got["sum"], ref)), c["name"]


def test_reference_matches_oracle(generated, oracle):
    check_against_oracle(*generated, oracle)


def test_case_generator_promises(generated):
    precision, table, cases, ps = generated
    w = rc.window(precision)
    assert len(cases) < 64                                    # one engine of 64 histograms, some left untouched
    names = {c["name"] for c in cases}
    assert len(names) == len(cases)
    for c in cases:
        assert c["total"] == sum(c["hist"].values()) < 2 ** 64, c["name"]
        assert all(-32768 <= k <= 32767 for k in c["hist"]), c["name"]
        inside = all(-w < k < w for k in c["hist"])
        assert inside == (c["form"] == "window"), c["name"]
        assert rc.expected_flag(c["hist"], precision) == (1 if inside else 3)
    window_totals = {c["total"] for c in cases if c["form"] == "window"}
    assert set(rc.REQUIRED_TOTALS) <= window_totals
    dense_totals = {c["total"] for c in cases if c["form"] == "dense"}
    assert {t + 1 for t in rc.REQUIRED_TOTALS} <= dense_totals          # the dense form of each: one more count
    for k in (0, 1, -1, w - 1, -(w - 1), w, -w, -32768, 32767):
        assert "single_%d" % k in names, k
    every = next(c for c in cases if c["name"] == "every_window_key")["hist"]
    assert sorted(every) == list(range(-(w - 1), w)) and all(every.values())
    alt = next(c for c in cases if c["name"] == "alternating")["hist"]
    assert all((k in alt) == ((k + w - 1) % 2 == 0) for k in range(-(w - 1), w))
    assert any(c["total"] == 0 and c["hist"] for c in cases)           # zero-count merges

    # percentile batches: at most LH_MAX_PERCENTILES each, one full and one empty reduction, every special p
    batches = rc.percentile_batches(ps)
    assert all(len(b) <= rc.MAX_PERCENTILES for b in batches)
    assert any(len(b) == rc.MAX_PERCENTILES for b in batches) and batches[-1] == []
    bits = {np.float64(p).view(np.uint64) for p in ps}
    assert all(np.float64(p).view(np.uint64) in bits for p in rc.SPECIAL_PS)

    # every non-empty case has p values exactly on a crossing float64(s) / float64(total) and one ulp on either side
    for c in cases:
        ref = rc.Reference(c["hist"], table)
        hits = 0
        for s in ref.cums:
            q = rc.go_div(float(s), ref.count)
            hits += all(np.float64(x).view(np.uint64) in bits
                        for x in (math.nextafter(q, -math.inf), q, math.nextafter(q, math.inf)))
        assert hits >= min(ref.nnz, 1), c["name"]

    # totals of 2^60 and more with count-1 runs: some p puts the threshold farther from ceil(p * total) than the walk of
    # percentile_threshold reaches, on histograms the window path reduces at precisions <= 146
    forced = [c["name"] for c in cases if c["form"] == "window" and c["total"] >= 2 ** 60
              and any(rc.forces_bisection(c["total"], p) for p in ps)]
    assert len(forced) >= 3, forced

    # magnitudes stay finite except where a bucket decompresses to +-Inf on purpose
    infs = []
    for c in cases:
        ref = rc.Reference(c["hist"], table)
        if isinstance(ref.sum, float):
            infs.append(ref.sum)
        else:
            assert ref.abs_sum < 2 ** 1000, c["name"]
    if precision <= 46:
        assert math.inf in infs and -math.inf in infs and any(math.isnan(x) for x in infs)
    else:
        assert not infs


def test_window_path_switch():
    assert rc.window(100) == 4368                              # lh_device.cuh: 4368 at precision 100
    assert rc.window_path(146) and not rc.window_path(147)
    assert rc.window_path(46) and not rc.window_path(250)


def test_threshold_rule():
    assert rc.threshold(3, 0.5) == 2 and rc.threshold(3, -0.0) == 0 and rc.threshold(3, 1.0) == 3
    assert rc.threshold(3, math.nextafter(1.0, 2.0)) is None and rc.threshold(3, math.nan) is None
    assert rc.threshold(0, 0.0) is None
    t = 2 ** 60
    s = rc.threshold(t, 0.75)
    assert float(s) / float(t) >= 0.75 > float(s - 1) / float(t)
    assert rc.forces_bisection(2 ** 64 - 1, float(2 ** 64 - 5000) / float(2 ** 64 - 1))
    assert not rc.forces_bisection(1000, 0.5)


def test_wrapped_reference_matches_oracle(wrapped, oracle):
    """Go's uint64 total and running counts wrap at 2^64: the reference and the oracle agree on every wrapped case."""
    check_against_oracle(*wrapped, oracle)


def test_wrapped_case_generator_promises(wrapped):
    precision, table, cases, ps = wrapped
    w = rc.window(precision)
    assert len(cases) < 64
    names = {c["name"] for c in cases}
    assert len(names) == len(cases)
    refs = {c["name"]: rc.Reference(c["hist"], table, c["name"]) for c in cases}
    for c in cases:
        assert c["total"] == sum(c["hist"].values()) >= 2 ** 64, c["name"]          # the exact sum wraps
        assert all(0 < n < 2 ** 64 for n in c["hist"].values()) and all(-32768 <= k <= 32767 for k in c["hist"])
        inside = all(-w < k < w for k in c["hist"])
        assert inside == (c["form"] == "window"), c["name"]
        assert refs[c["name"]].count == c["total"] % 2 ** 64
    for form in ("window", "dense"):
        totals = {c["total"] % 2 ** 64 for c in cases if c["form"] == form}
        assert set(rc.WRAPPED_TOTALS) <= totals, form
        assert any(c["wraps"] == 2 for c in cases if c["form"] == form), form
    # total 0 with a non-zero sum (average +-Inf) and with an exact zero sum (average 0 / 0 = NaN), in both forms
    zero = [refs[c["name"]] for c in cases if c["total"] % 2 ** 64 == 0 and c["form"] != "outside"]
    assert sum(r.sum == 0 for r in zero) >= 2 and sum(isinstance(r.sum, Fraction) and r.sum != 0 for r in zero) >= 2
    # a wrap only at the last bucket
    last = refs["wrap_at_last"]
    assert all(a < b for a, b in zip(last.cums, last.cums[1:-1])) and last.cums[-1] < last.cums[-2]

    # every window case has a p at which a bisection that assumes monotone running counts answers another bucket, and
    # the valleys do so at some p in [0, 1]: the running count at key 0 (the middle cell) is below the threshold
    # while an earlier bucket already satisfies the rule
    unit = [p for p in ps if 0.0 <= p <= 1.0]
    for c in cases:
        ref = refs[c["name"]]
        if c["form"] == "window":
            assert any(rc.monotone_search(ref, p, w) != ref.percentile(p) for p in ps), c["name"]
    for name in ("valley", "two_wraps", "wrap_at_warp_end", "wrap_in_warp", "wrap_in_row"):
        ref = refs[name]
        at0 = ref.cums[max(i for i, k in enumerate(ref.order) if k <= 0)]
        valley = [p for p in unit if ref.percentile(p) < 0 and at0 < max(rc.threshold(ref.count, p), 1)]
        assert valley and all(rc.monotone_search(ref, p, w) > 0 for p in valley), name

    # every dense-path case whose total is not 0 has a p at which the first warp (2048 keys) whose end-of-warp running
    # count satisfies the rule holds no bucket that does; with a total of 0 every non-empty running count gives +Inf,
    # and the count alone no longer tells an empty histogram
    for c in cases:
        ref = refs[c["name"]]
        if c["form"] != "window" and ref.count:
            assert any(rc.end_of_warp_owner(ref, p) != ref.percentile(p) for p in ps), c["name"]
    for name in ("wrap_at_warp_end", "wrap_in_warp", "wrap_in_row"):
        ref = refs[name + "+%d" % w]
        assert any(rc.end_of_warp_owner(ref, p) != ref.percentile(p) for p in unit), name
        ks = [k for k in ref.order if -2048 <= k < 0]
        at = dict(zip(ref.order, ref.cums))
        assert any(at[b] < at[a] for a, b in zip(ks, ks[1:])), name                   # the wrap lies in warp 15
    row = [k for k in refs["wrap_in_row"].order if k < 0]
    assert len({(k + 32768) // 32 for k in row}) == 1                                  # ... inside one 32-key row
    end = refs["wrap_at_warp_end"]
    assert dict(zip(end.order, end.cums))[-1] == 0                                     # ... ending at the warp's end
    assert any(c["form"] == "outside" and refs[c["name"]].count == 0 and c["hist"] for c in cases)

    # crossings: every case has p on each crossing float64(s) / float64(total) of a bucket whose count is not 1 and
    # one ulp on either side; some lie above 1, so 1.5 and +Inf answer too; NaN never does
    bits = {np.float64(p).view(np.uint64) for p in ps}
    for c in cases:
        ref = refs[c["name"]]
        for k, q in zip(ref.order, ref.ratios):
            if c["hist"][k] != 1:
                assert all(np.float64(x).view(np.uint64) in bits
                           for x in (math.nextafter(q, -math.inf), q, math.nextafter(q, math.inf))), c["name"]
    assert 1.5 in ps and math.inf in ps and any(math.isnan(p) for p in ps)
    assert any(r.percentile(1.5) is not None for r in refs.values())
    assert any(r.percentile(math.inf) is not None for r in refs.values())
    if precision <= 46:
        inf = refs["inf_wrap"]
        assert math.isinf(float(table[-32768 & 0xFFFF])) and math.isinf(float(table[32767]))
        assert math.isnan(inf.sum)
