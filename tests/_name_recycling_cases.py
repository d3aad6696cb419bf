"""Cases for the recycling of name ids (loghisto_b200/host/metric_system.h, NameTable), shared by
tests/test_name_recycling_cpu.py (the mirror over the oracle-backed stub) and tests/test_gpu_name_recycling.py (the
real library).  Every case takes the test file's `MS` factory: MS(max_histograms=..., max_counters=...).

A name used in interval k holds its id through k+1 and k+2; the id is free for k+3.  So the distinct names used in
any three consecutive intervals must fit the table, and whatever fits is never dropped."""
import ctypes
import os
import subprocess
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGG = ("_agg_avg", "_agg_count", "_agg_sum")


def _compare_interval(raw, m, rraw, rm):
    assert raw["Histograms"] == rraw["Histograms"]
    assert raw["Counters"] == rraw["Counters"] and raw["Rates"] == rraw["Rates"]
    got_keys = {k for k in m if not k.endswith(AGG)}
    ref_keys = {k for k in rm if not k.endswith(AGG)}
    assert got_keys == ref_keys
    for k in got_keys:
        if k.endswith(("_sum", "_avg")):
            assert abs(m[k] - rm[k]) <= 1e-12 * abs(rm[k]), k
        else:
            assert m[k] == rm[k], k


def churn_matches_oracle(MS, oracle):
    """60 intervals through a table of 24: 4 fresh histogram and 4 fresh counter names per interval (240 of each),
    2 permanent names, and names that come back after 1, 2 and 5 idle intervals (their ids are freed and re-taken in
    between).  Every interval's raw set and processed metrics equal the oracle's port of metrics.go, which has no
    limit; the cumulative Counters and the _agg_* aggregates carry on by name across a change of id."""
    rng = np.random.default_rng(11)
    ms = MS(max_histograms=24, max_counters=24)
    agg = MS(max_histograms=24, max_counters=24)        # the reaper's aggregates over the same sets, by name
    ref = oracle.OracleMetricSystem()
    try:
        for k in range(60):
            names = ["fresh%d_%d" % (k, j) for j in range(4)] + ["perm0", "perm1"]
            names += ["gap%d" % g for g in (1, 2, 5) if k % (g + 1) == 0]
            for nm in rng.permutation(names):
                for v in np.exp(rng.uniform(-4, 20, int(rng.integers(1, 6)))):
                    ms.Histogram("h_" + nm, float(v))
                    ref.Histogram("h_" + nm, float(v))
                amt = int(rng.integers(0, 2 ** 40)) if rng.random() < 0.8 else 0
                ms.Counter("c_" + nm, amt)
                ref.Counter("c_" + nm, amt)
            raw, m = ms.collect_and_process()
            rraw, rm = ref.collect_and_process()
            _compare_interval(raw, m, rraw, rm)
            am = agg.processMetrics(raw, aggregates=True)
            agg_keys = {x for x in rm if x.endswith(AGG)}
            assert agg_keys == {x for x in am if x.endswith(AGG)}
            for x in agg_keys:
                if x.endswith("_agg_count"):
                    assert am[x] == rm[x], x
                else:   # sums truncated to uint64 once per interval from sums that agree to 1e-12
                    assert abs(am[x] - rm[x]) <= 1e-12 * abs(rm[x]) + k + 1, x
        assert len(raw["Counters"]) == 240 + 2 + 3
        assert ms.dropped() == 0
    finally:
        ref.close()


def bound_drops(MS, kind):
    """Table of 4, 4 fresh names per interval: a name holds its id for two more intervals, so the names of intervals
    1 and 2 find no free id, those of interval 3 take the ids of interval 0's names, and so on."""
    ms = MS(max_histograms=4, max_counters=4)
    drops, before = [], 0
    for k in range(7):
        names = ["n%d_%d" % (k, j) for j in range(4)]
        for j, nm in enumerate(names):
            if kind == "histogram":
                ms.Histogram(nm, 1.0 + j)
            else:
                ms.Counter(nm, j + 1)
        raw, _ = ms.collect_and_process()
        d = ms.dropped()
        drops.append(d - before)
        before = d
        got = raw["Histograms"] if kind == "histogram" else raw["Rates"]
        assert set(got) == (set(names) if drops[-1] == 0 else set()), k
    assert drops == [0, 4, 4, 0, 4, 4, 0]


# Table of 3.  A is used in interval 0 only, so its id is free from interval 3 on; P holds its id throughout and X,
# last used in interval 1, is still retiring in interval 3.  B, new in interval 3, must take A's old id; in interval 4
# A comes back, its (id, generation) pair is stale, and it takes X's id, freed at collection 3.
SCHEDULE = [["P", "A", "X"], ["P", "X"], ["P"], ["P", "B"], ["P", "A"]]
VALUES = {"P": 1.0, "A": 1000.0, "X": 50.0, "B": 1e6}       # histogram values in distinct buckets
AMOUNTS = {"P": 1, "A": 1000, "X": 50, "B": 10 ** 6}


def stale_thread_cache(MS, oracle, kind):
    """One thread: its name cache still holds A's pair when B has A's old id.  A and B stay separate."""
    ms = MS(max_histograms=3, max_counters=3)
    for k, names in enumerate(SCHEDULE):
        for nm in names:
            if kind == "histogram":
                ms.Histogram(nm, VALUES[nm])
            else:
                ms.Counter(nm, AMOUNTS[nm])
        raw, _ = ms.collect_and_process()
        if kind == "histogram":
            assert raw["Histograms"] == {nm: {oracle.compress(VALUES[nm]): 1} for nm in names}, k
        else:
            assert raw["Rates"] == {nm: AMOUNTS[nm] for nm in names}, k
    assert ms.dropped() == 0


def timer_across_collections(MS, oracle):
    """StartTimer("A") interns A; the token's id is freed and handed to B before Stop().  The duration still lands
    under A, and B holds only its own value."""
    ms = MS(max_histograms=3, max_counters=3)
    timer = None
    for k, names in enumerate(SCHEDULE):
        for nm in names:
            if nm != "A":
                ms.Histogram(nm, VALUES[nm])
            elif timer is None:
                timer = ms.StartTimer("A")
            else:
                timer.Stop()
        raw, _ = ms.collect_and_process()
        want = {nm: {oracle.compress(VALUES[nm]): 1} for nm in names if nm != "A"}
        got = dict(raw["Histograms"])
        if k == len(SCHEDULE) - 1:
            assert sum(got.pop("A", {}).values()) == 1
        assert got == want, k
    assert ms.dropped() == 0


def _primes(n, start=1009):
    out, x = [], start
    while len(out) < n:
        if all(x % p for p in range(2, int(x ** 0.5) + 1)):
            out.append(x)
        x += 1
    return out


def build_race_driver(out_dir):
    so = os.path.join(str(out_dir), "libname_race_driver.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-pthread",
                    os.path.join(ROOT, "tests", "name_race_driver.c"), "-o", so], check=True)
    return so


def race(MS, oracle, driver_so, threads=16, nnames=240, window=16):
    """`threads` threads call Histogram / Counter (tests/name_race_driver.c) over a window of names that moves one
    name per collection, while this thread collects about every millisecond: ids are retired, freed and re-taken
    under load.  Name i records 1000*1.05^i (a bucket of its own) and counter amount p_i (distinct primes), so every
    interval's histogram of name i holds only key k_i and its rate is a multiple of p_i; summed over the intervals
    both equal what the threads recorded for i.  The table holds window + 8 names, more than the window can use in
    three intervals, so nothing is dropped."""
    values = [1000.0 * 1.05 ** i for i in range(nnames)]
    keys = [oracle.compress(v) for v in values]
    assert len(set(keys)) == nnames
    amounts = _primes(nnames)
    hnames = ["rh%d" % i for i in range(nnames)]
    cnames = ["rc%d" % i for i in range(nnames)]
    hidx = {nm: i for i, nm in enumerate(hnames)}
    cidx = {nm: i for i, nm in enumerate(cnames)}
    ms = MS(max_histograms=window + 8, max_counters=window + 8)

    lib = ctypes.CDLL(driver_so)
    vp = ctypes.c_void_p
    lib.race_start.restype = vp
    lib.race_start.argtypes = [vp, vp, vp, vp, vp, vp, vp, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
    lib.race_advance.restype = ctypes.c_int
    lib.race_advance.argtypes = [vp]
    lib.race_finish.argtypes = [vp, vp, vp]
    hn = (ctypes.c_char_p * nnames)(*[x.encode() for x in hnames])
    cn = (ctypes.c_char_p * nnames)(*[x.encode() for x in cnames])
    vals = np.array(values, dtype=np.float64)
    amts = np.array(amounts, dtype=np.uint64)
    hfn = ctypes.cast(ms._lib.lhms_histogram, vp)
    cfn = ctypes.cast(ms._lib.lhms_counter, vp)

    hist_total = np.zeros(nnames, dtype=np.int64)
    rate_total = np.zeros(nnames, dtype=np.int64)

    def absorb(raw):
        for nm, m in raw["Histograms"].items():
            i = hidx[nm]
            assert set(m) == {keys[i]}, (nm, m)
            hist_total[i] += m[keys[i]]
        for nm, r in raw["Rates"].items():
            i = cidx[nm]
            assert r % amounts[i] == 0, (nm, r)
            rate_total[i] += r // amounts[i]

    h = lib.race_start(ms._h, hfn, cfn, ctypes.cast(hn, vp), ctypes.cast(cn, vp), vals.ctypes.data, amts.ctypes.data,
                       nnames, window, threads)
    collections, collecting, t0 = 0, 0.0, time.perf_counter()
    try:
        while True:
            t1 = time.perf_counter()
            raw, _ = ms.collect_and_process()
            collecting += time.perf_counter() - t1
            absorb(raw)
            collections += 1
            if lib.race_advance(h):
                break
            time.sleep(0.001)
    finally:
        hcalls = np.zeros(nnames, dtype=np.uint64)
        ccalls = np.zeros(nnames, dtype=np.uint64)
        lib.race_finish(h, hcalls.ctypes.data, ccalls.ctypes.data)
    raw, _ = ms.collect_and_process()
    absorb(raw)
    print("race: %d Histogram + %d Counter calls, %d collections in %.2f s (%.2f s inside collect_and_process)"
          % (hcalls.sum(), ccalls.sum(), collections, time.perf_counter() - t0, collecting))
    assert collections >= nnames - window
    assert ms.dropped() == 0
    assert hcalls.sum() > 0 and ccalls.sum() > 0
    assert (hist_total == hcalls.astype(np.int64)).all()
    assert (rate_total == ccalls.astype(np.int64)).all()
    for i, nm in enumerate(cnames):
        assert raw["Counters"].get(nm, 0) == int(ccalls[i]) * amounts[i], nm
