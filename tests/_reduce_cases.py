"""Constructed histograms and an exact reference for the snapshot reduction (K3 `k_reduce`) and export (K4).

Shared by tests/test_reduce_reference.py, which checks the reference against the oracle on the CPU, and
tests/test_gpu_reduce.py, which checks the engine against it.  Histograms built from sample streams never reach the
places where a percentile threshold can be off by one bucket: totals beyond 2^53 (where float64(sofar) has plateaus),
p values on an exact ratio sofar/total or one ulp beside it, counts >= 2^32, keys just outside the fast window.  The
cases here are built bucket by bucket (merge triples) to land on them.
"""
from __future__ import annotations

import math
import random
from fractions import Fraction

import numpy as np

INT32_MIN = -2 ** 31
MAX_PERCENTILES = 32                 # LH_MAX_PERCENTILES
REDUCE_SMEM_BYTES = 100 * 1024       # k_reduce keeps the 2*win-1 window cells (uint64) in this much shared memory
PRECISIONS = (46, 100, 146, 147, 250)
# 146 is the largest precision whose window fits (window path for histograms with window keys only), 147 the smallest
# that always takes the dense path; at 46 and below the top keys decompress to +-Inf.

SPECIAL_PS = [0.0, -0.0, 5e-324, -math.inf, 0.5, 0.99, 1.0 - 2.0 ** -53, 1.0, math.nextafter(1.0, 2.0), math.inf, math.nan]

# window-form totals every precision must cover (the dense form of each adds one count)
REQUIRED_TOTALS = (1, 2, 3, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 3,
                   2 ** 60 - 12345, 2 ** 60 + 2 ** 41 + 7, 2 ** 64 - 2)

_SCALE = 2 ** 1074                   # every finite float64 is an integer multiple of 2^-1074


def window(precision: int) -> int:
    """Fast-window length at `precision` (make_prec in lh_api.cu): window keys are -(win-1) .. win-1."""
    return math.floor(precision * 63.0 * 0.6931471805599453 + 0.5) + 1


def window_path(precision: int) -> bool:
    """Does k_reduce reduce a histogram whose keys all lie in the window from shared memory at this precision?"""
    return (2 * window(precision) - 1) * 8 <= REDUCE_SMEM_BYTES


def expected_flag(hist: dict, precision: int) -> int:
    """The histogram's flag after merging `hist` (zero counts included): 0 untouched, 1 window keys only, 3 otherwise."""
    if not hist:
        return 0
    w = window(precision)
    return 1 if all(-w < k < w for k in hist) else 3


class Reference:
    """processHistograms + percentile (metrics.go:336-356, 406-418) on one {int16 key: count} histogram, restated
    independently of the oracle's key-ordered loop: buckets sorted by decompressed value as metrics.go:409 sorts
    (ties, which occur only at +-Inf for precisions <= 46, broken by key), running count and total as Python ints,
    the rule float64(sofar) / float64(total) >= p in Python floats (correctly rounded int -> float, IEEE division),
    and the sum of decompress(key) * count as an exact rational."""

    def __init__(self, hist: dict, table: np.ndarray, name: str = ""):
        self.name = name
        items = sorted(((float(table[k & 0xFFFF]), k, c) for k, c in hist.items() if c), key=lambda t: (t[0], t[1]))
        self.order = [k for _, k, _ in items]
        self.table = table
        self.count = sum(c for _, _, c in items)
        self.nnz = len(items)
        self.cums = []
        ratios = []
        sofar = 0
        for _, _, c in items:
            sofar += c
            self.cums.append(sofar)
            ratios.append(float(sofar) / float(self.count))
        self.ratios = np.array(ratios, dtype=np.float64)
        exact, mag, infs = 0, 0, set()
        for v, _, c in items:
            if math.isinf(v):
                infs.add(v)
                continue
            num, den = v.as_integer_ratio()
            t = num * (_SCALE // den) * c
            exact += t
            mag += abs(t)
        if infs:
            self.sum = math.nan if len(infs) == 2 else infs.pop()      # an Inf term decides the float sum
        else:
            self.sum = Fraction(exact, _SCALE)
        self.abs_sum = Fraction(mag, _SCALE)                           # sum of |terms| over the finite terms
        by_key = sorted((k, c) for k, c in hist.items() if c)
        self.keys = np.array([k for k, _ in by_key], dtype=np.int16)
        self.counts = np.array([c for _, c in by_key], dtype=np.uint64)

    def percentile(self, p: float):
        """Key of the first bucket (in value order) whose running count satisfies the rule; None where percentile()
        returns its error (p > 1, NaN, empty histogram)."""
        hit = np.flatnonzero(self.ratios >= p)
        return self.order[hit[0]] if hit.size else None

    def results(self, ps) -> dict:
        keys = [self.percentile(p) for p in ps]
        return {"keys": keys, "values": [math.nan if k is None else float(self.table[k & 0xFFFF]) for k in keys],
                "count": self.count, "sum": self.sum, "abs_sum": self.abs_sum, "nnz": self.nnz}


def reference(hist: dict, ps, table: np.ndarray) -> dict:
    """Keys (None = percentile() error), values, count, exact sum and sum of |terms| of `hist` for percentiles `ps`."""
    return Reference(hist, table).results(ps)


def sum_ok(got: float, ref: Reference) -> bool:
    """A float64 sum of the histogram's terms decompress(k) * float64(count) against the exact sum.

    Each term suffers at most nnz + 1 roundings (int -> float, product, nnz - 1 additions in any order), so
    |got - exact| <= gamma(nnz + 1) * sum |terms| <= (nnz + 2) * 2^-53 * sum |terms| for nnz < 2^26 (recursive
    summation, Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2).  When a bucket
    decompresses to +-Inf the sum is that Inf, or NaN when both signs are present."""
    if isinstance(ref.sum, float):
        return math.isnan(got) if math.isnan(ref.sum) else got == ref.sum
    if not math.isfinite(got):
        return False
    return abs(Fraction(got) - ref.sum) <= Fraction(ref.nnz + 2, 2 ** 53) * ref.abs_sum


def same_bits(got, want) -> np.ndarray:
    """Elementwise: equal bit patterns, or both NaN (absent percentiles; NaN payloads are not compared)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return np.where(np.isnan(want), np.isnan(got), got.view(np.uint64) == want.view(np.uint64))


def dense(hist: dict) -> np.ndarray:
    """uint64[65536] indexed by (uint16)key."""
    out = np.zeros(65536, dtype=np.uint64)
    for k, c in hist.items():
        out[k & 0xFFFF] += np.uint64(c)
    return out


def sparse(counts: np.ndarray) -> dict:
    """{int16 key: count} of the non-empty buckets of a uint64[65536] histogram indexed by (uint16)key."""
    return {(int(i) ^ 0x8000) - 0x8000: int(counts[i]) for i in np.flatnonzero(counts)}


def threshold(total: int, p: float):
    """Smallest s in [0, total] with float(s) / float(total) >= p (the rule as a threshold on the running count), or
    None when no s satisfies it."""
    ft = float(total)
    if not total or not ft / ft >= p:
        return None
    lo, hi = 0, total
    while lo < hi:
        mid = (lo + hi) // 2
        if float(mid) / ft >= p:
            hi = mid
        else:
            lo = mid + 1
    return lo


def forces_bisection(total: int, p: float) -> bool:
    """Is the threshold more than 8 below or 16 above ceil(p * total)?  percentile_threshold (lh_kernels.cuh) walks
    at most that far from this estimate before it falls back to bisection."""
    s = threshold(total, p)
    if s is None or not p > 0.0:
        return False
    est = math.ceil(p * float(total))
    est = total if est >= float(total) else est
    return s < est - 8 or s > est + 16


# ------------------------------------------------------------------------------------------------ case generator
def _giants_and_ones(total: int, giants: int, run: int, start: int, rng: random.Random) -> dict:
    """Consecutive keys from `start`: a run of count-1 buckets, a giant bucket, a run, ..., a run.  The count-1 buckets
    barely move float64(sofar) / float64(total), so past 2^53 the first bucket satisfying the rule lies many buckets
    away from ceil(p * total)."""
    ones = run * (giants + 1)
    rest = total - ones
    assert rest >= giants
    cuts = sorted(rng.randrange(1, rest) for _ in range(giants - 1))
    sizes = [b - a for a, b in zip([0] + cuts, cuts + [rest])]
    hist, k = {}, start
    for g in range(giants + 1):
        for _ in range(run):
            hist[k] = 1
            k += 1
        if g < giants:
            hist[k] = sizes[g]
            k += 1
    return hist


def make_cases(precision: int, table: np.ndarray, seed: int) -> list:
    """The constructed histograms for one precision, deterministic in (precision, seed).  Each case is a dict with
    name, hist {int16 key: count} (zero counts are merged as such), total, and form: "window" (every key inside the
    fast window), "dense" (the same histogram plus one count at an out-of-window key) or "outside" (a shape that
    needs out-of-window keys).  The caller's reference includes every count."""
    rng = random.Random(seed * 1_000_003 + precision)
    w = window(precision)
    K = w - 1
    ncells = 2 * w - 1
    finite = lambda k: math.isfinite(float(table[k & 0xFFFF]))      # noqa: E731
    extras = [k for k in (w, -w, -32768, 32767) if finite(k)]        # out-of-window keys of the dense forms
    base = []

    # totals: 1, 2, 3 and around 2^32, 2^53, 2^60, 2^64, from a few giant buckets among runs of count-1 buckets
    base.append(("total_1", {rng.randrange(-K, K + 1): 1}))
    base.append(("total_2", {-1: 1, 1: 1}))
    base.append(("total_3", {-K: 1, 0: 1, K: 1}))
    for total, giants, run in ((2 ** 32 - 1, 1, 300), (2 ** 32, 1, 300), (2 ** 32 + 1, 1, 300),
                               (2 ** 53 - 1, 2, 500), (2 ** 53, 2, 500), (2 ** 53 + 1, 2, 500), (2 ** 53 + 3, 2, 500),
                               (2 ** 60 - 12345, 3, 700), (2 ** 60 + 2 ** 41 + 7, 3, 700), (2 ** 64 - 2, 2, 1300)):
        run = min(run, (ncells - giants) // (giants + 1))
        start = rng.randrange(-K, K + 2 - run * (giants + 1) - giants)
        base.append(("total_%#x" % total, _giants_and_ones(total, giants, run, start, rng)))

    # shapes
    big = [1, 2 ** 32 + 7, 2 ** 63 + 5, 12345, 2 ** 64 - 2]
    for i, k in enumerate((0, 1, -1, K, -K)):
        base.append(("single_%d" % k, {k: big[i]}))
    base.append(("every_window_key", {k: rng.randrange(1, 2 ** 40) for k in range(-K, K + 1)}))
    base.append(("alternating", {k: rng.randrange(1, 2 ** 20) for k in range(-K, K + 1, 2)}))
    base.append(("two_far_window", {-K: rng.randrange(1, 2 ** 62), K: rng.randrange(1, 2 ** 62)}))

    cases = []
    for i, (name, hist) in enumerate(base):
        cases.append({"name": name, "hist": hist, "form": "window"})
        extra = extras[i % len(extras)]
        d = dict(hist)
        d[extra] = d.get(extra, 0) + 1
        cases.append({"name": name + "+%d" % extra, "hist": d, "form": "dense"})

    # shapes that need out-of-window keys; at precisions <= 46 the last three hold +-Inf buckets on purpose
    for i, k in enumerate((w, -w, -32768, 32767)):
        cases.append({"name": "single_%d" % k, "hist": {k: big[i + 1]}, "form": "outside"})
    cases.append({"name": "two_far", "hist": {-32768: rng.randrange(1, 2 ** 62), 32767: rng.randrange(1, 2 ** 62)},
                  "form": "outside"})
    cases.append({"name": "inf_mix", "hist": {-32768: 5, -32767: 2, 0: 10, K: 3, 32767: 2}, "form": "outside"})
    # a count-0 triple raises the flag but adds nothing: the histogram must read as untouched
    cases.append({"name": "zero_count_window", "hist": {3: 0}, "form": "window"})
    cases.append({"name": "zero_count_outside", "hist": {-32768: 0}, "form": "outside"})
    for c in cases:
        c["total"] = sum(c["hist"].values())
    return cases


def percentile_pool(cases: list, table: np.ndarray, seed: int) -> list:
    """SPECIAL_PS, then for a sample of crossings s of each case (the first bucket, the middle of the count-1 run after
    the largest bucket, one at random): q = float(s) / float(total) and the doubles on either side of it."""
    rng = random.Random(seed)
    pool = list(SPECIAL_PS)
    for c in cases:
        ref = Reference(c["hist"], table)
        n = ref.nnz
        if not n:
            continue
        counts = [c["hist"][k] for k in ref.order]
        top = max(range(n), key=counts.__getitem__)
        end = top + 1
        while end < n and counts[end] == 1:
            end += 1
        for i in sorted({0, min(n - 1, top + 1 + (end - top - 1) // 2), rng.randrange(n)}):
            q = float(ref.cums[i]) / float(ref.count)
            pool += [math.nextafter(q, -math.inf), q, math.nextafter(q, math.inf)]
    return pool


def percentile_batches(pool: list) -> list:
    """The pool in reductions of at most MAX_PERCENTILES each, then one reduction with no percentiles."""
    return [pool[i:i + MAX_PERCENTILES] for i in range(0, len(pool), MAX_PERCENTILES)] + [[]]


def merge_triples(cases: list):
    """(ids, keys, counts) that build case i in histogram id i."""
    ids, keys, counts = [], [], []
    for i, c in enumerate(cases):
        for k, n in c["hist"].items():
            ids.append(i)
            keys.append(k)
            counts.append(n)
    return (np.array(ids, dtype=np.uint32), np.array(keys, dtype=np.int16), np.array(counts, dtype=np.uint64))
