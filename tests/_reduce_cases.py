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
    (ties, which occur only at +-Inf for precisions <= 46, broken by key), running count and total as Go's uint64 (mod
    2^64), the rule float64(sofar) / float64(total) >= p in Python floats (correctly rounded int -> float, IEEE
    division: x / 0.0 is +Inf and 0 / 0.0 NaN when the total wraps to 0), and the sum of decompress(key) * count as an
    exact rational."""

    def __init__(self, hist: dict, table: np.ndarray, name: str = ""):
        self.name = name
        self.table = table
        self.nnz = sum(1 for c in hist.values() if c)
        self._rank([(k, c) for k, c in hist.items() if c])
        exact, mag, infs = 0, 0, set()
        for k, c in hist.items():
            v = float(table[k & 0xFFFF])
            if not c:
                continue
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

    def _rank(self, entries):
        """Value order, running counts and rule ratios of the (key, count) entries percentile() sorts."""
        items = sorted(((float(self.table[k & 0xFFFF]), k, c) for k, c in entries), key=lambda t: (t[0], t[1]))
        self.order = [k for _, k, _ in items]
        self.count = sum(c for _, _, c in items) % 2 ** 64
        self.cums = []
        ratios = []
        sofar = 0
        for _, _, c in items:
            sofar = (sofar + c) % 2 ** 64
            self.cums.append(sofar)
            ratios.append(go_div(float(sofar), self.count))
        self.ratios = np.array(ratios, dtype=np.float64)

    def percentile(self, p: float):
        """Key of the first bucket (in value order) whose running count satisfies the rule; None where percentile()
        returns its error (no bucket satisfies it: p above every ratio, NaN, an empty histogram)."""
        hit = np.flatnonzero(self.ratios >= p)
        return self.order[hit[0]] if hit.size else None

    def results(self, ps) -> dict:
        keys = [self.percentile(p) for p in ps]
        return {"keys": keys, "values": [math.nan if k is None else float(self.table[k & 0xFFFF]) for k in keys],
                "count": self.count, "sum": self.sum, "abs_sum": self.abs_sum, "nnz": self.nnz}


def reference(hist: dict, ps, table: np.ndarray) -> dict:
    """Keys (None = percentile() error), values, count, exact sum and sum of |terms| of `hist` for percentiles `ps`."""
    return Reference(hist, table).results(ps)


def go_div(x: float, count: int) -> float:
    """Go's x / float64(count) in IEEE arithmetic (metrics.go:356, 413): x / 0.0 is +-Inf, 0 / 0.0 and NaN / y NaN."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(x) / np.float64(float(count)))


def avg_of(s: float, ref: "Reference") -> float:
    """The average processHistograms reports beside a float64 sum `s` of the histogram: s / float64(total)."""
    return go_div(s, ref.count)


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


def _split_wrapping(total: int, parts: int, floor: int, rng: random.Random) -> list:
    """`parts` counts in [floor, 2^64 - 1] summing to `total` exactly."""
    assert parts * floor <= total <= parts * (2 ** 64 - 1)
    while True:
        cuts = sorted(rng.randrange(total + 1) for _ in range(parts - 1))
        sizes = [b - a for a, b in zip([0] + cuts, cuts + [total])]
        if all(floor <= x < 2 ** 64 for x in sizes):
            return sizes


def _wrapping_run(wrapped: int, giants: int, run: int, start: int, rng: random.Random) -> dict:
    """_giants_and_ones whose exact sum is 2^64 + `wrapped`: the running count wraps at one of the giant buckets, and
    past 2^53 the count-1 runs barely move float64(sofar) / float64(total)."""
    hist, k = {}, start
    sizes = _split_wrapping(2 ** 64 + wrapped - run * (giants + 1), giants, 2, rng)
    for g in range(giants + 1):
        for _ in range(run):
            hist[k] = 1
            k += 1
        if g < giants:
            hist[k] = sizes[g]
            k += 1
    return hist


WRAPPED_TOTALS = (0, 1, 2, 12345, 2 ** 53 - 1, 2 ** 53 + 1, 2 ** 60 + 2 ** 41 + 7)   # totals mod 2^64 every precision covers


def make_wrapped_cases(precision: int, table: np.ndarray, seed: int) -> list:
    """Histograms whose counts sum to 2^64 or more, so that Go's uint64 total and running counts (metrics.go:406-418)
    wrap: the running count is no longer monotone in the bucket order and the total may be 0.  Cases as make_cases
    gives them (name, hist, form, total = the exact sum) plus `wraps`, the number of times the running count passes
    2^64.  Every window case has a dense form that holds the same running counts at the window keys: one count moves
    from the last window bucket to the out-of-window key w, so that the total stays (the zero-sum case moves its two
    buckets to -w and w instead).

    The window shapes put a wrap where a search that assumes monotone running counts goes wrong: a "valley", where
    the running count at key 0 (the window's middle cell, where a bisection over the window starts) is below the
    threshold of some p in [0, 1] while an earlier bucket already satisfies the rule, and wraps at the end of warp
    15 (keys -2048 .. -1 of the dense path's 2 048-key warps), inside it and inside one 32-key row, so that warp 15's
    end-of-warp running count fails some p that a bucket inside it satisfies.  The runs of count-1 buckets lie in warp
    15 too, so that the running count at its end is the total while earlier ones exceed it."""
    rng = random.Random(seed * 1_000_003 + precision + 7)
    w = window(precision)
    K = w - 1
    H = 2 ** 63
    a, b = (K * 9) // 10, K // 2                      # every key below is inside the window for K >= 2009
    base = [
        # total 0: ratios x / 0.0 = +Inf (every p but NaN), 0 / 0.0 = NaN; the average is +-Inf, or NaN for a zero sum
        ("wrap0_sum", {-7: H, 9: H}),
        ("wrap0_zero_sum", {-b: H, b: H}),
        ("valley", {-1800: H, -10: H, a: 5}),
        ("wrap_at_last", {-1900: H, -1000: 2 ** 62, -2: H}),
        ("two_wraps", {-1900: H + 1, -1000: H + 1, -5: H, -3: H, a: 5}),
        ("wrap_at_warp_end", {-100: H, -1: H, 5: 3}),
        ("wrap_in_warp", {-1500: H + 10, -700: H, -3: 1, 600: 4}),
        ("wrap_in_row", {-37: H, -35: H, -33: 2, 900: 3}),
    ]
    for wrapped, giants, run in ((0, 2, 300), (1, 2, 300), (2, 2, 300), (12345, 3, 200), (2 ** 53 - 1, 2, 500),
                                 (2 ** 53 + 1, 2, 500), (2 ** 60 + 2 ** 41 + 7, 3, 400)):
        start = rng.randrange(-min(K, 2048), 1 - run * (giants + 1) - giants)      # inside warp 15 and the window
        base.append(("wrap_total_%#x" % wrapped, _wrapping_run(wrapped, giants, run, start, rng)))

    cases = []
    for name, hist in base:
        cases.append({"name": name, "hist": hist, "form": "window"})
        d = dict(hist)
        if name == "wrap0_zero_sum":                       # a zero sum in any summation order
            d = {-w: H, w: H}
        else:
            last = max(d)
            d[last] -= 1
            if not d[last]:
                del d[last]
            d[w] = 1
        cases.append({"name": name + "+%d" % w, "hist": d, "form": "dense"})
    # the dense path's own shapes: a wrap inside a warp outside the window, and at precision 46
    # +-Inf buckets (the ends of the key range) with a wrap between them
    k0 = -32768 + 2048 * ((32768 - w) // 2048 - 1)                    # first key of a warp wholly below -w
    cases.append({"name": "far_warp_wrap", "hist": {k0 + 100: H, k0 + 1000: H, -k0 - 100: 5}, "form": "outside"})
    cases.append({"name": "inf_wrap", "hist": {-32768: 3, -5: H, -3: H, 32767: 2}, "form": "outside"})
    cases.append({"name": "inf_wrap_to_0", "hist": {-32767: H, -32766: H}, "form": "outside"})
    for c in cases:
        c["total"] = sum(c["hist"].values())
        c["wraps"] = c["total"] >> 64
    return cases


def wrapped_percentile_pool(cases: list, table: np.ndarray, seed: int) -> list:
    """percentile_pool's sample, 1.5, and every crossing float64(s) / float64(total) of a bucket whose count is not 1,
    with the doubles on either side; each value once."""
    pool = percentile_pool(cases, table, seed) + [1.5]
    for c in cases:
        ref = Reference(c["hist"], table)
        for k, q in zip(ref.order, ref.ratios):
            if c["hist"][k] != 1:
                pool += [math.nextafter(q, -math.inf), q, math.nextafter(q, math.inf)]
    seen, out = set(), []
    for p in pool:
        b = np.float64(p).view(np.uint64)
        if b not in seen:
            seen.add(b)
            out.append(p)
    return out


def monotone_search(ref: Reference, p: float, w: int):
    """What a search that assumes monotone running counts answers for a window histogram: the integer threshold of
    the rule on the wrapped total (None when float64(total) / float64(total) fails p, or the total is 0), then a
    bisection of the 2w-1 window cells for the first running count at or above it."""
    T = threshold(ref.count, p)
    if T is None:
        return None
    T = max(T, 1)
    run, cells = 0, []
    at = dict(zip(ref.order, ref.cums))
    for k in range(-(w - 1), w):
        run = at.get(k, run)
        cells.append(run)
    lo, hi = 0, len(cells) - 1
    while lo < hi:
        mid = (lo + hi) // 2
        if cells[mid] >= T:
            hi = mid
        else:
            lo = mid + 1
    return lo - (w - 1)


def end_of_warp_owner(ref: Reference, p: float):
    """What the dense path answers when percentile p's owner is the first 2048-key warp with a non-zero total whose
    running count at its end satisfies the rule: the first non-empty bucket of that warp that satisfies it."""
    warps = {}
    for k, s in zip(ref.order, ref.cums):
        warps.setdefault((k + 32768) // 2048, []).append((k, s))
    prev = 0
    for wi in sorted(warps):
        end = warps[wi][-1][1]
        if (end - prev) % 2 ** 64 and go_div(float(end), ref.count) >= p:
            return next((k for k, s in warps[wi] if go_div(float(s), ref.count) >= p), None)
        prev = end
    return None


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
            q = float(ref.ratios[i])
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
