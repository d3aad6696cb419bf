"""The FP32 bucket estimate behind every fast path, checked for every input at every precision, and int64 nanosecond
samples at bucket boundaries through every int64 route.

Every ingest path decides a sample's bucket with an FP32 estimate of P ln(1+|v|) and runs the exact FP64 path only when
the estimate lies within eps of a bucket boundary, so bit-exact counts rest on the estimate's error staying below eps
for every input.  The estimate depends on v only through its sign and (exponent, top 23 mantissa bits) of x = 1+|v|,
so lh_fastpath_certify can visit all 2^29 such cells of [1, 2^64) at every precision 1 ... 250, through each shipped
form of the estimate, and compare with FP64 ln at both ends of each cell.  Bar: no unflagged cell has a double whose
bucket differs from Go's, no slot falls outside its sub-histogram, everything outside the window is flagged, nothing
is flagged without a boundary within eps, and the error stays below eps/2 everywhere.

Timer samples are int64 nanoseconds converted as Go's float64(ns), round-to-nearest-even.  The last test feeds integers
that round onto, next to, and (as exact ties) either side of every bucket boundary of the window through every int64
route, each reference key taken from Python's float(int) and the oracle."""
import math
import time

import numpy as np
import pytest

import _ingest_routes as R
from test_gpu_ingest_routes import check, reference

pytestmark = pytest.mark.gpu

PRECISIONS = range(1, 251)
# the four shipped forms of the estimate, in lh_certify_form row order
FORMS = ("fast_candidate", "packed, sign folded (K1 bulk)", "packed, positive-only (K1 bulk default, keyed small)",
         "slot index, positive-only (keyed write-combining)")
POSITIVE_ONLY = (False, False, True, True)
DELTA = 2.0 ** -30                     # bucket units: FP64 ln errs by far less
WINDOW_CELLS = 63 << 23                # cells of x in [1, 2^63)
SEED = 0x10C415C0


def eps(precision):
    """Half-width of the band the fast paths hand to the exact path (Prec::thresh = 0.5 - eps, make_prec)."""
    return 2.0 ** -12 * max(1.0, precision / 100.0)


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_every_cell_at_every_precision(lh):
    """Every cell of every shipped form at every precision 1 ... 250 (one context sweeps them all)."""
    with lh.Engine(device=0) as eng:
        t0 = time.perf_counter()
        rows = eng.fastpath_certify(1, 250)
        wall = time.perf_counter() - t0
    assert rows.shape == (250, 4)
    for i, p in enumerate(PRECISIONS):
        for f, name in enumerate(FORMS):
            r, what = rows[i, f], (p, name)
            # both signs of every window cell were seen (one sign for the positive-only forms)
            assert int(r["samples"]) == WINDOW_CELLS * (1 if POSITIVE_ONLY[f] else 2), what
            assert int(r["input_mismatch"]) == 0, what
            assert int(r["wrong"]) == 0, (what, int(r["wrong"]))
            assert int(r["out_of_range"]) == 0, (what, int(r["out_of_range"]))
            assert int(r["unflagged_outside"]) == 0, (what, int(r["unflagged_outside"]))
            assert int(r["over_flagged"]) == 0, (what, int(r["over_flagged"]))
            assert r["min_margin"] >= DELTA, (what, float(r["min_margin"]))
            assert r["max_err"] < eps(p) / 2, (what, float(r["max_err"]))
            assert 0 < int(r["flagged"]) < int(r["samples"]) // 100, (what, int(r["flagged"]))
    print("\nlh_fastpath_certify, precisions 1..250, 4 forms: %.2f s wall" % wall)
    for f, name in enumerate(FORMS):
        err, margin = rows["max_err"][:, f], rows["min_margin"][:, f]
        ratio = np.array([eps(p) for p in PRECISIONS]) / err
        frac = rows["flagged"][:, f].astype(np.float64) / rows["samples"][:, f]
        print("  %-52s max_err %.3e (P=%d)  min eps/max_err %.1f (P=%d)  min_margin %.3e (P=%d)  flagged %.4f %% (P=%d)"
              % (name, err.max(), err.argmax() + 1, ratio.min(), ratio.argmin() + 1, margin.min(), margin.argmin() + 1,
                 100 * frac.max(), frac.argmax() + 1))


def test_decompress_table_and_window_thresholds_at_every_precision(lh, oracle):
    """At every precision 1 ... 250: the decompress table bit for bit, and every bucket boundary of the window +-3 ulp,
    both signs, through both evaluators of lh_compress_f64."""
    offs = np.arange(-3, 4, dtype=np.int64)
    bisect_cpu = 0.0
    for p in PRECISIONS:
        t0 = time.process_time()
        T = R.thresholds(oracle, p, R.window(p) - 1)
        bisect_cpu += time.process_time() - t0
        bits = (T[:, None].astype(np.int64) + offs[None, :]).reshape(-1).astype(np.uint64)
        vals = np.concatenate([bits, bits | np.uint64(0x8000000000000000)]).view(np.float64)
        want = oracle.compress_many(vals, p)
        with lh.Engine(device=0, precision=p) as eng:
            for mode in (0, 1):
                got = eng.compress(vals, mode)
                bad = np.nonzero(got != want)[0]
                assert bad.size == 0, (p, mode, bad.size, vals[bad[:5]], got[bad[:5]], want[bad[:5]])
            tab = eng.decompress_table()
        assert (tab.view(np.uint64) == oracle.decompress_table(p).view(np.uint64)).all(), p
    print("\noracle bisection of the window thresholds, precisions 1..250: %.1f s CPU" % bisect_cpu)


INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def boundary_nanos(oracle, precision):
    """int64 values around every window threshold T_k >= 1: floor(T_k) - 1, floor(T_k), ceil(T_k), and for T_k >= 2^53
    (where float64(ns) rounds) the ties T_k - ulp/2 and T_k + ulp/2 (round-to-nearest-even picks a side) and
    T_k - ulp/2 +- 1; both signs, plus INT64_MIN and +-INT64_MAX."""
    T = R.thresholds(oracle, precision, R.window(precision) - 1).view(np.float64)
    out = set()
    for t in T[T >= 1.0]:
        f = math.floor(t)
        out.update((f - 1, f, math.ceil(t)))
        if t >= 2.0 ** 53:
            ti = int(t)
            below = ti - int(np.nextafter(t, 0.0))        # the gap to the double below T_k ...
            above = int(np.nextafter(t, np.inf)) - ti     # ... and above (they differ at a power of two)
            tie = ti - below // 2
            out.update((tie - 1, tie, tie + 1, ti + above // 2))
    pos = sorted(out)
    return np.array(pos + [-n for n in pos] + [INT64_MIN, INT64_MAX, -INT64_MAX], dtype=np.int64)


@pytest.mark.parametrize("precision", [100, 1, 147, 250])
def test_int64_nanoseconds_at_bucket_boundaries(lh, oracle, sms, precision):
    """The boundary integers (repeated past 2^17 samples, with a ragged tail) through lh_ingest_keyed_i64ns_u16 on the
    few-histogram, vector and write-combining kernels, the int64 segment of lh_ingest_keyed_pair_u16,
    lh_ingest_keyed_i64ns_u16_host, int64 items of lh_ingest_batch and of a graph recorder: the named kernel ran, and
    every bucket of every histogram equals Go's float64(ns) bucketed by the oracle."""
    import torch
    ns0 = boundary_nanos(oracle, precision)
    n = ns0.size * -(-(1 << 17) // ns0.size) + 5
    ns = np.resize(ns0, n)
    keys = oracle.compress_many(np.array([float(int(x)) for x in ns], dtype=np.float64), precision).view(np.uint16)
    rng = np.random.default_rng(SEED ^ precision)
    label = "P=%d" % precision

    # few histograms: the shared-memory kernel, fed from device memory and from the host
    H = 3
    ids = rng.integers(0, H, n).astype(np.uint32)
    ref = reference(H, ids, keys)
    with lh.Engine(device=0, max_histograms=H, precision=precision) as e:
        d_i, d_n = e.upload(ids.astype(np.uint16)), e.upload(ns)
        before = e.stats()["dropped"]
        e.ingest_keyed_i64ns_u16(d_i, d_n, n)
        assert e.keyed_kernel_name() == R.keyed_route(H, n, precision, sms).kernel == R.SMALL, label
        check(e, H, ref, before, (label, "i64ns_u16 small"))
        e.ingest_keyed_i64ns_u16_host(ids.astype(np.uint16), ns)
        assert e.keyed_kernel_name() == R.keyed_route(H, n, precision, sms).kernel == R.SMALL, label
        check(e, H, ref, before, (label, "i64ns_u16_host"))

    # many histograms: the vector kernel, the write-combining kernel alone and as a fused pair, batches, a graph recorder
    H = 300
    ids = rng.integers(0, H, n).astype(np.uint32)
    ref = reference(H, ids, keys)
    with lh.Engine(device=0, max_histograms=H, precision=precision) as e:
        d_i, d_n = e.upload(ids.astype(np.uint16)), e.upload(ns)
        for mode, kernel in ((1, R.VEC), (2, R.WC)):
            e.tune("keyed_mode", mode)
            before = e.stats()["dropped"]
            e.ingest_keyed_i64ns_u16(d_i, d_n, n)
            assert e.keyed_kernel_name() == R.keyed_route(H, n, precision, sms, keyed_mode=mode).kernel == kernel, label
            check(e, H, ref, before, (label, "i64ns_u16", kernel))
        # the float64 segment carries float64(ns) itself, so both segments add the same counts
        d_f = e.upload(np.array([float(int(x)) for x in ns], dtype=np.float64))
        want = R.pair_route(H, n, n, precision, sms, keyed_mode=2)
        assert want.wc is not None and want.wc.taken2 > 0, label
        before = e.stats()["dropped"]
        e.ingest_keyed_pair_u16(d_i, d_f, n, d_i, d_n, n)
        assert e.keyed_kernel_name() == want.kernel == R.WC, label
        check(e, H, reference(H, np.concatenate([ids, ids]), np.concatenate([keys, keys])), before, (label, "pair"))

        # int64 items: contiguous slices of the samples, each under one histogram id
        t = torch.from_numpy(ns).cuda()
        cuts = np.linspace(0, n, 8).astype(np.int64)
        hids = [0, 1, 150, H - 1, 7, 298, 42]
        item_ids = np.repeat(np.array(hids, np.uint32), np.diff(cuts))
        before = e.stats()["dropped"]
        e.ingest_batch([(h, t[a:b]) for h, a, b in zip(hids, cuts[:-1], cuts[1:])])
        check(e, H, reference(H, item_ids, keys), before, (label, "batch"))
        targets = [H - 1 - h for h in hids]
        with e.graph_recorder(targets, ()) as gr:
            gr.ingest([(i, t[a:b]) for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))])
            torch.cuda.synchronize()
            before = e.stats()["dropped"]
            check(e, H, reference(H, np.repeat(np.array(targets, np.uint32), np.diff(cuts)), keys), before,
                  (label, "graph recorder"))
