"""The device API (include/loghisto_b200_device.cuh) as callers build and launch it, against the oracle.

The header is compiled by other people's nvcc commands and launched with other people's grids.  build_device_client()
builds one client, tests/device_matrix_client.cu, under each flag set of build.DEVICE_MATRIX: the library's own device
flags (ref), --use_fast_math, -G, -maxrregcount=32, -rdc=true over two translation units, and PTX for compute_90 and
compute_70 that the driver JITs at load.  tests/test_device_api_builds_cpu.py checks that each library is what its
name says.  Here every variant runs, and the bar is exact equality throughout:

- the FP32 estimate (lh::fast_candidate) gives the same outputs as ref for every (exponent, 23-bit prefix) cell of
  1 + |v| and both signs, at every precision 1 ... 250, compared through per-CTA hashes; ref's keys equal the library's
  own lh_compress_f64 (which the exhaustive certificate covers), and a Prec one float ulp off changes the hashes;
- lh::key16_of and lh::exact_key16 equal the oracle on edge inputs at precisions 1, 2, 100, 147 and 250;
- lh::record / record_ns / count, lh::BlockHistogram and lh::BlockRecorder leave every bucket of every row, the counter
  deltas and `dropped` equal to the oracle, over 1-D and 3-D blocks, grids with idle CTAs, divergent trip counts and
  lanes that leave early, table sizes 0 ... 16384, shared memory at non-zero offsets, repeated flushes and two tables
  in one CTA;
- lh::raw_percentile / raw_rank / raw_bucket_count and lh::read_histogram answer as the library's grid calls on boards
  built from tests/_reduce_cases.py, wrapped cases included;
- in the -rdc=true build, kernels of both translation units record into one scope."""
import ctypes as C
import functools
import os
import time

import numpy as np
import pytest

import _reduce_cases as rc
from _ingest_routes import epsilon_band_values, thresholds
from loghisto_b200 import build

pytestmark = pytest.mark.gpu

VARIANTS = list(build.DEVICE_MATRIX)
SEED = 0xB111D5
INT32_MIN = -(1 << 31)
UNBOUND = 0xFFFFFFFF
PS = [0.5]

EST_GRID, EST_THREADS = 4096, 256            # the estimate launch: 2^29 / 4096 = 131072 cells per CTA
CELLS_PER_CTA = (1 << 29) // EST_GRID
PRECISIONS = list(range(1, 251))
KEY_PRECISIONS = [1, 2, 100, 147, 250]
BLOCK_PRECISIONS = [1, 100, 250]

# (grid, (bx, by, bz)): 1-D and 3-D blocks, and grids with more threads than samples (idle CTAs)
SHAPES = [(264, (1, 1, 1)), (264, (31, 1, 1)), (264, (33, 1, 1)), (132, (96, 1, 1)), (132, (1000, 1, 1)),
          (132, (1024, 1, 1)), (132, (7, 5, 3)), (132, (32, 2, 16)), (264, (1, 1, 64)),
          (30000, (96, 1, 1)), (2048, (1024, 1, 1)), (9000, (32, 2, 16))]
PATTERNS = {0: "every lane", 1: "divergent trip counts", 2: "early return"}
TABLE_SIZES = [0, 31, 32, 33, 4096, 16384]


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@functools.lru_cache(maxsize=None)
def client(variant):
    """The variant's library, with the launchers' signatures."""
    from loghisto_b200 import _lib
    path = build.matrix_lib(variant)
    assert os.path.exists(path), "build() did not produce " + path
    lib = C.CDLL(path)
    rp, vp, sz, u32, i32 = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t, C.c_uint32, C.c_int
    sigs = {
        "lhm_set_device": [i32],
        "lhm_estimate": [rp, i32, u32, u32, vp, vp, vp],
        "lhm_estimate_cells": [rp, i32, u32, u32, vp, vp, vp, vp],
        "lhm_keys": [rp, vp, sz, vp, vp, vp],
        "lhm_record": [rp, i32, i32, vp, vp, sz, u32, u32, u32, u32, vp],
        "lhm_block_histogram": [rp, vp, vp, sz, sz, i32, u32, u32, u32, u32, u32, vp],
        "lhm_block_recorder": [rp, i32, vp, vp, sz, sz, i32, u32, u32, i32, u32, u32, u32, u32, vp],
        "lhm_raw_percentiles": [C.POINTER(_lib.lh_raw_board), vp, vp, sz, vp, vp, vp, vp],
        "lhm_raw_ranks": [C.POINTER(_lib.lh_raw_board), vp, vp, sz, vp, vp, vp, vp],
        "lhm_raw_bucket_counts": [C.POINTER(_lib.lh_raw_board), vp, vp, sz, vp, vp, vp],
        "lhm_read_histograms": [C.POINTER(_lib.lh_board), vp, sz, vp, vp, vp],
        "lhm_record_part2": [rp, vp, vp, sz, u32, u32, vp],
    }
    for name, args in sigs.items():
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = C.c_int
    assert lib.lhm_set_device(0) == 0
    return lib


@functools.lru_cache(maxsize=None)
def recorder_of(precision):
    """A copy of the recorder lh_record_begin hands out at `precision`: its precision block is what the launchers of
    the estimate and of the keys read (the scope is closed again; they record nothing)."""
    import loghisto_b200 as lh
    from loghisto_b200 import _lib
    with lh.Engine(device=0, precision=precision) as eng:
        rec = eng.record_begin()
        copy = _lib.lh_recorder.from_buffer_copy(rec)
        eng.record_end(rec)
    return copy


# ---------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=None)
def edge_values(precision):
    """Every bucket threshold of the finite range +-3 ulp, both signs; the epsilon-band inputs; +-0, +-Inf, NaN payloads
    of both signs, +-2^63 and the double below it, +-1e300."""
    from oracle import oracle
    kmax = int(np.floor(precision * np.log1p(1.7976931348623157e308) + 0.5))
    T = thresholds(oracle, precision, kmax)
    bits = (T[:, None].astype(np.int64) + np.arange(-3, 4, dtype=np.int64)[None, :]).reshape(-1).astype(np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(1 << 63)])
    nan_bits = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, 0x7FF4000000000000,
                         0x7FF8000000000001], dtype=np.uint64)
    nans = np.concatenate([nan_bits, nan_bits | np.uint64(1 << 63)]).view(np.float64)
    special = np.array([0.0, -0.0, np.inf, -np.inf, 2.0 ** 63, -2.0 ** 63, np.nextafter(2.0 ** 63, 0),
                        -np.nextafter(2.0 ** 63, 0), 1e300, -1e300], dtype=np.float64)
    return np.concatenate([bits.view(np.float64), epsilon_band_values(oracle, precision), nans, special])


STREAMS = (0, 1, 2, 8)                            # U, L, S, N (U with a random sign)


@functools.lru_cache(maxsize=None)
def values(precision, n_stream=50_000):
    """Streams U / L / S / N and the edge values, shuffled so that each warp sees a mix."""
    from oracle import oracle
    v = np.concatenate([oracle.gen_stream(k, n_stream, SEED ^ k ^ precision) for k in STREAMS] + [edge_values(precision)])
    return np.ascontiguousarray(np.random.default_rng(SEED ^ precision).permutation(v))


@functools.lru_cache(maxsize=None)
def keys_of(precision):
    from oracle import oracle
    return oracle.compress_many(values(precision), precision).view(np.uint16).astype(np.int64)


@functools.lru_cache(maxsize=None)
def nanos():
    """int64 durations: the timer stream with both signs, and values where float64(ns) rounds."""
    from oracle import oracle
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, 300_000, SEED).view(np.int64).copy()
    ns[::3] *= -1
    big = np.array([2 ** 53 + 1, 2 ** 53 + 3, 2 ** 60 + 12345, 2 ** 62 - 1, 2 ** 63 - 1, -(2 ** 63), -(2 ** 53) - 1,
                    -(2 ** 61) - 777, 0, 1, -1], dtype=np.int64)
    return np.concatenate([ns, np.repeat(big, 7)])


@functools.lru_cache(maxsize=None)
def nano_keys(precision):
    from oracle import oracle
    return oracle.compress_many(nanos().astype(np.float64), precision).view(np.uint16).astype(np.int64)


def ids_for(n, H, seed):
    """ids in [0, H) with every 97th >= H (H, H + 5 and 0xFFFFFFFF): dropped and counted."""
    from oracle import oracle
    ids = oracle.gen_ids(0, n, H, seed).astype(np.uint32)
    bad = np.array([H, H + 5, UNBOUND], dtype=np.uint32)
    ids[::97] = bad[np.arange(ids[::97].size) % 3]
    return ids


def hist_ref(H, ids, keys, fed):
    keep = fed & (ids < H)
    flat = ids[keep].astype(np.int64) * 65536 + keys[keep]
    return np.bincount(flat, minlength=H * 65536).astype(np.uint64).reshape(H, 65536)


def fed_mask(pattern, n, threads):
    """Which samples a k_record pattern feeds (device_matrix_client.cu): all of them for patterns 0 and 1; for pattern 2
    thread g's run [g * base, (g + 1) * base) up to its sample (uint32(g) * 2654435761) % (base + 2)."""
    if pattern != 2:
        return np.ones(n, dtype=bool)
    base = -(-n // threads)
    i = np.arange(n, dtype=np.uint64)
    g, k = i // np.uint64(base), i % np.uint64(base)
    stop = ((g * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) % np.uint64(base + 2)
    return k < stop


def dense(sp, H):
    out = np.zeros((H, 65536), dtype=np.uint64)
    hid = np.repeat(np.arange(H), np.diff(sp.offsets.astype(np.int64)))
    out[hid, sp.keys.view(np.uint16)] = sp.counts
    return out


def snapshot(eng, H):
    """(dense rows, counter deltas, dropped so far) of the interval."""
    _, sp = eng.snapshot(PS)
    eng.sync()
    return dense(sp, H), sp.counter_deltas.copy(), eng.stats()["dropped"]


class Cases:
    """Runs every case and fails once at the end, naming each case whose check failed, so that a defect shows the
    shapes and patterns it breaks and the ones it leaves alone."""

    def __init__(self):
        self.n, self.failed = 0, []

    def run(self, what, check, *args):
        self.n += 1
        try:
            check(*args)
        except AssertionError as e:
            self.failed.append("%s: %s" % (what, str(e).splitlines()[0][:400]))

    def check(self):
        assert not self.failed, "%d of %d cases failed:\n  %s" % (len(self.failed), self.n, "\n  ".join(self.failed))


def assert_rows(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d cells differ, first (row, uint16 key, got, want): %s" % (
        what, len(bad), [(int(h), int(k), int(got[h, k]), int(want[h, k])) for h, k in bad[:4]])


# ---------------------------------------------------------------- the estimate, cell by cell
_ref_hashes = {}


def estimate_hashes(torch, variant, precisions, c1_ulps=0):
    """[len(precisions), EST_GRID] uint64 per-CTA hashes, and the number of representatives that left their cell."""
    lib = client(variant)
    hashes = torch.zeros((len(precisions), EST_GRID), dtype=torch.int64, device="cuda")
    left = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for j, p in enumerate(precisions):
        assert lib.lhm_estimate(C.byref(recorder_of(p)), c1_ulps, EST_GRID, EST_THREADS, hashes[j].data_ptr(),
                                left.data_ptr(), stream) == 0, (variant, p)
    torch.cuda.synchronize()
    return hashes.cpu().numpy().view(np.uint64), int(left.item())


def ref_hashes(torch, precisions):
    missing = [p for p in precisions if p not in _ref_hashes]
    if missing:
        h, left = estimate_hashes(torch, "ref", missing)
        assert left == 0
        _ref_hashes.update(zip(missing, h))
    return np.stack([_ref_hashes[p] for p in precisions])


def cell_outputs(torch, variant, precision, c_lo, n, c1_ulps=0):
    """(idx, slow, w bits) of cells [c_lo, c_lo + n), both signs: entry 2j + s is cell c_lo + j, sign s."""
    idx = torch.empty(2 * n, dtype=torch.int32, device="cuda")
    slow = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    w = torch.empty(2 * n, dtype=torch.float32, device="cuda")
    assert client(variant).lhm_estimate_cells(C.byref(recorder_of(precision)), c1_ulps, c_lo, n, idx.data_ptr(),
                                              slow.data_ptr(), w.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    return idx.cpu().numpy().view(np.uint32), slow.cpu().numpy(), w.cpu().numpy().view(np.uint32)


def drill_down(torch, variant, precision, cta, c1_ulps=0, limit=4):
    """The cells of CTA `cta` whose outputs differ between ref and `variant`, named."""
    c_lo = cta * CELLS_PER_CTA
    a = cell_outputs(torch, "ref", precision, c_lo, CELLS_PER_CTA)
    b = cell_outputs(torch, variant, precision, c_lo, CELLS_PER_CTA, c1_ulps)
    diff = np.nonzero((a[1] != b[1]) | ((a[1] == 0) & ((a[0] != b[0]) | (a[2] != b[2]))))[0]
    named = []
    for e in diff[:limit]:
        c = c_lo + int(e) // 2
        x = float(np.uint64(0x3FF0000000000000 + (c << 29)).view(np.float64))
        named.append("cell %d (x = %r, exponent %d, prefix 0x%06x, %s): ref (idx %d, slow %d, w 0x%08x) vs "
                     "(idx %d, slow %d, w 0x%08x)" % (c, x, c >> 23, c & 0x7FFFFF,
                                                      "-v" if e & 1 else "+v", a[0][e], a[1][e], a[2][e],
                                                      b[0][e], b[1][e], b[2][e]))
    return diff.size, named


def compare_estimates(torch, variant, precisions, c1_ulps=0):
    """None when every CTA hash equals ref's at every precision, else a message naming the first differing cells."""
    want = ref_hashes(torch, precisions)
    got, left = estimate_hashes(torch, variant, precisions, c1_ulps)
    assert left == 0, (variant, left)
    bad = np.argwhere(got != want)
    if not bad.size:
        return None
    j, cta = (int(x) for x in bad[0])
    n, named = drill_down(torch, variant, precisions[j], cta, c1_ulps)
    return ("%s: %d CTA hashes differ from ref over %d precisions; at P = %d, CTA %d has %d differing outputs: %s"
            % (variant, len(bad), len(set(bad[:, 0])), precisions[j], cta, n, "; ".join(named)))


@pytest.mark.parametrize("variant", VARIANTS)
def test_estimate_equals_ref_in_every_cell(torch, variant):
    """fast_candidate's outputs (slow, and idx and the bits of w where not slow) for both signs of every cell of
    1 + |v|, hashed per CTA, equal ref's at every precision 1 ... 250, and no representative's 1 + |v| leaves its
    cell."""
    t0 = time.perf_counter()
    msg = compare_estimates(torch, variant, PRECISIONS)
    print("\n%s: estimate over %d precisions x 2^30 inputs: %.2f s" % (variant, len(PRECISIONS), time.perf_counter() - t0))
    assert msg is None, msg


def test_estimate_comparison_can_fail(torch):
    """The comparison is not vacuous: ref with c1 one float ulp higher changes the hashes, and the drill-down names
    the cells whose outputs moved."""
    for p in (85, 100, 141):
        msg = compare_estimates(torch, "ref", [p], c1_ulps=1)
        assert msg is not None and "cell " in msg, (p, msg)
    print("\n" + msg)


@pytest.mark.parametrize("precision", KEY_PRECISIONS)
def test_ref_keys_equal_the_library_compress(lh, torch, precision):
    """ref's key16_of and exact_key16 give the keys of the library's own lh_compress_f64 (mode 0: key16_of, mode 1:
    exact_key16) on the edge and stream inputs, tying the ref build to the certified one."""
    vals = values(precision)
    fast, exact = client_keys(torch, "ref", precision, vals)
    with lh.Engine(device=0, precision=precision) as eng:
        for mode, got in ((0, fast), (1, exact)):
            want = eng.compress(vals, mode).view(np.uint16)
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, (precision, mode, bad.size, vals[bad[:4]], got[bad[:4]], want[bad[:4]])


def client_keys(torch, variant, precision, vals):
    v = torch.from_numpy(vals).cuda()
    fast = torch.empty(vals.size, dtype=torch.int16, device="cuda")
    exact = torch.empty(vals.size, dtype=torch.int16, device="cuda")
    assert client(variant).lhm_keys(C.byref(recorder_of(precision)), v.data_ptr(), vals.size, fast.data_ptr(),
                                    exact.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    return fast.cpu().numpy().view(np.uint16), exact.cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("variant", VARIANTS)
def test_keys_equal_the_oracle(oracle, torch, variant):
    """key16_of and exact_key16 equal the oracle's compress on the edge and stream inputs at P = 1, 2, 100, 147, 250."""
    for p in KEY_PRECISIONS:
        vals = values(p)
        want = keys_of(p).astype(np.uint16)
        for name, got in zip(("key16_of", "exact_key16"), client_keys(torch, variant, p, vals)):
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, (variant, p, name, bad.size, vals[bad[:4]], got[bad[:4]], want[bad[:4]])


# ---------------------------------------------------------------- recording
@pytest.mark.parametrize("variant", VARIANTS)
def test_record_matches_oracle(lh, oracle, variant):
    """lh::record, record_ns and count under every launch shape and pattern: every bucket of every row, the counter
    deltas and `dropped` equal the oracle."""
    lib = client(variant)
    P, H, Cn = 100, 23, 7
    vals, keys = values(P), keys_of(P)
    ns, nkeys = nanos(), nano_keys(P)
    ids = ids_for(vals.size, H, SEED)
    nids = ids_for(ns.size, H, SEED ^ 1)
    rng = np.random.default_rng(SEED)
    amounts = rng.integers(0, 2 ** 63, ns.size, dtype=np.uint64) * np.uint64(2) + np.uint64(1)   # wraps many times
    cids = rng.integers(0, Cn + 2, ns.size).astype(np.uint32)
    cids[::101] = UNBOUND
    with lh.Engine(device=0, max_histograms=H, max_counters=Cn, precision=P) as eng:
        d = {k: eng.upload(a) for k, a in (("v", vals), ("i", ids), ("ns", ns), ("ni", nids), ("a", amounts), ("ci", cids))}

        def case(grid, block, pattern):
            T = grid * block[0] * block[1] * block[2]
            before = eng.stats()["dropped"]
            with eng.recording() as rec:
                for op, (di, dv, n) in enumerate(((d["i"], d["v"], vals.size), (d["ni"], d["ns"], ns.size),
                                                  (d["ci"], d["a"], ns.size))):
                    assert lib.lhm_record(C.byref(rec), op, pattern, di.ptr, dv.ptr, n, grid, *block,
                                          eng.ingest_stream) == 0, "launch failed"
            got, deltas, now = snapshot(eng, H)
            fv, fn = fed_mask(pattern, vals.size, T), fed_mask(pattern, ns.size, T)
            assert_rows(got, hist_ref(H, ids, keys, fv) + hist_ref(H, nids, nkeys, fn), "buckets")
            keep = fn & (cids < Cn)
            assert (deltas == oracle.counter_add(cids[keep], amounts[keep], Cn)).all(), "counter deltas"
            want = int((fv & (ids >= H)).sum() + (fn & (nids >= H)).sum() + (fn & (cids >= Cn)).sum())
            assert now - before == want, "dropped %d, want %d" % (now - before, want)

        cases = Cases()
        for grid, block in SHAPES:
            for pattern, pname in PATTERNS.items():
                cases.run((variant, grid, block, pname), case, grid, block, pattern)
        cases.check()


BLOCK_SHAPES = [s for _, s in SHAPES[:9]]          # these kernels size their grids to the samples, plus idle CTAs


@pytest.mark.parametrize("variant", VARIANTS)
def test_block_histogram_matches_oracle(lh, variant):
    """One BlockHistogram per CTA, its shared memory 16 bytes into the dynamic shared memory, flushed 3 times; CTAs
    bound to ids >= H drop their samples, and the last CTAs get none."""
    lib = client(variant)
    H, chunk, flushes, off = 19, 6007, 3, 16
    cases = Cases()
    for P in BLOCK_PRECISIONS:
        vals, keys = values(P), keys_of(P)
        n = vals.size
        grid = -(-n // chunk) + 3
        block_ids = ids_for(grid, H, SEED ^ P)
        ids = np.repeat(block_ids, chunk)[:n]
        want = hist_ref(H, ids, keys, np.ones(n, dtype=bool))
        with lh.Engine(device=0, max_histograms=H, precision=P) as eng:
            d_v, d_b = eng.upload(vals), eng.upload(block_ids)

            def case(block):
                before = eng.stats()["dropped"]
                with eng.recording() as rec:
                    assert lib.lhm_block_histogram(C.byref(rec), d_b.ptr, d_v.ptr, n, chunk, flushes, off, grid, *block,
                                                   eng.ingest_stream) == 0, "launch failed"
                got, _, now = snapshot(eng, H)
                assert_rows(got, want, "buckets")
                assert now - before == int((ids >= H).sum()), "dropped"

            for block in BLOCK_SHAPES:
                cases.run((variant, P, block), case, block)
    cases.check()


def recorder_cases():
    """(shape, table size, op, two tables): every shape with every table size; record_ns at every other size; two
    tables on every other shape where two fit in shared memory."""
    out = []
    for s, shape in enumerate(BLOCK_SHAPES):
        for t, entries in enumerate(TABLE_SIZES):
            out.append((shape, entries, t % 2, int(s % 2 == 1 and entries <= 4096)))
    return out


@pytest.mark.parametrize("variant", VARIANTS)
def test_block_recorder_matches_oracle(lh, variant):
    """BlockRecorder tables asked for 0, 31, 32, 33, 4096 and 16384 entries, 8 bytes into the dynamic shared memory,
    flushed 3 times, alone or two per CTA over disjoint shared memory, under every shape; the last CTAs get no samples."""
    lib = client(variant)
    H, chunk, flushes, off = 23, 6007, 3, 8
    cases = Cases()
    for P in BLOCK_PRECISIONS:
        srcs = ((values(P), keys_of(P)), (nanos(), nano_keys(P)))
        ids = [ids_for(a.size, H, SEED ^ P ^ j) for j, (a, _) in enumerate(srcs)]
        want = [hist_ref(H, i, k, np.ones(i.size, dtype=bool)) for i, (_, k) in zip(ids, srcs)]
        with lh.Engine(device=0, max_histograms=H, precision=P) as eng:
            dev = [(eng.upload(i), eng.upload(a)) for i, (a, _) in zip(ids, srcs)]

            def case(block, entries, op, dual):
                n = srcs[op][0].size
                grid = -(-n // chunk) + 2
                before = eng.stats()["dropped"]
                with eng.recording() as rec:
                    assert lib.lhm_block_recorder(C.byref(rec), op, dev[op][0].ptr, dev[op][1].ptr, n, chunk, flushes,
                                                  entries, off, dual, grid, *block, eng.ingest_stream) == 0, "launch"
                got, _, now = snapshot(eng, H)
                assert_rows(got, want[op], "buckets")
                assert now - before == int((ids[op] >= H).sum()), "dropped"

            for block, entries, op, dual in recorder_cases():
                what = (variant, P, block, entries, ("record", "record_ns")[op], "two tables" if dual else "one table")
                cases.run(what, case, block, entries, op, dual)
    cases.check()


def test_rdc_kernels_of_both_units_record_into_one_scope(lh):
    """-rdc=true: a kernel of the first translation unit records the first half of the samples and one of the second
    unit the rest, in one scope; the interval equals the oracle."""
    lib = client("rdc")
    P, H = 147, 29
    vals, keys = values(P), keys_of(P)
    ids = ids_for(vals.size, H, SEED ^ 7)
    half = vals.size // 2
    with lh.Engine(device=0, max_histograms=H, precision=P) as eng:
        d_v, d_i = eng.upload(vals), eng.upload(ids)
        with eng.recording() as rec:
            assert lib.lhm_record(C.byref(rec), 0, 0, d_i.ptr, d_v.ptr, half, 264, 256, 1, 1, eng.ingest_stream) == 0
            assert lib.lhm_record_part2(C.byref(rec), d_i.ptr + 4 * half, d_v.ptr + 8 * half, vals.size - half, 264,
                                        256, eng.ingest_stream) == 0
        got, _, dropped = snapshot(eng, H)
        assert_rows(got, hist_ref(H, ids, keys, np.ones(vals.size, dtype=bool)), "rdc")
        assert dropped == int((ids >= H).sum())


# ---------------------------------------------------------------- reads
HIST_ROW = np.dtype([("count", "<u8"), ("sum", "<f8"), ("avg", "<f8"), ("present", "<u4"), ("reserved", "<u4"),
                     ("pvals", "<f8", (32,)), ("pkeys", "<i4", (32,))])


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def to_cuda(torch, a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def kernel_reads(torch, lib, fn, board, rows, inp, in_dtype, out_dtypes):
    """One query per (rows[i], inp[i]) through a launcher of the client; the outputs as numpy arrays."""
    r, x = to_cuda(torch, rows, np.uint32), to_cuda(torch, inp, in_dtype)
    outs = [torch.empty(len(rows), dtype=dt, device="cuda") for dt in out_dtypes]
    assert getattr(lib, fn)(C.byref(board), r.data_ptr(), x.data_ptr(), len(rows), *[o.data_ptr() for o in outs],
                            torch.cuda.current_stream().cuda_stream) == 0, fn
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


@functools.lru_cache(maxsize=None)
def board_cases(precision):
    from oracle import oracle
    table = oracle.decompress_table(precision)
    plain = rc.make_cases(precision, table, SEED)
    wrapped = rc.make_wrapped_cases(precision, table, SEED)
    return ((plain, rc.percentile_pool(plain, table, SEED)), (wrapped, rc.wrapped_percentile_pool(wrapped, table, SEED)))


@pytest.mark.parametrize("variant", VARIANTS)
def test_reads_equal_the_grid_calls(lh, torch, variant):
    """raw_percentile, raw_rank and raw_bucket_count from the variant's kernels equal RawBoard.percentiles / .ranks and
    the export, and read_histogram equals Board.read(), on boards of tests/_reduce_cases.py cases (plain and wrapped)
    at P = 100 and 147.  Rows past the board answer as empty, with publish number 0."""
    import torch as T
    lib = client(variant)
    H = 64
    for P in (100, 147):
        for cases, pool in board_cases(P):
            what = (variant, P, cases[0]["name"])
            assert len(cases) < H
            ids, keys, counts = rc.merge_triples(cases)
            hid = list(range(H - 1)) + [UNBOUND]
            rng = np.random.default_rng(SEED + P)
            ps = np.array(list(pool)[:512] + list(rng.random(128) * 1.1 - 0.05) + [float("nan")], dtype=np.float64)
            labels = list(ps[:32])
            with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=P) as eng, \
                    eng.raw_board(H) as rb, eng.board(H, 1) as bd:
                eng.merge_counts_host(ids, keys, counts)
                eng.snapshot_begin()
                try:
                    rb.publish(hid)
                    eng.snapshot_reduce(labels)
                    bd.publish(hid, [0])
                    sp = eng.snapshot_export()
                finally:
                    eng.snapshot_end()
                # percentiles: every row x every p, and two rows past the board
                gk, gv, _ = (t.cpu().numpy() for t in rb.percentiles(to_cuda(torch, ps, np.float64)))
                T.cuda.synchronize()
                rows = np.concatenate([np.repeat(np.arange(H), ps.size), [H, UNBOUND]])
                pp = np.concatenate([np.tile(ps, H), [0.5, 0.5]])
                kk, kv, kp = kernel_reads(torch, lib, "lhm_raw_percentiles", rb.board, rows, pp, np.float64,
                                          (T.int32, T.float64, T.int64))
                assert (kk[:-2] == gk.ravel()).all() and (bits(kv[:-2]) == bits(gv.ravel())).all(), what
                assert (kk[-2:] == INT32_MIN).all() and np.isnan(kv[-2:]).all(), what
                assert (kp[:-2] == 1).all() and (kp[-2:] == 0).all(), what
                # ranks of the edge values
                vals = np.concatenate([edge_values(P)[::37], [0.0, -0.0, np.nan, np.inf, -np.inf, 1e300]])
                gr, gt, _ = (t.cpu().numpy() for t in rb.ranks(to_cuda(torch, vals, np.float64)))
                rows = np.repeat(np.arange(H), vals.size)
                kr, kt, kp = kernel_reads(torch, lib, "lhm_raw_ranks", rb.board, rows, np.tile(vals, H), np.float64,
                                          (T.int64, T.int64, T.int64))
                assert (kr == gr.ravel()).all() and (kt == np.repeat(gt, vals.size)).all() and (kp == 1).all(), what
                # bucket counts of every key of every row
                rows = np.repeat(np.arange(H), 65536)
                allkeys = np.tile(np.arange(-32768, 32768), H)
                bc, bp = kernel_reads(torch, lib, "lhm_raw_bucket_counts", rb.board, rows, allkeys, np.int32,
                                      (T.int64, T.int64))
                want = np.zeros((H, 65536), dtype=np.uint64)
                hrow = np.repeat(np.arange(H), np.diff(sp.offsets.astype(np.int64)))
                want[hrow, sp.keys.astype(np.int64) + 32768] = sp.counts
                assert (bc.view(np.uint64) == want.ravel()).all() and (bp == 1).all(), what
                # processed rows
                v = {k: x.cpu().numpy() for k, x in bd.read().items()}
                T.cuda.synchronize()
                rows = np.concatenate([np.arange(H), [H, H + 7]]).astype(np.uint32)
                out = T.zeros(rows.size * HIST_ROW.itemsize, dtype=T.uint8, device="cuda")
                pub = T.zeros(rows.size, dtype=T.int64, device="cuda")
                assert lib.lhm_read_histograms(C.byref(bd.board), to_cuda(torch, rows, np.uint32).data_ptr(), rows.size,
                                               out.data_ptr(), pub.data_ptr(), T.cuda.current_stream().cuda_stream) == 0
                T.cuda.synchronize()
                hr, pub = out.cpu().numpy().view(HIST_ROW), pub.cpu().numpy()
                assert (pub[:H] == int(v["collection"])).all() and (pub[H:] == 0).all(), what
                assert (hr["count"][:H] == v["count"].view(np.uint64)).all(), what
                assert (bits(hr["sum"][:H]) == bits(v["sum"])).all() and (bits(hr["avg"][:H]) == bits(v["avg"])).all()
                assert (hr["present"][:H] == v["present"]).all(), what
                assert (bits(hr["pvals"][:H]) == bits(v["pvals"])).all() and (hr["pkeys"][:H] == v["pkeys"]).all(), what
                assert (hr[H:].view(np.uint8) == 0).all(), what
