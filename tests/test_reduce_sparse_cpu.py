"""lh_reduce_sparse_host's semantics without a GPU: the Go-map reference (zero-count keys kept) against the oracle's
percentile() on (value, count) pairs, and processMetrics of the C++ mirror on sets it did not collect, over the
oracle-backed stub of the C ABI (tests/stub_abi/lh_stub.c) plus its lh_reduce_sparse_host
(tests/stub_abi/lh_stub_reduce_sparse.c)."""
import ctypes
import math
import os
import random
import subprocess

import numpy as np
import pytest

import _process_metrics_cases as pmc
import _reduce_cases as rc
from _go_map_reference import GoMapReference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
SEED = 0x5BA25E


@pytest.fixture(scope="module")
def stub_host_lib():
    """The host mirror linked against the stub with lh_reduce_sparse_host (own file names in tests/_build)."""
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_rs.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_rs.so")
    inc = os.path.join(ROOT, "include")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", inc,
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub.c"),
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub_reduce_sparse.c"),
                    os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", inc,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_rs", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return host


@pytest.fixture()
def MS(stub_host_lib, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_host_lib)))
    made = []

    def make(interval_s=3600.0, **kw):
        ms = m.MetricSystem(interval_s, False, max_histograms=kw.get("max_histograms", 64),
                            max_counters=kw.get("max_counters", 64))
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


def go_map_cases(precision: int, table: np.ndarray, rng: random.Random) -> list:
    """Maps with zero-count keys: below, inside and above the non-empty ones, at both ends of the key range (+-Inf at
    precisions <= 46), all zero, and large totals."""
    w = rc.window(precision)
    cases = [
        {-5: 0, 0: 3, 7: 2},
        {0: 3, 4: 0, 7: 2},
        {-w - 3: 0, 0: 3, w - 1: 1},
        {-32768: 0, 5: 4},
        {32767: 0, 5: 4, -3: 2},
        {-32768: 0, -32767: 0, 32767: 0, 1: 1},
        {1: 0, -2: 0},
        {-32768: 0},
        {3: 2 ** 63, -9: 0, 10: 2 ** 63 - 1},
    ]
    for _ in range(20):                   # finite sums: |decompress| below e^175 times counts below 2^40
        keys = rng.sample(range(-4 * w, 4 * w), rng.randrange(1, 40))
        cases.append({k: rng.choice([0, 0, 1, rng.randrange(2 ** 40)]) for k in keys})
    return cases


@pytest.mark.parametrize("precision", [46, 100])
def test_go_map_reference_matches_oracle_percentile(oracle, precision):
    table = oracle.decompress_table(precision)
    rng = random.Random(SEED + precision)
    cases = go_map_cases(precision, table, rng)
    ps = list(rc.SPECIAL_PS) + [0.25, 0.75, 1e-300, -1e-300]
    for hist in cases:
        ref = GoMapReference(hist, table)
        values = [float(table[k & 0xFFFF]) for k in hist]
        counts = list(hist.values())
        total = sum(counts) % 2 ** 64
        for p in ps:
            key = ref.percentile(p)
            try:
                got = oracle.percentile(total, values, counts, p)
            except ValueError:
                assert key is None, (hist, p)
                continue
            assert key is not None, (hist, p)
            assert rc.same_bits(got, float(table[key & 0xFFFF])), (hist, p, got, key)
        # Go's sum, in any order: Inf * 0 is NaN
        go_sum = sum(v * float(c) for v, c in zip(values, counts))
        assert rc.sum_ok(go_sum, ref), (hist, go_sum, ref.sum)


def test_go_map_mode_differs_only_on_zero_counts(oracle):
    table = oracle.decompress_table(46)
    hist = {-32768: 0, -7: 0, 2: 5, 9: 1}
    go, dense = GoMapReference(hist, table), rc.Reference(hist, table)
    assert go.percentile(0.0) == -32768 and dense.percentile(0.0) == 2
    assert go.percentile(0.5) == dense.percentile(0.5) == 2
    assert math.isnan(go.sum) and not isinstance(dense.sum, float)
    assert go.count == dense.count == 6 and go.nnz == dense.nnz == 2
    assert GoMapReference({5: 0}, table).percentile(0.0) is None


def test_stub_reduce_sparse_zero_count_rules(stub_host_lib, oracle):
    """The stub's lh_reduce_sparse_host (what the CPU mirror tests run on) against the Go-map reference at precision 100,
    on shuffled, split entries."""
    lib = ctypes.CDLL(stub_host_lib)
    table = oracle.decompress_table(100)
    rng = random.Random(SEED)
    cases = go_map_cases(100, table, rng)
    offsets, keys, counts = [0], [], []
    for hist in cases:
        entries = []
        for k, c in hist.items():
            a = rng.randrange(2 ** 64)
            entries += [(k, a), (k, (c - a) % 2 ** 64)] if rng.random() < 0.5 else [(k, c)]
        rng.shuffle(entries)
        keys += [k for k, _ in entries]
        counts += [c for _, c in entries]
        offsets.append(len(keys))
    ps = np.array(rc.SPECIAL_PS + [0.5, 0.9], dtype=np.float64)
    n, npct = len(cases), ps.size
    offs = np.array(offsets, np.uint32)
    ks, cs = np.array(keys, np.int16), np.array(counts, np.uint64)
    out_c, sums, avgs = np.zeros(n, np.uint64), np.zeros(n), np.zeros(n)
    pk, pv = np.zeros((n, npct), np.int32), np.zeros((n, npct))
    lib.lh_create.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
    from loghisto_b200 import _lib as L
    cfg = L.lh_config(ctypes.sizeof(L.lh_config), 0, 1, 1, 0, 0, 0, 100)
    h = ctypes.c_void_p()
    assert lib.lh_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    fn = lib.lh_reduce_sparse_host
    fn.argtypes = L.SIGNATURES["lh_reduce_sparse_host"][1]
    try:
        assert fn(h, n, offs.ctypes.data, ks.ctypes.data, cs.ctypes.data, ps.ctypes.data, npct, out_c.ctypes.data,
                  sums.ctypes.data, avgs.ctypes.data, pk.ctypes.data, pv.ctypes.data) == 0
        bad = offs.copy()
        bad[1], bad[2] = bad[2], bad[1]
        assert fn(h, n, bad.ctypes.data, ks.ctypes.data, cs.ctypes.data, ps.ctypes.data, npct, 0, 0, 0, 0, 0) == -1
        assert fn(h, n, offs.ctypes.data, ks.ctypes.data, cs.ctypes.data, ps.ctypes.data, 33, 0, 0, 0, 0, 0) == -1
        assert fn(h, n, offs.ctypes.data, None, cs.ctypes.data, ps.ctypes.data, npct, 0, 0, 0, 0, 0) == -1
    finally:
        lib.lh_destroy.argtypes = [ctypes.c_void_p]
        lib.lh_destroy(h)
    for i, hist in enumerate(cases):
        ref = GoMapReference(hist, table, str(hist))
        want = ref.results(ps)
        assert int(out_c[i]) == ref.count, hist
        assert list(pk[i]) == [rc.INT32_MIN if k is None else k for k in want["keys"]], hist
        assert rc.same_bits(pv[i], want["values"]).all(), hist
        assert rc.sum_ok(float(sums[i]), ref), hist
        assert rc.same_bits(avgs[i], sums[i] / float(ref.count) if ref.count else math.nan), hist


def test_kat1_bare_keys(MS):
    pmc.check_kat1_bare_keys(MS)


def test_union_of_two_systems(MS):
    pmc.check_union_of_two_systems(MS)


def test_empty_map(MS):
    pmc.check_empty_map(MS)


def test_collected_set_fed_back(MS):
    pmc.check_collected_set_fed_back(MS)
