"""Joined ranks (MetricSystem.join_ranks) on the CPU: the C++ mirror over the TEST-ONLY oracle-backed stub of the C ABI
(tests/stub_abi/lh_stub_ranks.c), whose all-reduce sums the stub contexts of one process through the maps, one thread
per rank.  Covers the byte-sorted union and its cut at the bounds with drop counts, the maps after churn (one name at
different and recycled ids per rank), Counter(name, 0) in Rates, the configuration refusal at join on every rank
alike, a failed exchange on every rank followed by a summed collection, the stub's validation of both ABI calls, the
Python argument errors, the lhms_ranks_* bindings, and a mirror over a stub without the calls.
tests/test_gpu_ranks.py runs the real library."""
import ctypes
import os
import random
import re
import subprocess
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUBS = ("lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c")
CALLS = ["lh_snapshot_rows", "lh_snapshot_allreduce_rows"]
ABSENT = 0xFFFFFFFF
LH_ERR_INVALID, LH_ERR_STATE, LH_ERR_RANGE = -1, -5, -6


def build_pair(tag, stub_main):
    stub = os.path.join(BUILD, "liblh_stub_ranks%s.so" % tag)
    host = os.path.join(BUILD, "libloghisto_host_stub_ranks%s.so" % tag)
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in (stub_main,) + STUBS] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_ranks%s" % tag, "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return ctypes.CDLL(stub), host


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    s, host = build_pair("", "lh_stub_ranks.c")
    s.lh_stub_rows_calls.restype = ctypes.c_uint64
    return s, host


@pytest.fixture
def MS(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    made = []

    def make(max_histograms=16, max_counters=16, precision=0):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=max_counters, precision=precision)
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


class Exchange:
    """An all-gather between rank threads; fail=True makes every rank's callback raise before the barrier."""

    def __init__(self, world):
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)
        self.fail = False

    def for_rank(self, r):
        def allgather(mine):
            if self.fail:
                raise RuntimeError("exchange down")
            self.slots[r] = bytes(mine)
            self.barrier.wait(timeout=60)
            out = list(self.slots)
            self.barrier.wait(timeout=60)
            return out
        return allgather


def on_ranks(world, fn):
    out, errs = [None] * world, [None] * world

    def run(r):
        try:
            out[r] = fn(r)
        except BaseException as e:
            errs[r] = e
    ts = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out, errs


def joined(MS, world, **kw):
    ex = Exchange(world)
    systems = [MS(**kw) for _ in range(world)]
    _, errs = on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r)))
    assert errs == [None] * world
    return systems, ex


def collect(systems):
    got, errs = on_ranks(len(systems), lambda r: systems[r].collect_and_process())
    assert errs == [None] * len(systems)
    return got


def test_union_is_byte_sorted_and_cut_at_the_bounds_with_drops_counted(MS):
    systems, _ = joined(MS, 2, max_histograms=4, max_counters=3)
    # byte order puts "B" < "a" < "b"; rank 0 interns in reverse order so its ids do not follow the union
    names0, names1 = ["b2", "a1", "B0"], ["b2", "c3", "a1", "zz"]
    for i, n in enumerate(names0):
        for _ in range(i + 1):
            systems[0].Histogram(n, 5.0)
    for i, n in enumerate(names1):
        for _ in range(10 * (i + 1)):
            systems[1].Histogram(n, 7.0)
    for n, a in (("k3", 4), ("k1", 0), ("K0", 2)):
        systems[0].Counter(n, a)
    for n, a in (("k2", 5), ("k9", 6)):
        systems[1].Counter(n, a)
    before = [ms.dropped() for ms in systems]
    got = collect(systems)
    kept = sorted(set(names0 + names1))[:4]
    assert kept == ["B0", "a1", "b2", "c3"]
    for raw, _ in got:
        assert sorted(raw["Histograms"]) == kept
        assert sum(raw["Histograms"]["b2"].values()) == 1 + 10
        assert sum(raw["Histograms"]["a1"].values()) == 2 + 30
        assert raw["Rates"] == {"K0": 2, "k1": 0, "k2": 5}
    # rank 1 recorded 40 samples under "zz"; rank 0 counter "k3" (4), rank 1 "k9" (6)
    assert [systems[r].dropped() - before[r] for r in range(2)] == [4, 40 + 6]
    assert [ms.ranks_info()["names_dropped"] for ms in systems] == [3, 3]


def test_maps_after_churn_equal_one_system_seeing_every_sample(MS):
    """Rank 0 interns a, b, c and rank 1 c, b, a, so one name sits at different ids.  a and b then idle on rank 0 for
    three intervals, which frees their ids (NameTable), and d, e take them over while rank 1 keeps a and b; the last
    intervals mix names at random.  Every collection must equal one unjoined system fed every rank's samples."""
    world = 2
    systems, _ = joined(MS, world, max_histograms=5, max_counters=4)   # 5 names: never full, ids still recycled
    ref = MS(max_histograms=64, max_counters=64)
    rng = random.Random(7)
    plan = [(["a", "b", "c"], ["c", "b", "a"]), (["c"], ["a", "b"]), (["c"], ["b"]), (["c"], ["a"]),
            (["d", "e"], ["a", "b"]), (["d", "a"], ["e", "b"])]
    plan += [(rng.sample("abcde", 2), rng.sample("abcde", 2)) for _ in range(6)]
    for interval, per_rank in enumerate(plan):
        for r, names in enumerate(per_rank):
            for n in names:
                for _ in range(rng.randint(1, 5)):
                    v = rng.lognormvariate(2, 2)
                    systems[r].Histogram(n, v)
                    ref.Histogram(n, v)
            c = "k%d" % rng.randint(0, 2)
            a = rng.randint(0, 3)
            systems[r].Counter(c, a)
            ref.Counter(c, a)
        got = collect(systems)
        want_raw, want = ref.collect_and_process()
        for raw, metrics in got:
            assert raw["Histograms"] == want_raw["Histograms"], interval
            assert raw["Rates"] == want_raw["Rates"], interval
            assert raw["Counters"] == want_raw["Counters"], interval
            assert metrics == want, interval
    assert all(ms.ranks_info()["summed"] == len(plan) for ms in systems)
    assert all(ms.dropped() == 0 for ms in systems)


def test_counter_zero_is_in_rates_on_every_rank(MS):
    systems, _ = joined(MS, 2)
    systems[1].Counter("z", 0)
    for raw, _ in collect(systems):
        assert raw["Rates"] == {"z": 0} and raw["Counters"] == {"z": 0}


def test_configuration_mismatch_is_refused_on_every_rank_alike(MS, stub_libs):
    ex = Exchange(2)
    systems = [MS(max_histograms=4), MS(max_histograms=8)]
    _, errs = on_ranks(2, lambda r: systems[r].join_ranks(r, 2, ex.for_rank(r)))
    assert all(isinstance(e, ValueError) and "max_histograms" in str(e) for e in errs), errs
    for ms in systems:   # nothing was imported: the systems still collect alone
        assert ms.ranks_info()["world"] == 0
        ms.Histogram("h", 1.0)
        raw, _ = ms.collect_and_process()
        assert sum(raw["Histograms"]["h"].values()) == 1


def test_failed_exchange_on_every_rank_then_a_summed_collection(MS, stub_libs, capfd):
    systems, ex = joined(MS, 3)
    calls = stub_libs[0].lh_stub_rows_calls()
    for r, ms in enumerate(systems):
        ms.Histogram("h", float(r + 1))
        ms.Counter("c", r + 1)
    ex.fail = True
    for r, (raw, _) in enumerate(collect(systems)):
        assert sum(raw["Histograms"]["h"].values()) == 1
        assert raw["Rates"] == {"c": r + 1}
        assert systems[r].ranks_info()["status"] == 3
    assert stub_libs[0].lh_stub_rows_calls() == calls      # nothing launched anywhere
    assert "exchange down" in capfd.readouterr().err
    ex.fail = False
    for ms in systems:
        ms.Histogram("h", 2.0)
        ms.Counter("c", 1)
    for r, (raw, _) in enumerate(collect(systems)):
        assert sum(raw["Histograms"]["h"].values()) == 3
        assert raw["Rates"] == {"c": 3}
        assert raw["Counters"] == {"c": (r + 1) + 3}   # the cumulative store keeps the rank-local interval
    assert all(ms.ranks_info()["status"] == 0 and ms.ranks_info()["summed"] == 1 for ms in systems)


class lh_config(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("device", ctypes.c_int32), ("max_histograms", ctypes.c_uint32),
                ("max_counters", ctypes.c_uint32), ("staging_bytes", ctypes.c_uint64), ("staging_slots", ctypes.c_uint32),
                ("flags", ctypes.c_uint32), ("precision", ctypes.c_uint32), ("reserved", ctypes.c_uint32 * 3)]


def test_abi_validation(stub_libs):
    """The stub validates both calls as the header states, before anything is launched."""
    s = stub_libs[0]
    vp, u32 = ctypes.c_void_p, ctypes.c_uint32
    s.lh_create.restype = s.lh_comm_import.restype = s.lh_snapshot_begin.restype = ctypes.c_int
    s.lh_snapshot_rows.restype = s.lh_snapshot_allreduce_rows.restype = ctypes.c_int
    s.lh_snapshot_rows.argtypes = [vp, vp, vp, vp]
    s.lh_snapshot_allreduce_rows.argtypes = [vp, ctypes.c_uint64, vp, u32, vp, u32, vp, vp]
    s.lh_comm_import.argtypes = [vp, u32, u32, vp]
    s.lh_comm_export.argtypes = [vp, vp]
    s.lh_snapshot_begin.argtypes = s.lh_snapshot_end.argtypes = s.lh_destroy.argtypes = [vp]
    H, C = 4, 2
    cfg = lh_config(ctypes.sizeof(lh_config), 0, H, C, 0, 0, 0, 0)
    ctxs = []
    for _ in range(2):
        c = vp()
        assert s.lh_create(ctypes.byref(cfg), ctypes.byref(c)) == 0
        ctxs.append(c)
    c = ctxs[0]
    hm = np.tile(np.arange(H, dtype=np.uint32), (2, 1))
    cm = np.tile(np.arange(C, dtype=np.uint32), (2, 1))
    fr = np.array([1, 1], np.uint32)

    def ar(seq=1, frozen=fr, n=H, h=hm, nc=C, cmap=cm):
        return s.lh_snapshot_allreduce_rows(c, seq, frozen.ctypes.data if frozen is not None else None, n,
                                            h.ctypes.data if h is not None else None, nc,
                                            cmap.ctypes.data if cmap is not None else None, None)
    try:
        touched = np.zeros(H, np.uint8)
        assert s.lh_snapshot_rows(c, touched.ctypes.data, None, None) == LH_ERR_STATE     # no snapshot
        assert s.lh_snapshot_begin(c) == 0
        assert ar() == LH_ERR_STATE                                                     # no lh_comm_import
        assert s.lh_snapshot_end(c) == 0
        handles = (ctypes.c_uint8 * (2 * 1024))()
        for r, x in enumerate(ctxs):
            assert s.lh_comm_export(x, ctypes.byref(handles, r * 1024)) == 0
        for r, x in enumerate(ctxs):
            assert s.lh_comm_import(x, r, 2, handles) == 0
        assert ar() == LH_ERR_STATE                                                     # no snapshot
        assert s.lh_snapshot_begin(c) == 0                                              # freezes half 1
        frozen = ctypes.c_uint32(9)
        assert s.lh_snapshot_rows(c, touched.ctypes.data, None, ctypes.byref(frozen)) == 0 and frozen.value == 1
        before = s.lh_stub_rows_calls()
        assert ar(n=H + 1, h=np.zeros((2, H + 1), np.uint32)) == LH_ERR_INVALID
        assert ar(nc=C + 1, cmap=np.zeros((2, C + 1), np.uint32)) == LH_ERR_INVALID
        assert ar(h=None) == LH_ERR_INVALID
        assert ar(cmap=None) == LH_ERR_INVALID
        assert ar(frozen=None) == LH_ERR_INVALID
        assert ar(frozen=np.array([1, 2], np.uint32)) == LH_ERR_INVALID
        assert ar(frozen=np.array([0, 1], np.uint32)) == LH_ERR_INVALID                # not this snapshot's half
        assert ar(seq=0) == LH_ERR_INVALID                                              # not above the last
        bad = hm.copy(); bad[1, 2] = H
        assert ar(h=bad) == LH_ERR_RANGE
        bad = cm.copy(); bad[0, 1] = C
        assert ar(cmap=bad) == LH_ERR_RANGE
        assert s.lh_stub_rows_calls() == before                                        # nothing was launched
        s.lh_snapshot_end(c)
    finally:
        for x in ctxs:
            s.lh_destroy(x)


def test_argument_errors_are_raised_before_any_call(MS):
    ms = MS()
    never = lambda mine: pytest.fail("allgather called")   # noqa: E731
    with pytest.raises(TypeError):
        ms.join_ranks(0, 2, None)
    for rank, world in ((0, 1), (2, 2), (-1, 2), (0, 17)):
        with pytest.raises(ValueError):
            ms.join_ranks(rank, world, never)
    assert ms.ranks_info() == {"rank": 0, "world": 0, "status": 0, "summed": 0, "bytes_from_peers": 0,
                               "names_dropped": 0}


def test_join_after_a_collection_is_refused(MS):
    ms = MS()
    ms.collect_and_process()
    with pytest.raises(RuntimeError, match="collected already"):
        ms.join_ranks(0, 2, lambda mine: pytest.fail("allgather called"))


def test_bindings_and_weak_symbols(stub_libs):
    from loghisto_b200 import _lib
    import loghisto_b200.metric_system as m
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    for nm in CALLS:
        assert re.search(r"LH_API lh_status %s\(" % nm, hdr), nm
        assert nm in _lib.SIGNATURES, nm
        assert "#pragma weak " + nm in src, nm
    names = re.findall(r"LHMS_API [\w *]+?(lhms_ranks_\w+)\(", src)
    assert names == ["lhms_ranks_join", "lhms_ranks_info"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm


def test_mirror_over_a_stub_without_the_calls(monkeypatch):
    """The calls are bound weakly: over a C ABI without them join_ranks refuses before any exchange, and the system
    still collects its own interval."""
    import loghisto_b200.metric_system as m
    _, host = build_pair("_old", "lh_stub.c")
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        with pytest.raises(RuntimeError, match="no row-mapped all-reduce"):
            ms.join_ranks(0, 2, lambda mine: pytest.fail("allgather called"))
        ms.Histogram("h", 3.0)
        ms.Counter("c", 0)
        raw, _ = ms.collect_and_process()
        assert sum(raw["Histograms"]["h"].values()) == 1
        assert raw["Rates"] == {"c": 0}
        assert ms.ranks_info()["world"] == 0
    finally:
        ms.close()
