"""Joined ranks through the caller's all-reduce (MetricSystem.join_ranks(..., allreduce)) on the CPU: the C++ mirror over
the TEST-ONLY oracle-backed stub (tests/stub_abi/lh_stub_rows_pack.c, whose "device" payloads are host memory), one
thread per rank, with an in-process numpy uint64 all-reduce.  Covers the payload layout every rank agrees on (one rank
dense, another window-only on the same name), one callback per collection and none when nothing was touched, a failed
exchange, a raising callback, the refusals at join, a stub without the calls and the C shim driven from C.
tests/test_gpu_ranks_allreduce.py runs the real library."""
import ctypes
import os
import random
import subprocess
import threading

import numpy as np
import pytest

from test_ranks_cpu import BUILD, INC, ROOT, Exchange, build_pair, on_ranks

WIN100 = 4368   # fast-window half-width at precision 100: a window row is 2 * WIN100 - 1 words


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    s, host = build_pair("_pack", "lh_stub_rows_pack.c")
    s.lh_stub_pack_calls.restype = s.lh_stub_unpack_calls.restype = s.lh_stub_rows_calls.restype = ctypes.c_uint64
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


def words_at(ptr, n):
    return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint64)), shape=(n,)) if n else np.zeros(0, np.uint64)


class Reduce:
    """An element-wise uint64 all-reduce between rank threads over the stub's host payloads; records every call.
    fail=True makes every rank's callback raise before the barrier."""

    def __init__(self, world):
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)
        self.fail = False
        self.calls = [[] for _ in range(world)]

    def for_rank(self, r):
        def allreduce(send, recv, n, stream):
            self.calls[r].append(n)
            if self.fail:
                raise RuntimeError("transport down")
            self.slots[r] = words_at(send, n).copy()
            self.barrier.wait(timeout=60)
            total = np.zeros(n, np.uint64)
            for s in self.slots:
                total += s                      # uint64: wraps as the contract asks
            words_at(recv, n)[:] = total
            self.barrier.wait(timeout=60)
        return allreduce


def joined(MS, world, **kw):
    ex, red = Exchange(world), Reduce(world)
    systems = [MS(**kw) for _ in range(world)]
    _, errs = on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r), red.for_rank(r)))
    assert errs == [None] * world, errs
    return systems, ex, red


def collect(systems):
    got, errs = on_ranks(len(systems), lambda r: systems[r].collect_and_process())
    assert errs == [None] * len(systems), errs
    return got


def test_every_rank_agrees_on_the_layout_with_one_rank_dense(MS):
    systems, _, red = joined(MS, 3)
    systems[0].Histogram("x", 1e100)          # beyond the window: rank 0's row is dense
    systems[1].Histogram("x", 5.0)            # window only on ranks 1 and 2
    systems[2].Histogram("x", 6.0)
    systems[1].Histogram("y", 7.0)
    for r, ms in enumerate(systems):
        ms.Counter("c%d" % (r % 2), r + 1)
    got = collect(systems)
    want_words = 65536 + (2 * WIN100 - 1) + 2      # x dense, y window, counters c0 and c1
    assert [c for c in red.calls] == [[want_words]] * 3
    for raw, _ in got:
        assert {k: sum(v.values()) for k, v in raw["Histograms"].items()} == {"x": 3, "y": 1}
        assert raw["Rates"] == {"c0": 1 + 3, "c1": 2}
    assert all(ms.ranks_info()["bytes_from_peers"] == 8 * want_words for ms in systems)


def test_collections_equal_one_system_seeing_every_sample(MS, stub_libs):
    """Names at different and recycled ids per rank, values in and beyond the window, counters and Counter(name, 0)."""
    world = 2
    systems, _, red = joined(MS, world, max_histograms=5, max_counters=4)
    ref = MS(max_histograms=64, max_counters=64)
    rng = random.Random(11)
    rows_calls = stub_libs[0].lh_stub_rows_calls()
    plan = [(["a", "b", "c"], ["c", "b", "a"]), (["c"], ["a", "b"]), (["c"], ["b"]), (["c"], ["a"]),
            (["d", "e"], ["a", "b"]), (["d", "a"], ["e", "b"])]
    plan += [(rng.sample("abcde", 2), rng.sample("abcde", 2)) for _ in range(6)]
    for interval, per_rank in enumerate(plan):
        for r, names in enumerate(per_rank):
            for n in names:
                for _ in range(rng.randint(1, 5)):
                    v = rng.choice([rng.lognormvariate(2, 2), 1e100, -3e90])
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
    assert red.calls == [[red.calls[0][i] for i in range(len(plan))]] * world   # once per collection, same sizes
    assert all(ms.ranks_info()["summed"] == len(plan) and ms.ranks_info()["status"] == 0 for ms in systems)
    assert stub_libs[0].lh_stub_rows_calls() == rows_calls                     # the peer all-reduce never ran


def test_no_callback_when_nothing_was_touched(MS, stub_libs):
    systems, _, red = joined(MS, 2)
    packs = stub_libs[0].lh_stub_pack_calls()
    for raw, _ in collect(systems):
        assert raw["Histograms"] == {} and raw["Rates"] == {}
    assert red.calls == [[], []]
    assert stub_libs[0].lh_stub_pack_calls() == packs + 2     # every rank packed an empty payload
    assert all(ms.ranks_info()["status"] == 0 for ms in systems)


def test_failed_exchange_gives_status_3_and_no_callback(MS, stub_libs):
    systems, ex, red = joined(MS, 3)
    packs = stub_libs[0].lh_stub_pack_calls()
    for r, ms in enumerate(systems):
        ms.Histogram("h", float(r + 1))
        ms.Counter("c", r + 1)
    ex.fail = True
    for r, (raw, _) in enumerate(collect(systems)):
        assert sum(raw["Histograms"]["h"].values()) == 1
        assert raw["Rates"] == {"c": r + 1}
        assert systems[r].ranks_info()["status"] == 3
    assert red.calls == [[], [], []] and stub_libs[0].lh_stub_pack_calls() == packs
    ex.fail = False
    for ms in systems:
        ms.Histogram("h", 2.0)
    for raw, _ in collect(systems):
        assert sum(raw["Histograms"]["h"].values()) == 3
    assert all(ms.ranks_info()["status"] == 0 and ms.ranks_info()["summed"] == 1 for ms in systems)


def test_raising_callback_gives_own_counts_under_job_wide_names_then_sums_again(MS, capfd):
    systems, _, red = joined(MS, 2)
    systems[0].Histogram("a", 1.0)
    systems[1].Histogram("b", 2.0)
    systems[1].Histogram("b", 3.0)
    systems[0].Counter("c", 4)
    red.fail = True
    got = collect(systems)
    assert {k: sum(v.values()) for k, v in got[0][0]["Histograms"].items()} == {"a": 1}
    assert {k: sum(v.values()) for k, v in got[1][0]["Histograms"].items()} == {"b": 2}
    assert got[0][0]["Rates"] == {"c": 4} and got[1][0]["Rates"] == {"c": 0}    # the job-wide row, this rank's count
    assert [ms.ranks_info()["status"] for ms in systems] == [4, 4]
    assert [ms.ranks_info()["bytes_from_peers"] for ms in systems] == [0, 0]
    assert "transport down" in capfd.readouterr().err
    red.fail = False
    systems[0].Histogram("b", 1.0)
    systems[1].Histogram("b", 1.0)
    for raw, _ in collect(systems):
        assert {k: sum(v.values()) for k, v in raw["Histograms"].items()} == {"b": 2}
    assert all(ms.ranks_info()["status"] == 0 and ms.ranks_info()["summed"] == 1 for ms in systems)


@pytest.mark.parametrize("mismatch", ["transport", "max_histograms", "max_counters", "precision"])
def test_ranks_that_disagree_are_refused_on_every_rank(MS, mismatch):
    ex, red = Exchange(2), Reduce(2)
    kw = [dict(), dict()]
    if mismatch != "transport":
        kw[1][mismatch] = {"max_histograms": 8, "max_counters": 8, "precision": 250}[mismatch]
    systems = [MS(**kw[0]), MS(**kw[1])]

    def join(r):
        reduce = None if (mismatch == "transport" and r == 0) else red.for_rank(r)
        systems[r].join_ranks(r, 2, ex.for_rank(r), reduce)
    _, errs = on_ranks(2, join)
    assert all(isinstance(e, ValueError) and mismatch in str(e) for e in errs), errs
    for ms in systems:
        assert ms.ranks_info()["world"] == 0


def test_a_non_callable_allreduce_is_a_type_error(MS):
    ms = MS()
    with pytest.raises(TypeError):
        ms.join_ranks(0, 2, lambda mine: pytest.fail("allgather called"), 42)
    assert ms.ranks_info()["world"] == 0


def test_mirror_over_a_library_without_the_calls(monkeypatch):
    import loghisto_b200.metric_system as m
    _, host = build_pair("_nopack", "lh_stub_ranks.c")
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    ms = m.MetricSystem(1e-6, False, max_histograms=4, max_counters=4)
    try:
        with pytest.raises(RuntimeError, match="lh_snapshot_pack_rows"):
            ms.join_ranks(0, 2, lambda mine: pytest.fail("allgather called"), lambda *a: pytest.fail("allreduce called"))
        ms.Histogram("h", 3.0)
        raw, _ = ms.collect_and_process()
        assert sum(raw["Histograms"]["h"].values()) == 1
    finally:
        ms.close()


def test_bindings_and_weak_symbols(stub_libs):
    import re
    from loghisto_b200 import _lib
    hdr = open(os.path.join(INC, "loghisto_b200.h")).read()
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    for nm in ("lh_snapshot_row_levels", "lh_snapshot_pack_rows", "lh_snapshot_unpack_rows"):
        assert re.search(r"LH_API lh_status %s\(" % nm, hdr), nm
        assert nm in _lib.SIGNATURES, nm
        assert "#pragma weak " + nm in src, nm
    import loghisto_b200.metric_system as m
    assert m._bind(ctypes.CDLL(stub_libs[1])).lhms_ranks_join_allreduce.argtypes is not None


C_DRIVER = r"""
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

typedef void (*sink_fn)(void *, uint32_t, const void *, uint64_t);
typedef void (*emit_fn)(void *, int, const char *, int, uint64_t, double);
void *lhms_new(int64_t, int, uint32_t, uint32_t, char *, int);
void lhms_free(void *);
void lhms_histogram(void *, const char *, double);
void lhms_counter(void *, const char *, uint64_t);
int lhms_collect_and_process(void *, emit_fn, void *, char *, int);
void lhms_ranks_info(void *, uint64_t *);
int lhms_ranks_join_allreduce(void *, uint32_t, uint32_t,
                              int (*)(void *, const void *, uint64_t, sink_fn, void *),
                              int (*)(void *, const uint64_t *, uint64_t *, uint64_t, void *), void *, char *, int);

static pthread_barrier_t bar;
static char gathered[2][4096]; static uint64_t glen[2];
static const uint64_t *sends[2]; static uint64_t nwords[2];
static double count_h[2], rate_c[2];

static int gather(void *user, const void *mine, uint64_t len, sink_fn sink, void *sctx) {
    int r = (int)(intptr_t)user;
    memcpy(gathered[r], mine, len); glen[r] = len;
    pthread_barrier_wait(&bar);
    for (uint32_t k = 0; k < 2; k++) sink(sctx, k, gathered[k], glen[k]);
    pthread_barrier_wait(&bar);
    return 0;
}
static int reduce(void *user, const uint64_t *send, uint64_t *recv, uint64_t n, void *stream) {
    int r = (int)(intptr_t)user;
    (void)stream;
    sends[r] = send; nwords[r] = n;
    pthread_barrier_wait(&bar);
    if (nwords[0] != nwords[1]) return 1;
    for (uint64_t i = 0; i < n; i++) recv[i] = sends[0][i] + sends[1][i];
    pthread_barrier_wait(&bar);
    return 0;
}
struct out { int r; };
static void emit(void *ctx, int kind, const char *name, int key, uint64_t u, double f) {
    int r = ((struct out *)ctx)->r;
    (void)key;
    if (kind == 3 && !strcmp(name, "h_count")) count_h[r] = f;   /* processed metric */
    if (kind == 1 && !strcmp(name, "c")) rate_c[r] = (double)u;  /* raw rate */
}
static void *rank_main(void *arg) {
    int r = (int)(intptr_t)arg;
    char err[256] = "";
    void *ms = lhms_new(1000, 0, 8, 8, err, sizeof err);
    if (lhms_ranks_join_allreduce(ms, r, 2, gather, reduce, (void *)(intptr_t)r, err, sizeof err) != 0) {
        fprintf(stderr, "join: %s\n", err); return (void *)1;
    }
    for (int i = 0; i <= r; i++) lhms_histogram(ms, "h", 10.0 * (i + 1));
    lhms_counter(ms, "c", 5 + r);
    struct out o = {r};
    if (lhms_collect_and_process(ms, emit, &o, err, sizeof err) != 0) { fprintf(stderr, "collect: %s\n", err); return (void *)1; }
    uint64_t info[6];
    lhms_ranks_info(ms, info);
    printf("rank %d count %g rate %g status %llu summed %llu bytes %llu\n", r, count_h[r], rate_c[r],
           (unsigned long long)info[2], (unsigned long long)info[3], (unsigned long long)info[4]);
    lhms_free(ms);
    return NULL;
}
int main(void) {
    pthread_t t[2];
    pthread_barrier_init(&bar, NULL, 2);
    for (intptr_t r = 0; r < 2; r++) pthread_create(&t[r], NULL, rank_main, (void *)r);
    int rc = 0;
    for (int r = 0; r < 2; r++) { void *x; pthread_join(t[r], &x); rc |= x != NULL; }
    return rc;
}
"""


def test_c_shim_driven_from_c(stub_libs):
    src = os.path.join(BUILD, "ranks_allreduce_driver.c")
    exe = os.path.join(BUILD, "ranks_allreduce_driver")
    with open(src, "w") as f:
        f.write(C_DRIVER)
    host = stub_libs[1]
    subprocess.run(["gcc", "-std=gnu11", "-O1", src, "-o", exe, host, "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    words = (2 * WIN100 - 1) + 1
    for r in range(2):
        assert "rank %d count 3 rate 11 status 0 summed 1 bytes %d" % (r, 8 * words) in res.stdout, res.stdout
