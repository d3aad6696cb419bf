"""Graph recorders (lh_graph_recorder_*): recording from kernels captured into CUDA graphs and replayed, drained into the
interval of every collection.

The captured kernels live in tests/graph_record_client.cu, a separate CUDA library built by build() that knows the
engine only through its public headers.  Bar: every bucket equal to the oracle over exactly the replays each interval
received, nothing lost or counted twice while collections run beside replays, labels by name under MetricSystem, and
collections from another thread during a capture in torch's default (global) mode."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from test_gpu_device_record import PS, SEED, dense_all, edge_inputs

pytestmark = pytest.mark.gpu

PRECISIONS = [50, 100, 200]
UNBOUND = 0xFFFFFFFF
LH_ERR_INVALID, LH_ERR_RANGE = -1, -6
K1_MIN = 1 << 20            # kBatchK1Min in lh_api.cu: F64 items this long take the single-histogram kernel


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def client():
    from loghisto_b200 import _lib, build
    assert os.path.exists(build.GRAPH_CLIENT_LIB), "build() did not produce " + build.GRAPH_CLIENT_LIB
    lib = C.CDLL(build.GRAPH_CLIENT_LIB)
    rp, vp, sz, u32 = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t, C.c_uint32
    lib.grc_set_device.argtypes = [C.c_int]
    lib.grc_prepare.argtypes = [u32, u32]
    lib.grc_step.argtypes = [rp, vp, vp, sz, vp, vp, sz, vp, vp, sz, u32, u32, sz, vp]
    for name in ("grc_set_device", "grc_prepare", "grc_step"):
        getattr(lib, name).restype = C.c_int
    assert lib.grc_set_device(0) == 0
    assert lib.grc_prepare(100 * 1024, 4096) == 0   # BlockHistogram at precision 200 takes 68 KiB
    return lib


class Step:
    """The inputs of one client step (grc_step) on the device, and what one replay of it adds, by local id."""

    def __init__(self, lh, oracle, torch, k, kc, precision, seed, n=200_003, n_ns=50_001, n_c=30_001, entries=4096):
        rng = np.random.default_rng(seed)
        vals = np.concatenate([oracle.gen_stream(lh.STREAM_S, n, seed), edge_inputs(precision),
                               np.array([np.nan, np.inf, -np.inf, 2.0 ** 63, -(2.0 ** 63), 1.8e308, -1.8e308])])
        self.n = vals.size
        ids = rng.integers(0, k, self.n).astype(np.uint32)
        ids[::97] = k + 1                           # dropped and counted
        ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n_ns, seed ^ 1).view(np.int64).copy()
        ns[::3] *= -1
        ns_ids = rng.integers(0, k, n_ns).astype(np.uint32)
        cids = rng.integers(0, kc + 1, n_c).astype(np.uint32)     # id kc: dropped and counted
        amounts = rng.integers(0, 2 ** 40, n_c, dtype=np.uint64)
        self.bh_id, self.entries, self.k, self.kc = k - 1, entries, k, kc
        signed = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}
        dev = lambda a: torch.from_numpy(a.view(signed.get(a.dtype, a.dtype)).copy()).cuda()
        self.t = [dev(ids), dev(vals), dev(ns_ids), dev(ns), dev(cids), dev(amounts)]
        keep = ids < k
        want = np.zeros((k, 65536), dtype=np.uint64)
        keys = oracle.compress_many(vals, precision).view(np.uint16)
        np.add.at(want, (ids[keep], keys[keep]), 2)                     # lh::record and BlockRecorder
        np.add.at(want, (np.full(self.n, self.bh_id), keys), 1)         # BlockHistogram
        nkeys = oracle.compress_many(ns.astype(np.float64), precision).view(np.uint16)
        np.add.at(want, (ns_ids, nkeys), 1)
        self.want = want
        self.want_c = np.zeros(kc, dtype=np.uint64)
        np.add.at(self.want_c, cids[cids < kc], amounts[cids < kc])
        self.dropped = 2 * int((~keep).sum()) + int((cids >= kc).sum())

    def launch(self, client, rec, stream):
        ids, vals, ns_ids, ns, cids, amounts = (int(x.data_ptr()) for x in self.t)
        assert client.grc_step(C.byref(rec), ids, vals, self.n, ns_ids, ns, self.t[3].numel(), cids, amounts,
                               self.t[4].numel(), self.bh_id, self.entries, 8191, stream) == 0


def capture(torch, fn, stream=None):
    g = torch.cuda.CUDAGraph()
    s = stream or torch.cuda.Stream()
    with torch.cuda.graph(g, stream=s):
        fn(torch.cuda.current_stream().cuda_stream)
    return g


def interval(eng, H):
    red, sp = eng.snapshot(PS)
    eng.sync()
    return dense_all(sp, H), sp.counter_deltas.copy()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("entries", [0, 4096])
def test_replays_land_in_the_interval_they_ran_in(lh, oracle, torch, client, precision, entries):
    """Captured once, replayed 0, 1, 2 and 3 times between collections: each interval == the oracle over exactly the
    replays before it, under the ids the rows are bound to (local i -> H - 1 - i), counters included."""
    H, C_, k, kc = 9, 5, 6, 3
    step = Step(lh, oracle, torch, k, kc, precision, SEED ^ precision, entries=entries)
    hmap, cmap = [H - 1 - i for i in range(k)], [C_ - 1 - i for i in range(kc)]
    with lh.Engine(device=0, max_histograms=H, max_counters=C_, precision=precision) as eng:
        with eng.graph_recorder(hmap, cmap) as gr:
            g = capture(torch, lambda s: step.launch(client, gr.recorder, s))
            for reps in (0, 1, 2, 3):
                for _ in range(reps):
                    g.replay()
                torch.cuda.synchronize()
                got, ctr = interval(eng, H)
                for i in range(k):
                    assert (got[hmap[i]] == step.want[i] * np.uint64(reps)).all(), (precision, reps, i)
                for h in set(range(H)) - set(hmap):
                    assert not got[h].any()
                for i in range(kc):
                    assert int(ctr[cmap[i]]) == int(step.want_c[i]) * reps
            assert eng.stats()["dropped"] == 6 * step.dropped
            gr.close(stream=0)
        got, ctr = interval(eng, H)
        assert not got.any() and not ctr.any()


def test_concurrent_collections_lose_nothing(lh, oracle, torch, client):
    """Two graphs share one recorder and replay on two streams while another thread collects without pause: the sum
    over every interval plus the close's final drain == the oracle over every replay, counters included.  Replays go
    on, one round of 4 pairs queued behind the one running, until at least `reps` pairs have been replayed and the
    collector has finished `min_collections` collections since the first replay, however fast either side runs."""
    H, C_, k, kc, reps, min_collections = 6, 3, 6, 3, 40, 3
    a = Step(lh, oracle, torch, k, kc, 100, SEED ^ 11, n=100_003)
    b = Step(lh, oracle, torch, k, kc, 100, SEED ^ 12, n=60_001)
    with lh.Engine(device=0, max_histograms=H, max_counters=C_) as eng:
        total, total_c, n_iv = np.zeros((H, 65536), np.uint64), np.zeros(C_, np.uint64), [0]
        stop = threading.Event()
        errors = []

        def collector():
            try:
                while not stop.is_set():
                    got, ctr = interval(eng, H)
                    total[:] += got
                    total_c[:] += ctr
                    n_iv[0] += 1
            except BaseException as ex:   # pragma: no cover - reported below
                errors.append(ex)

        gr = eng.graph_recorder(list(range(k)), list(range(kc)))
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        g1 = capture(torch, lambda s: a.launch(client, gr.recorder, s), s1)
        g2 = capture(torch, lambda s: b.launch(client, gr.recorder, s), s2)
        th = threading.Thread(target=collector)
        th.start()
        pairs, first, prev = 0, n_iv[0], None
        while (pairs < reps or n_iv[0] - first < min_collections) and pairs < 100 * reps and not errors:
            for _ in range(4):
                with torch.cuda.stream(s1):
                    g1.replay()
                with torch.cuda.stream(s2):
                    g2.replay()
                pairs += 1
            ev = (torch.cuda.Event(), torch.cuda.Event())
            ev[0].record(s1)
            ev[1].record(s2)
            if prev is not None:          # keep one round queued: the collector runs while replays are in flight
                prev[0].synchronize()
                prev[1].synchronize()
            prev = ev
        torch.cuda.synchronize()
        stop.set()
        th.join()
        assert not errors, errors
        assert n_iv[0] - first >= min_collections, (n_iv[0] - first, pairs)
        gr.close(stream=0)
        got, ctr = interval(eng, H)
        total += got
        total_c += ctr
        assert (total == (a.want + b.want) * np.uint64(pairs)).all()
        assert (total_c == (a.want_c + b.want_c) * np.uint64(pairs)).all()
        assert eng.stats()["dropped"] == pairs * (a.dropped + b.dropped)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_captured_tensor_ingest(lh, oracle, torch, precision):
    """MetricSystem.graph_recorder(...).histograms captured in torch.cuda.graph: float64 and int64-ns items of 0, 1,
    kBatchK1Min - 1 and kBatchK1Min + 3 samples (both routes).  The static inputs are rewritten between replays; each
    interval == the oracle over the contents replayed into it."""
    from loghisto_b200.metric_system import MetricSystem
    lens = {"f0": 0, "f1": 1, "fm": K1_MIN - 1, "fk": K1_MIN + 3, "n1": 1, "nk": K1_MIN + 3}
    ms = MetricSystem(3600, max_histograms=8, max_counters=2, precision=precision)
    try:
        with ms.graph_recorder(histograms=list(lens)) as gr:
            bufs = {nm: torch.zeros(n, dtype=torch.int64 if nm[0] == "n" else torch.float64, device="cuda")
                    for nm, n in lens.items()}
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                gr.histograms(bufs)
            for rnd in range(3):
                contents = {}
                for j, (nm, n) in enumerate(lens.items()):
                    seed = SEED ^ (rnd << 8) ^ j
                    if nm[0] == "n":
                        v = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, seed).view(np.int64).copy()
                        v[::5] *= -1
                        contents[nm] = v.astype(np.float64)
                    else:
                        v = oracle.gen_stream(lh.STREAM_S, n, seed).copy()
                        contents[nm] = v
                    bufs[nm].copy_(torch.from_numpy(v))
                reps = rnd + 1
                for _ in range(reps):
                    g.replay()
                torch.cuda.synchronize()
                raw, _ = ms.collect_and_process()
                for nm, v in contents.items():
                    if v.size == 0:
                        assert nm not in raw["Histograms"]
                        continue
                    keys, cnt = np.unique(oracle.compress_many(v, precision), return_counts=True)
                    want = {int(kk): int(c) * reps for kk, c in zip(keys, cnt)}
                    assert raw["Histograms"][nm] == want, (precision, rnd, nm)
        assert ms.dropped() == 0
    finally:
        ms.close()


def test_names(lh, oracle, torch, client):
    """Two recorders share a name; other names churn through recycling while a recorder stays open and its name keeps
    labelling its counts; with a full table a new name is unbound and drops exactly its drained samples; close() drains
    leftovers into the next collection."""
    from loghisto_b200.metric_system import MetricSystem
    # two ids for the recorders' names, three for the host names of intervals k, k - 1 and k - 2: the ids of older ones
    # are recycled
    ms = MetricSystem(3600, max_histograms=5, max_counters=2)
    full = MetricSystem(3600, max_histograms=2, max_counters=2)
    try:
        x = torch.from_numpy(oracle.gen_stream(0, 10_001, SEED)).cuda()
        y = torch.from_numpy(oracle.gen_stream(1, 7_001, SEED)).cuda()

        def want_of(*arrs):
            v = np.concatenate([a.cpu().numpy() for a in arrs])
            keys, cnt = np.unique(oracle.compress_many(v), return_counts=True)
            return {int(kk): int(c) for kk, c in zip(keys, cnt)}
        with ms.graph_recorder(histograms=["shared", "mine"]) as g1, ms.graph_recorder(histograms=["shared"]) as g2:
            ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(ga):
                g1.histograms({"shared": x, "mine": y})
            with torch.cuda.graph(gb):
                g2.histograms({"shared": y})
            for it in range(8):                     # a new host name every interval: ids recycle around the recorders
                ms.Histogram("churn%d" % it, 5.0)
                ga.replay()
                gb.replay()
                torch.cuda.synchronize()
                raw, _ = ms.collect_and_process()
                assert raw["Histograms"]["shared"] == want_of(x, y), it
                assert raw["Histograms"]["mine"] == want_of(y), it
                assert raw["Histograms"]["churn%d" % it] == {oracle.compress(5.0): 1}, it
            ga.replay()
            torch.cuda.synchronize()
        raw, _ = ms.collect_and_process()           # the closes drained the last replay
        assert raw["Histograms"]["shared"] == want_of(x) and raw["Histograms"]["mine"] == want_of(y)
        assert ms.dropped() == 0
        for nm in ("a", "b"):                       # every id is held by a name used this interval
            full.Histogram(nm, 1.0)
        with full.graph_recorder(histograms=["late"]) as g3:
            gc = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gc):
                g3.histograms({"late": x})
            gc.replay()
            gc.replay()
            torch.cuda.synchronize()
            raw, _ = full.collect_and_process()
            assert set(raw["Histograms"]) == {"a", "b"}
            assert full.dropped() == 2 * x.numel()
        raw, _ = full.collect_and_process()
        assert raw["Histograms"] == {} and full.dropped() == 2 * x.numel()
    finally:
        ms.close()
        full.close()


def test_scope_and_graph_recorder_write_one_name(lh, oracle, torch):
    """A record scope and a graph recorder write the same name in one interval: the metrics equal the oracle port of
    metrics.go fed with every sample."""
    import importlib.util
    from loghisto_b200.metric_system import MetricSystem
    spec = importlib.util.spec_from_file_location("name_recycling_cases",
                                                  os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                               "_name_recycling_cases.py"))
    cases = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cases)
    ms = MetricSystem(3600, max_histograms=4, max_counters=2)
    ref = oracle.OracleMetricSystem()
    try:
        a = oracle.gen_stream(2, 3001, SEED ^ 5)
        b = oracle.gen_stream(1, 2003, SEED ^ 6)
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        torch.cuda.synchronize()
        with ms.graph_recorder(histograms=["x"]) as gr:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                gr.histograms({"x": tb})
            g.replay()
            with ms.recording(histograms=["x"]) as s:
                s.histograms({"x": ta})
            ms.Histogram("x", 12.5)
            torch.cuda.synchronize()
            raw, m = ms.collect_and_process()
        for v in np.concatenate([a, b, [12.5]]):
            ref.Histogram("x", float(v))
        rraw, rm = ref.collect_and_process()
        cases._compare_interval(raw, m, rraw, rm)
    finally:
        ms.close()
        ref.close()


def test_collection_from_another_thread_during_a_global_capture(lh, oracle, torch):
    """torch.cuda.graph captures in cudaStreamCaptureModeGlobal: a collection from another thread while it captures
    succeeds, the capture too, and the replay's samples arrive in the next collection."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(3600, max_histograms=4, max_counters=2)
    try:
        v = oracle.gen_stream(0, 5003, SEED ^ 7)
        t = torch.from_numpy(v).cuda()
        ms.Histogram("host", 3.0)
        out, errors = {}, []

        def collect():
            try:
                out["raw"], _ = ms.collect_and_process()
            except BaseException as ex:   # pragma: no cover - reported below
                errors.append(ex)
        with ms.graph_recorder(histograms=["g"]) as gr:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                gr.histograms({"g": t})
                th = threading.Thread(target=collect)
                th.start()
                th.join()
            assert not errors, errors
            assert out["raw"]["Histograms"] == {"host": {oracle.compress(3.0): 1}}
            g.replay()
            torch.cuda.synchronize()
            raw, _ = ms.collect_and_process()
        keys, cnt = np.unique(oracle.compress_many(v), return_counts=True)
        assert raw["Histograms"] == {"g": {int(kk): int(c) for kk, c in zip(keys, cnt)}}
    finally:
        ms.close()


def test_two_contexts_allreduce(lh, oracle, torch, client):
    """Two contexts on one GPU, each with a graph recorder: after lh_snapshot_allreduce every rank holds the sums a
    single context gets from both replays."""
    H, C_, k, kc = 6, 3, 6, 3
    steps = [Step(lh, oracle, torch, k, kc, 100, SEED ^ (21 + r), n=80_001) for r in range(2)]
    engs = [lh.Engine(device=0, max_histograms=H, max_counters=C_) for _ in range(2)]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, 2, handles)
        grs = [e.graph_recorder(list(range(k)), list(range(kc))) for e in engs]
        graphs = [capture(torch, lambda s, r=r: steps[r].launch(client, grs[r].recorder, s)) for r in range(2)]
        for g in graphs:
            g.replay()
        torch.cuda.synchronize()
        for e in engs:
            e.snapshot_begin()
            e.snapshot_allreduce(True)
        want = steps[0].want + steps[1].want
        want_c = steps[0].want_c + steps[1].want_c
        for e in engs:
            red = e.snapshot_reduce(PS)
            sp = e.snapshot_export()
            e.sync()
            got = dense_all(sp, H)
            assert (got[:k] == want).all()
            assert (sp.counter_deltas[:kc] == want_c).all()
            e.snapshot_end()
        for gr in grs:
            gr.close(stream=0)
    finally:
        for e in engs:
            e.close()


def test_validation(lh, torch, client):
    """Ids out of range at create / bind, destroyed and foreign handles, lh_record_end on a graph recorder, and an
    ingest refused by validation: each returns its status and enqueues nothing."""
    from loghisto_b200 import _lib as L
    with lh.Engine(device=0, max_histograms=4, max_counters=2) as eng, lh.Engine(device=0, max_histograms=4) as other:
        lib = eng.lib
        g = L.lh_graph_recorder()
        ids = lambda *x: (C.c_uint32 * len(x))(*x)
        assert lib.lh_graph_recorder_create(eng.h, 5, 0, None, None, C.byref(g)) == LH_ERR_RANGE
        assert lib.lh_graph_recorder_create(eng.h, 1, 3, None, None, C.byref(g)) == LH_ERR_RANGE
        assert lib.lh_graph_recorder_create(eng.h, 2, 0, ids(0, 4), None, C.byref(g)) == LH_ERR_RANGE
        assert lib.lh_graph_recorder_create(eng.h, 0, 0, None, None, C.byref(g)) == LH_ERR_INVALID
        gr = eng.graph_recorder([0, UNBOUND], [1])
        assert lib.lh_graph_recorder_bind(eng.h, C.byref(gr.g), ids(0, 7), None) == LH_ERR_RANGE
        assert lib.lh_graph_recorder_bind(eng.h, C.byref(gr.g), None, ids(2)) == LH_ERR_RANGE
        assert lib.lh_record_end(eng.h, C.byref(gr.recorder)) == LH_ERR_INVALID
        assert lib.lh_graph_recorder_bind(other.h, C.byref(gr.g), ids(0, 0), None) == LH_ERR_INVALID   # foreign
        x = torch.ones(100, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        launches = eng.stats()["kernel_launches"]
        bad = (L.lh_batch_item * 2)(L.lh_batch_item(x.data_ptr(), 100, 0, 0), L.lh_batch_item(x.data_ptr(), 100, 2, 0))
        assert lib.lh_graph_recorder_ingest(eng.h, C.byref(gr.g), bad, 2, 0) == LH_ERR_RANGE
        bad[1] = L.lh_batch_item(x.data_ptr(), 100, 1, 7)
        assert lib.lh_graph_recorder_ingest(eng.h, C.byref(gr.g), bad, 2, 0) == LH_ERR_INVALID
        assert eng.stats()["kernel_launches"] == launches
        gr.ingest([(0, x)], stream=0)
        eng.sync()
        red, sp = eng.snapshot(PS)
        assert int(red.counts[0]) == 100 and int(red.counts.sum()) == 100
        assert eng.stats()["samples"] == 0
        gr.close(stream=0)
        for call in (lambda: lib.lh_graph_recorder_bind(eng.h, C.byref(gr.g), None, None),
                     lambda: lib.lh_graph_recorder_ingest(eng.h, C.byref(gr.g), bad, 1, 0),
                     lambda: lib.lh_graph_recorder_destroy(eng.h, C.byref(gr.g), 0)):
            assert call() == LH_ERR_INVALID
