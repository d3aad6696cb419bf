"""Job-wide MetricSystem collections (MetricSystem.join_ranks) and the row-mapped peer all-reduce behind them
(lh_snapshot_rows / lh_snapshot_allreduce_rows).

World 2, 3 and 4 run as one thread per rank in this process, rank r on device r % device_count(), so one H100 runs
every case; the all-gather is a barrier between the threads.  Ranks intern their names in different orders, share some
names and keep others private, and churn them over several intervals, so the same name sits at different and recycled
ids on different ranks.  Every joined collection must equal, bucket for bucket, what one unjoined system reports after
seeing every rank's samples, and be identical on every rank.

No test needs K5's 10 s timeout: every rank reaches each collective, and the failure case fails the exchange on every
rank, which launches nothing."""
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PS = {"%s_p50": 0.5, "%s_p99": 0.99}


@pytest.fixture(scope="module")
def ndev():
    import torch
    n = torch.cuda.device_count()
    assert n >= 1
    return n


class Exchange:
    """An all-gather between rank threads.  fail=True makes every rank's callback raise before the barrier."""

    def __init__(self, world):
        self.world = world
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)
        self.fail = False

    def for_rank(self, r):
        def allgather(mine):
            if self.fail:
                raise RuntimeError("exchange down")
            self.slots[r] = bytes(mine)
            self.barrier.wait(timeout=120)
            out = list(self.slots)
            self.barrier.wait(timeout=120)
            return out
        return allgather


def on_ranks(world, fn):
    """fn(r) on one thread per rank; returns the results in rank order and raises the first error."""
    out, errs = [None] * world, []

    def run(r):
        try:
            out[r] = fn(r)
        except BaseException as e:   # pragma: no cover - reported below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]
    return out


def joined_systems(world, ndev, precision, H=256, C=64):
    from loghisto_b200.metric_system import MetricSystem
    ex = Exchange(world)
    systems = [MetricSystem(3600.0, device=r % ndev, max_histograms=H, max_counters=C, precision=precision)
               for r in range(world)]
    for ms in systems:
        ms.SpecifyPercentiles(PS)
    on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r)))
    return systems, ex


def interval_plan(world, interval, n_names, rng):
    """{rank: [(name, values)]} and {rank: {counter: amount}} for one interval: shared names on every rank, private
    names on one, names that come and go with the interval, each rank in its own order."""
    plan, ctrs = {}, {}
    shared = ["shared.%03d" % i for i in range(n_names)]
    for r in range(world):
        names = list(shared)
        names += ["rank%d.only.%d" % (r, i) for i in range(3)]
        names += ["churn.%d.%d" % (interval % 3, i) for i in range(2) if (i + r + interval) % 2 == 0]
        rng.shuffle(names)
        items = []
        for n in names:
            k = rng.randint(1, 40)
            vals = [rng.lognormvariate(3, 2) for _ in range(k)]
            if rng.random() < 0.2:
                vals.append(rng.choice([1e100, 1e-100, -1e90]))   # out of the window: dense rows
            items.append((n, vals))
        plan[r] = items
        ctrs[r] = {"c.shared": rng.randint(0, 9), "c.rank%d" % r: rng.randint(1, 9), "c.zero": 0,
                   "c.churn.%d" % (interval % 2): rng.randint(1, 5)}
    return plan, ctrs


def feed(ms, items, ctrs):
    for n, vals in items:
        for v in vals:
            ms.Histogram(n, v)
    for n, a in ctrs.items():
        ms.Counter(n, a)


def reference(precision, H, C):
    from loghisto_b200.metric_system import MetricSystem
    ref = MetricSystem(3600.0, device=0, max_histograms=H * 4, max_counters=C * 4, precision=precision)
    ref.SpecifyPercentiles(PS)
    return ref


@pytest.mark.parametrize("precision", [100, 250])
@pytest.mark.parametrize("world", [2, 3, 4])
# rows per collection: n_names + 3 * world + up to 2.  K5 takes the two-shot form from 16 rows at precision 100 and
# from 7 at precision 250, so world 2 and 3 at precision 100 with 4 names run one-shot and every other case two-shot.
@pytest.mark.parametrize("n_names", [4, 40])
def test_joined_collections_equal_one_system_seeing_every_sample(ndev, precision, world, n_names):
    rng = random.Random(1000 * world + n_names + precision)
    systems, ex = joined_systems(world, ndev, precision)
    ref = reference(precision, 256, 64)
    try:
        for interval in range(6):
            plan, ctrs = interval_plan(world, interval, n_names, rng)
            on_ranks(world, lambda r: feed(systems[r], plan[r], ctrs[r]))
            for r in range(world):
                feed(ref, plan[r], ctrs[r])
            got = on_ranks(world, lambda r: systems[r].collect_and_process())
            want_raw, want = ref.collect_and_process()
            for r, (raw, metrics) in enumerate(got):
                assert raw["Histograms"] == want_raw["Histograms"], (interval, r)
                assert raw["Rates"] == want_raw["Rates"], (interval, r)
                assert raw["Counters"] == want_raw["Counters"], (interval, r)
                assert "c.zero" in raw["Rates"]
                assert metrics == want, (interval, r)
                info = systems[r].ranks_info()
                assert info["status"] == 0 and info["world"] == world and info["rank"] == r
                assert info["summed"] == interval + 1
    finally:
        for ms in systems:
            ms.close()
        ref.close()


def test_union_over_the_bound_keeps_the_first_names_and_counts_the_rest(ndev):
    world, H = 2, 8
    systems, ex = joined_systems(world, ndev, 100, H=H, C=8)
    try:
        # rank 0: a0..a5, rank 1: b0..b5 -> union of 12, the first 8 in byte order kept (a0..a5, b0, b1)
        counts = {}
        for r, p in enumerate("ab"):
            for i in range(6):
                for k in range(i + 1):
                    systems[r].Histogram("%s%d" % (p, i), 10.0 + k)
                counts["%s%d" % (p, i)] = i + 1
        before = [ms.dropped() for ms in systems]
        got = on_ranks(world, lambda r: systems[r].collect_and_process())
        kept = sorted(counts)[:H]
        for raw, _ in got:
            assert sorted(raw["Histograms"]) == kept
            for n in kept:
                assert sum(raw["Histograms"][n].values()) == counts[n]
        dropped = [systems[r].dropped() - before[r] for r in range(world)]
        assert dropped == [0, sum(counts[n] for n in counts if n not in kept)]
        assert all(ms.ranks_info()["names_dropped"] == 4 for ms in systems)
    finally:
        for ms in systems:
            ms.close()


def test_failed_exchange_on_every_rank_collects_alone_then_sums_again(ndev):
    world = 3
    systems, ex = joined_systems(world, ndev, 100)
    try:
        for r in range(world):
            systems[r].Histogram("h", float(r + 1))
            systems[r].Counter("c", r + 1)
        ex.fail = True
        got = on_ranks(world, lambda r: systems[r].collect_and_process())
        for r, (raw, _) in enumerate(got):
            assert sum(raw["Histograms"]["h"].values()) == 1
            assert raw["Rates"] == {"c": r + 1}
            assert systems[r].ranks_info()["status"] == 3
        ex.fail = False
        for r in range(world):
            systems[r].Histogram("h", float(r + 1))
            systems[r].Counter("c", 1)
        got = on_ranks(world, lambda r: systems[r].collect_and_process())
        for r, (raw, _) in enumerate(got):
            assert sum(raw["Histograms"]["h"].values()) == world
            assert raw["Rates"] == {"c": world}
            assert systems[r].ranks_info()["status"] == 0
    finally:
        for ms in systems:
            ms.close()


@pytest.mark.parametrize("H", [4, 64])   # one-shot and two-shot at precision 100
def test_identity_maps_equal_the_identity_allreduce(ndev, H):
    """lh_snapshot_allreduce_rows with identity maps over H rows gives bit-identical results to lh_snapshot_allreduce
    on the same arrays."""
    import loghisto_b200 as lh
    world, C = 2, 16
    rng = np.random.default_rng(H)
    engs = [lh.Engine(device=r % ndev, max_histograms=H, max_counters=C, precision=100) for r in range(world)]
    try:
        handles = b"".join(e.comm_export() for e in engs)
        for r, e in enumerate(engs):
            e.comm_import(r, world, handles)
        shares = []
        for r in range(world):
            ids = rng.integers(0, H, 4000).astype(np.uint32)
            keys = rng.integers(-9000, 9000, 4000).astype(np.int16)
            keys[:50] = rng.integers(-32768, 32767, 50)
            counts = rng.integers(1, 1 << 40, 4000).astype(np.uint64)
            cids = rng.integers(0, C, 100).astype(np.uint16)
            amts = rng.integers(0, 1 << 50, 100).astype(np.uint64)
            shares.append((ids, keys, counts, cids, amts))
        results = []
        for mapped in (False, True):
            for r, e in enumerate(engs):
                ids, keys, counts, cids, amts = shares[r]
                e.merge_counts_host(ids, keys, counts)
                e.counter_add_u16_host(cids, amts)
                e.sync()
            for e in engs:
                e.snapshot_begin()
            if mapped:
                frozen = [e.snapshot_rows()[2] for e in engs]
                ident_h = np.tile(np.arange(H, dtype=np.uint32), (world, 1))
                ident_c = np.tile(np.arange(C, dtype=np.uint32), (world, 1))
                seq = max(e.comm_info()["allreduces"] for e in engs) + 1
                for e in engs:
                    assert e.snapshot_allreduce_rows(seq, frozen, ident_h, ident_c) == seq
            else:
                for e in engs:
                    e.snapshot_allreduce(True)
            per = []
            for e in engs:
                red = e.snapshot_reduce([0.5, 0.99])
                sp = e.snapshot_export()
                per.append((red, sp, e.comm_info()["status"]))
                e.snapshot_end()
            results.append(per)
        for (ra, sa, st_a), (rb, sb, st_b) in zip(*results):
            assert st_a == st_b == 0
            for f in ("counts", "sums", "avgs", "pkeys", "pvals"):
                assert np.array_equal(np.asarray(getattr(ra, f)).view(np.uint8), np.asarray(getattr(rb, f)).view(np.uint8)), f
            for f in ("offsets", "keys", "counts", "counter_deltas"):
                assert np.array_equal(np.asarray(getattr(sa, f)), np.asarray(getattr(sb, f))), f
    finally:
        for e in engs:
            e.close()


def capture(torch, fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        fn()
    return g


def test_scopes_graphs_and_subscriptions_read_job_wide_rows(ndev, oracle):
    """Rank 0 records through a record scope's keyed samples and counter adds, rank 1 through Histogram() and a graph
    recorder's replays, on streams U and L.  Rank 1's processed and raw device subscriptions must read the job-wide
    rows: every value equals what one unjoined system fed every sample reports."""
    import torch
    world = 2
    systems, ex = joined_systems(world, ndev, 100, H=16, C=8)
    ref = reference(100, 16, 8)
    dev0, dev1 = torch.device("cuda", 0), torch.device("cuda", 1 % ndev)
    labels = sorted(PS.items())
    hnames = ["lat", "tok", "r1only", "never"]
    try:
        with systems[1].raw_device_subscription(histograms=hnames) as rsub, \
                systems[1].device_subscription(histograms=hnames, counters=["steps"]) as psub, \
                systems[1].graph_recorder(histograms=["lat", "r1only"], counters=["steps"]) as g:
            gvals_np = np.array([1.5, 2.5e3, 7.0, 1e100, 0.25])
            with torch.cuda.device(dev1):
                gid = torch.tensor([0, 1, 0, 1, 0], dtype=torch.int32, device=dev1)
                gvals = torch.tensor(gvals_np, dtype=torch.float64, device=dev1)
                cid = torch.zeros(2, dtype=torch.int32, device=dev1)
                cam = torch.tensor([3, 4], dtype=torch.int64, device=dev1)
                graph = capture(torch, lambda: (g.keyed(gid, gvals), g.counters(cid, cam)))
            ps_t = torch.tensor([p for _, p in labels], dtype=torch.float64, device=dev1)
            for j in range(4):
                kind = (oracle.STREAM_U, oracle.STREAM_L)[j % 2]
                x = oracle.gen_stream(kind, 5000, 31 + j)
                ids = (np.arange(x.size) % 3 == 0).astype(np.int32)          # 1: "lat", 0: "tok"
                with torch.cuda.device(dev0):
                    t_ids, t_x = torch.tensor(ids, device=dev0), torch.tensor(x, device=dev0)
                    t_cid = torch.zeros(3, dtype=torch.int32, device=dev0)
                    t_am = torch.tensor([1, 2, j], dtype=torch.int64, device=dev0)
                    torch.cuda.synchronize(dev0)
                    with systems[0].recording(histograms=["tok", "lat"], counters=["steps"]) as s:
                        s.keyed(t_ids, t_x)
                        s.counters(t_cid, t_am)
                    torch.cuda.synchronize(dev0)
                ref.HistogramMany("tok", x[ids == 0])
                ref.HistogramMany("lat", x[ids == 1])
                ref.Counter("steps", 3 + j)
                y = oracle.gen_stream(kind, 700, 77 + j)
                systems[1].HistogramMany("lat", y)
                ref.HistogramMany("lat", y)
                with torch.cuda.device(dev1):
                    for _ in range(j + 1):
                        graph.replay()
                    torch.cuda.synchronize(dev1)
                for _ in range(j + 1):
                    ref.HistogramMany("lat", gvals_np[[0, 2, 4]])
                    ref.HistogramMany("r1only", gvals_np[[1, 3]])
                    ref.Counter("steps", 7)
                got = on_ranks(world, lambda r: systems[r].collect_and_process())
                want_raw, want = ref.collect_and_process()
                for r, (raw, metrics) in enumerate(got):
                    assert raw["Histograms"] == want_raw["Histograms"], (j, r)
                    assert raw["Rates"] == want_raw["Rates"] and raw["Counters"] == want_raw["Counters"], (j, r)
                    assert metrics == want, (j, r)
                with torch.cuda.device(dev1):
                    keys, vals, _ = rsub.percentiles(ps_t)
                    views = psub.read()
                    torch.cuda.synchronize(dev1)
                vals, counts = vals.cpu().numpy(), views["count"].cpu().numpy()
                rates = views["rate"].cpu().numpy()
                for i, nm in enumerate(hnames):
                    if nm not in want_raw["Histograms"]:
                        assert counts[i] == 0, (j, nm)
                        continue
                    assert counts[i] == want[nm + "_count"], (j, nm)
                    for c, (label, _) in enumerate(labels):
                        assert vals[i, c] == want[label % nm], (j, nm, label)
                assert rates[0] == want_raw["Rates"]["steps"]
    finally:
        for ms in systems:
            ms.close()
        ref.close()


def test_abi_validation_before_any_launch(ndev):
    """lh_snapshot_rows and lh_snapshot_allreduce_rows refuse bad calls with nothing launched, so no rank is left in a
    collective."""
    import loghisto_b200 as lh
    from loghisto_b200 import _lib as L
    from loghisto_b200.engine import LhError
    H, C, world = 4, 2, 2
    engs = [lh.Engine(device=r % ndev, max_histograms=H, max_counters=C, precision=100) for r in range(world)]
    hm = np.tile(np.arange(H, dtype=np.uint32), (world, 1))
    cm = np.tile(np.arange(C, dtype=np.uint32), (world, 1))

    def status(fn):
        with pytest.raises(LhError) as e:
            fn()
        return e.value.status
    try:
        e = engs[0]
        assert status(e.snapshot_rows) == L.LH_ERR_STATE                               # no snapshot
        e.snapshot_begin()
        fr = [e.snapshot_rows()[2]] * world
        assert status(lambda: e.snapshot_allreduce_rows(1, fr, hm, cm)) == L.LH_ERR_STATE   # no lh_comm_import
        e.snapshot_end()
        handles = b"".join(x.comm_export() for x in engs)
        for r, x in enumerate(engs):
            x.comm_import(r, world, handles)
        assert status(lambda: e.snapshot_allreduce_rows(1, [0, 0], hm, cm)) == L.LH_ERR_STATE   # no snapshot
        e.snapshot_begin()
        f = e.snapshot_rows()[2]
        fr = [f, f]
        assert status(lambda: e.snapshot_allreduce_rows(1, fr, np.zeros((world, H + 1), np.uint32), cm)) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_allreduce_rows(1, fr, hm, np.zeros((world, C + 1), np.uint32))) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_allreduce_rows(1, [f, 2], hm, cm)) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_allreduce_rows(1, [f ^ 1, f], hm, cm)) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_allreduce_rows(0, fr, hm, cm)) == L.LH_ERR_INVALID   # seq not above the last
        bad = hm.copy()
        bad[1, 3] = H
        assert status(lambda: e.snapshot_allreduce_rows(1, fr, bad, cm)) == L.LH_ERR_RANGE
        bad = cm.copy()
        bad[0, 0] = C
        assert status(lambda: e.snapshot_allreduce_rows(1, fr, hm, bad)) == L.LH_ERR_RANGE
        assert e.comm_info()["allreduces"] == 0                                          # nothing was launched
        e.snapshot_end()
    finally:
        for x in engs:
            x.close()


def _gloo_rank(rank, world, path, out):
    import torch.distributed as dist
    from loghisto_b200.distributed import rank_allgather
    from loghisto_b200.metric_system import MetricSystem
    dist.init_process_group("gloo", init_method="file://" + path, rank=rank, world_size=world)
    try:
        group = dist.new_group(backend="gloo")
        ms = MetricSystem(3600.0, device=rank, max_histograms=8, max_counters=8)
        ms.join_ranks(rank, world, rank_allgather(group))
        ms.Histogram("h.%d" % rank, 1.0)
        ms.Histogram("shared", float(rank + 1))
        ms.Counter("c", rank + 1)
        raw, _ = ms.collect_and_process()
        out.put((rank, {k: sum(v.values()) for k, v in raw["Histograms"].items()}, raw["Rates"], ms.ranks_info()["status"]))
        ms.close()
    finally:
        dist.destroy_process_group()


def test_processes_join_through_a_gloo_group(ndev, tmp_path):
    if ndev < 2:
        pytest.skip("needs 2 GPUs: one process per GPU")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    ps = [ctx.Process(target=_gloo_rank, args=(r, world, str(tmp_path / "store"), out)) for r in range(world)]
    for p in ps:
        p.start()
    res = sorted(out.get(timeout=300) for _ in range(world))
    for p in ps:
        p.join(timeout=60)
    for rank, hists, rates, status in res:
        assert hists == {"h.0": 1, "h.1": 1, "shared": 2} and rates == {"c": 3} and status == 0, rank
