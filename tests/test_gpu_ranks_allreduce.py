"""Job-wide MetricSystem collections through the caller's all-reduce (join_ranks(..., allreduce)) and the kernels behind
them (lh_snapshot_row_levels / lh_snapshot_pack_rows / lh_snapshot_unpack_rows).

Ranks run as threads of this process (rank r on device r % device_count(), so one H100 runs every case), with an
in-process all-reduce: each rank copies its payload to the host on the snapshot stream, the threads sum the payloads as
uint64 with numpy, and each rank copies the sums back on that stream.  The scenarios of tests/test_gpu_ranks.py run
unchanged over this transport, and every collection must also equal, bit for bit, the same plan through peer-joined
systems.  Two processes on one card join through distributed.rank_allreduce over a gloo group.

Every case succeeds or fails on every rank alike: the failure cases fail the exchange, or the all-reduce before its
first barrier, on every rank."""
import random
import threading

import numpy as np
import pytest

import test_gpu_ranks as gr

pytestmark = pytest.mark.gpu

WIN = {100: 4368, 250: 10918}   # fast-window half-width per precision: a window row is 2 * win - 1 words


@pytest.fixture(scope="module")
def ndev():
    import torch
    n = torch.cuda.device_count()
    assert n >= 1
    return n


class DeviceReduce:
    """The element-wise uint64 all-reduce between rank threads; records each rank's n_words.  fail=True makes every
    rank's callback raise before it touches a buffer."""

    def __init__(self, world):
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)
        self.fail = False
        self.calls = [[] for _ in range(world)]

    def for_rank(self, r):
        import torch
        from loghisto_b200.distributed import _CudaView

        def allreduce(send, recv, n, stream):
            self.calls[r].append(n)
            if self.fail:
                raise RuntimeError("transport down")
            ts = torch.as_tensor(_CudaView(send, n))
            tr = torch.as_tensor(_CudaView(recv, n))
            s = torch.cuda.ExternalStream(stream, device=ts.device)
            s.synchronize()                                   # the pack ran
            self.slots[r] = ts.cpu().numpy().view(np.uint64)
            self.barrier.wait(timeout=120)
            total = np.zeros(n, np.uint64)
            for x in self.slots:
                total += x
            self.barrier.wait(timeout=120)
            with torch.cuda.stream(s):
                tr.copy_(torch.from_numpy(total.view(np.int64)).pin_memory(), non_blocking=True)
            s.synchronize()
        return allreduce


def joined_allreduce(world, ndev, precision, H=256, C=64):
    """test_gpu_ranks.joined_systems, joined through DeviceReduce."""
    from loghisto_b200.metric_system import MetricSystem
    ex, red = gr.Exchange(world), DeviceReduce(world)
    systems = [MetricSystem(3600.0, device=r % ndev, max_histograms=H, max_counters=C, precision=precision)
               for r in range(world)]
    for ms in systems:
        ms.SpecifyPercentiles(gr.PS)
    gr.on_ranks(world, lambda r: systems[r].join_ranks(r, world, ex.for_rank(r), red.for_rank(r)))
    ex.reduce = red
    return systems, ex


@pytest.fixture
def over_allreduce(monkeypatch):
    monkeypatch.setattr(gr, "joined_systems", joined_allreduce)


@pytest.mark.parametrize("precision", [100, 250])
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("n_names", [4, 40])
def test_collections_equal_one_system_seeing_every_sample(ndev, over_allreduce, precision, world, n_names):
    gr.test_joined_collections_equal_one_system_seeing_every_sample(ndev, precision, world, n_names)


def test_union_over_the_bound_drops_and_counts_as_the_peer_path(ndev, over_allreduce):
    gr.test_union_over_the_bound_keeps_the_first_names_and_counts_the_rest(ndev)


def test_failed_exchange_collects_alone_then_sums_again(ndev, over_allreduce):
    gr.test_failed_exchange_on_every_rank_collects_alone_then_sums_again(ndev)


def test_scopes_graphs_and_subscriptions_read_job_wide_rows(ndev, over_allreduce, oracle):
    gr.test_scopes_graphs_and_subscriptions_read_job_wide_rows(ndev, oracle)


@pytest.mark.parametrize("precision", [100, 250])
@pytest.mark.parametrize("world", [2, 4])
def test_bit_identical_to_the_peer_path(ndev, precision, world):
    """The same plan through allreduce-joined and peer-joined systems: raw Histograms, Rates, Counters and processed
    metrics agree exactly, collection by collection, and each payload has the size its levels
    give."""
    rng = random.Random(7 * world + precision)
    a, ex_a = joined_allreduce(world, ndev, precision)
    p, _ = gr.joined_systems(world, ndev, precision)
    try:
        for interval in range(4):
            plan, ctrs = gr.interval_plan(world, interval, 12, rng)
            gr.on_ranks(world, lambda r: (gr.feed(a[r], plan[r], ctrs[r]), gr.feed(p[r], plan[r], ctrs[r])))
            got_a = gr.on_ranks(world, lambda r: a[r].collect_and_process())
            got_p = gr.on_ranks(world, lambda r: p[r].collect_and_process())
            for r in range(world):
                raw_a, m_a = got_a[r]
                raw_p, m_p = got_p[r]
                for k in ("Histograms", "Rates", "Counters"):
                    assert raw_a[k] == raw_p[k], (interval, r, k)
                assert m_a == m_p, (interval, r)
                assert a[r].ranks_info()["status"] == 0
            sizes = {calls[-1] for calls in ex_a.reduce.calls}
            assert len(sizes) == 1
            assert a[0].ranks_info()["bytes_from_peers"] == 8 * sizes.pop()
    finally:
        for ms in a + p:
            ms.close()


def test_dense_rows_beyond_2_63_on_one_rank(ndev):
    """Rank 0 records values at and beyond 2^63 (dense row), rank 1 only window values under the same name: the agreed
    level is 3, and the collection equals one system that saw every sample."""
    world = 2
    systems, ex = joined_allreduce(world, ndev, 100, H=8, C=4)
    ref = gr.reference(100, 8, 4)
    try:
        big = [2.0 ** 63, 2.0 ** 63 * 1.5, 2.0 ** 64, 1e300]
        small = [1.0, 2.5, 1000.0]
        for v in big:
            systems[0].Histogram("d", v)
            ref.Histogram("d", v)
        for v in small:
            systems[1].Histogram("d", v)
            ref.Histogram("d", v)
            systems[1].Histogram("w", v)
            ref.Histogram("w", v)
        got = gr.on_ranks(world, lambda r: systems[r].collect_and_process())
        want_raw, want = ref.collect_and_process()
        for raw, metrics in got:
            assert raw["Histograms"] == want_raw["Histograms"]
            assert metrics == want
        assert ex.reduce.calls == [[65536 + 2 * WIN[100] - 1]] * world
    finally:
        for ms in systems:
            ms.close()
        ref.close()


def test_raising_allreduce_gives_own_counts_then_sums_again(ndev):
    world = 3
    systems, ex = joined_allreduce(world, ndev, 100, H=16, C=8)
    try:
        for r in range(world):
            systems[r].Histogram("h", float(r + 1))
            systems[r].Histogram("r%d" % r, 1.0)
            systems[r].Counter("c", r + 1)
        ex.reduce.fail = True
        got = gr.on_ranks(world, lambda r: systems[r].collect_and_process())
        for r, (raw, _) in enumerate(got):
            assert {k: sum(v.values()) for k, v in raw["Histograms"].items()} == {"h": 1, "r%d" % r: 1}
            assert raw["Rates"] == {"c": r + 1}
            assert systems[r].ranks_info()["status"] == 4
        ex.reduce.fail = False
        for r in range(world):
            systems[r].Histogram("h", float(r + 1))
            systems[r].Counter("c", 1)
        got = gr.on_ranks(world, lambda r: systems[r].collect_and_process())
        for raw, _ in got:
            assert {k: sum(v.values()) for k, v in raw["Histograms"].items()} == {"h": world}
            assert raw["Rates"] == {"c": world}
        assert all(ms.ranks_info()["status"] == 0 and ms.ranks_info()["summed"] == 1 for ms in systems)
    finally:
        for ms in systems:
            ms.close()


# ---- the ABI through Engine ------------------------------------------------------------------------------------------
def _payload(send, n):
    import torch
    from loghisto_b200.distributed import _CudaView
    torch.cuda.synchronize()
    return torch.as_tensor(_CudaView(send, n)).cpu().numpy().view(np.uint64).copy()


def _shares(rng, H, C):
    ids = rng.integers(0, H, 3000).astype(np.uint32)
    keys = rng.integers(-4000, 4000, 3000).astype(np.int16)
    keys[:20] = rng.integers(-32768, 32767, 20)          # out of the window: dense rows
    counts = rng.integers(1, 1 << 40, 3000).astype(np.uint64)
    cids = rng.integers(0, C, 50).astype(np.uint16)
    amts = rng.integers(0, 1 << 50, 50).astype(np.uint64)
    return ids, keys, counts, cids, amts


def _feed(e, share):
    ids, keys, counts, cids, amts = share
    e.merge_counts_host(ids, keys, counts)
    e.counter_add_u16_host(cids, amts)
    e.sync()


def _layout_cells(level, win):
    if level == 0:
        return np.zeros(0, np.int64)
    if level == 3:
        return np.arange(65536)
    return np.concatenate([np.arange(win), np.arange(65536 - (win - 1), 65536)])


def test_pack_layout_and_unpack_of_a_host_sum_equal_one_context(ndev):
    """The packed send buffer equals the frozen cells (lh_snapshot_copy_histogram) in the stated layout; unpack(1) of
    a host-computed sum of two contexts' payloads equals a single context that merged both; unpack(0) gives own
    counts; counts that wrap past 2^64 wrap as uint64."""
    import loghisto_b200 as lh
    H, C, win = 24, 8, WIN[100]
    rng = np.random.default_rng(5)
    engs = [lh.Engine(device=0, max_histograms=H, max_counters=C, precision=100) for _ in range(3)]
    try:
        shares = [_shares(rng, H, C), _shares(rng, H, C)]
        # one row whose sum wraps past 2^64 in a window cell and in a dense cell
        wrap_ids, wrap_keys = np.array([3, 3], np.uint32), np.array([5, -30000], np.int16)
        big = np.array([(1 << 63) + 7, (1 << 63) + 11], np.uint64)
        for e, share in zip(engs[:2], shares):
            _feed(e, share)
            e.merge_counts_host(wrap_ids, wrap_keys, big)
            e.sync()
        for share in shares:                                  # engs[2]: one context holding the merged counts
            _feed(engs[2], share)
            engs[2].merge_counts_host(wrap_ids, wrap_keys, big)
        engs[2].sync()
        for e in engs:
            e.snapshot_begin()
        lv = [engs[0].snapshot_row_levels(), engs[1].snapshot_row_levels()]
        agreed = np.maximum(lv[0], lv[1])
        rows = np.arange(H, dtype=np.uint32)
        crow = np.arange(C, dtype=np.uint32)
        pay = []
        for k, e in enumerate(engs[:2]):
            before = e.stats()
            send, recv, n, stream = e.snapshot_pack_rows(rows, agreed, crow)
            assert stream != 0 and send != 0 and recv != 0
            want_n = sum(_layout_cells(int(x), win).size for x in agreed) + C
            assert n == want_n
            p = _payload(send, n)
            at = 0
            for g in range(H):
                cells = _layout_cells(int(agreed[g]), win)
                if cells.size:
                    assert np.array_equal(p[at:at + cells.size], e.snapshot_copy_histogram(g)[cells]), (k, g)
                at += cells.size
            pay.append((e, send, recv, n, p))
            assert e.stats()["kernel_launches"] == before["kernel_launches"] + 1
        import torch
        from loghisto_b200.distributed import _CudaView
        total = pay[0][4] + pay[1][4]                         # uint64: wraps
        e0, _, recv0, n0, _ = pay[0]
        torch.as_tensor(_CudaView(recv0, n0)).copy_(torch.from_numpy(total.view(np.int64)))
        torch.cuda.synchronize()
        e0.snapshot_unpack_rows(True)
        e1 = pay[1][0]
        own = [e1.snapshot_copy_histogram(g) for g in range(H)]
        e1.snapshot_unpack_rows(False)
        ps = [0.5, 0.99]
        red0, sp0 = e0.snapshot_reduce(ps), e0.snapshot_export()
        red2, sp2 = engs[2].snapshot_reduce(ps), engs[2].snapshot_export()
        for f in ("counts", "sums", "avgs", "pkeys", "pvals"):
            assert np.array_equal(np.asarray(getattr(red0, f)).view(np.uint8), np.asarray(getattr(red2, f)).view(np.uint8)), f
        for f in ("offsets", "keys", "counts", "counter_deltas"):
            assert np.array_equal(np.asarray(getattr(sp0, f)), np.asarray(getattr(sp2, f))), f
        row3 = e0.snapshot_copy_histogram(3)
        assert agreed[3] == 3 and row3[5] < (1 << 63) and row3[35536] < (1 << 63)   # both sums wrapped past 2^64
        assert np.array_equal(row3, engs[2].snapshot_copy_histogram(3))
        # unpack(0): this context's own rows under the job-wide ones (every own cell lies in the agreed layout)
        for g in range(H):
            assert np.array_equal(e1.snapshot_copy_histogram(g), own[g]), g
        for e in engs:
            e.snapshot_end()
    finally:
        for e in engs:
            e.close()


def test_errors_before_any_launch(ndev):
    import loghisto_b200 as lh
    from loghisto_b200 import _lib as L
    from loghisto_b200.engine import LhError
    H, C = 4, 2
    e = lh.Engine(device=0, max_histograms=H, max_counters=C, precision=100)

    def status(fn):
        with pytest.raises(LhError) as x:
            fn()
        return x.value.status
    rows, lv, cr = np.arange(H, dtype=np.uint32), np.ones(H, np.uint8), np.arange(C, dtype=np.uint32)
    try:
        assert status(e.snapshot_row_levels) == L.LH_ERR_STATE                           # no snapshot
        assert status(lambda: e.snapshot_pack_rows(rows, lv, cr)) == L.LH_ERR_STATE
        assert status(lambda: e.snapshot_unpack_rows(True)) == L.LH_ERR_STATE
        e.merge_counts_host(np.array([1], np.uint32), np.array([3], np.int16), np.array([2], np.uint64))
        e.sync()
        e.snapshot_begin()
        assert status(lambda: e.snapshot_unpack_rows(True)) == L.LH_ERR_STATE            # no pack
        before = e.stats()
        assert status(lambda: e.snapshot_pack_rows(np.arange(H + 1, dtype=np.uint32), np.ones(H + 1, np.uint8), cr)) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_pack_rows(rows, lv, np.arange(C + 1, dtype=np.uint32))) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_pack_rows(rows, np.array([1, 2, 1, 1], np.uint8), cr)) == L.LH_ERR_INVALID
        assert status(lambda: e.snapshot_pack_rows(np.array([0, 1, 2, H], np.uint32), lv, cr)) == L.LH_ERR_RANGE
        assert status(lambda: e.snapshot_pack_rows(rows, lv, np.array([0, C], np.uint32))) == L.LH_ERR_RANGE
        C_ = __import__("ctypes")
        out = C_.c_void_p()
        n = C_.c_uint64()
        rc = e.lib.lh_snapshot_pack_rows(e.h, H, rows.ctypes.data, None, 0, None, C_.byref(out), C_.byref(out),
                                         C_.byref(n), C_.byref(out))
        assert rc == L.LH_ERR_INVALID                                                     # NULL levels with rows
        rc = e.lib.lh_snapshot_pack_rows(e.h, 0, None, None, 0, None, None, C_.byref(out), C_.byref(n), C_.byref(out))
        assert rc == L.LH_ERR_INVALID                                                     # NULL output pointer
        assert e.stats() == before                                                        # nothing launched or copied
        absent = np.full(H, L.LH_ROW_ABSENT, np.uint32)
        absent[1] = 1
        e.snapshot_pack_rows(absent, lv, cr)
        assert status(lambda: e.snapshot_pack_rows(rows, lv, cr)) == L.LH_ERR_STATE       # packed already
        e.snapshot_unpack_rows(False)
        assert status(lambda: e.snapshot_unpack_rows(False)) == L.LH_ERR_STATE            # unpacked already
        assert status(e.snapshot_row_levels) == L.LH_ERR_STATE
        assert e.snapshot_copy_histogram(1)[3] == 2 and e.snapshot_copy_histogram(0).sum() == 0
        e.snapshot_end()
        # a snapshot that packs without an unpack reads its own frozen arrays
        e.merge_counts_host(np.array([2], np.uint32), np.array([4], np.int16), np.array([9], np.uint64))
        e.sync()
        e.snapshot_begin()
        e.snapshot_pack_rows(np.zeros(1, np.uint32), np.ones(1, np.uint8), np.zeros(0, np.uint32))
        assert e.snapshot_copy_histogram(2)[4] == 9
        e.snapshot_end()
    finally:
        e.close()


# ---- processes -------------------------------------------------------------------------------------------------------
def _process_rank(rank, world, path, backend, out):
    import torch.distributed as dist
    from loghisto_b200.distributed import rank_allgather, rank_allreduce
    from loghisto_b200.metric_system import MetricSystem
    import torch
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method="file://" + path, rank=rank, world_size=world)
    try:
        gather = dist.new_group(backend="gloo")
        group = dist.new_group(backend=backend)
        ms = MetricSystem(3600.0, device=dev, max_histograms=8, max_counters=8)
        ms.join_ranks(rank, world, rank_allgather(gather), rank_allreduce(group))
        res = []
        for k in range(2):
            ms.Histogram("h.%d" % rank, 1.0)
            ms.Histogram("shared", float(rank + 1))
            ms.Histogram("big", 1e100 if rank == 0 else 3.0)
            ms.Counter("c", rank + 1 + k)
            raw, m = ms.collect_and_process()
            res.append(({n: sum(v.values()) for n, v in raw["Histograms"].items()}, raw["Rates"],
                        ms.ranks_info()["status"], m["shared_p99"] if "shared_p99" in m else None))
        out.put((rank, res))
        ms.close()
    except BaseException as e:
        out.put((rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def _run_processes(tmp_path, backend):
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    ps = [ctx.Process(target=_process_rank, args=(r, world, str(tmp_path / "store"), backend, out)) for r in range(world)]
    try:
        for p in ps:
            p.start()
        res = sorted(out.get(timeout=300) for _ in range(world))
    finally:
        for p in ps:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    assert [p.exitcode for p in ps] == [0] * world
    for rank, r in res:
        assert not isinstance(r, str), (rank, r)
        for k, (hists, rates, status, _) in enumerate(r):
            assert hists == {"h.0": 1, "h.1": 1, "shared": 2, "big": 2}, (rank, k)
            assert rates == {"c": 3 + 2 * k} and status == 0, (rank, k)
    assert res[0][1] == res[1][1]


def test_two_processes_on_one_card_through_a_gloo_group(ndev, tmp_path):
    _run_processes(tmp_path, "gloo")


def test_two_processes_through_an_nccl_group(ndev, tmp_path):
    if ndev < 2:
        pytest.skip("needs 2 GPUs: NCCL runs one rank per GPU")
    _run_processes(tmp_path, "nccl")
