"""Captured keyed samples, counter adds and GPU-timed spans of graph recorders (lh_graph_recorder_ingest_keyed_*,
lh_graph_recorder_counter_add_*, lh_graph_recorder_timer_*), recorded inside torch.cuda.graph captures and replayed.

Bar: every collection equal, bit for bit, to the oracle times the number of replays it received; dropped samples and
ops counted exactly once per replay; durations equal to the oracle's buckets of what the stops wrote; every refusal
returns its status with nothing enqueued."""
import numpy as np
import pytest

from test_gpu_device_record import PS, SEED, dense_all

pytestmark = pytest.mark.gpu

LH_ERR_INVALID, LH_ERR_RANGE = -1, -6
NS = [1, 7, 8, 9, (1 << 16) - 1, (1 << 16) + 1, 10 ** 6 + 3]
OFFSETS = [(0, 0), (1, 0), (0, 1)]          # start of (ids, values) in elements past an aligned allocation


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def capture(torch, fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        fn()
    return g


def collect(eng, H):
    _, sp = eng.snapshot(PS)
    eng.sync()
    return dense_all(sp, H), sp.counter_deltas.copy(), eng.stats()["dropped"]


def dev_at(torch, a, off):
    """`a` on the device, starting `off` elements past the start of its allocation."""
    t = torch.empty(a.size + off, dtype=getattr(torch, a.dtype.name), device="cuda")
    t[off:] = torch.from_numpy(a).cuda()
    return t[off:]


def sample_values(rng, n, kind):
    if kind == "f64":
        v = rng.lognormal(0.0, 6.0, n) * rng.choice([-1.0, 1.0], n)
        special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.8e308, 5e-324, 1.0])
        v[: min(n, special.size)] = special[: min(n, special.size)]
        return v
    v = rng.integers(-(1 << 40), 1 << 62, n, dtype=np.int64)
    v[: min(n, 3)] = np.array([0, -1, (1 << 63) - 1])[: min(n, 3)]
    return v


@pytest.mark.parametrize("precision", [100, 250])
@pytest.mark.parametrize("kind", ["f64", "i64"])
@pytest.mark.parametrize("id_dtype", [np.uint16, np.uint32])
def test_keyed_replays_equal_the_oracle(lh, oracle, torch, precision, kind, id_dtype):
    """Every n and alignment: captured once, replayed 1 then 2 times, one collection after each.  Each collection's
    rows == R x the oracle's keyed ingest (local i -> context id H - 1 - i); dropped grows by R x the ids >= k."""
    H, k = 8, 5
    hmap = [H - 1 - i for i in range(k)]
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=precision) as eng:
        for n in NS:
            for off_i, off_v in OFFSETS:
                rng = np.random.default_rng([SEED, precision, n, off_i, off_v, id_dtype(0).itemsize])
                ids = rng.integers(0, k + 3, n).astype(id_dtype)
                vals = sample_values(rng, n, kind)
                keep = ids < k
                keys = oracle.compress_many(vals.astype(np.float64), precision).view(np.uint16)
                want = np.zeros((H, 65536), dtype=np.uint64)
                np.add.at(want, (np.array(hmap)[ids[keep].astype(np.int64)], keys[keep]), 1)
                d_ids, d_vals = dev_at(torch, ids.view(np.int16 if id_dtype is np.uint16 else np.int32), off_i), dev_at(torch, vals, off_v)
                if id_dtype is np.uint16:
                    d_ids = d_ids.view(torch.uint16)
                with eng.graph_recorder(hmap) as gr:
                    g = capture(torch, lambda: gr.keyed(d_ids, d_vals))
                    torch.cuda.synchronize()
                    d0 = eng.stats()["dropped"]
                    for reps in (1, 2):
                        for _ in range(reps):
                            g.replay()
                        torch.cuda.synchronize()
                        got, _, d1 = collect(eng, H)
                        assert np.array_equal(got, want * np.uint64(reps)), (n, off_i, off_v, reps)
                        assert d1 - d0 == reps * int((~keep).sum()), (n, off_i, off_v, reps)
                        d0 = d1


@pytest.mark.parametrize("id_dtype", [np.uint16, np.uint32])
def test_counter_replays_wrap_and_drop(lh, torch, id_dtype):
    """Amounts that wrap 2^64 and ids >= kc: each collection's deltas == R x the sum mod 2^64, dropped += R x the ops
    with id >= kc."""
    C_, kc = 6, 3
    cmap = [C_ - 1 - i for i in range(kc)]
    with lh.Engine(device=0, max_histograms=1, max_counters=C_) as eng:
        for n in (1, 9, (1 << 16) + 1, 10 ** 6 + 3):
            for off_i, off_a in OFFSETS:
                rng = np.random.default_rng([SEED, n, off_i, off_a])
                ids = rng.integers(0, kc + 2, n).astype(id_dtype)
                amounts = rng.integers(0, 1 << 64, n, dtype=np.uint64)
                want = np.zeros(C_, dtype=np.uint64)
                keep = ids < kc
                np.add.at(want, np.array(cmap)[ids[keep].astype(np.int64)], amounts[keep])
                d_ids = dev_at(torch, ids.view(np.int16 if id_dtype is np.uint16 else np.int32), off_i)
                if id_dtype is np.uint16:
                    d_ids = d_ids.view(torch.uint16)
                d_amt = dev_at(torch, amounts.view(np.int64), off_a)
                with eng.graph_recorder([], cmap) as gr:
                    g = capture(torch, lambda: gr.counters(d_ids, d_amt))
                    torch.cuda.synchronize()
                    d0 = eng.stats()["dropped"]
                    for reps in (1, 2):
                        for _ in range(reps):
                            g.replay()
                        torch.cuda.synchronize()
                        _, ctr, d1 = collect(eng, 1)
                        with np.errstate(over="ignore"):
                            assert np.array_equal(ctr, want * np.uint64(reps)), (n, off_i, off_a, reps)
                        assert d1 - d0 == reps * int((~keep).sum())
                        d0 = d1


def test_counters_and_keyed_under_metric_system_names(lh, oracle, torch):
    """By name: counters land in Rates, name_rate and the cumulative Counters; keyed samples under the histogram of
    their local id; a negative int32 id is dropped and counted."""
    from loghisto_b200.metric_system import MetricSystem
    ms = MetricSystem(3600, max_histograms=8, max_counters=8)
    try:
        with ms.graph_recorder(histograms=["h0", "h1"], counters=["tokens", "experts"]) as g:
            ids = torch.tensor([0, 1, 1, 0, 1, 2, -1], dtype=torch.int32, device="cuda")
            amounts = torch.tensor([5, 7, 1, 2, 3, 100, 100], dtype=torch.int64, device="cuda")
            vals = torch.tensor([1.5, 2.5, 2.5, 1e9, 3.0, 4.0, 5.0], dtype=torch.float64, device="cuda")
            graph = capture(torch, lambda: (g.counters(ids, amounts), g.keyed(ids, vals)))
            total = 0
            for reps in (1, 3):
                for _ in range(reps):
                    graph.replay()
                torch.cuda.synchronize()
                raw, m = ms.collect_and_process()
                total += reps * 7
                assert raw["Rates"] == {"tokens": reps * 7, "experts": reps * 11}
                assert m["tokens_rate"] == reps * 7 and m["experts_rate"] == reps * 11
                assert raw["Counters"]["tokens"] == total
                c = oracle.compress
                assert raw["Histograms"] == {"h0": {c(1.5): reps, c(1e9): reps},
                                             "h1": {c(2.5): 2 * reps, c(3.0): reps}}
            assert ms.dropped() == 4 * 4         # 2 ops and 2 samples per replay, 4 replays
    finally:
        ms.close()


def sleep_cycles_ns(torch, cycles):
    """The least time `cycles` SM cycles take, in ns of %globaltimer: at the maximum SM clock (clock_rate, kHz), less
    1 %, since %globaltimer does not count SM cycles (on an H100 80GB HBM3 at 700 W a 2 M-cycle spin measured
    1.00496 ms of it, 0.5 % under 2 M cycles at 1 980 MHz)."""
    return 0.99 * cycles / (torch.cuda.get_device_properties(0).clock_rate * 1e3) * 1e9


def test_timer_spans_equal_the_oracle_of_their_durations(lh, oracle, torch):
    """start, torch.cuda._sleep(c), stop with out=: after each replay `out` holds the span, every span at least c
    cycles at the maximum SM clock, and each collection's row is the oracle's buckets of exactly those spans."""
    H, cycles = 4, 2_000_000
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        with eng.graph_recorder([2]) as gr:
            out = torch.zeros(1, dtype=torch.int64, device="cuda")

            def body():
                gr.start_timer(0)
                torch.cuda._sleep(cycles)
                gr.stop_timer(0, out=out)
            g = capture(torch, body)
            for reps in (1, 3):
                spans = []
                for _ in range(reps):
                    g.replay()
                    torch.cuda.synchronize()
                    spans.append(int(out.item()))
                got, _, _ = collect(eng, H)
                want = np.zeros(65536, dtype=np.uint64)
                np.add.at(want, oracle.compress_many(np.array(spans, dtype=np.float64)).view(np.uint16), 1)
                assert np.array_equal(got[2], want) and not got[[0, 1, 3]].any()
                assert min(spans) >= sleep_cycles_ns(torch, cycles), spans


def test_nested_and_cross_stream_spans(lh, oracle, torch):
    """Nested spans of two names (timer() around an inner span), and a span started on one stream and stopped on
    another that joins it inside the capture: each records exactly what its stop wrote."""
    H = 4
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        with eng.graph_recorder([0, 1, 3]) as gr:
            outs = torch.zeros(3, dtype=torch.int64, device="cuda")
            side = torch.cuda.Stream()

            def body():
                main = torch.cuda.current_stream()
                gr.start_timer(0)
                gr.start_timer(1)
                torch.cuda._sleep(500_000)
                gr.stop_timer(1, out=outs[1:2])
                torch.cuda._sleep(500_000)
                gr.stop_timer(0, out=outs[0:1])
                gr.start_timer(2)                               # on main ...
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    torch.cuda._sleep(500_000)
                    gr.stop_timer(2, out=outs[2:3])             # ... stopped on side, joined back below
                main.wait_stream(side)
            g = capture(torch, body)
            spans = []
            for _ in range(2):
                g.replay()
                torch.cuda.synchronize()
                spans.append(outs.cpu().numpy().copy())
            got, _, _ = collect(eng, H)
            spans = np.array(spans)
            assert (spans[:, 0] > spans[:, 1]).all() and (spans[:, 2] > 0).all()
            for local, row in ((0, 0), (1, 1), (2, 3)):
                want = np.zeros(65536, dtype=np.uint64)
                np.add.at(want, oracle.compress_many(spans[:, local].astype(np.float64)).view(np.uint16), 1)
                assert np.array_equal(got[row], want), local


def test_stop_without_start_drops_one_per_replay(lh, torch):
    with lh.Engine(device=0, max_histograms=2, max_counters=1) as eng:
        with eng.graph_recorder([0]) as gr:
            g = capture(torch, lambda: gr.stop_timer(0))
            torch.cuda.synchronize()
            d0 = eng.stats()["dropped"]
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize()
            got, _, d1 = collect(eng, 2)
            assert d1 - d0 == 3 and not got.any()


def test_histograms_and_keyed_in_one_graph_add_up(lh, oracle, torch):
    H = 3
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as eng:
        with eng.graph_recorder([1, 2]) as gr:
            a = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64, device="cuda")
            ids = torch.tensor([0, 1, 1], dtype=torch.int32, device="cuda")
            g = capture(torch, lambda: (gr.ingest([(0, a)]), gr.keyed(ids, a)))
            for _ in range(2):
                g.replay()
            torch.cuda.synchronize()
            got, _, _ = collect(eng, H)
            c = lambda v: oracle.compress(v) & 0xFFFF
            want = np.zeros((H, 65536), dtype=np.uint64)
            for v in (1.0, 2.0, 3.0, 1.0):
                want[1, c(v)] += 2
            for v in (2.0, 3.0):
                want[2, c(v)] += 2
            assert np.array_equal(got, want)


def test_refusals_enqueue_nothing(lh, torch):
    """Each failed check returns its status, with no launch and the recorder's rows untouched."""
    import ctypes as C
    from loghisto_b200 import _lib as L
    with lh.Engine(device=0, max_histograms=4, max_counters=2) as eng:
        gr = eng.graph_recorder([0, 1], [0])
        lib, h, g = eng.lib, eng.h, C.byref(gr.g)
        ids = torch.zeros(8, dtype=torch.int32, device="cuda")
        vals = torch.ones(8, dtype=torch.float64, device="cuda")
        amt = torch.ones(8, dtype=torch.int64, device="cuda")
        ip, vp, ap = ids.data_ptr(), vals.data_ptr(), amt.data_ptr()
        foreign = L.lh_graph_recorder()
        C.memmove(C.byref(foreign), C.byref(gr.g), C.sizeof(foreign))
        foreign.handle ^= 1
        torch.cuda.synchronize()
        launches = eng.stats()["kernel_launches"]
        cases = [
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u32(h, C.byref(foreign), ip, vp, 0, 8, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u32(h, g, ip, vp, 2, 8, None)),        # kind
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u32(h, g, None, vp, 0, 8, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u32(h, g, ip, None, 0, 8, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u32(h, g, ip + 2, vp, 0, 4, None)),    # ids alignment
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u16(h, g, ip + 1, vp, 0, 4, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_ingest_keyed_u16(h, g, ip, vp + 4, 0, 4, None)),    # values
            (0, lib.lh_graph_recorder_ingest_keyed_u16(h, g, ip, vp, 0, 0, None)),                     # n = 0
            (LH_ERR_INVALID, lib.lh_graph_recorder_counter_add_u32(h, C.byref(foreign), ip, ap, 8, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_counter_add_u16(h, g, None, ap, 8, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_counter_add_u16(h, g, ip, ap + 4, 4, None)),
            (0, lib.lh_graph_recorder_counter_add_u16(h, g, ip, ap, 0, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_timer_start(h, C.byref(foreign), 0, None)),
            (LH_ERR_RANGE, lib.lh_graph_recorder_timer_start(h, g, 2, None)),
            (LH_ERR_RANGE, lib.lh_graph_recorder_timer_stop(h, g, 2, None, None)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_timer_stop(h, g, 0, None, ap + 4)),
            (LH_ERR_INVALID, lib.lh_graph_recorder_timer_stop(h, C.byref(foreign), 0, None, None)),
        ]
        assert [st for _, st in cases] == [want for want, _ in cases]
        assert eng.stats()["kernel_launches"] == launches
        torch.cuda.synchronize()
        got, ctr, _ = collect(eng, 4)
        assert not got.any() and not ctr.any()
        gr.close()
        assert lib.lh_graph_recorder_ingest_keyed_u16(h, g, ip, vp, 0, 8, None) == LH_ERR_INVALID  # destroyed
        assert lib.lh_graph_recorder_timer_start(h, g, 0, None) == LH_ERR_INVALID
