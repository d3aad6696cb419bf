"""Random sequences of MetricSystem calls (tests/_ms_sequences.py) on an H100: host calls on three threads, record scopes
with device arrays, graph recorders captured with torch.cuda.graph and replayed 0-3 times, device and window raw
subscriptions, torch-tensor device gauges, and collections, each checked exactly against the model: the RawMetricSet,
the dropped delta, every scope's bindings, every processed metric (percentile keys and values bit for bit, sums within
the summation bound, averages bit for bit), every open board read with read(), every raw board's percentiles at the
label ps and one-ulp neighbours of crossings and its ranks at bucket thresholds against the window model, and the
gauges bit for bit.  Every stream the ops used is synchronised before each collection, so each interval is exact.

LH_MS_SEQUENCE_SEEDS (comma-separated integers) adds seeds for a longer run; the default seeds stay fixed.

Single changes to the library that these runs catch (first failing collection per run, default seeds):
  k_board_publish leaving `present` set on a row whose name is absent: 0x3a5 and 0x3a6 at (100, 12, 8), collections
    10 and 13, and 0x3a5 at (46, 24, 16), collection 17 (the (250, 64, 24) run does not catch it);
  k_raw_publish_window not removing the leaving interval when the row is unbound in the entering one: all four runs;
  k_graph_drain not clearing a drained cell: all four runs.
tests/test_ms_sequences_cpu.py covers recycle() freeing a retiring id a collection early."""
import numpy as np
import pytest

import _ms_sequences as S
from test_gpu_op_sequences import GIB, ProcessMemory, View

pytestmark = pytest.mark.gpu

TORCH_DTYPES = {"float64": "float64", "float32": "float32", "float16": "float16", "bfloat16": "bfloat16",
                "int64": "int64", "int32": "int32", "uint64": "uint64"}


class GpuBackend:
    """The pools uploaded once; graph recorders' calls captured once with torch.cuda.graph and replayed; boards read
    with DeviceSubscription.read; raw queries through RawDeviceSubscription; gauges are one-element tensors."""

    full_boards = True
    counter_drop = "amount"

    def __init__(self, torch, cfg, pools):
        import loghisto_b200.metric_system as m
        self.torch, self.pools = torch, pools
        self.ms = m.MetricSystem(1.0, False, max_histograms=cfg.H, max_counters=cfg.C, precision=cfg.precision)
        self.dev = {n: torch.from_numpy(a.view({2: np.int16, 4: np.int32, 8: np.int64}[a.dtype.itemsize])).cuda()
                    for n, a in pools.arrays().items()}
        self.dev_vals = torch.from_numpy(pools.vals).cuda()
        self.graphs, self.gauges, self.reads = {}, {}, {}
        self.capture_stream = torch.cuda.Stream()
        torch.cuda.synchronize()

    def stream(self):
        return None

    def graph_stream(self):
        return None

    def array(self, pool, off, n):
        d = self.dev[pool]
        return View(d.data_ptr() + off * d.element_size(), n, getattr(self.pools, pool).dtype)

    def scope_histogram(self, scope, name, off, n):
        scope.histogram(name, self.dev_vals[off:off + n])

    def new_graph(self, op, g):
        torch = self.torch
        cg = torch.cuda.CUDAGraph()
        spans = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for c in op["calls"] if c[0] == "timer"]
        torch.cuda.synchronize()
        with torch.cuda.graph(cg, stream=self.capture_stream):
            t = iter(spans)
            for c in op["calls"]:
                if c[0] == "timer":
                    g.start_timer(op["hnames"][c[1]])
                    g.stop_timer(op["hnames"][c[1]], out=next(t))
                elif c[0] == "histograms":
                    g.histograms([(op["hnames"][li], self.array(vk, off, n)) for li, vk, off, n in c[1]])
                elif c[0] == "keyed":
                    g.keyed(self.array("lids16" if c[1] == 2 else "lids32", c[3], c[5]), self.array(c[2], c[4], c[5]))
                else:
                    g.counters(self.array("clids16" if c[1] == 2 else "clids32", c[2], c[4]),
                               self.array("amounts", c[3], c[4]))
        self.graphs[op["gid"]] = (cg, spans)

    def replay(self, gid, times):
        """Each replay on its own, its spans read back before the next overwrites them."""
        cg, spans = self.graphs[gid]
        out = []
        for _ in range(times):
            cg.replay()
            self.torch.cuda.synchronize()
            out.append([int(d.item()) for d in spans])
        return out

    def gpu_timer(self, name):
        d = self.torch.full((1,), -1, dtype=self.torch.int64, device="cuda")
        self.ms.StartGpuTimer(name).Stop(out=d)
        self.torch.cuda.synchronize()
        return int(d.item())

    def drop_graph(self, gid):
        del self.graphs[gid]

    def board(self, sub):
        """read(), and a read captured into a CUDA graph when the subscription opened, replayed now: both images
        must be the same bytes."""
        torch = self.torch
        if id(sub) not in self.reads:
            buf = torch.zeros(sub.board.bytes, dtype=torch.uint8, device="cuda")
            cg = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(cg, stream=self.capture_stream):
                sub.read(out=buf)
            self.reads[id(sub)] = (sub, cg, buf)
        _, cg, buf = self.reads[id(sub)]
        v = sub.read()
        buf.zero_()
        cg.replay()
        torch.cuda.synchronize()
        image = v["image"].cpu().numpy().tobytes()
        if buf.cpu().numpy().tobytes() != image:
            raise S.Mismatch("the captured lh_board_read differs from read()")
        return S.parse_board(image, sub.board.k)

    def raw_query(self, sub, ps, values):
        torch = self.torch
        keys, vals, _ = sub.percentiles(torch.tensor(ps, dtype=torch.float64, device="cuda"))
        ranks, totals, _ = sub.ranks(torch.tensor(values, dtype=torch.float64, device="cuda"))
        torch.cuda.synchronize()
        return (keys.cpu().numpy(), vals.cpu().numpy(), ranks.cpu().numpy().view(np.uint64),
                totals.cpu().numpy().view(np.uint64))

    def _write(self, t, bits):
        t.view(self.torch.uint8).copy_(self.torch.tensor(list(bits), dtype=self.torch.uint8))

    def gauge(self, name, dtype, bits):
        t = self.torch.empty(1, dtype=getattr(self.torch, TORCH_DTYPES[dtype]), device="cuda")
        self._write(t, bits)
        self.torch.cuda.synchronize()
        self.ms.RegisterDeviceGauge(name, t)
        self.gauges[name] = t

    def write_gauge(self, name, bits):
        self._write(self.gauges[name], bits)

    def drop_gauge(self, name):
        self.gauges.pop(name, None)

    def sync(self):
        self.torch.cuda.synchronize()

    def close(self):
        self.torch.cuda.synchronize()
        self.graphs.clear()
        self.reads.clear()
        self.ms.close()


@pytest.mark.parametrize("cfg,seed", S.ALL_RUNS,
                         ids=["p%d-H%d-C%d-%#x" % (c.precision, c.H, c.C, s) for c, s in S.ALL_RUNS])
def test_random_metric_system_sequences(oracle, cfg, seed):
    import torch
    mem = ProcessMemory()
    torch.cuda.synchronize()
    base, free0 = mem.used(), torch.cuda.mem_get_info()[0]
    pools = S.Pools(oracle, cfg, seed)
    runner = S.Runner(oracle, cfg, seed, GpuBackend(torch, cfg, pools), pools=pools)
    try:
        runner.run(S.gen(seed, cfg))
        used, device = mem.used(), free0 - torch.cuda.mem_get_info()[0]
    finally:
        runner.close()
    print("device memory in use grew by %.3f GiB (the whole device)" % (device / GIB))
    if base is None or used is None:
        print("device memory of this process: not reported by NVML")
    else:
        print("device memory of this process grew by %.3f GiB" % ((used - base) / GIB))
