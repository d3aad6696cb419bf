"""Random sequences of ingest calls, tuning changes, graph replays and snapshots (tests/_op_sequences.py), each interval
checked exactly against the per-interval model: every bucket of every row, counts, percentile keys and values of every
touched histogram, sums and averages, counter deltas, the dropped tally, and reduce_sparse of the export against the
interval's reduction.  After every keyed, pair or counter call, keyed_kernel_name() is the route model's prediction.

State that lives across calls and intervals (touched flags, the uint32 hot window and its fold, the double-buffered
arrays, graph-recorder rows, the last keyed route, tuning) is exercised in orders no fixed test writes down; a count
that leaks into the next interval fails that interval.  On a count mismatch the interval is re-run alone in a fresh
engine with a snapshot after every op, and the first op whose effect is wrong is named.

LH_OP_SEQUENCE_SEEDS (comma-separated integers) adds seeds for a longer run; the default seeds stay fixed."""
import os

import numpy as np
import pytest

import _op_sequences as S
from _op_sequences import PS

pytestmark = pytest.mark.gpu

EXTRA = [int(x, 0) for x in os.environ.get("LH_OP_SEQUENCE_SEEDS", "").split(",") if x.strip()]
RUNS = S.RUNS + [(c, s) for c in S.CONFIGS for s in EXTRA]
GIB = 1 << 30


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


class View:
    """A device view (address, length, numpy dtype) with __cuda_array_interface__, for batch items and graph calls."""

    def __init__(self, ptr, n, dtype):
        self.ptr, self.n, self.dtype = ptr, n, np.dtype(dtype)

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.n,), "typestr": self.dtype.str, "data": (self.ptr, False), "version": 3}


class Runner:
    """Issues ops on one engine: the pools uploaded once, three torch streams, live graph recorders by id."""

    def __init__(self, lh, torch, e, pools, cfg):
        self.lh, self.torch, self.e, self.pools, self.cfg = lh, torch, e, pools, cfg
        self.dev = {name: e.upload(a) for name, a in pools.arrays().items()}
        torch.cuda.synchronize()
        self.streams = [None] + [torch.cuda.Stream() for _ in range(3)]
        self.graphs = {}
        self.kernel = ""

    def at(self, pool, off):
        d = self.dev[pool]
        return d.ptr + off * d.dtype.itemsize

    def view(self, pool, off, n):
        return View(self.at(pool, off), n, self.dev[pool].dtype)

    def close(self):
        for gr, g in self.graphs.values():
            gr.close()
        self.graphs.clear()
        self.e.sync()
        self.torch.cuda.synchronize()
        for d in self.dev.values():
            d.free()

    def tune(self, t):
        for k, v in t.items():
            self.e.tune(k, v)

    def issue(self, op):
        """Issue one op; returns True when it ran a keyed, pair or counter ingest call (its kernel name is checked)."""
        e, o, st, p = self.e, op["op"], self.streams[op["stream"]], self.pools
        if o == "k1":
            e.tune("k1", op["variant"])
            e.ingest_f64(op["hid"], self.at("vals", op["voff"]), op["n"], st)
        elif o == "keyed":
            self.tune(op["tune"])
            ip, vp = S.KINDS[op["form"]]
            fn = {"f64_u16": e.ingest_keyed_f64_u16, "f64_u32": e.ingest_keyed_f64_u32, "i64ns_u16": e.ingest_keyed_i64ns_u16}
            fn[op["form"]](self.at(ip, op["ioff"]), self.at(vp, op["voff"]), op["n"], st)
            return True
        elif o == "pair":
            self.tune(op["tune"])
            e.ingest_keyed_pair_u16(self.at("ids16", op["iof"]), self.at("vals", op["vof"]), op["nf"],
                                    self.at("ids16", op["ion"]), self.at("ns", op["von"]), op["nn"], st)
            return True
        elif o == "batch":
            e.ingest_batch([(h, self.view(vk, off, n)) for h, vk, off, n in op["items"]], st)
        elif o == "counter":
            ip = "cids16" if op["width"] == 2 else "cids32"
            (e.counter_add_u16 if op["width"] == 2 else e.counter_add_u32)(self.at(ip, op["ioff"]),
                                                                          self.at("amounts", op["aoff"]), op["n"], st)
            return True
        elif o == "mapped":
            self.tune(op["tune"])
            ip = "ids16" if op["width"] == 2 else "ids32"
            kind = self.lh._lib.LH_VALUES_F64 if op["vkind"] == "vals" else self.lh._lib.LH_VALUES_I64NS
            (e.ingest_keyed_mapped_u16 if op["width"] == 2 else e.ingest_keyed_mapped_u32)(
                op["map"], self.at(ip, op["ioff"]), self.at(op["vkind"], op["voff"]), kind, op["n"], st)
            return True
        elif o == "counter_mapped":
            ip = "cids16" if op["width"] == 2 else "cids32"
            (e.counter_add_mapped_u16 if op["width"] == 2 else e.counter_add_mapped_u32)(
                op["map"], self.at(ip, op["ioff"]), self.at("amounts", op["aoff"]), op["n"], st)
            return True
        elif o == "host":
            self.tune(op["tune"])
            f, n, i, v = op["form"], op["n"], op["ioff"], op["voff"]
            if f == "f64":
                e.ingest_f64_host(op["hid"], p.vals[v:v + n])
            elif f == "keyed_f64":
                e.ingest_keyed_f64_u16_host(p.ids16[i:i + n], p.vals[v:v + n])
            elif f == "keyed_ns":
                e.ingest_keyed_i64ns_u16_host(p.ids16[i:i + n], p.ns[v:v + n])
            else:
                e.counter_add_u16_host(p.cids16[i:i + n], p.amounts[v:v + n])
            return f != "f64"
        elif o == "staging":
            self.tune(op["tune"])
            f, n, i, v, io = op["form"], op["n"], op["ioff"], op["voff"], op["ids_offset"]
            s = e.staging_acquire()
            if f == "abandon":
                e.staging_abandon(s)
                return False
            if f == "counter":
                e.staging_view(s, np.uint64, n)[:] = p.amounts[v:v + n]
            else:
                e.staging_view(s, np.float64, n)[:] = p.vals[v:v + n]
            if f == "f64":
                e.staging_commit_f64(s, op["hid"], n)
                return False
            e.staging_view(s, np.uint16, n, io)[:] = (p.cids16 if f == "counter" else p.ids16)[i:i + n]
            (e.staging_commit_counter_u16 if f == "counter" else e.staging_commit_keyed_f64_u16)(s, n, io)
            return True
        elif o == "merge":
            e.merge_counts_host(op["ids"], op["keys"], op["counts"])
        elif o == "graph":
            self.replay(op, st)
        return False

    def replay(self, op, st):
        spec = op["graph"]
        if spec["gid"] not in self.graphs:
            torch = self.torch
            gr = self.e.graph_recorder(spec["hist"], spec["ctr"])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.Stream()):
                for c in spec["calls"]:
                    if c[0] == "ingest":
                        gr.ingest([(c[1], self.view(c[2], c[3], c[4]))])
                    elif c[0] == "keyed":
                        lp = "lids16" if c[1] == 2 else "lids32"
                        gr.keyed(self.view(lp, c[3], c[5]), self.view(c[2], c[4], c[5]))
                    else:
                        lp = "lids16" if c[1] == 2 else "lids32"
                        gr.counters(self.view(lp, c[2], c[4]), self.view("amounts", c[3], c[4]))
            torch.cuda.synchronize()
            self.graphs[spec["gid"]] = (gr, g)
        _, g = self.graphs[spec["gid"]]
        stream = st if st is not None else self.torch.cuda.current_stream()
        with self.torch.cuda.stream(stream):
            for _ in range(op["replays"]):
                g.replay()
        stream.synchronize()      # a replay belongs to the interval whose collection comes after it has run

    def snapshot(self, form, row):
        """The interval's (Reduced, Sparse or None, dense row `row` or None, counter deltas) through one of the three
        snapshot forms.  Without an export, the deltas are read from the frozen buffer (snapshot_device) after
        snapshot_copy_histogram has waited for the snapshot stream."""
        e = self.e
        if form == "plain":
            red, sp = e.snapshot(PS, export=True)
            return red, sp, None, sp.counter_deltas
        e.snapshot_begin()
        try:
            if form == "async":
                red = e.snapshot_result(e.snapshot_reduce_async(PS))
                sp = e.snapshot_export()
                return red, sp, None, sp.counter_deltas
            dense = e.snapshot_copy_histogram(row)
            deltas = np.zeros(self.cfg.C, np.uint64)
            e._check(e.lib.lh_memcpy_d2h(e.h, deltas.ctypes.data, e.snapshot_device().d_counters, deltas.nbytes))
            return e.snapshot_reduce(PS), None, dense, deltas
        finally:
            e.snapshot_end()


class ProcessMemory:
    """Device memory this process holds, as NVML reports it per process; None where NVML does not list this process
    (for instance from inside a PID namespace) or reports no figure for it."""

    def __init__(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.handles = [pynvml.nvmlDeviceGetHandleByIndex(i) for i in range(pynvml.nvmlDeviceGetCount())]
        except Exception:
            self.nv = None

    def used(self):
        if self.nv is None:
            return None
        total, seen = 0, False
        for h in self.handles:
            for p in self.nv.nvmlDeviceGetComputeRunningProcesses(h):
                if p.pid == os.getpid() and p.usedGpuMemory is not None:
                    total += p.usedGpuMemory
                    seen = True
        return total if seen else None


def check_interval(e, want, red, sp, dense, deltas, row, dropped_before, what):
    if sp is not None:
        S.check(e, want, what, dropped_before, snap=(red, sp), every=True)
        back = e.reduce_sparse(sp, PS)
        for f in ("counts", "sums", "avgs", "pvals"):
            assert (getattr(back, f).view(np.uint64) == getattr(red, f).view(np.uint64)).all(), (what, "reduce_sparse", f)
        assert (back.pkeys == red.pkeys).all(), (what, "reduce_sparse", "pkeys")
    else:
        assert (dense == want.dense(row)).all(), (what, "row", row, np.flatnonzero(dense != want.dense(row))[:5])
        S.check_reduced(red, want, what, every=True)
        assert (deltas == want.counters).all(), (what, "counters", np.nonzero(deltas != want.counters)[0][:5])
        assert e.stats()["dropped"] - dropped_before == want.dropped, (what, "dropped")


def describe(seed, cfg, i, interval):
    return "seed %#x %r interval %d (%s snapshot)\n  " % (seed, cfg, i, interval["snapshot"]) + \
        "\n  ".join(S.compact(op) for op in interval["ops"])


def localise(lh, torch, oracle, cfg, pools, interval):
    """The interval alone in a fresh engine, one snapshot after each op: the first op whose effect is wrong, or None."""
    with lh.Engine(device=0, max_histograms=cfg.H, max_counters=cfg.C, precision=cfg.precision,
                   staging_bytes=S.STAGING_BYTES) as e:
        run = Runner(lh, torch, e, pools, cfg)
        try:
            for j, op in enumerate(interval["ops"]):
                want = S.Want(oracle, cfg.H, cfg.C, cfg.precision)
                S.apply(want, op, pools)
                before = e.stats()["dropped"]
                run.issue(op)
                try:
                    S.check(e, want, "op %d" % j, before)
                except AssertionError as ex:
                    return "op %d: %s: %s" % (j, S.compact(op), ex)
            return None
        finally:
            run.close()


def run_sequence(lh, torch, oracle, cfg, seed, intervals=None, pools=None):
    """Every interval of gen(seed, cfg) (or the given ones), checked.  Returns the most device memory this process held
    beyond what it held before (None when NVML gives no per-process figure), and the most the whole device's use grew
    by, which counts other processes on the device too; both sampled after every op and every snapshot."""
    if intervals is None:
        pools, intervals = S.gen(seed, cfg, oracle)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mem = ProcessMemory()
    torch.cuda.synchronize()
    base, free0 = mem.used(), torch.cuda.mem_get_info()[0]
    peak, device_peak = None, 0

    def sample():
        nonlocal peak, device_peak
        used = mem.used()
        if base is not None and used is not None:
            peak = max(peak or 0, used - base)
        device_peak = max(device_peak, free0 - torch.cuda.mem_get_info()[0])
    failure = None
    with lh.Engine(device=0, max_histograms=cfg.H, max_counters=cfg.C, precision=cfg.precision,
                   staging_bytes=S.STAGING_BYTES) as e:
        run = Runner(lh, torch, e, pools, cfg)
        try:
            for i, interval in enumerate(intervals):
                what = describe(seed, cfg, i, interval)
                want = S.interval_want(oracle, cfg, pools, interval)
                before = e.stats()["dropped"]
                for j, op in enumerate(interval["ops"]):
                    if run.issue(op):
                        run.kernel = S.expected_kernel(op, cfg, run.kernel, sms)
                        assert e.keyed_kernel_name() == run.kernel, (what, "op %d kernel" % j, e.keyed_kernel_name())
                    sample()
                red, sp, dense, deltas = run.snapshot(interval["snapshot"], interval["row"])
                sample()
                try:
                    check_interval(e, want, red, sp, dense, deltas, interval["row"], before, what)
                except AssertionError as ex:
                    failure = (i, interval, ex)
                    break
        finally:
            run.close()
    if failure is not None:
        i, interval, ex = failure
        where = localise(lh, torch, oracle, cfg, pools, interval)
        raise AssertionError("%s\n%s\nre-run alone: %s" % (describe(seed, cfg, i, interval), ex,
                                                          where or "every op right on its own"))
    return peak, device_peak


@pytest.mark.parametrize("config,seed", RUNS, ids=["p%d-H%d-C%d-%#x" % (c + (s,)) for c, s in RUNS])
def test_random_op_sequences(lh, oracle, torch, config, seed):
    cfg = S.Config(*config, sms=torch.cuda.get_device_properties(0).multi_processor_count)
    peak, device_peak = run_sequence(lh, torch, oracle, cfg, seed)
    print("device memory in use grew by at most %.2f GiB (the whole device)" % (device_peak / GIB))
    if peak is None:
        print("device memory of this process: not reported by NVML")
    else:
        print("peak device memory of this process: %.2f GiB" % (peak / GIB))
        assert peak <= 3 * GIB, peak
