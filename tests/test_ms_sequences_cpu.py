"""Random sequences of MetricSystem calls (tests/_ms_sequences.py) on the CPU: the C++ mirror over the TEST-ONLY
oracle-backed stub of the C ABI with every feature the sequences use (record scopes, batches, mapped keyed and counter
calls, graph recorders, device and window raw boards, device gauges, GPU timers), each collection checked against the
model of the name tables and of what every op puts where.  Also: generation is deterministic and valid, the GPU runs
reach every op kind, drops, recycling under open subscriptions, recorder names bound late, long absences from raw
windows and every mapped keyed route, the model agrees with the oracle's own MetricSystem, and the checks fail on
every single perturbation.  tests/test_gpu_ms_sequences.py runs the same sequences on an H100.

recycle() (metric_system.cc) freeing a retiring id one collection early fails all four runs here (a scope binding
differs: seeds 0x3a5 and 0x3a6 at (100, 12, 8), collections 7 and 4; 0x3a5 at (46, 24, 16) and (250, 64, 24),
collection 2)."""
import ctypes
import copy
import math
import os
import subprocess

import numpy as np
import pytest

import _ingest_routes as R
import _ms_sequences as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
STUBS = ("lh_stub.c", "lh_stub_reduce_sparse.c", "lh_stub_record.c", "lh_stub_batch.c", "lh_stub_board.c",
         "lh_stub_raw_window.c", "lh_stub_gauges.c", "lh_stub_scope_keyed.c", "lh_stub_stream_timer.c")
GAUGE_CODE = dict(S.GAUGE_DTYPES)


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_ms_sequences.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_ms_sequences.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC] +
                   [os.path.join(ROOT, "tests", "stub_abi", f) for f in STUBS] +
                   [os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_ms_sequences", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    s = ctypes.CDLL(stub)
    s.lh_stub_gauge_alloc.restype = ctypes.c_void_p
    s.lh_stub_gauge_alloc.argtypes = [ctypes.c_size_t]
    s.lh_stub_gauge_free.argtypes = [ctypes.c_void_p]
    s.lh_stub_graph_set_clock.argtypes = [ctypes.c_uint64]
    return s, host


@pytest.fixture
def mslib(stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_libs[1])))
    return m


class HostArray:
    """A host numpy array posing as a device array (the stub reads host pointers)."""

    def __init__(self, a):
        self.a = a
        self.__cuda_array_interface__ = {"shape": (a.size,), "typestr": a.dtype.str, "data": (a.ctypes.data, False),
                                         "version": 3}


class CpuBackend:
    """Device arrays are views of the host pools, graph replays re-issue the recorder's calls, boards are read where
    the stub keeps them, raw queries go through the lhms_raw_subscription_* shim and gauges live in stub memory."""

    def __init__(self, m, stub, cfg, pools):
        self.m, self.stub, self.pools = m, stub, pools
        self.ms = m.MetricSystem(1e-6, False, max_histograms=cfg.H, max_counters=cfg.C, precision=cfg.precision)
        self.calls, self.cells = {}, {}
        self.full_boards = False                # the stub publishes counts, not reductions
        self.counter_drop = "ops"               # the stub drops an unbound recorder counter per op
        self.clock = 1000

    def stream(self):
        return None

    def graph_stream(self):
        return None

    def array(self, pool, off, n):
        return HostArray(getattr(self.pools, pool)[off:off + n])

    def scope_histogram(self, scope, name, off, n):
        a = self.pools.vals[off:off + n]      # RecordScope.histogram takes torch tensors only: its shim, directly
        assert self.ms._lib.lhms_record_ingest_f64(self.ms._h, ctypes.byref(scope.recorder), scope._hnames.index(name),
                                                   a.ctypes.data, n) == 0

    def new_graph(self, op, g):
        self.calls[op["gid"]] = (op, g)

    def replay(self, gid, times):
        op, g = self.calls[gid]
        out = []
        for _ in range(times):
            spans = []
            for c in op["calls"]:
                if c[0] == "timer":                      # the stub's device clock moves between start and stop
                    d = np.full(1, -1, np.int64)
                    self.stub.lh_stub_graph_set_clock(self.clock)
                    g.start_timer(op["hnames"][c[1]])
                    self.clock += 1 + (self.clock * 7919) % 999983
                    self.stub.lh_stub_graph_set_clock(self.clock)
                    g.stop_timer(op["hnames"][c[1]], out=HostArray(d))
                    spans.append(int(d[0]))
                elif c[0] == "histograms":
                    g.histograms([(op["hnames"][li], self.array(vk, off, n)) for li, vk, off, n in c[1]])
                elif c[0] == "keyed":
                    g.keyed(self.array("lids16" if c[1] == 2 else "lids32", c[3], c[5]), self.array(c[2], c[4], c[5]))
                else:
                    g.counters(self.array("clids16" if c[1] == 2 else "clids32", c[2], c[4]),
                               self.array("amounts", c[3], c[4]))
            out.append(spans)
        return out

    def gpu_timer(self, name):
        """StartGpuTimer, then Stop with its duration written to host memory (the stub's "device" memory; the
        Python Stop takes CUDA tensors only, so the shim directly)."""
        t = self.ms.StartGpuTimer(name)
        d = np.full(1, -1, np.int64)
        assert self.ms._lib.lhms_gpu_timer_stop(t._h, t._stream, d.ctypes.data) == 0
        t._free()
        return int(d[0])

    def drop_graph(self, gid):
        del self.calls[gid]

    def board(self, sub):
        b = sub.board
        return S.parse_board(bytes((ctypes.c_char * b.bytes).from_address(b.d_board)), b.k)

    def raw_query(self, sub, ps, values):
        k, L = sub.board.k, self.m._lib
        ps, values = np.ascontiguousarray(ps), np.ascontiguousarray(values)
        keys, vals, pub = np.zeros((k, ps.size), np.int32), np.zeros((k, ps.size)), np.zeros((k, ps.size), np.uint64)
        assert L.lhms_raw_subscription_percentiles(sub._h, ps.ctypes.data, ps.size, keys.ctypes.data, vals.ctypes.data,
                                                   pub.ctypes.data, None) == 0
        ranks, totals = np.zeros((k, values.size), np.uint64), np.zeros(k, np.uint64)
        rpub = np.zeros((k, values.size), np.uint64)
        assert L.lhms_raw_subscription_ranks(sub._h, values.ctypes.data, values.size, ranks.ctypes.data,
                                             totals.ctypes.data, rpub.ctypes.data, None) == 0
        return keys, vals, ranks, totals

    def gauge(self, name, dtype, bits):
        old = self.cells.pop(name, None)
        p = self.stub.lh_stub_gauge_alloc(8)
        ctypes.memmove(p, bits, len(bits))
        assert self.ms._lib.lhms_register_device_gauge(self.ms._h, name.encode(), p, GAUGE_CODE[dtype]) == 0
        self.cells[name] = p
        if old:
            self.stub.lh_stub_gauge_free(old)

    def write_gauge(self, name, bits):
        ctypes.memmove(self.cells[name], bits, len(bits))

    def drop_gauge(self, name):
        p = self.cells.pop(name, None)
        if p:
            self.stub.lh_stub_gauge_free(p)

    def sync(self):
        pass

    def close(self):
        self.ms.close()
        for p in self.cells.values():
            self.stub.lh_stub_gauge_free(p)
        self.cells.clear()


def cpu_cfg(cfg):
    """The configuration at precision 100, the only one the stub ingests at."""
    c = copy.copy(cfg)
    c.precision = 100
    return c


def run(oracle, m, stub, cfg, seed, check=True):
    """Every collection of the GPU run (cfg, seed), at precision 100."""
    ops = S.gen(seed, cfg)
    cfg = cpu_cfg(cfg)
    pools = S.Pools(oracle, cfg, seed)
    runner = S.Runner(oracle, cfg, seed, CpuBackend(m, stub, cfg, pools), pools=pools)
    try:
        return runner, runner.run(ops, check=check)
    finally:
        runner.close()


# ------------------------------------------------------------------------------------------------- generation
def _valid(op, cfg):
    o = op["op"]
    if o == "many":
        assert 0 <= op["off"] and op["off"] + op["n"] <= cfg.nv
    if o == "scope":
        assert op["hnames"] or not any(it[0] != "counters" for it in op["items"])
        for it in op["items"]:
            if it[0] == "histogram":
                assert it[1] < len(op["hnames"]) and it[2] + it[3] <= cfg.nv
            elif it[0] == "histograms":
                assert all(li < len(op["hnames"]) and off + n <= cfg.nv for li, _, off, n in it[1])
            elif it[0] == "keyed":
                assert it[1] in (2, 4) and it[3] + it[5] <= cfg.nl and it[4] + it[5] <= cfg.nv
            else:
                assert op["cnames"] and it[1] in (2, 4) and it[2] + it[4] <= 1 << 14 and it[3] + it[4] <= 1 << 14
    if o == "gopen":
        assert 1 <= len(op["hnames"]) <= cfg.H and len(op["cnames"]) <= cfg.C
    if o in ("sub", "raw"):
        assert len(op["hnames"]) <= cfg.H and (op["hnames"] or op.get("cnames"))
    if o == "raw":
        assert op["window"] in S.WINDOWS
    if o == "pct":
        assert len(op["labels"]) in (0, 3, 32) and all(lb.count("%s") == 1 for lb, _ in op["labels"])
    if "thread" in op:
        assert op["thread"] in (0, 1, 2)


def test_generation_is_deterministic_and_valid():
    for cfg, seed in S.ALL_RUNS:
        a, b = S.gen(seed, cfg), S.gen(seed, cfg)
        assert repr(a) == repr(b)          # repr: NaN labels compare unequal to themselves
        assert len(a) == cfg.collections
        for ops in a:
            for op in ops:
                _valid(op, cfg)
        assert repr(S.gen(seed + 1, cfg)) != repr(a)


def test_gpu_runs_reach_every_feature_and_route():
    """The GPU runs, by the generator and the route model: every op kind, the write-combining, vector and small keyed
    routes of mapped scope calls, K1 batch items, and pct label sets with p = 0, p = 1, p > 1 and NaN."""
    kinds, routes, k1, ps = set(), set(), 0, set()
    for cfg, seed in S.RUNS:
        for ops in S.gen(seed, cfg):
            for op in ops:
                kinds.add(op["op"])
                routes |= S.scope_routes(op, cfg)
                k1 += S.k1_items(op)
                for _, p in op.get("labels", ()):
                    ps.add("nan" if math.isnan(p) else "gt1" if p > 1 else p if p in (0.0, 1.0) else "mid")
                if op["op"] == "gauge":
                    kinds.add("gauge:" + op["dtype"])
                kinds |= {"graph:" + c[0] for c in op.get("calls", ())}
    assert kinds >= {"hist", "many", "counter", "timer", "gtimer", "pct", "scope", "gopen", "greplay", "gclose",
                     "sub", "subclose", "raw", "rawclose", "gauge", "gwrite", "gdel", "graph:timer", "graph:counters",
                     "graph:keyed", "graph:histograms"}
    assert {"gauge:" + d for d, _ in S.GAUGE_DTYPES} <= kinds
    assert {R.SMALL, R.VEC, R.WC} <= routes, routes
    assert k1 >= 1
    assert ps >= {0.0, 1.0, "nan", "gt1", "mid"}


# ------------------------------------------------------------------------------------------------- the runs
@pytest.fixture(scope="module")
def runs(oracle, stub_libs):
    """Every GPU run over the stub, each collection checked: {(cfg, seed): (the Mismatch or None, facts reached)}."""
    import loghisto_b200.metric_system as m
    saved = m._lib
    m._lib = m._bind(ctypes.CDLL(stub_libs[1]))
    out = {}
    try:
        for cfg, seed in S.RUNS:
            try:
                runner, _ = run(oracle, m, stub_libs[0], cfg, seed)
                out[(cfg, seed)] = (None, runner.seen)
            except S.Mismatch as e:
                out[(cfg, seed)] = (e, set())
    finally:
        m._lib = saved
    return out


@pytest.mark.parametrize("cfg,seed", S.RUNS, ids=["%d-%d-%d-%#x" % (c.precision, c.H, c.C, s) for c, s in S.RUNS])
def test_every_collection_equals_the_model(runs, cfg, seed):
    """The stub's collections equal the model's, collection by collection, through all of every run."""
    failure, _ = runs[(cfg, seed)]
    if failure is not None:
        raise failure


def test_runs_reach_every_state(runs):
    """Together the runs reach a drop, a recycled id under an open subscription, a recorder name unbound at a
    collection and bound at a later one, a recorder counter drained while unbound, a window row whose name is absent
    for longer than its window, and a window row whose name had no id in an interval of its window."""
    seen = set().union(*(facts for _, facts in runs.values()))
    assert {"drop", "recycled_under_subscription", "graph_unbound_then_bound", "recorder_counter_unbound",
            "window_absent_longer_than_w", "window_row_unbound"} <= seen, seen


def test_model_equals_the_oracle_system(oracle):
    """At precision 100 with no drops, the model's Histograms, Counters and Rates for Histogram, HistogramMany and
    Counter equal an accumulation through oracle.OracleMetricSystem."""
    cfg = S.Config(100, 64, 64, collections=12)
    pools = S.Pools(oracle, cfg, 5)
    model = S.Model(oracle, cfg, pools)
    ref = oracle.OracleMetricSystem()
    rng = np.random.default_rng(5)
    try:
        for j in range(cfg.collections):
            for _ in range(20):
                kind = rng.integers(0, 3)
                name = "h%d" % rng.integers(0, 6) if kind < 2 else "c%d" % rng.integers(0, 4)
                if kind == 0:
                    v = float(rng.choice(S.OS.SPECIALS)) if rng.random() < 0.3 else float(rng.normal(0, 1e3))
                    model.apply({"op": "hist", "name": name, "value": v})
                    ref.Histogram(name, v)
                elif kind == 1:
                    n = int(rng.integers(0, 300))
                    off = int(rng.integers(0, cfg.nv - n))
                    model.apply({"op": "many", "name": name, "off": off, "n": n, "vk": "vals"})
                    for v in pools.vals[off:off + n]:
                        ref.Histogram(name, float(v))
                else:
                    a = int(rng.choice(S.OS.AMOUNTS)) if rng.random() < 0.5 else int(rng.integers(0, 9))
                    model.apply({"op": "counter", "name": name, "amount": a})
                    ref.Counter(name, a)
            exp = model.collect()
            assert exp["want"].dropped == 0
            got, _ = ref.collect_and_process()
            for part in ("Histograms", "Counters", "Rates"):
                assert got[part] == exp["raw"][part], (j, part)
    finally:
        ref.close()


# ------------------------------------------------------------------------------------------------- the checks fail
@pytest.fixture(scope="module")
def recorded(oracle, stub_libs):
    """One short run's expectations and results, with what the boards and raw queries returned."""
    import loghisto_b200.metric_system as m
    saved = m._lib
    m._lib = m._bind(ctypes.CDLL(stub_libs[1]))
    try:
        ops = S.gen(S.SEEDS[0], S.CONFIGS[0])
        cfg = cpu_cfg(S.CONFIGS[0])
        pools = S.Pools(oracle, cfg, S.SEEDS[0])
        runner = S.Runner(oracle, cfg, S.SEEDS[0], CpuBackend(m, stub_libs[0], cfg, pools), pools=pools)
        boards, raws = [], []
        orig = runner.check

        def keep(j, ops, exp, raw, metrics, dropped, scope_ids, state):
            orig(j, ops, exp, raw, metrics, dropped, scope_ids, state)
            for sid, sub in runner.subs.items():
                boards.append((j, exp, metrics, runner.model.subs[sid], copy.deepcopy(runner.b.board(sub))))
            for rid, sub in runner.raws.items():
                ps, values = S.raw_queries(runner.model, rid, exp["labels"], cfg.precision)
                raws.append((j, rid, copy.deepcopy(runner.model.raws[rid]), [dict(h) for h in runner.model.raw_hist[rid]],
                             ps, values, runner.b.raw_query(sub, ps, values)))
        runner.check = keep
        try:
            history = runner.run(ops)
        finally:
            runner.close()
        return cfg, runner.model, history, boards, raws
    finally:
        m._lib = saved


def _fails(fn):
    with pytest.raises(S.Mismatch):
        fn()


def _pick(history, pred):
    for h in history:
        if pred(h):
            return h
    raise AssertionError("no collection fits")


def test_checks_fail_on_bucket_count_and_previous_collection(recorded):
    cfg, model, history, _, _ = recorded
    exp, raw, metrics, dropped, ids = _pick(history, lambda h: h[1]["Histograms"])
    S.check_collection(exp, raw, metrics, dropped, ids, "ok")
    for delta in (1, -1):
        bad = copy.deepcopy(raw)
        name = sorted(bad["Histograms"])[0]
        key = sorted(bad["Histograms"][name])[0]
        bad["Histograms"][name][key] += delta
        if bad["Histograms"][name][key] == 0:
            del bad["Histograms"][name][key]
        _fails(lambda: S.check_collection(exp, bad, metrics, dropped, ids, "+-1"))
    # a count moved to the previous collection: one sample of a name leaves this collection for the one before
    i = next(i for i in range(1, len(history)) if history[i][1]["Histograms"] and history[i - 1][1]["Histograms"])
    prev, cur = copy.deepcopy(history[i - 1][1]), copy.deepcopy(history[i][1])
    name = sorted(cur["Histograms"])[0]
    key = sorted(cur["Histograms"][name])[0]
    cur["Histograms"][name][key] -= 1
    prev["Histograms"].setdefault(name, {})
    prev["Histograms"][name][key] = prev["Histograms"][name].get(key, 0) + 1
    _fails(lambda: S.check_collection(history[i - 1][0], prev, history[i - 1][2], history[i - 1][3], history[i - 1][4], "prev"))
    _fails(lambda: S.check_collection(history[i][0], cur, history[i][2], history[i][3], history[i][4], "cur"))


def test_checks_fail_on_dropped_and_percentile_ulp(recorded):
    _, _, history, _, _ = recorded
    exp, raw, metrics, dropped, ids = _pick(history, lambda h: h[1]["Histograms"] and h[0]["labels"])
    for d in (1, -1):
        _fails(lambda: S.check_collection(exp, raw, metrics, dropped + d, ids, "dropped"))
    label, _ = exp["labels"][-1]
    name = sorted(exp["reduced"])[0]
    key = label.replace("%s", name, 1)
    if key in metrics:
        bad = dict(metrics)
        bad[key] = float(np.nextafter(bad[key], np.inf))
        _fails(lambda: S.check_collection(exp, raw, bad, dropped, ids, "ulp"))
    bad_ids = copy.deepcopy(ids)
    if bad_ids and bad_ids[0][0]:
        bad_ids[0][0][0] ^= 1
        _fails(lambda: S.check_collection(exp, raw, metrics, dropped, bad_ids, "ids"))


def test_checks_fail_on_a_row_bound_to_the_wrong_name(recorded):
    """A present row that shows another name's histogram of the collection, and an absent name's row left present."""
    _, _, _, boards, _ = recorded

    def other(b):
        exp, sub, rows = b[1], b[3], b[4][1]
        totals = {n: sum(h.values()) for n, h in exp["raw"]["Histograms"].items()}
        for i, n in enumerate(sub["hnames"]):
            if rows[i]["present"]:
                for m, t in totals.items():
                    if t != totals[n]:
                        return i, t
    j, exp, metrics, sub, image = next(b for b in boards if other(b))
    h, rows, crows = image
    S.check_board(exp, metrics, sub, image, "ok", full=False)
    i, t = other((j, exp, metrics, sub, image))
    bad = rows.copy()
    bad[i]["count"] = t
    _fails(lambda: S.check_board(exp, metrics, sub, (h, bad, crows), "wrong name", full=False))
    j, exp, metrics, sub, image = next(b for b in boards if any(n not in b[1]["raw"]["Histograms"] for n in b[3]["hnames"]))
    h, rows, crows = image
    i = next(i for i, n in enumerate(sub["hnames"]) if n not in exp["raw"]["Histograms"])
    bad = rows.copy()
    bad[i]["present"] = 1
    _fails(lambda: S.check_board(exp, metrics, sub, (h, bad, crows), "present left set", full=False))


def test_checks_fail_on_a_window_slot_not_aged_out(recorded, oracle):
    cfg, model, _, _, raws = recorded
    j, rid, sub, hist, ps, values, got = next(r for r in raws if len(r[3]) > r[2]["window"] and any(
        n in r[3][-r[2]["window"] - 1] for n in r[2]["hnames"]))
    m = S.Model(oracle, cfg, model.pools)
    m.raws[rid], m.raw_hist[rid] = sub, hist
    S.check_raw(m, rid, got, S.expected_raw(m, rid, ps, values, cfg.precision), "ok", ps)
    good = S.expected_raw(m, rid, ps, values, cfg.precision)
    m.raws[rid] = dict(sub, window=sub["window"] + 1)    # what a board that kept the leaving interval answers
    stale = S.expected_raw(m, rid, ps, values, cfg.precision)
    m.raws[rid] = sub
    _fails(lambda: S.check_raw(m, rid, stale, good, "not aged out", ps))


def test_checks_fail_on_a_gauge_ulp(recorded):
    cfg, model, history, _, _ = recorded
    exp, raw, metrics, dropped, ids = _pick(history, lambda h: any(math.isfinite(v) and v != 0 for v in h[1]["Gauges"].values()))
    name = next(n for n, v in raw["Gauges"].items() if math.isfinite(v) and v != 0)
    bad = copy.deepcopy(raw)
    bad["Gauges"][name] = float(np.nextafter(bad["Gauges"][name], 0.0))
    _fails(lambda: S.check_collection(exp, bad, metrics, dropped, ids, "gauge"))
