"""Seeded random sequences of MetricSystem calls, and the exact model of every collection they are checked against.

`gen(seed, cfg)` returns a list of collections, each a list of ops the Python layer accepts: Histogram, HistogramMany,
Counter, StartTimer / Stop, SpecifyPercentiles, record scopes (histogram, histograms, keyed, counters), graph recorders
opened, replayed 0-3 times and closed, device and raw device subscriptions (windows 1, 2, 3, 5) opened and closed, and
device gauges registered, rewritten and deregistered.  Names come from a small pool per configuration: permanent names,
names that come back after 1, 2 and 5 idle collections, and bursts of fresh names that overflow the name table, so ids
are dropped, retired, freed and handed to other names while scopes, recorders and subscriptions hold or watch them.

`Model` restates the contracts of loghisto_b200/host/metric_system.h: the name table of each kind (NameTable: free,
live, retiring), what each op puts into the open interval under which name, what is dropped and counted, and, at each
collection, the RawMetricSet, the processed metrics, the board rows and window sums of the subscriptions and the
gauges.  `Runner` issues the ops on a backend (the oracle-backed stub on the CPU, the real library on an H100) and
checks every collection against the model.  Values, nanoseconds, specials and counter amounts come from _op_sequences.
"""
from __future__ import annotations

import concurrent.futures
import math
import os

import numpy as np

import _ingest_routes as R
import _op_sequences as OS
import _reduce_cases as rc

UNBOUND = 0xFFFFFFFF
INT32_MIN = -(1 << 31)
MAX_PERCENTILES = 32
BATCH_K1_MIN = OS.BATCH_K1_MIN
H100_SMS = 132
WC_MIN_PAIRS = 1 << 22
WINDOWS = (1, 2, 3, 5)
# the percentile labels a MetricSystem starts with (metric_system.cc, the constructor; metrics.go:145-155)
DEFAULT_LABELS = [("%s_min", 0.0), ("%s_50", .5), ("%s_75", .75), ("%s_90", .9), ("%s_95", .95), ("%s_99", .99),
                  ("%s_99.9", .999), ("%s_99.99", .9999), ("%s_max", 1.0)]
# (name, numpy dtype or "bfloat16", LH_GAUGE_*)
GAUGE_DTYPES = [("float64", 0), ("float32", 1), ("float16", 2), ("bfloat16", 3), ("int64", 4), ("int32", 5),
                ("uint64", 6)]
GAUGE_FLOATS = [float("nan"), float("inf"), float("-inf"), 5e-324, -5e-324, 1e-40, -0.0, 0.0, 2.5, -7.25, 6.1e-05,
                1e-45, 3.4e38, 65504.0, 1.7976931348623157e308]
GAUGE_INTS = {"int64": [-(1 << 63), (1 << 63) - 1, (1 << 53) + 1, -1, 0],
              "int32": [-(1 << 31), (1 << 31) - 1, -1, 0, 7],
              "uint64": [(1 << 64) - 1, 1 << 63, (1 << 53) + 1, 0, 3]}


class Config:
    """One configuration: the system's (precision, max_histograms, max_counters), collections, pool sizes, and whether
    it issues the few large calls (write-combining keyed scopes, K1 batch items)."""

    def __init__(self, precision, H, C, collections=40, large=False):
        self.precision, self.H, self.C, self.collections, self.large = precision, H, C, collections, large
        self.nv = (WC_MIN_PAIRS + (1 << 16)) if large else (1 << 17)
        self.nl = self.nv

    def __repr__(self):
        return "Config(precision=%d, H=%d, C=%d)" % (self.precision, self.H, self.C)


# (100, 12, 8): recycling and drops every few collections; (46, 24, 16): +-Inf buckets, so sums and averages are Inf
# or NaN; (250, 64, 24): dense raw rows, reductions off the window path, and room for a scope of more than 44 names
CONFIGS = [Config(100, 12, 8), Config(46, 24, 16), Config(250, 64, 24, large=True)]
SEEDS = (0x3A5, 0x3A6)
RUNS = [(CONFIGS[0], SEEDS[0]), (CONFIGS[0], SEEDS[1]), (CONFIGS[1], SEEDS[0]), (CONFIGS[2], SEEDS[0])]
EXTRA = [int(x, 0) for x in os.environ.get("LH_MS_SEQUENCE_SEEDS", "").split(",") if x.strip()]
ALL_RUNS = RUNS + [(c, s) for c in CONFIGS for s in EXTRA]


# ------------------------------------------------------------------------------------------------------------- pools
class Pools:
    """Host arrays every array op reads a view of, and the oracle's keys of the value pools."""

    def __init__(self, oracle, cfg: Config, seed: int):
        rng = np.random.default_rng([seed, cfg.precision, cfg.H, cfg.C, 7])
        self.vals = OS._values(oracle, rng, cfg.nv, cfg.precision, seed)
        self.ns = OS._nanos(oracle, rng, cfg.nv, seed + 11)
        lids = rng.integers(0, 72, cfg.nl).astype(np.uint32)      # local ids: scopes hold up to ~52 names
        lids[rng.integers(0, cfg.nl, cfg.nl // 97)] = 65535
        self.lids16, self.lids32 = lids.astype(np.uint16), lids
        clids = rng.integers(0, 8, 1 << 14).astype(np.uint32)
        self.clids16, self.clids32 = clids.astype(np.uint16), clids
        amounts = rng.integers(0, 2 ** 64, 1 << 14, dtype=np.uint64)
        amounts[::3] = OS.AMOUNTS[rng.integers(0, OS.AMOUNTS.size, amounts[::3].size)]
        amounts[1::5] = rng.integers(0, 1 << 20, amounts[1::5].size).astype(np.uint64)
        amounts[2::11] = 0
        self.amounts = amounts
        self.keys_vals = oracle.compress_many(self.vals, cfg.precision).view(np.uint16)
        self.keys_ns = oracle.compress_many(self.ns.astype(np.float64), cfg.precision).view(np.uint16)

    def arrays(self) -> dict:
        return {n: getattr(self, n) for n in POOLS}


POOLS = ("vals", "ns", "lids16", "lids32", "clids16", "clids32", "amounts")
POOL_LEN = {"vals": "nv", "ns": "nv", "lids16": "nl", "lids32": "nl"}


# --------------------------------------------------------------------------------------------------------- generator
class _Names:
    """The name pool of one run: permanent names, names that return after 1, 2 and 5 idle collections, bursts of fresh
    names, and names that are only ever subscribed to or bound by scopes."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.hperm = ["hp%d" % i for i in range(3)]
        self.cperm = ["cp%d" % i for i in range(2)]
        self.hgap = {g: ["hg%d_%d" % (g, i) for i in range(2)] for g in (1, 2, 5)}
        self.cgap = {g: ["cg%d_%d" % (g, i) for i in range(2)] for g in (1, 2, 5)}
        self.bursts = 0

    def hactive(self, j):
        return self.hperm + [n for g, ns in self.hgap.items() if j % (g + 1) == 0 for n in ns]

    def cactive(self, j):
        return self.cperm + [n for g, ns in self.cgap.items() if j % (g + 1) == 0 for n in ns]

    def burst(self, prefix, m):
        self.bursts += 1
        return ["%s%d_%d" % (prefix, self.bursts, i) for i in range(m)]

    def universe(self, j):
        return self.hperm + [n for ns in self.hgap.values() for n in ns] + ["hb%d_0" % max(1, self.bursts),
                                                                             "hnever%d" % (j % 3)]


def _size(rng, cap):
    """Log-uniform from 0 to cap."""
    return min(int(2.0 ** rng.uniform(0, math.log2(cap + 1))) - 1, cap)


def _view(rng, pool_len, n):
    off = int(rng.integers(0, 4))
    base = int(rng.integers(0, max(1, (pool_len - n - off) // 16 + 1))) * 16
    assert base + off + n <= pool_len
    return base + off


def _labels(rng):
    """0, 3 or 32 labels, sorted as the system keeps them; p = 0 and p = 1 among them, now and then p > 1 and NaN."""
    m = int(rng.choice([0, 3, 32]))
    ps = list(rng.uniform(0, 1, m))
    if m:
        ps[0] = 0.0
        ps[-1] = 1.0
    if m > 2:
        pick = rng.random()
        if pick < 0.3:
            ps[1] = 1.5
        elif pick < 0.5:
            ps[1] = float("nan")
        elif pick < 0.7:
            ps[1] = float(np.nextafter(0.5, 1.0))
    return [("%%s_q%02d" % i, float(p)) for i, p in enumerate(ps)]


def _gauge_value(rng, dtype):
    pool = GAUGE_INTS.get(dtype, GAUGE_FLOATS)
    return pool[int(rng.integers(0, len(pool)))]          # by index: rng.choice would round big ints to float


def _scope_items(rng, cfg, hnames, cnames, big):
    items = []
    if big == "wc":                                             # at least 2^22 pairs: the write-combining route
        n = int(rng.integers(WC_MIN_PAIRS, WC_MIN_PAIRS + (1 << 15)))
        w = int(rng.choice([2, 4]))
        a = lambda: _view(rng, cfg.nv, n) & ~3                  # 32-byte aligned: the vector body covers it all
        items.append(("keyed", w, str(rng.choice(["vals", "ns"])), a(), a(), n))
    elif big == "k1":                                           # a float64 item of 2^20 samples or more: K1
        n = int(rng.integers(BATCH_K1_MIN, BATCH_K1_MIN + (1 << 16)))
        items.append(("histograms", [(int(rng.integers(0, len(hnames))), "vals", _view(rng, cfg.nv, n), n)]))
    for _ in range(int(rng.integers(1, 4))):
        what = str(rng.choice(["histogram", "histograms", "keyed", "counters"] if cnames else
                              ["histogram", "histograms", "keyed"]))
        if what == "histogram":
            n = _size(rng, 4096)
            items.append(("histogram", int(rng.integers(0, len(hnames))), _view(rng, cfg.nv, n), n))
        elif what == "histograms":
            arrs = []
            for _ in range(int(rng.integers(1, 4))):
                vk = str(rng.choice(["vals", "ns"]))
                n = _size(rng, 1 << 14)
                arrs.append((int(rng.integers(0, len(hnames))), vk, _view(rng, cfg.nv, n), n))
            items.append(("histograms", arrs))
        elif what == "keyed":
            # from about 2^14 pairs on, a scope of few names takes the small-table route
            n = int(rng.integers(1 << 14, 1 << 16)) if rng.random() < 0.3 else _size(rng, 1 << 14)
            w = int(rng.choice([2, 4]))
            items.append(("keyed", w, str(rng.choice(["vals", "ns"])), _view(rng, cfg.nl, n), _view(rng, cfg.nv, n), n))
        else:
            n = _size(rng, 512)
            items.append(("counters", int(rng.choice([2, 4])), _view(rng, 1 << 14, n), _view(rng, 1 << 14, n), n))
    return items


def _graph_calls(rng, cfg, k, kc):
    calls = []
    for _ in range(int(rng.integers(1, 4))):
        what = str(rng.choice(["histograms", "keyed", "timer", "counters"] if kc else ["histograms", "keyed", "timer"]))
        if what == "timer":                                     # GraphRecorder.timer(name): a span per replay
            calls.append(("timer", int(rng.integers(0, k))))
            continue
        n = max(1, _size(rng, 1 << 12))
        if what == "histograms":
            calls.append(("histograms", [(int(rng.integers(0, k)), str(rng.choice(["vals", "ns"])),
                                          _view(rng, cfg.nv, n), n)]))
        elif what == "keyed":
            calls.append(("keyed", int(rng.choice([2, 4])), str(rng.choice(["vals", "ns"])), _view(rng, cfg.nl, n),
                          _view(rng, cfg.nv, n), n))
        else:
            calls.append(("counters", int(rng.choice([2, 4])), _view(rng, 1 << 14, n), _view(rng, 1 << 14, n), n))
    return calls


CROWD_AT = (11, 27)


def _crowd(rng, cfg, j, ids):
    """At CROWD_AT[i]: more fresh names than either table holds, then a recorder and a window-5 raw subscription on
    the last of them (unbound at this collection), the recorder replayed with counter adds; three collections later,
    when the crowd's ids are free again, samples under those names (so the raw row has an unbound interval and one
    with data in the same window).  The raw subscription stays open to the end."""
    ops = []
    for c in CROWD_AT:
        hn = ["hc%d_%d" % (c, i) for i in range(cfg.H + 3)]
        cn = ["cc%d_%d" % (c, i) for i in range(cfg.C + 3)]
        if j == c:
            ops += [{"op": "hist", "name": n, "value": float(i), "thread": i % 3} for i, n in enumerate(hn)]
            ops += [{"op": "counter", "name": n, "amount": i + 1, "thread": i % 3} for i, n in enumerate(cn)]
            calls = [("counters", 2, _view(rng, 1 << 14, 300), _view(rng, 1 << 14, 300), 300),
                     ("histograms", [(0, "vals", _view(rng, cfg.nv, 100), 100)]), ("timer", 1)]
            ops.append({"op": "gopen", "gid": ids["graph"], "hnames": hn[-2:], "cnames": cn[-2:], "calls": calls})
            ops.append({"op": "greplay", "gid": ids["graph"], "times": 2})
            ops.append({"op": "gclose", "gid": ids["graph"]})
            ids["graph"] += 1
            ops.append({"op": "raw", "rid": ids["raw"], "hnames": ["hp0"] + hn[-2:], "window": 5})
            ids["raw"] += 1
        if j == c + 3:
            ops += [{"op": "hist", "name": n, "value": 3.0, "thread": 0} for n in hn[-2:]]
    return ops


OP_WEIGHTS = {"hist": 8, "many": 8, "counter": 7, "timer": 2, "gtimer": 2, "pct": 1, "scope": 5, "gopen": 1.5, "greplay": 4,
              "gclose": 1, "sub": 1.2, "subclose": .6, "raw": 1.5, "rawclose": .7, "gauge": 1.2, "gwrite": 1.5,
              "gdel": .5}
P_OPS = np.array(list(OP_WEIGHTS.values())) / sum(OP_WEIGHTS.values())


def gen(seed: int, cfg: Config):
    """[collection: [op, ...]]; every op a dict with "op" and its arguments, host ops with "thread" (0-2)."""
    rng = np.random.default_rng([seed, cfg.precision, cfg.H, cfg.C, 2])
    nm = _Names(cfg)
    out = []
    open_graphs, open_subs, open_raws, gauges = [], [], [], {}
    ids = {"graph": 0, "sub": 0, "raw": 0, "gauge": 0}
    big_at = {3: "wc", 9: "k1", 22: "wc", 30: "k1"} if cfg.large else {}
    burst, burst_left = [], 0
    for j in range(cfg.collections):
        ops = []
        th = lambda: int(rng.integers(0, 3))
        if burst_left == 0 and rng.random() < 0.3:              # a burst of fresh names, some past the table
            m = int(rng.integers(2, cfg.H + 4))
            burst, burst_left = nm.burst("hb", m), int(rng.choice([1, 1, 2, 3]))
        hact = nm.hactive(j) + (burst if burst_left else [])
        cact = nm.cactive(j) + ([b.replace("hb", "cb") for b in burst[:cfg.C // 2 + 2]] if burst_left else [])
        hold = burst if burst_left else []                      # the burst this collection uses
        burst_left = max(0, burst_left - 1)
        for c in nm.cperm:                                      # permanent counters never lose their ids
            ops.append({"op": "counter", "name": c, "amount": [0, 1, 2 ** 64 - 1, 1 << 32, 5][int(rng.integers(0, 5))],
                        "thread": th()})
        for h in nm.hperm:
            ops.append({"op": "hist", "name": h, "value": float(rng.choice(OS.SPECIALS)) if rng.random() < 0.2
                        else float(rng.uniform(-5, 1e6)), "thread": th()})
        ops += _crowd(rng, cfg, j, ids)
        for i in range(int(rng.integers(3, 12))):
            kind = "scope" if i == 0 and j in big_at else str(rng.choice(list(OP_WEIGHTS), p=P_OPS))
            op = {"op": kind}
            if kind == "hist":
                op.update(name=str(rng.choice(hact)), value=float(rng.choice(OS.SPECIALS)) if rng.random() < 0.3
                          else float(rng.normal(0, 1e4)), thread=th())
            elif kind == "many":
                n = _size(rng, 2000)
                op.update(name=str(rng.choice(hact)), off=_view(rng, cfg.nv, n), n=n, vk=str(rng.choice(["vals", "ns"])),
                          thread=th())
            elif kind == "counter":
                a = int(rng.choice(OS.AMOUNTS)) if rng.random() < 0.4 else [0, 1, 3, 1 << 31][int(rng.integers(0, 4))]
                op.update(name=str(rng.choice(cact)), amount=a, thread=th())
            elif kind in ("timer", "gtimer"):
                op.update(name=str(rng.choice(hact)), thread=th())
            elif kind == "pct":
                op.update(labels=_labels(rng))
            elif kind == "scope":
                big = big_at.pop(j, None)
                if big == "wc":                                 # more than 44 names: the write-combining route
                    hn = list(dict.fromkeys(nm.universe(j) + hact + nm.burst("hw", 48)))[:52]
                else:
                    pool = nm.universe(j) + hact + nm.burst("hs", int(rng.integers(0, 3)))
                    hn = [str(x) for x in rng.choice(pool, int(rng.integers(1, 7)))]
                cn = [str(x) for x in rng.choice(cact + ["cnever"], int(rng.integers(0, 4)))]
                op.update(hnames=hn, cnames=cn, items=_scope_items(rng, cfg, hn, cn, big), thread=th())
            elif kind == "gopen":
                if len(open_graphs) >= 3:
                    continue
                pool = nm.universe(j) + hact + nm.burst("hq", int(rng.integers(0, 3)))
                cpool = nm.cperm + cact
                if hold and rng.random() < 0.6:                 # the burst's last names: likely past the table
                    pool = hold[-3:] + nm.hperm
                    cpool = [b.replace("hb", "cb") for b in hold[-3:]] + nm.cperm
                hn = [str(x) for x in rng.choice(pool, int(rng.integers(1, 5)))]
                cn = [str(x) for x in rng.choice(cpool, int(rng.integers(0, 3)))]
                op.update(gid=ids["graph"], hnames=hn, cnames=cn, calls=_graph_calls(rng, cfg, len(hn), len(cn)))
                ids["graph"] += 1
                open_graphs.append(op)
            elif kind == "greplay":
                if not open_graphs:
                    continue
                op.update(gid=open_graphs[int(rng.integers(0, len(open_graphs)))]["gid"], times=int(rng.integers(0, 4)))
            elif kind == "gclose":
                if not open_graphs:
                    continue
                op.update(gid=open_graphs.pop(int(rng.integers(0, len(open_graphs))))["gid"])
            elif kind == "sub":
                if len(open_subs) >= 3:
                    continue
                pool = nm.universe(j) + hact
                hn = [str(x) for x in rng.choice(pool, int(rng.integers(0, 5)))]
                cn = [str(x) for x in rng.choice(nm.cperm + [c for cs in nm.cgap.values() for c in cs] + cact +
                                                 ["cnever"], int(rng.integers(0 if hn else 1, 4)))]
                op.update(sid=ids["sub"], hnames=hn[:cfg.H], cnames=cn[:cfg.C])
                ids["sub"] += 1
                open_subs.append(op["sid"])
            elif kind == "subclose":
                if not open_subs:
                    continue
                op.update(sid=open_subs.pop(int(rng.integers(0, len(open_subs)))))
            elif kind == "raw":
                if len(open_raws) >= 4:
                    continue
                pool = nm.universe(j) + hact + hold[-2:]
                hn = [str(x) for x in rng.choice(pool, int(rng.integers(1, 6)))]
                op.update(rid=ids["raw"], hnames=hn[:cfg.H], window=int(rng.choice(WINDOWS)))
                ids["raw"] += 1
                open_raws.append(op["rid"])
            elif kind == "rawclose":
                if not open_raws:
                    continue
                op.update(rid=open_raws.pop(int(rng.integers(0, len(open_raws)))))
            elif kind == "gauge":
                name = "g%d" % int(rng.integers(0, 4))
                dtype = GAUGE_DTYPES[ids["gauge"] % len(GAUGE_DTYPES)][0]    # every dtype in turn
                ids["gauge"] += 1
                op.update(name=name, dtype=dtype, value=_gauge_value(rng, dtype))
                gauges[name] = dtype
            elif kind == "gwrite":
                if not gauges:
                    continue
                name = sorted(gauges)[int(rng.integers(0, len(gauges)))]
                op.update(name=name, value=_gauge_value(rng, gauges[name]))
            else:
                if not gauges:
                    continue
                name = sorted(gauges)[int(rng.integers(0, len(gauges)))]
                op.update(name=name)
                del gauges[name]
            ops.append(op)
        out.append(ops)
    return out


def compact(op) -> str:
    """One line per op for failure messages."""
    skip = ("op", "items", "calls")
    s = op["op"] + "(" + ", ".join("%s=%s" % (k, v) for k, v in op.items() if k not in skip)
    if "items" in op:
        s += ", items=%s" % [(it[0],) + tuple(x for x in it[1:] if not isinstance(x, list)) for it in op["items"]]
    return s + ")"


def scope_routes(op, cfg, sms=H100_SMS) -> set:
    """The keyed kernels the route model predicts for a scope's keyed items (k = the scope's histogram names)."""
    out = set()
    for it in op.get("items", ()):
        if it[0] == "keyed" and it[5]:
            k = len(op["hnames"])
            out.add(R.keyed_route(k, it[5], cfg.precision, sms, id_bytes=it[1], vals_addr=(it[4] * 8) & 31,
                                  ids_addr=(it[3] * it[1]) & 31).kernel)
    return out


def k1_items(op) -> int:
    return sum(1 for it in op.get("items", ()) if it[0] == "histograms"
               for _, vk, _, n in it[1] if vk == "vals" and n >= BATCH_K1_MIN)


# ------------------------------------------------------------------------------------------------------------ model
FREE, LIVE, RETIRING = 0, 1, 2


class Table:
    """NameTable of metric_system.h, restated: each id free, live or retiring."""

    def __init__(self, capacity):
        self.capacity = capacity
        self.ids, self.names, self.state, self.used, self.free = {}, [], [], [], []

    def intern(self, name, mark=True):
        """A lookup that creates or revives the name: its id, or None when no id is free.  A live name found by the
        read-locked fast path is not marked used (metric_system.cc, intern); every other lookup is (intern_locked)."""
        if name in self.ids:
            i = self.ids[name]
            if self.state[i] == LIVE and not mark:
                return i
        elif self.free:
            i = self.free.pop()                       # the last id freed is taken first (intern_locked: free_ids.back())
            self.names[i] = name
            self.ids[name] = i
        elif len(self.names) < self.capacity:
            i = len(self.names)
            self.names.append(name)
            self.state.append(FREE)
            self.used.append(0)
            self.ids[name] = i
        else:
            return None
        self.state[i], self.used[i] = LIVE, 1
        return i

    def lookup(self, name):
        """Histogram / Counter / StartTimer: the read-locked fast path for a live name, else intern."""
        return self.intern(name, mark=False)

    def recycle(self, landed):
        """The three transitions of metric_system.h:477-480; `landed`: names a sample or counter op landed for."""
        for i in range(len(self.names)):
            live_now = self.names[i] in landed or self.used[i]
            self.used[i] = 0
            if self.state[i] == RETIRING and not live_now:
                del self.ids[self.names[i]]
                self.names[i] = ""
                self.state[i] = FREE
                self.free.append(i)
            elif self.state[i] == LIVE and not live_now:
                self.state[i] = RETIRING
            elif self.state[i] == RETIRING:
                self.state[i] = LIVE

    def describe(self):
        st = {FREE: "free", LIVE: "live", RETIRING: "retiring"}
        return {n: (st[self.state[i]], i) for n, i in sorted(self.ids.items())}


def gauge_bits(dtype, value):
    """(raw bytes as stored, float64 the collection reports) of a gauge value written as `dtype`."""
    if dtype == "bfloat16":
        import torch
        t = torch.tensor([value], dtype=torch.float64).to(torch.bfloat16)
        return t.view(torch.int16).numpy().tobytes(), float(t.to(torch.float64)[0])
    a = np.array([value], dtype=dtype) if dtype in GAUGE_INTS else np.array([value], np.float64).astype(dtype)
    return a.tobytes(), float(a.astype(np.float64)[0])


class Want:
    """What one collection must hold."""

    def __init__(self):
        self.hist = {}            # name -> [uint16 key arrays]
        self.deltas = {}          # counter name -> uint64 delta
        self.touched = set()      # counter names touched on the host
        self.dropped = 0
        self.unbound = set()      # histogram names whose host samples found no id
        self.scope_ids = []       # per scope op: (histogram ids, counter ids)

    def add(self, name, keys, times=1):
        if len(keys) and times:
            self.hist.setdefault(name, []).append(np.tile(np.asarray(keys, np.uint16), times))

    def count(self, name, amounts, times=1):
        s = int(np.sum(np.asarray(amounts, np.uint64), dtype=np.uint64)) * times
        self.deltas[name] = (self.deltas.get(name, 0) + s) % (1 << 64)

    def dense(self, name):
        return np.bincount(np.concatenate(self.hist[name]).astype(np.int64), minlength=65536).astype(np.uint64)


class Model:
    """The whole MetricSystem as its header describes it, one collection at a time."""

    def __init__(self, oracle, cfg: Config, pools: Pools, counter_drop="amount"):
        """counter_drop: what a recorder counter row drained while unbound adds to the dropped tally: its drained
        amount (the library, lh_graph_recorder_bind) or one per counter op (the CPU stub)."""
        self.oracle, self.cfg, self.pools, self.counter_drop = oracle, cfg, pools, counter_drop
        self.ht, self.ct = Table(cfg.H), Table(cfg.C)
        self.labels = list(DEFAULT_LABELS)
        self.store = {}           # Counters: cumulative per name
        self.graphs = {}          # gid -> op, in the order they were opened
        self.pending = {}         # gid -> [per replay since the last drain: [duration of each timer call]]
        self.subs, self.raws = {}, {}
        self.raw_hist = {}        # rid -> [per-collection {name: dense}]
        self.gauges = {}          # name -> (dtype, bits, float64)
        self.want = Want()
        self.table = oracle.decompress_table(cfg.precision)
        self.unbound, self.events = set(), set()   # recorder names found unbound; facts the coverage test asserts
        self.raw_unbound = {}     # rid -> name -> collections (indices into raw_hist) at which the name had no id

    def keys(self, vk, off, n):
        return (self.pools.keys_vals if vk == "vals" else self.pools.keys_ns)[off:off + n]

    # ---- one op
    def host_hist(self, name, keys):
        if not len(keys):                       # HistogramMany of nothing looks nothing up (lhms_histogram_many)
            return
        if self.ht.lookup(name) is None:
            self.want.dropped += len(keys)
            self.want.unbound.add(name)
        else:
            self.want.add(name, keys)

    def host_counter(self, name, amount):
        if self.ct.lookup(name) is None:
            self.want.dropped += 1
        else:
            self.want.touched.add(name)
            self.want.count(name, [amount])

    def bind_graph(self, g):
        """bind_graph: every name interned (created or revived) and used; None where no id is free."""
        hids = [self.ht.intern(n) for n in g["hnames"]]
        for n, i in zip(g["hnames"], hids):
            if i is None:
                self.unbound.add((g["gid"], n))
            elif (g["gid"], n) in self.unbound:
                self.events.add("graph_unbound_then_bound")
        return hids, [self.ct.intern(n) for n in g["cnames"]]

    def drain(self, gid, hids, cids):
        """What the replays since the last drain recorded, under the names bound now (unbound rows dropped)."""
        g, replays = self.graphs[gid], self.pending.get(gid, [])
        self.pending[gid] = []
        r = len(replays)
        if not r:
            return
        p, w = self.pools, self.want
        kc = len(g["cnames"])
        timers = 0
        for c in g["calls"]:
            if c[0] == "timer":                         # one span per replay: float64(duration ns) under the name
                ns = [rep[timers] for rep in replays]
                timers += 1
                keys = self.oracle.compress_many(np.array(ns, np.float64), self.cfg.precision).view(np.uint16)
                self._local(hids, g["hnames"], [c[1]] * r, keys)
            elif c[0] == "histograms":
                for li, vk, off, n in c[1]:
                    self._local(hids, g["hnames"], [li] * n, self.keys(vk, off, n), r)
            elif c[0] == "keyed":
                lids = (p.lids16 if c[1] == 2 else p.lids32)[c[3]:c[3] + c[5]]
                self._local(hids, g["hnames"], lids, self.keys(c[2], c[4], c[5]), r)
            else:
                lids = (p.clids16 if c[1] == 2 else p.clids32)[c[2]:c[2] + c[4]].astype(np.int64)
                am = p.amounts[c[3]:c[3] + c[4]]
                w.dropped += int((lids >= kc).sum()) * r
                for li in range(kc):
                    sel = am[lids == li]
                    if not sel.size:
                        continue
                    if cids[li] is not None:
                        w.count(g["cnames"][li], sel, r)
                    elif self.counter_drop == "amount":  # the row's drained (wrapping) sum
                        w.dropped += int(np.sum(sel, dtype=np.uint64)) * r % (1 << 64)
                        self.events.add("recorder_counter_unbound")
                    else:
                        w.dropped += sel.size * r
                        self.events.add("recorder_counter_unbound")

    def _local(self, ids, names, lids, keys, times=1):
        """Samples under local ids: id l < k is name l when bound; ids past the names, or under unbound names, are
        dropped and counted."""
        lids = np.asarray(lids, np.int64)
        keys = np.asarray(keys)
        k = len(names)
        self.want.dropped += int((lids >= k).sum()) * times
        for li in range(k):
            sel = keys[lids == li]
            if not sel.size:
                continue
            if ids[li] is None:
                self.want.dropped += sel.size * times
            else:
                self.want.add(names[li], sel, times)

    def apply(self, op, got=None):
        """Add the op's effect.  `got`: what the call returned (a timer's duration in ns)."""
        o, p, w = op["op"], self.pools, self.want
        if o == "hist":
            self.host_hist(op["name"], self.oracle.compress_many(np.array([op["value"]]), self.cfg.precision).view(np.uint16))
        elif o == "many":
            self.host_hist(op["name"], self.keys(op["vk"], op["off"], op["n"]) if op["vk"] == "vals" else
                           self.oracle.compress_many(p.ns[op["off"]:op["off"] + op["n"]].astype(np.float64),
                                                     self.cfg.precision).view(np.uint16))
        elif o == "counter":
            self.host_counter(op["name"], op["amount"])
        elif o == "timer":
            self.host_hist(op["name"], self.oracle.compress_many(np.array([float(got)]), self.cfg.precision).view(np.uint16))
        elif o == "gtimer":
            # GpuTimerToken::Stop binds the name through a record scope at the stop (BeginRecording): unbound, the
            # sample is dropped and counted; bound, float64(duration ns) lands under it
            i = self.ht.intern(op["name"], mark=False)
            if i is None:
                w.dropped += 1
            else:
                self.ht.used[i] = 1
                w.add(op["name"], self.oracle.compress_many(np.array([float(got)]), self.cfg.precision).view(np.uint16))
        elif o == "pct":
            self.labels = sorted(op["labels"])[:MAX_PERCENTILES]
        elif o == "scope":
            # BeginRecording: every histogram name, then every counter name, interned; bound ids used (pin_names)
            hids = [self.ht.intern(n, mark=False) for n in op["hnames"]]
            cids = [self.ct.intern(n, mark=False) for n in op["cnames"]]
            for t, ids_ in ((self.ht, hids), (self.ct, cids)):
                for i in ids_:
                    if i is not None:
                        t.used[i] = 1
            w.scope_ids.append(([UNBOUND if i is None else i for i in hids], [UNBOUND if i is None else i for i in cids]))
            hn, cn = op["hnames"], op["cnames"]
            for it in op["items"]:
                if it[0] == "histogram":
                    self._local(hids, hn, [it[1]] * it[3], self.keys("vals", it[2], it[3]))
                elif it[0] == "histograms":
                    for li, vk, off, n in it[1]:
                        self._local(hids, hn, [li] * n, self.keys(vk, off, n))
                elif it[0] == "keyed":
                    lids = (p.lids16 if it[1] == 2 else p.lids32)[it[3]:it[3] + it[5]]
                    self._local(hids, hn, lids, self.keys(it[2], it[4], it[5]))
                else:
                    lids = (p.clids16 if it[1] == 2 else p.clids32)[it[2]:it[2] + it[4]].astype(np.int64)
                    am = p.amounts[it[3]:it[3] + it[4]]
                    w.dropped += int((lids >= len(cn)).sum())
                    for li in range(len(cn)):
                        sel = am[lids == li]
                        if not sel.size:
                            continue
                        if cids[li] is None:
                            w.dropped += sel.size
                        else:
                            w.count(cn[li], sel)
        elif o == "gopen":
            self.graphs[op["gid"]] = op
            self.pending[op["gid"]] = []
            self.bind_graph(op)
        elif o == "greplay":
            self.pending[op["gid"]] += got          # the timer durations of each replay
        elif o == "gclose":
            hids, cids = self.bind_graph(self.graphs[op["gid"]])   # Close: bind, then the final drain
            self.drain(op["gid"], hids, cids)
            del self.graphs[op["gid"]]
            del self.pending[op["gid"]]
        elif o == "sub":
            self.subs[op["sid"]] = op
        elif o == "subclose":
            del self.subs[op["sid"]]
        elif o == "raw":
            self.raws[op["rid"]] = op
            self.raw_hist[op["rid"]] = []
        elif o == "rawclose":
            del self.raws[op["rid"]]
            del self.raw_hist[op["rid"]]
        elif o in ("gauge", "gwrite"):
            dtype = op["dtype"] if o == "gauge" else self.gauges[op["name"]][0]
            self.gauges[op["name"]] = (dtype,) + gauge_bits(dtype, op["value"])
        elif o == "gdel":
            del self.gauges[op["name"]]
        else:
            raise AssertionError("unknown op " + o)

    # ---- the collection
    def collect(self):
        """collectRawMetrics + processMetrics: returns the expected (raw, metrics, want) and opens the next interval."""
        for gid, g in list(self.graphs.items()):   # open recorders rebound, in the order they were opened, then drained
            hids, cids = self.bind_graph(g)         # (metric_system.cc, collectRawMetrics: bind_graph before the snapshot)
            self.drain(gid, hids, cids)
        w = self.want
        hist = {n: w.dense(n) for n in w.hist}
        hist = {n: d for n, d in hist.items() if d.any()}
        rates = {n: d for n, d in w.deltas.items() if d or n in w.touched}
        for n in w.touched:
            rates.setdefault(n, 0)
        self.ht.recycle(set(hist))
        self.ct.recycle({n for n, d in rates.items() if d or n in w.touched})
        for n, d in rates.items():
            self.store[n] = (self.store.get(n, 0) + d) % (1 << 64)
        raw = {"Counters": dict(self.store), "Rates": rates,
               "Histograms": {n: rc.sparse(d) for n, d in hist.items()},
               "Gauges": {n: g[2] for n, g in self.gauges.items()}}
        metrics, reduced = {}, {}
        ps = [p for _, p in self.labels]
        for n, d in hist.items():
            ref = self.oracle.process_histogram(d, ps, self.cfg.precision)
            reduced[n] = (ref, rc.Reference(raw["Histograms"][n], self.table))
            for (label, _), k, v in zip(self.labels, ref["pkeys"], ref["pvals"]):
                if k != INT32_MIN:
                    metrics[label.replace("%s", n, 1)] = float(v)
        for n, t in self.store.items():
            metrics[n] = float(t)
        for n, d in rates.items():
            metrics[n + "_rate"] = float(d)
        metrics.update(raw["Gauges"])
        for rid, hs in self.raw_hist.items():
            hs.append({n: hist[n] for n in self.raws[rid]["hnames"] if n in hist})
        exp = {"raw": raw, "metrics": metrics, "reduced": reduced, "labels": list(self.labels), "want": w,
               "hist": hist}
        self.want = Want()
        return exp

    def window(self, rid, name):
        """A raw row's sum over the last `window` collections since the subscription opened."""
        w = self.raws[rid]["window"]
        out = np.zeros(65536, np.uint64)
        for h in self.raw_hist[rid][-w:]:
            if name in h:
                out += h[name]
        return out

    def describe(self):
        return {"histograms": self.ht.describe(), "counters": self.ct.describe()}


# ------------------------------------------------------------------------------------------------------------ checks
class Mismatch(AssertionError):
    pass


# the board layout of include/loghisto_b200.h (tests/test_device_subscription_cpu.py checks it against a C compiler)
BOARD_HDR = np.dtype([("seq", "<u8"), ("publishes", "<u8"), ("np", "<u4"), ("reserved", "<u4", (3,)),
                      ("percentiles", "<f8", (MAX_PERCENTILES,))])
BOARD_ROW = np.dtype([("count", "<u8"), ("sum", "<f8"), ("avg", "<f8"), ("present", "<u4"), ("reserved", "<u4"),
                      ("pvals", "<f8", (MAX_PERCENTILES,)), ("pkeys", "<i4", (MAX_PERCENTILES,))])
BOARD_CTR = np.dtype([("rate", "<u8"), ("total", "<u8"), ("present", "<u4"), ("reserved", "<u4")])


def parse_board(image: bytes, k: int):
    """(header, histogram rows, counter rows) of a board image."""
    raw = np.frombuffer(image, dtype=np.uint8)
    h = raw[:BOARD_HDR.itemsize].view(BOARD_HDR)[0]
    rows = raw[BOARD_HDR.itemsize:BOARD_HDR.itemsize + k * BOARD_ROW.itemsize].view(BOARD_ROW)
    crows = raw[BOARD_HDR.itemsize + k * BOARD_ROW.itemsize:].view(BOARD_CTR)
    return h, rows, crows


def _first_diff(got: dict, want: dict):
    for k in sorted(set(got) | set(want), key=str):
        if k not in got or k not in want:
            return k, got.get(k, "<absent>"), want.get(k, "<absent>")
        g, w = got[k], want[k]
        if isinstance(w, dict):
            d = _first_diff(g, w)
            if d:
                return (k,) + d
        elif isinstance(w, float):
            if not rc.same_bits(g, w):
                return k, g, w
        elif g != w:
            return k, g, w
    return None


def check_collection(exp, got_raw, got_metrics, dropped, scope_ids, what):
    """The collection's RawMetricSet, dropped delta, scope bindings and processed metrics against the model."""
    raw, w = exp["raw"], exp["want"]
    for part in ("Histograms", "Counters", "Rates", "Gauges"):
        d = _first_diff(got_raw[part], raw[part])
        if d:
            raise Mismatch("%s: %s differ at %s" % (what, part, d))
    if dropped != w.dropped % (1 << 64):          # the tally is a uint64: drained counter amounts wrap it
        raise Mismatch("%s: dropped %d, want %d" % (what, dropped, w.dropped % (1 << 64)))
    if scope_ids != w.scope_ids:
        raise Mismatch("%s: scope bindings %s, want %s" % (what, scope_ids, w.scope_ids))
    metrics = dict(got_metrics)
    for n, (ref, r) in exp["reduced"].items():
        cnt, s, a = metrics.pop(n + "_count", None), metrics.pop(n + "_sum", None), metrics.pop(n + "_avg", None)
        if cnt != float(r.count):
            raise Mismatch("%s: %s_count %r, want %r" % (what, n, cnt, float(r.count)))
        if s is None or not rc.sum_ok(s, r):
            raise Mismatch("%s: %s_sum %r, exact %r" % (what, n, s, r.sum))
        if not rc.same_bits(a, rc.avg_of(s, r)):
            raise Mismatch("%s: %s_avg %r, want %r" % (what, n, a, rc.avg_of(s, r)))
    d = _first_diff(metrics, exp["metrics"])
    if d:
        raise Mismatch("%s: processed metric %s" % (what, d))


def check_board(exp, got_metrics, sub, image, what, full=True):
    """A device subscription's board: header, histogram rows as processMetrics reports them, counter rows.  Without
    `full` (the stub's boards, which carry counts only): presence, counts and counter rows."""
    h, rows, crows = image
    raw, labels = exp["raw"], exp["labels"]
    if full and h["np"] != len(labels):
        raise Mismatch("%s: board np %d, want %d" % (what, h["np"], len(labels)))
    for i, n in enumerate(sub["hnames"]):
        row = rows[i]
        if n not in raw["Histograms"]:
            if row["present"] != 0 or row["count"] != 0:
                raise Mismatch("%s: board row %d (%s) present %d count %d for an absent name" %
                               (what, i, n, row["present"], row["count"]))
            continue
        ref, r = exp["reduced"][n]
        if row["present"] != 1 or int(row["count"]) != r.count:
            raise Mismatch("%s: board row %d (%s) present %d count %d, want %d" % (what, i, n, row["present"],
                                                                                  row["count"], r.count))
        if not full:
            continue
        if not (rc.same_bits(row["sum"], got_metrics[n + "_sum"]) and rc.same_bits(row["avg"], got_metrics[n + "_avg"])):
            raise Mismatch("%s: board row %d (%s) sum/avg" % (what, i, n))
        np_ = len(labels)
        if not ((row["pkeys"][:np_] == ref["pkeys"]).all() and
                rc.same_bits(row["pvals"][:np_], ref["pvals"]).all()):
            raise Mismatch("%s: board row %d (%s) percentiles %s / %s, want %s / %s" % (
                what, i, n, list(row["pkeys"][:np_]), list(row["pvals"][:np_]), list(ref["pkeys"]), list(ref["pvals"])))
    for i, n in enumerate(sub["cnames"]):
        c = crows[i]
        want = (int(n in raw["Rates"]), raw["Rates"].get(n, 0), raw["Counters"].get(n, 0))
        got = (int(c["present"]), int(c["rate"]), int(c["total"]))
        if got != want:
            raise Mismatch("%s: board counter row %d (%s) (present, rate, total) %s, want %s" % (what, i, n, got, want))


def raw_queries(model, rid, labels, precision):
    """(ps, values) for one raw board: the label ps, and the crossings of each row's buckets with the doubles beside
    them; values at and one ulp below each row's bucket thresholds."""
    ps = {0.0, 0.5, 0.99, 1.0} | {p for _, p in labels if 0 <= p <= 1}
    values = {-1.0, 0.0, 1.0}
    table = model.table
    for n in model.raws[rid]["hnames"]:
        d = model.window(rid, n)
        nz = np.flatnonzero(d)
        if not nz.size:
            continue
        keys = np.sort(((nz.astype(np.int64) ^ 0x8000) - 0x8000))
        total = int(d.sum(dtype=np.uint64))
        for k in keys[[0, keys.size // 2, -1]]:
            run = int(sum(int(d[kk & 0xFFFF]) for kk in keys if kk <= k))
            q = run / total
            ps |= {q, float(np.nextafter(q, 0.0)), float(np.nextafter(q, 2.0))}
            v = float(table[int(k) & 0xFFFF])
            if math.isfinite(v):
                values |= {v, float(np.nextafter(v, -np.inf))}
    return np.array(sorted(p for p in ps if p <= 1.0)[:256]), np.array(sorted(values))


def expected_raw(model, rid, ps, values, precision):
    """Keys, values, ranks and totals a raw board answers, from the window model."""
    names = model.raws[rid]["hnames"]
    kv = model.oracle.compress_many(values, precision).astype(np.int64)
    keys = np.full((len(names), ps.size), INT32_MIN, np.int32)
    vals = np.full((len(names), ps.size), np.nan)
    ranks = np.zeros((len(names), values.size), np.uint64)
    totals = np.zeros(len(names), np.uint64)
    for i, n in enumerate(names):
        d = model.window(rid, n)
        totals[i] = d.sum(dtype=np.uint64)
        if not totals[i]:
            continue
        ref = model.oracle.process_histogram(d, ps, precision)
        keys[i], vals[i] = ref["pkeys"], ref["pvals"]
        signed = (np.arange(65536) ^ 0x8000) - 0x8000
        for j, k in enumerate(kv):
            ranks[i, j] = d[signed <= k].sum(dtype=np.uint64)
    return keys, vals, ranks, totals


def check_raw(model, rid, got, want, what, ps):
    gk, gv, gr, gt = got
    wk, wv, wr, wt = want
    names = model.raws[rid]["hnames"]
    for i, n in enumerate(names):
        if int(gt[i]) != int(wt[i]):
            raise Mismatch("%s: raw board %d row %d (%s) total %d, want %d" % (what, rid, i, n, gt[i], wt[i]))
        bad = np.flatnonzero((gk[i] != wk[i]) | ~rc.same_bits(gv[i], wv[i]))
        if bad.size:
            j = bad[0]
            raise Mismatch("%s: raw board %d row %d (%s) p=%r: %d / %r, want %d / %r" % (
                what, rid, i, n, float(ps[j]), gk[i][j], gv[i][j], wk[i][j], wv[i][j]))
        bad = np.flatnonzero(gr[i].astype(np.uint64) != wr[i])
        if bad.size:
            raise Mismatch("%s: raw board %d row %d (%s) rank %d at value #%d, want %d" % (
                what, rid, i, n, gr[i][bad[0]], bad[0], wr[i][bad[0]]))


def check_gauges(model, got_raw, what):
    want = {n: g[2] for n, g in model.gauges.items()}
    d = _first_diff(got_raw["Gauges"], want)
    if d:
        raise Mismatch("%s: gauge %s" % (what, d))


# ------------------------------------------------------------------------------------------------------------ runner
class Runner:
    """Issues one run's ops on a backend and checks every collection.

    A backend provides: ms (the MetricSystem), array(pool, off, n) (a device array of a pool view),
    scope_histogram(scope, name, off, n) (RecordScope.histogram of a view of the float64 pool), full_boards (whether
    boards carry sums and percentiles), new_graph(op, g)
    (capture or remember the recorder's calls) and replay(gid, times) (-> per replay, the duration in ns of each timer
    call, read from its out= array), gpu_timer(name) (StartGpuTimer then Stop(out=...) on one stream -> the duration
    in ns), counter_drop (Model's), board(sub) (the board image (header, histogram
    rows, counter rows)), raw_query(sub, ps, values) ((keys, vals, ranks, totals) as numpy), gauge(name, dtype, bits)
    (a registered device cell written with those bytes), write_gauge(name, bits), sync() (every stream the ops used),
    and close()."""

    def __init__(self, oracle, cfg, seed, backend, pools=None, model=None):
        self.oracle, self.cfg, self.seed, self.b = oracle, cfg, seed, backend
        self.pools = pools or Pools(oracle, cfg, seed)
        self.model = model or Model(oracle, cfg, self.pools, backend.counter_drop)
        self.workers = [concurrent.futures.ThreadPoolExecutor(max_workers=1) for _ in range(3)]
        self.graphs, self.subs, self.raws = {}, {}, {}
        self.seen = set()          # facts the coverage test asserts

    def close(self):
        for g in list(self.graphs.values()):
            g.close()
        for s in list(self.subs.values()) + list(self.raws.values()):
            s.close()
        for w in self.workers:
            w.shutdown()
        self.b.close()

    def _host(self, op, fn):
        return self.workers[op["thread"]].submit(fn).result()

    def issue(self, op, scope_ids):
        ms, o, b = self.b.ms, op["op"], self.b
        got = None
        if o == "hist":
            self._host(op, lambda: ms.Histogram(op["name"], op["value"]))
        elif o == "many":
            a = getattr(self.pools, op["vk"])[op["off"]:op["off"] + op["n"]]
            self._host(op, lambda: ms.HistogramMany(op["name"], a.astype(np.float64)))
        elif o == "counter":
            self._host(op, lambda: ms.Counter(op["name"], op["amount"]))
        elif o == "timer":
            got = self._host(op, lambda: ms.StartTimer(op["name"]).Stop())
        elif o == "gtimer":
            got = self._host(op, lambda: b.gpu_timer(op["name"]))
        elif o == "pct":
            ms.SpecifyPercentiles(dict(op["labels"]))
        elif o == "scope":
            def run():
                with ms.recording(b.stream(), histograms=op["hnames"], counters=op["cnames"]) as s:
                    hn = op["hnames"]
                    scope_ids.append(([s.histogram_ids[n] for n in hn], [s.counter_ids[n] for n in op["cnames"]]))
                    for it in op["items"]:
                        if it[0] == "histogram":
                            b.scope_histogram(s, hn[it[1]], it[2], it[3])
                        elif it[0] == "histograms":
                            s.histograms([(hn[li], b.array(vk, off, n)) for li, vk, off, n in it[1]])
                        elif it[0] == "keyed":
                            s.keyed(b.array("lids16" if it[1] == 2 else "lids32", it[3], it[5]), b.array(it[2], it[4], it[5]))
                        else:
                            s.counters(b.array("clids16" if it[1] == 2 else "clids32", it[2], it[4]),
                                       b.array("amounts", it[3], it[4]))
            self._host(op, run)
        elif o == "gopen":
            g = _open_graph(ms, op["hnames"], op["cnames"])
            self.graphs[op["gid"]] = g
            b.new_graph(op, g)
        elif o == "greplay":
            got = b.replay(op["gid"], op["times"])
        elif o == "gclose":
            b.sync()
            self.graphs.pop(op["gid"]).close(b.graph_stream())
            b.drop_graph(op["gid"])
        elif o == "sub":
            self.subs[op["sid"]] = ms.device_subscription(histograms=op["hnames"], counters=op["cnames"])
        elif o == "subclose":
            b.sync()
            self.subs.pop(op["sid"]).close()
        elif o == "raw":
            self.raws[op["rid"]] = ms.raw_device_subscription(histograms=op["hnames"], window=op["window"])
        elif o == "rawclose":
            b.sync()
            self.raws.pop(op["rid"]).close()
        elif o == "gauge":
            b.gauge(op["name"], op["dtype"], gauge_bits(op["dtype"], op["value"])[0])
        elif o == "gwrite":
            b.write_gauge(op["name"], gauge_bits(self.model.gauges[op["name"]][0], op["value"])[0])
        elif o == "gdel":
            ms.DeregisterGaugeFunc(op["name"])
            b.drop_gauge(op["name"])
        return got

    def note(self, op):
        """Facts the coverage test asserts, from the model's state before the op."""
        m = self.model
        if op["op"] in ("sub", "raw"):
            for n in op["hnames"]:
                if n in m.ht.ids:
                    self.seen.add(("watch_id", n, m.ht.ids[n]))

    def run(self, collections, check=True):
        """Every collection issued and checked; returns the model's expectations and what came back."""
        history = []
        for j, ops in enumerate(collections):
            scope_ids = []
            before = self.b.ms.dropped()
            for op in ops:
                self.note(op)
                got = self.issue(op, scope_ids)
                self.model.apply(op, got)
            self.b.sync()
            exp = self.model.collect()
            raw, metrics = self.b.ms.collect_and_process()
            self.b.sync()
            dropped = (self.b.ms.dropped() - before) % (1 << 64)   # a drained recorder counter adds its amount
            state = self.model.describe()
            history.append((exp, raw, metrics, dropped, scope_ids))
            self._coverage(j, exp)
            if check:
                self.check(j, ops, exp, raw, metrics, dropped, scope_ids, state)
        return history

    def _coverage(self, j, exp):
        m = self.model
        if exp["want"].dropped:
            self.seen.add("drop")
        for key in list(self.seen):
            if isinstance(key, tuple) and key[0] == "watch_id":
                n, i = key[1], key[2]
                if i < len(m.ht.names) and m.ht.names[i] and m.ht.names[i] != n and \
                        any(n in s["hnames"] for s in list(m.subs.values()) + list(m.raws.values())):
                    self.seen.add("recycled_under_subscription")
        self.seen |= m.events
        for rid, r in m.raws.items():
            hs = m.raw_hist[rid]
            for n in r["hnames"]:
                if n not in m.ht.ids:
                    m.raw_unbound.setdefault(rid, {}).setdefault(n, set()).add(len(hs) - 1)
                gone = m.raw_unbound.get(rid, {}).get(n, set())
                w = r["window"]
                if any(i >= len(hs) - w for i in gone) and any(n in h for h in hs[-w:]):
                    self.seen.add("window_row_unbound")   # one interval of the window without an id, one with data
            for n in r["hnames"]:
                run = 0
                for h in hs:
                    run = 0 if n in h else run + 1
                if run > r["window"] and any(n in h for h in hs):
                    self.seen.add("window_absent_longer_than_w")

    def check(self, j, ops, exp, raw, metrics, dropped, scope_ids, state):
        what = "%r seed %#x collection %d" % (self.cfg, self.seed, j)
        try:
            check_collection(exp, raw, metrics, dropped, scope_ids, what)
            check_gauges(self.model, raw, what)
            for sid, sub in self.subs.items():
                check_board(exp, metrics, self.model.subs[sid], self.b.board(sub), what + " board %d" % sid,
                            self.b.full_boards)
            for rid, sub in self.raws.items():
                ps, values = raw_queries(self.model, rid, exp["labels"], self.cfg.precision)
                got = self.b.raw_query(sub, ps, values)
                check_raw(self.model, rid, got, expected_raw(self.model, rid, ps, values, self.cfg.precision), what, ps)
        except Mismatch as e:
            lines = [str(e), "ops of this collection:"] + ["  " + compact(op) for op in ops]
            lines.append("name table after it: %s" % state)
            raise Mismatch("\n".join(lines)) from None


def _open_graph(ms, hnames, cnames):
    import loghisto_b200.metric_system as m
    return m.GraphRecorder(ms, hnames, cnames)
