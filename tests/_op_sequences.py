"""Seeded random sequences of engine calls, and the exact per-interval model they are checked against.

`gen(seed, config)` returns the pools (host arrays every call reads a view of) and a list of intervals, each a list of
ops: K1 ingest under every variant, keyed ingest of every id width and value type under changing tuning, the fused
pair, batches, counters, mapped keyed and counter calls, the host-fed entry points, the staging ring, merges and
graph recorders replayed 0-3 times, each on one of three streams or the ingest stream.  Every op is a call the C ABI
accepts: values 8-byte aligned, ids naturally aligned, every view inside its pool, kinds and widths matched.

`Want` is what one interval must hold, `check` / `check_reduced` compare a snapshot with it.  `apply(want, op, pools)`
adds one op's effect; `expected_kernel(op, ...)` is the keyed kernel the route model (_ingest_routes) predicts for it.
Nothing here needs a GPU.
"""
from __future__ import annotations

import math

import numpy as np

import _ingest_routes as R
import _reduce_cases as rc

PS = [0.0, 0.5, 0.99, 1.0]
UNBOUND = 0xFFFFFFFF                          # LH_GRAPH_UNBOUND
MAP_MAX = 4096                                # LH_MAP_MAX: entries of a mapped call's map
BATCH_K1_MIN = R._int_expr(R._src("lh_api.cu"), r"constexpr size_t kBatchK1Min = ([^;]+);", {})
STAGING_BYTES = 1 << 20                       # the engines' staging slots: host calls past ~100k samples take chunks
SPECIALS = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, np.inf, -np.inf, np.nan, 2.0 ** 63,
                     2.0 ** 64, -(2.0 ** 63), 1.7976931348623157e308, -1.0, -1e-300], np.float64)
AMOUNTS = np.array([2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, 1 << 63, 0xFFFFFFFF00000001], np.uint64)   # carry out of a half

# (precision, H, C): between them, every route of the route model (tests/test_op_sequences_cpu.py checks it)
CONFIGS = [(100, 40, 64), (100, 1024, 8193), (1, 1024, 8192), (250, 600, 64), (147, 300, 1024)]
SEEDS = (0x5E9, 0x5EA)
# the (config, seed) runs of tests/test_gpu_op_sequences.py: the cheapest configuration with both seeds, the others with
# the first; the route coverage test walks the same list
RUNS = [(c, s) for c in CONFIGS for s in (SEEDS if c == CONFIGS[0] else SEEDS[:1])]
H100_SMS = 132


class Config:
    """One generator configuration: the engine's (precision, H, C), the number of intervals and the pool sizes."""

    def __init__(self, precision, H, C, intervals=30, nv=(1 << 24) + 64, nc=(1 << 22) + 64, nl=(1 << 20) + 64,
                 big=1 << 24, sms=H100_SMS):
        self.precision, self.H, self.C, self.intervals = precision, H, C, intervals
        self.nv, self.nc, self.nl, self.big, self.sms = nv, nc, nl, big, sms

    def __repr__(self):
        return "Config(precision=%d, H=%d, C=%d)" % (self.precision, self.H, self.C)


# ------------------------------------------------------------------------------------------------------------- pools
def _bad_ids16(H):
    return np.array([H, 65535, min(H + 1, 65535)], np.uint32)


def _fill_ids(rng, n, H, block=4096):
    """ids in blocks: uniform below H, Zipf-skewed (its tail past H) or a single id."""
    out = np.empty(n, np.uint32)
    for a in range(0, n, block):
        m = min(block, n - a)
        kind = rng.integers(0, 3)
        if kind == 0:
            out[a:a + m] = rng.integers(0, H, m)
        elif kind == 1:
            out[a:a + m] = np.minimum(rng.zipf(1.3, m) - 1, 65535)
        else:
            out[a:a + m] = rng.integers(0, H)
    return out


def _values(oracle, rng, n, precision, seed, block=4096):
    """Streams U / L / S / N and timer ns (as float64) block by block, long runs of one value, specials, and values on
    and one ulp beside bucket boundaries, of both signs."""
    streams = [oracle.STREAM_U, oracle.STREAM_L, oracle.STREAM_S, oracle.STREAM_N]
    nb = (n + block - 1) // block
    which = rng.integers(0, 6, nb)
    out = np.empty(n, np.float64)
    for k, st in enumerate(streams):
        sel = np.flatnonzero(which == k)
        if sel.size:
            g = oracle.gen_stream(st, nb * block, seed + k)[:n]
            mask = np.repeat(which == k, block)[:n]
            out[mask] = g[mask]
    mask = np.repeat(which == 4, block)[:n]
    out[mask] = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, seed + 7).view(np.int64)[mask].astype(np.float64)
    T = R.thresholds(oracle, precision, R.window(precision) + 40).view(np.float64)
    edges = np.concatenate([T, np.nextafter(T, 0.0), np.nextafter(T, np.inf)])
    edges = np.concatenate([edges, -edges])
    for b in np.flatnonzero(which == 5):                       # runs: one value over a whole block
        pick = rng.integers(0, 3)
        v = SPECIALS[rng.integers(0, SPECIALS.size)] if pick == 0 else edges[rng.integers(0, edges.size)] if pick == 1 \
            else out[b * block - 1] if b else 1.0
        out[b * block:(b + 1) * block] = v
    pos = rng.integers(0, n, n // 997)
    out[pos] = SPECIALS[rng.integers(0, SPECIALS.size, pos.size)]
    pos = rng.integers(0, n, n // 251)
    out[pos] = edges[rng.integers(0, edges.size, pos.size)]
    return out


def _nanos(oracle, rng, n, seed):
    ns = oracle.gen_stream(oracle.STREAM_TIMER_NS, n, seed).view(np.int64).copy()
    ns[::5] *= -1
    pos = rng.integers(0, n, n // 499)
    ns[pos] = np.array([0, -1, 1, (1 << 63) - 1, -(1 << 63), 1 << 53, (1 << 53) + 1, 1 << 62], np.int64)[
        rng.integers(0, 8, pos.size)]
    for a in rng.integers(0, max(1, n - 8192), 4):             # a few long runs
        ns[a:a + 8192] = ns[a]
    return ns


class Pools:
    """The host arrays every op reads a view of (the device copies are uploaded once per engine), and the oracle's keys
    of the value pools, so the model of an op is a slice."""

    def __init__(self, oracle, cfg: Config, seed: int):
        rng = np.random.default_rng([seed, cfg.precision, cfg.H, cfg.C])
        H, C = cfg.H, cfg.C
        self.vals = _values(oracle, rng, cfg.nv, cfg.precision, seed)
        self.ns = _nanos(oracle, rng, cfg.nv, seed + 11)
        ids = _fill_ids(rng, cfg.nv, H)
        pos = rng.integers(0, cfg.nv, cfg.nv // 389)
        ids[pos] = _bad_ids16(H)[rng.integers(0, 3, pos.size)]
        self.ids16 = ids.astype(np.uint16)
        ids32 = ids.copy()
        pos = rng.integers(0, cfg.nv, cfg.nv // 401)
        ids32[pos] = R.high_ids(H, int(rng.integers(0, H)))[rng.integers(0, 3, pos.size)]
        self.ids32 = ids32
        cids = _fill_ids(rng, cfg.nc, min(C, 65536))
        pos = rng.integers(0, cfg.nc, cfg.nc // 97)
        cids[pos] = np.array([C, 65535, min(C + 7, 65535)], np.uint32)[rng.integers(0, 3, pos.size)]
        self.cids16 = cids.astype(np.uint16)
        cids32 = cids.copy()
        pos = rng.integers(0, cfg.nc, cfg.nc // 101)
        cids32[pos] = R.high_ids(min(C, 65536), int(rng.integers(0, min(C, 65536))))[rng.integers(0, 3, pos.size)]
        self.cids32 = cids32
        amounts = rng.integers(0, 2 ** 64, cfg.nc, dtype=np.uint64)
        amounts[::3] = AMOUNTS[rng.integers(0, AMOUNTS.size, amounts[::3].size)]
        amounts[1::5] = rng.integers(0, 1 << 20, amounts[1::5].size).astype(np.uint64)
        self.amounts = amounts
        lids = rng.integers(0, 12, cfg.nl).astype(np.uint32)     # local ids of graph recorders (k <= 8)
        self.lids16, self.lids32 = lids.astype(np.uint16), lids
        self.keys_v = oracle.compress_many(self.vals, cfg.precision).view(np.uint16)
        self.keys_ns = oracle.compress_many(self.ns.astype(np.float64), cfg.precision).view(np.uint16)

    def arrays(self) -> dict:
        return {n: getattr(self, n) for n in POOLS}


# pool name -> the value pool whose keys it carries (for values) or None
POOLS = ("vals", "ns", "ids16", "ids32", "cids16", "cids32", "amounts", "lids16", "lids32")
KEYS_OF = {"vals": "keys_v", "ns": "keys_ns"}


# --------------------------------------------------------------------------------------------------------- generator
def _size(rng, cfg, cap):
    """Log-uniform from 0 to about 2^24 (bounded by cap); now and then one past 2^22 (the write-combining kernel)."""
    if rng.random() < 0.12 and cap > (1 << 22):
        return int(rng.integers(1 << 22, min(cap, cfg.big) + 1))
    return min(int(2.0 ** rng.uniform(0, math.log2(min(cap, cfg.big) + 1))) - 1, cap)


def _view(rng, pool_len, n):
    """Start of an n-element view: a multiple of 16 elements plus 0-3, inside the pool."""
    off = int(rng.integers(0, 4))
    base = int(rng.integers(0, max(1, (pool_len - n - off) // 16 + 1))) * 16
    assert base + off + n <= pool_len
    return base + off


def _tuning(rng):
    return dict(keyed_mode=int(rng.integers(0, 3)), wc_spt=int(rng.choice([3, 4, 6, 8])),
                kp_chunk=int(rng.choice([65536, 1 << 20, 16 << 20, 64 << 20])),
                wc_flush=int(rng.choice([4096, 8192, R.DEFAULTS["wc_flush"], 65536])))


# the values lh_tune accepts for the keys the generator sets
TUNE_OK = {"keyed_mode": lambda v: 0 <= v <= 2, "wc_spt": lambda v: v in (3, 4, 6, 8),
           "kp_chunk": lambda v: 1 << 16 <= v <= 1 << 28, "wc_flush": lambda v: 4096 <= v <= 65536}


def _map(rng, k, limit):
    """A map of k entries: rows below limit (repeats allowed) and about one in eight unbound."""
    m = rng.integers(0, limit, k).astype(np.int64)
    m[rng.random(k) < 0.125] = UNBOUND
    return [int(x) for x in m]


KINDS = {"f64_u16": ("ids16", "vals"), "f64_u32": ("ids32", "vals"), "i64ns_u16": ("ids16", "ns")}
WEIGHTS = {"k1": 3, "keyed": 6, "pair": 2, "batch": 2, "counter": 3, "mapped": 5, "counter_mapped": 2, "host": 2,
           "staging": 2, "merge": 1, "graph": 2}


def _op(rng, cfg, k1_slots, graphs):
    kind = rng.choice(list(WEIGHTS), p=np.array(list(WEIGHTS.values())) / sum(WEIGHTS.values()))
    op = {"op": str(kind), "stream": int(rng.integers(0, 4))}        # 0: the ingest stream, 1-3: torch streams
    H, C = cfg.H, cfg.C
    if kind == "k1":
        n = _size(rng, cfg, cfg.nv - 4)
        op.update(variant=int(rng.choice(k1_slots)), hid=int(rng.integers(0, H)), n=n, voff=_view(rng, cfg.nv, n))
    elif kind == "keyed":
        n = _size(rng, cfg, cfg.nv - 4)
        form = str(rng.choice(list(KINDS)))
        op.update(form=form, tune=_tuning(rng), n=n, ioff=_view(rng, cfg.nv, n), voff=_view(rng, cfg.nv, n))
    elif kind == "pair":
        nf, nn = _size(rng, cfg, cfg.nv // 2), _size(rng, cfg, cfg.nv // 2)
        if rng.random() < 0.5:                  # both arrays 32-byte aligned: the fused launch is possible
            a = lambda m: _view(rng, cfg.nv, m) & ~3
        else:
            a = lambda m: _view(rng, cfg.nv, m)
        op.update(tune=_tuning(rng), nf=nf, nn=nn, iof=a(nf), vof=a(nf), ion=a(nn), von=a(nn))
    elif kind == "batch":
        items = []
        for _ in range(int(rng.integers(1, 5))):
            f64 = rng.random() < 0.7
            if f64 and rng.random() < 0.5 and cfg.nv > 3 * BATCH_K1_MIN:
                n = int(rng.integers(BATCH_K1_MIN, 3 * BATCH_K1_MIN))
            else:
                n = _size(rng, cfg, min(BATCH_K1_MIN - 1, cfg.nv - 4))
            items.append((int(rng.integers(0, H)), "vals" if f64 else "ns", _view(rng, cfg.nv, n), n))
        op.update(items=items)
    elif kind == "counter":
        n = _size(rng, cfg, cfg.nc - 4)
        op.update(width=int(rng.choice([2, 4])), n=n, ioff=_view(rng, cfg.nc, n), aoff=_view(rng, cfg.nc, n))
    elif kind == "mapped":
        n = _size(rng, cfg, cfg.nv - 4)
        k = int(rng.choice([0, 1, 5, 40, 300, 1500, MAP_MAX], p=[.04, .1, .16, .2, .2, .15, .15]))
        op.update(width=int(rng.choice([2, 4])), vkind=str(rng.choice(["vals", "ns"])), map=_map(rng, k, H),
                  tune=_tuning(rng), n=n, ioff=_view(rng, cfg.nv, n), voff=_view(rng, cfg.nv, n))
    elif kind == "counter_mapped":
        n = _size(rng, cfg, cfg.nc - 4)
        k = int(rng.choice([0, 1, 7, 100, MAP_MAX]))
        op.update(width=int(rng.choice([2, 4])), map=_map(rng, k, C), n=n, ioff=_view(rng, cfg.nc, n),
                  aoff=_view(rng, cfg.nc, n))
    elif kind == "host":
        form = str(rng.choice(["f64", "keyed_f64", "keyed_ns", "counter"]))
        pool = cfg.nc if form == "counter" else cfg.nv
        n = _size(rng, cfg, min(pool - 4, 1 << 19))
        op.update(form=form, tune=_tuning(rng), hid=int(rng.integers(0, H)), n=n, ioff=_view(rng, pool, n),
                  voff=_view(rng, pool, n))
        op["stream"] = 0
    elif kind == "staging":
        form = str(rng.choice(["f64", "keyed", "counter", "abandon"]))
        per = STAGING_BYTES // (8 if form == "f64" else 10)
        n = int(min(_size(rng, cfg, per), per - 16))
        pool = cfg.nc if form == "counter" else cfg.nv
        ids_offset = ((n * 8 + 15) // 16) * 16 + 16 * int(rng.integers(0, 3))
        if ids_offset + 2 * n > STAGING_BYTES:
            ids_offset = ((n * 8 + 15) // 16) * 16
        op.update(form=form, tune=_tuning(rng), hid=int(rng.integers(0, H)), n=n, ids_offset=ids_offset, ioff=_view(rng, pool, n),
                  voff=_view(rng, pool, n))
        op["stream"] = 0
    elif kind == "merge":
        m = int(rng.integers(1, 65))
        ids = rng.integers(0, H + 2, m)
        w = R.window(cfg.precision)
        keys = np.where(rng.random(m) < 0.5, rng.integers(-w + 1, w, m), rng.integers(-32768, 32768, m))
        counts = rng.integers(1, 1 << 40, m, dtype=np.uint64)
        counts[::4] = np.array([2 ** 32 - 1, 2 ** 32 + 1, 1], np.uint64)[rng.integers(0, 3, counts[::4].size)]
        op.update(ids=[int(x) for x in ids], keys=[int(x) for x in keys], counts=[int(x) for x in counts])
        op["stream"] = 0
    else:                                                      # graph recorder: a new one, or replay a live one
        if graphs and rng.random() < 0.5:
            spec = graphs[int(rng.integers(0, len(graphs)))]
        else:
            k, kc = int(rng.integers(1, 9)), int(rng.integers(0, 5))
            calls = []
            for _ in range(int(rng.integers(1, 4))):
                what = str(rng.choice(["ingest", "keyed", "counters"] if kc else ["ingest", "keyed"]))
                n = max(1, _size(rng, cfg, min(cfg.nl - 4, 1 << 20)))
                if what == "ingest":
                    vk = str(rng.choice(["vals", "ns"]))
                    calls.append(("ingest", int(rng.integers(0, k)), vk, _view(rng, cfg.nv, n), n))
                elif what == "keyed":
                    calls.append(("keyed", int(rng.choice([2, 4])), str(rng.choice(["vals", "ns"])),
                                  _view(rng, cfg.nl, n), _view(rng, cfg.nv, n), n))
                else:
                    calls.append(("counters", int(rng.choice([2, 4])), _view(rng, cfg.nl, n), _view(rng, cfg.nc, n), n))
            spec = {"gid": len(graphs), "hist": [int(x) for x in rng.integers(0, H, k)],
                    "ctr": [int(x) for x in rng.integers(0, C, kc)], "calls": calls}
            graphs.append(spec)
        op.update(graph=spec, replays=int(rng.integers(0, 4)))
    return op


def gen(seed: int, cfg: Config, oracle=None):
    """(Pools or None without an oracle, [interval: {"ops": [...], "snapshot": "plain" | "async" | "copy", "row": r}])."""
    rng = np.random.default_rng([seed, cfg.precision, cfg.H, cfg.C, 1])
    k1_slots = [i for i, (name, _, _) in enumerate(R.k1_variants(cfg.precision)) if not name.startswith("probe")]
    graphs, intervals = [], []
    for _ in range(cfg.intervals):
        ops = [_op(rng, cfg, k1_slots, graphs) for _ in range(int(rng.integers(2, 9)))]
        form = str(rng.choice(["plain", "async", "copy"]))
        intervals.append({"ops": ops, "snapshot": form, "row": int(rng.integers(0, cfg.H))})
    return (Pools(oracle, cfg, seed) if oracle is not None else None), intervals


def compact(op) -> str:
    """One line per op for failure messages."""
    skip = ("op", "graph", "map", "ids", "keys", "counts")
    s = op["op"] + "(" + ", ".join("%s=%s" % (k, v) for k, v in op.items() if k not in skip)
    if "map" in op:
        s += ", map=[k=%d, unbound=%d]" % (len(op["map"]), sum(1 for x in op["map"] if x == UNBOUND))
    if "graph" in op:
        g = op["graph"]
        s += ", graph=%d hist=%s ctr=%s calls=%s" % (g["gid"], g["hist"], g["ctr"], g["calls"])
    if "ids" in op:
        s += ", triples=%d" % len(op["ids"])
    return s + ")"


# ------------------------------------------------------------------------------------------------------ validity
def views(op, cfg: Config):
    """[(pool name, start, n, element bytes, kind)] of every array an op reads; kind is "value", "id" or "amount"."""
    o = op["op"]
    out = []
    if o == "k1":
        out.append(("vals", op["voff"], op["n"], 8, "value"))
    elif o == "keyed":
        ip, vp = KINDS[op["form"]]
        out += [(ip, op["ioff"], op["n"], 2 if ip == "ids16" else 4, "id"), (vp, op["voff"], op["n"], 8, "value")]
    elif o == "pair":
        out += [("ids16", op["iof"], op["nf"], 2, "id"), ("vals", op["vof"], op["nf"], 8, "value"),
                ("ids16", op["ion"], op["nn"], 2, "id"), ("ns", op["von"], op["nn"], 8, "value")]
    elif o == "batch":
        out += [(vk, off, n, 8, "value") for _, vk, off, n in op["items"]]
    elif o in ("counter", "counter_mapped"):
        ip = "cids16" if op["width"] == 2 else "cids32"
        out += [(ip, op["ioff"], op["n"], op["width"], "id"), ("amounts", op["aoff"], op["n"], 8, "amount")]
    elif o == "mapped":
        ip = "ids16" if op["width"] == 2 else "ids32"
        out += [(ip, op["ioff"], op["n"], op["width"], "id"), (op["vkind"], op["voff"], op["n"], 8, "value")]
    elif o in ("host", "staging"):
        counter = op["form"] == "counter"
        vp = "amounts" if counter else ("ns" if op["form"] == "keyed_ns" else "vals")
        out.append((vp, op["voff"], op["n"], 8, "amount" if counter else "value"))
        if op["form"] not in ("f64", "abandon"):
            out.append(("cids16" if counter else "ids16", op["ioff"], op["n"], 2, "id"))
    elif o == "graph":
        for c in op["graph"]["calls"]:
            if c[0] == "ingest":
                out.append((c[2], c[3], c[4], 8, "value"))
            elif c[0] == "keyed":
                out += [("lids16" if c[1] == 2 else "lids32", c[3], c[5], c[1], "id"), (c[2], c[4], c[5], 8, "value")]
            else:
                out += [("lids16" if c[1] == 2 else "lids32", c[2], c[4], c[1], "id"), ("amounts", c[3], c[4], 8, "amount")]
    return out


POOL_LEN = {"vals": "nv", "ns": "nv", "ids16": "nv", "ids32": "nv", "cids16": "nc", "cids32": "nc", "amounts": "nc",
            "lids16": "nl", "lids32": "nl"}
POOL_BYTES = {"vals": 8, "ns": 8, "ids16": 2, "ids32": 4, "cids16": 2, "cids32": 4, "amounts": 8, "lids16": 2,
              "lids32": 4}


# --------------------------------------------------------------------------------------------------------- model
class Want:
    """What one interval of one context must hold: (id * 65536 + key) counts, counters and dropped samples, with the
    keys from the oracle's compress at the context's precision."""

    def __init__(self, oracle, H, C=1, precision=100):
        self.oracle, self.H, self.C, self.precision = oracle, H, C, precision
        self.parts = []
        self.counters = np.zeros(C, np.uint64)
        self.dropped = 0

    def hist_keys(self, ids, keys, times=1):
        """Samples whose keys are known (uint16 bit patterns) into histograms `ids`; ids >= H dropped."""
        ids = np.asarray(ids).astype(np.int64)
        ok = ids < self.H
        flat = ids[ok] * 65536 + np.asarray(keys)[ok].astype(np.int64)
        u, c = np.unique(flat, return_counts=True)
        self.parts.append((u, c.astype(np.uint64) * np.uint64(times)))
        self.dropped += int((~ok).sum()) * times

    def hist(self, ids, vals, times=1):
        self.hist_keys(ids, self.oracle.compress_many(np.asarray(vals, np.float64), self.precision).view(np.uint16), times)

    def single(self, hid, vals, times=1):
        self.hist(np.full(len(vals), hid), vals, times)

    def mapped(self, hmap, local, keys, times=1):
        """Keyed samples under local ids: local id l < len(hmap) is histogram hmap[l]; a local id past the map or an
        unbound entry drops the sample (and counts it)."""
        rows = np.append(np.asarray(hmap, np.int64), UNBOUND)
        local = np.asarray(local).astype(np.int64)
        self.hist_keys(rows[np.minimum(local, len(hmap))], keys, times)

    def counter(self, ids, amounts, times=1):
        ids = np.asarray(ids).astype(np.int64)
        ok = ids < self.C
        amounts = np.asarray(amounts, np.uint64)[ok]
        for _ in range(times):
            self.oracle.counter_add(ids[ok].astype(np.uint32), amounts, self.C, self.counters)
        self.dropped += int((~ok).sum()) * times

    def counter_mapped(self, cmap, local, amounts, times=1):
        rows = np.append(np.asarray(cmap, np.int64), UNBOUND)
        self.counter(rows[np.minimum(np.asarray(local).astype(np.int64), len(cmap))], amounts, times)

    def merge(self, ids, keys, counts):
        """lh_merge_counts_host triples: ids >= H dropped (one each), the rest added as they are."""
        ids = np.asarray(ids, np.int64)
        ok = ids < self.H
        flat = ids[ok] * 65536 + (np.asarray(keys, np.int64)[ok] & 0xFFFF)
        self.parts.append((flat, np.asarray(counts, np.uint64)[ok]))
        self.dropped += int((~ok).sum())

    def sparse(self):
        """(sorted id * 65536 + key, count) of the non-empty buckets; kept until the next part is added."""
        if not self.parts:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        if getattr(self, "_n", -1) != len(self.parts):
            u, inv = np.unique(np.concatenate([p[0] for p in self.parts]), return_inverse=True)
            c = np.zeros(u.size, np.uint64)
            np.add.at(c, inv, np.concatenate([p[1] for p in self.parts]))
            nz = c != 0
            self._sparse, self._n = (u[nz], c[nz]), len(self.parts)
        return self._sparse

    def dense(self, h):
        u, c = self.sparse()
        a, b = np.searchsorted(u, [h * 65536, (h + 1) * 65536])
        out = np.zeros(65536, np.uint64)
        out[u[a:b] & 0xFFFF] = c[a:b]
        return out


def _sl(pools, name, off, n):
    return getattr(pools, name)[off:off + n]


def _keys(pools, name, off, n):
    return getattr(pools, KEYS_OF[name])[off:off + n]


def apply(want: Want, op, pools: Pools, times=None):
    """Add what `op` puts into the interval (a graph op: `times` replays of its captured calls, default its own)."""
    o = op["op"]
    if o == "k1":
        want.hist_keys(np.full(op["n"], op["hid"]), _keys(pools, "vals", op["voff"], op["n"]))
    elif o == "keyed":
        ip, vp = KINDS[op["form"]]
        want.hist_keys(_sl(pools, ip, op["ioff"], op["n"]), _keys(pools, vp, op["voff"], op["n"]))
    elif o == "pair":
        want.hist_keys(_sl(pools, "ids16", op["iof"], op["nf"]), _keys(pools, "vals", op["vof"], op["nf"]))
        want.hist_keys(_sl(pools, "ids16", op["ion"], op["nn"]), _keys(pools, "ns", op["von"], op["nn"]))
    elif o == "batch":
        for hid, vk, off, n in op["items"]:
            want.hist_keys(np.full(n, hid), _keys(pools, vk, off, n))
    elif o == "counter":
        ip = "cids16" if op["width"] == 2 else "cids32"
        want.counter(_sl(pools, ip, op["ioff"], op["n"]), _sl(pools, "amounts", op["aoff"], op["n"]))
    elif o == "mapped":
        ip = "ids16" if op["width"] == 2 else "ids32"
        want.mapped(op["map"], _sl(pools, ip, op["ioff"], op["n"]), _keys(pools, op["vkind"], op["voff"], op["n"]))
    elif o == "counter_mapped":
        ip = "cids16" if op["width"] == 2 else "cids32"
        want.counter_mapped(op["map"], _sl(pools, ip, op["ioff"], op["n"]), _sl(pools, "amounts", op["aoff"], op["n"]))
    elif o in ("host", "staging"):
        f, n = op["form"], op["n"]
        if f == "f64":
            want.hist_keys(np.full(n, op["hid"]), _keys(pools, "vals", op["voff"], n))
        elif f in ("keyed_f64", "keyed"):
            want.hist_keys(_sl(pools, "ids16", op["ioff"], n), _keys(pools, "vals", op["voff"], n))
        elif f == "keyed_ns":
            want.hist_keys(_sl(pools, "ids16", op["ioff"], n), _keys(pools, "ns", op["voff"], n))
        elif f == "counter":
            want.counter(_sl(pools, "cids16", op["ioff"], n), _sl(pools, "amounts", op["voff"], n))
    elif o == "merge":
        want.merge(op["ids"], op["keys"], op["counts"])
    elif o == "graph":
        g, r = op["graph"], op["replays"] if times is None else times
        if r == 0:
            return
        for c in g["calls"]:
            if c[0] == "ingest":
                want.hist_keys(np.full(c[4], g["hist"][c[1]]), _keys(pools, c[2], c[3], c[4]), r)
            elif c[0] == "keyed":
                ip = "lids16" if c[1] == 2 else "lids32"
                want.mapped(g["hist"], _sl(pools, ip, c[3], c[5]), _keys(pools, c[2], c[4], c[5]), r)
            else:
                ip = "lids16" if c[1] == 2 else "lids32"
                want.counter_mapped(g["ctr"], _sl(pools, ip, c[2], c[4]), _sl(pools, "amounts", c[3], c[4]), r)
    else:
        raise AssertionError("unknown op " + o)


def interval_want(oracle, cfg, pools, interval) -> Want:
    w = Want(oracle, cfg.H, cfg.C, cfg.precision)
    for op in interval["ops"]:
        apply(w, op, pools)
    return w


# ------------------------------------------------------------------------------------------------------ routes
def _addr(off, nbytes):
    return (off * nbytes) & 31


def expected_kernel(op, cfg: Config, previous: str, sms: int = H100_SMS) -> str:
    """keyed_kernel_name() after `op`, from the route model (the hot window never fills: a sequence's keyed calls hold
    far fewer than 2^32 - 2^30 samples per interval).  Ops that run no keyed ingest leave `previous`."""
    o, p = op["op"], cfg.precision
    if o == "keyed":
        ip, vp = KINDS[op["form"]]
        ib = 2 if ip == "ids16" else 4
        return R.keyed_route(cfg.H, op["n"], p, sms, id_bytes=ib, vals_addr=_addr(op["voff"], 8),
                             ids_addr=_addr(op["ioff"], ib), previous=previous, **op["tune"]).kernel
    if o == "mapped":
        if op["n"] == 0:
            return previous
        if not op["map"]:
            return R.SCALAR                                    # no ids in play: the scalar kernel drops every sample
        return R.keyed_route(len(op["map"]), op["n"], p, sms, id_bytes=op["width"], vals_addr=_addr(op["voff"], 8),
                             ids_addr=_addr(op["ioff"], op["width"]), **op["tune"]).kernel
    if o == "pair":
        return pair_kernel(op, cfg, previous, sms)
    if o == "host" and op["form"] in ("keyed_f64", "keyed_ns") and op["n"]:
        per = (STAGING_BYTES // 10) & ~15
        last = op["n"] - (op["n"] - 1) // per * per
        return R.keyed_route(cfg.H, last, p, sms, **op["tune"]).kernel
    if o == "staging" and op["form"] == "keyed" and op["n"]:
        return R.keyed_route(cfg.H, op["n"], p, sms, ids_addr=op["ids_offset"] & 31, **op["tune"]).kernel
    return previous


def pair_kernel(op, cfg, previous, sms=H100_SMS):
    """launch_keyed_pair: fused when both arrays are vector-aligned and the route model's pair_route fuses them, else
    the float64 array then the int64 one through launch_keyed, each at its own address."""
    t, p = op["tune"], cfg.precision
    if not op["nf"] and not op["nn"]:
        return previous
    aligned = all(_addr(op[v], 8) == 0 and (_addr(op[i], 2) & 7) == 0 for v, i in (("vof", "iof"), ("von", "ion")))
    if aligned:
        r = R.pair_route(cfg.H, op["nf"], op["nn"], p, sms, **t)
        if "apart" not in r.extra:
            return r.kernel
    k = previous
    for n, v, i in ((op["nf"], "vof", "iof"), (op["nn"], "von", "ion")):
        k = R.keyed_route(cfg.H, n, p, sms, vals_addr=_addr(op[v], 8), ids_addr=_addr(op[i], 2), previous=k, **t).kernel
    return k


def routes(op, cfg: Config, sms: int = H100_SMS) -> set:
    """Every route (kernel tag) the op takes, for the coverage test: "k1:<slot>", keyed kernels ("wc:<spt>" for the
    write-combining one), "pair:fused", "batch:k1" / "batch:kernel", counter kernels and the mapped forms."""
    o, p, out = op["op"], cfg.precision, set()

    def keyed(k, tune):
        spt = tune["wc_spt"]                                   # as with_wc_shape resolves it
        return "wc:%d" % (spt if spt in (3, 4, 6) else 8) if k == R.WC else k
    if o == "k1":
        out.add("k1:%d" % op["variant"])
    elif o == "keyed":
        out.add(keyed(expected_kernel(op, cfg, "", sms), op["tune"]))
    elif o == "pair":
        k = pair_kernel(op, cfg, "", sms)
        aligned = all(_addr(op[v], 8) == 0 and (_addr(op[i], 2) & 7) == 0 for v, i in (("vof", "iof"), ("von", "ion")))
        if aligned and "apart" not in R.pair_route(cfg.H, op["nf"], op["nn"], p, sms, **op["tune"]).extra:
            out.add("pair:fused")
        else:
            out.add(keyed(k, op["tune"]))
    elif o == "batch":
        for _, vk, _, n in op["items"]:
            if n:
                out.add("batch:k1" if vk == "vals" and n >= BATCH_K1_MIN else "batch:kernel")
    elif o == "counter":
        if op["n"]:
            out.add(R.counter_route(cfg.C, op["n"], id_bytes=op["width"], amounts_addr=_addr(op["aoff"], 8),
                                    ids_addr=_addr(op["ioff"], op["width"])).kernel)
    elif o == "mapped":
        k = expected_kernel(op, cfg, "", sms)
        if k:
            out.add("mapped:" + keyed(k, op["tune"]))
    elif o == "counter_mapped":
        if op["n"]:
            out.add("mapped:" + R.COUNTER_SMEM)
    return out


# ------------------------------------------------------------------------------------------------------ checks
def check_reduced(red, want, what, every=False):
    """Counts of every histogram; the percentile keys and values of the first and last three touched ones (every
    touched one with `every`) against the oracle; sums and averages of the first and last three."""
    u, c = want.sparse()
    totals = np.zeros(want.H, np.uint64)
    np.add.at(totals, u >> 16, c)
    assert (red.counts == totals).all(), (what, "counts", np.nonzero(red.counts != totals)[0][:5])
    hs = np.unique(u >> 16)
    few = np.unique(np.concatenate([hs[:3], hs[-3:]]))
    table = None
    for h in (hs if every else few):
        dense = want.dense(h)
        ref = want.oracle.process_histogram(dense, PS, want.precision)
        assert (red.pkeys[h] == ref["pkeys"]).all(), (what, "percentile keys", int(h))
        assert (red.pvals[h].view(np.uint64) == ref["pvals"].view(np.uint64)).all(), (what, "percentile values", int(h))
        if h in few:
            if table is None:
                table = want.oracle.decompress_table(want.precision)
            r = rc.Reference(rc.sparse(dense), table)
            s = float(red.sums[h])
            assert rc.sum_ok(s, r), (what, "sum", int(h), s, float(r.sum))
            assert rc.same_bits(red.avgs[h], rc.avg_of(s, r)), (what, "average", int(h))


def check(e, want, what, dropped_before=None, snap=None, every=False):
    """The interval (a fresh snapshot, or `snap` = (Reduced, Sparse)) equals `want` bucket for bucket."""
    red, sp = snap if snap is not None else e.snapshot(PS)
    u, c = want.sparse()
    flat = np.repeat(np.arange(want.H, dtype=np.int64), np.diff(sp.offsets.astype(np.int64))) * 65536 + sp.keys.view(np.uint16)
    order = np.argsort(flat, kind="stable")
    assert flat.size == u.size and (flat[order] == u).all(), (what, "buckets", flat.size, u.size)
    assert (sp.counts[order] == c).all(), (what, "bucket counts", np.nonzero(sp.counts[order] != c)[0][:5])
    check_reduced(red, want, what, every)
    assert (sp.counter_deltas == want.counters).all(), (what, "counters", np.nonzero(sp.counter_deltas != want.counters)[0][:5])
    if dropped_before is not None:
        assert e.stats()["dropped"] - dropped_before == want.dropped, (what, "dropped", e.stats()["dropped"] - dropped_before, want.dropped)
