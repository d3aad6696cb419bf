"""The op-sequence generator and model of tests/_op_sequences.py, without a GPU: the same seed gives the same calls,
every call is one the C ABI accepts, the default seeds reach every route the route model knows, the model agrees with
a separate accumulation through the oracle, and `check` fails on every single-count perturbation of a snapshot."""
import copy

import numpy as np
import pytest

import _ingest_routes as R
import _op_sequences as S
import _reduce_cases as rc
from loghisto_b200.engine import Reduced, Sparse

TINY = dict(intervals=6, nv=(1 << 16) + 64, nc=(1 << 14) + 64, nl=(1 << 12) + 64, big=1 << 15)


def default_runs():
    return [(seed, S.Config(*c)) for c in S.CONFIGS for seed in S.SEEDS]


def test_same_seed_same_ops():
    for seed, cfg in default_runs()[:3]:
        assert S.gen(seed, cfg)[1] == S.gen(seed, cfg)[1]
    a, b = S.gen(S.SEEDS[0], S.Config(*S.CONFIGS[0]))[1], S.gen(S.SEEDS[1], S.Config(*S.CONFIGS[0]))[1]
    assert a != b


@pytest.mark.parametrize("run", range(len(S.CONFIGS) * len(S.SEEDS)))
def test_every_op_is_valid(run):
    """Views inside their pools; values / amounts 8-byte elements, ids of the call's width; ids of histogram calls
    below H, maps within LH_MAP_MAX and their bound rows below H (C); staging layouts inside the slot."""
    seed, cfg = default_runs()[run]
    _, intervals = S.gen(seed, cfg)
    lengths = {name: getattr(cfg, attr) for name, attr in S.POOL_LEN.items()}
    for iv in intervals:
        assert iv["snapshot"] in ("plain", "async", "copy") and 0 <= iv["row"] < cfg.H
        for op in iv["ops"]:
            assert op["stream"] in (0, 1, 2, 3), op
            for pool, off, n, nbytes, kind in S.views(op, cfg):
                assert 0 <= off and n >= 0 and off + n <= lengths[pool], (S.compact(op), pool)
                assert S.POOL_BYTES[pool] == nbytes, (S.compact(op), pool)
                assert (kind == "id") == pool.endswith(("16", "32")), (S.compact(op), pool)
            if "tune" in op:
                assert set(op["tune"]) == set(S.TUNE_OK) and all(S.TUNE_OK[k](v) for k, v in op["tune"].items()), op
            if "hid" in op:
                assert 0 <= op["hid"] < cfg.H
            if op["op"] == "batch":
                assert all(0 <= h < cfg.H and vk in ("vals", "ns") for h, vk, _, _ in op["items"])
            if "map" in op:
                limit = cfg.H if op["op"] == "mapped" else cfg.C
                assert len(op["map"]) <= S.MAP_MAX and all(x == S.UNBOUND or 0 <= x < limit for x in op["map"])
            if op["op"] == "staging":
                per = S.STAGING_BYTES // (8 if op["form"] == "f64" else 10)
                assert op["n"] <= per and op["stream"] == 0
                if op["form"] in ("keyed", "counter"):
                    o = op["ids_offset"]
                    assert o % 16 == 0 and o >= 8 * op["n"] and o + 2 * op["n"] <= S.STAGING_BYTES
            if op["op"] == "merge":
                assert all(-32768 <= k < 32768 for k in op["keys"]) and all(0 < c < 2 ** 64 for c in op["counts"])
            if op["op"] == "graph":
                g = op["graph"]
                assert 1 <= len(g["hist"]) <= 8 and all(0 <= h < cfg.H for h in g["hist"])
                assert all(0 <= c < cfg.C for c in g["ctr"]) and 0 <= op["replays"] <= 3
                for c in g["calls"]:
                    assert c[0] != "ingest" or 0 <= c[1] < len(g["hist"])
                    assert c[0] != "counters" or g["ctr"]


def test_default_seeds_reach_every_route():
    """Across the runs of tests/test_gpu_op_sequences.py, the route model sends some call to every K1 slot, to each
    keyed kernel (the write-combining one at every wc_spt), to the fused pair, both batch routes, both counter kernels
    and the mapped small / write-combining / counter forms."""
    seen = set()
    for config, seed in S.RUNS:
        cfg = S.Config(*config)
        for iv in S.gen(seed, cfg)[1]:
            for op in iv["ops"]:
                seen |= S.routes(op, cfg)
    k1 = {"k1:%d" % i for i, (name, _, _) in enumerate(R.k1_variants(100)) if not name.startswith("probe")}
    need = k1 | {R.SCALAR, R.SMALL, R.VEC, "wc:3", "wc:4", "wc:6", "wc:8", "pair:fused", "batch:k1", "batch:kernel",
                 R.COUNTER_SMEM, R.COUNTER_GLOBAL, "mapped:" + R.SMALL, "mapped:wc:3", "mapped:wc:4", "mapped:wc:6",
                 "mapped:wc:8", "mapped:" + R.COUNTER_SMEM}
    assert need <= seen, sorted(need - seen)


def oracle_intervals(oracle, cfg, pools, intervals):
    """Each interval as dense [H][65536] counts, counters and dropped, from the oracle over the ops' arrays,
    independently of Want.  At precision 100 keyed samples go through oracle.ingest_keyed and int64 nanoseconds through
    oracle.ingest_keyed_i64, which converts them itself; the oracle's keyed entry points have no other precision, so
    elsewhere oracle.ingest takes each histogram's samples, int64 ones converted with numpy as the model does."""
    out = []
    for iv in intervals:
        dense = np.zeros((cfg.H, 65536), np.uint64)
        ctr = np.zeros(cfg.C, np.uint64)
        dropped = [0]

        def keyed(ids, vals, times=1):
            ids = np.asarray(ids, np.uint32)
            dropped[0] += int((ids >= cfg.H).sum()) * times
            ok = ids < cfg.H
            vals = np.asarray(vals)[ok]
            one = np.zeros((cfg.H, 65536), np.uint64)
            if cfg.precision == 100:
                (oracle.ingest_keyed_i64 if vals.dtype == np.int64 else oracle.ingest_keyed)(ids[ok], vals, cfg.H, one)
            else:
                for h in np.unique(ids[ok]):
                    oracle.ingest(vals[ids[ok] == h].astype(np.float64), one[h], precision=cfg.precision)
            dense[:] += one * np.uint64(times)

        def counters(ids, amounts, times=1):
            ids = np.asarray(ids, np.uint32)
            dropped[0] += int((ids >= cfg.C).sum()) * times
            for _ in range(times):
                oracle.counter_add(ids[ids < cfg.C], np.asarray(amounts, np.uint64)[ids < cfg.C], cfg.C, ctr)

        def remap(m, local):
            rows = np.append(np.asarray(m, np.int64), S.UNBOUND).astype(np.uint32)
            return rows[np.minimum(np.asarray(local, np.int64), len(m))]
        p = pools
        for op in iv["ops"]:
            o = op["op"]
            if o == "k1":
                keyed(np.full(op["n"], op["hid"]), p.vals[op["voff"]:op["voff"] + op["n"]])
            elif o == "keyed":
                ip, vp = S.KINDS[op["form"]]
                keyed(getattr(p, ip)[op["ioff"]:op["ioff"] + op["n"]], getattr(p, vp)[op["voff"]:op["voff"] + op["n"]])
            elif o == "pair":
                keyed(p.ids16[op["iof"]:op["iof"] + op["nf"]], p.vals[op["vof"]:op["vof"] + op["nf"]])
                keyed(p.ids16[op["ion"]:op["ion"] + op["nn"]], p.ns[op["von"]:op["von"] + op["nn"]])
            elif o == "batch":
                for h, vk, off, n in op["items"]:
                    keyed(np.full(n, h), getattr(p, vk)[off:off + n])
            elif o == "counter":
                ids = (p.cids16 if op["width"] == 2 else p.cids32)[op["ioff"]:op["ioff"] + op["n"]]
                counters(ids, p.amounts[op["aoff"]:op["aoff"] + op["n"]])
            elif o == "mapped":
                ids = (p.ids16 if op["width"] == 2 else p.ids32)[op["ioff"]:op["ioff"] + op["n"]]
                keyed(remap(op["map"], ids), getattr(p, op["vkind"])[op["voff"]:op["voff"] + op["n"]])
            elif o == "counter_mapped":
                ids = (p.cids16 if op["width"] == 2 else p.cids32)[op["ioff"]:op["ioff"] + op["n"]]
                counters(remap(op["map"], ids), p.amounts[op["aoff"]:op["aoff"] + op["n"]])
            elif o in ("host", "staging"):
                f, n, i, v = op["form"], op["n"], op["ioff"], op["voff"]
                if f == "f64":
                    keyed(np.full(n, op["hid"]), p.vals[v:v + n])
                elif f in ("keyed", "keyed_f64"):
                    keyed(p.ids16[i:i + n], p.vals[v:v + n])
                elif f == "keyed_ns":
                    keyed(p.ids16[i:i + n], p.ns[v:v + n])
                elif f == "counter":
                    counters(p.cids16[i:i + n], p.amounts[v:v + n])
            elif o == "merge":
                for h, k, c in zip(op["ids"], op["keys"], op["counts"]):
                    if h < cfg.H:
                        dense[h, k & 0xFFFF] += np.uint64(c)
                    else:
                        dropped[0] += 1
            elif o == "graph":
                g, r = op["graph"], op["replays"]
                for c in g["calls"] if r else ():
                    if c[0] == "ingest":
                        keyed(np.full(c[4], g["hist"][c[1]]), getattr(p, c[2])[c[3]:c[3] + c[4]], r)
                    elif c[0] == "keyed":
                        lids = (p.lids16 if c[1] == 2 else p.lids32)[c[3]:c[3] + c[5]]
                        keyed(remap(g["hist"], lids), getattr(p, c[2])[c[4]:c[4] + c[5]], r)
                    else:
                        lids = (p.lids16 if c[1] == 2 else p.lids32)[c[2]:c[2] + c[4]]
                        counters(remap(g["ctr"], lids), p.amounts[c[3]:c[3] + c[4]], r)
        out.append((dense, ctr, dropped[0]))
    return out


@pytest.mark.parametrize("config", [(100, 40, 64), (250, 600, 64), (1, 30, 9000)])
def test_model_equals_oracle_accumulation(oracle, config):
    cfg = S.Config(*config, **TINY)
    pools, intervals = S.gen(S.SEEDS[0], cfg, oracle)
    for i, (iv, (dense, ctr, dropped)) in enumerate(zip(intervals, oracle_intervals(oracle, cfg, pools, intervals))):
        w = S.interval_want(oracle, cfg, pools, iv)
        u, c = w.sparse()
        got = np.zeros((cfg.H, 65536), np.uint64)
        got[u >> 16, u & 0xFFFF] = c
        assert (got == dense).all(), (config, i)
        assert (w.counters == ctr).all() and w.dropped == dropped, (config, i)


# ------------------------------------------------------------------------------------------------ the checker itself
class FakeEngine:
    def __init__(self, dropped):
        self._d = dropped

    def stats(self):
        return {"dropped": self._d}


def snapshot_of(want, ps=S.PS):
    """(Reduced, Sparse) a correct engine would return for `want`: export from the model, reduction from the oracle,
    sums from the exact reference rounded once."""
    u, c = want.sparse()
    H = want.H
    offsets = np.zeros(H + 1, np.uint32)
    np.add.at(offsets, (u >> 16) + 1, 1)
    offsets = np.cumsum(offsets).astype(np.uint32)
    keys = (u & 0xFFFF).astype(np.uint16).view(np.int16)
    red = Reduced(np.zeros(H, np.uint64), np.zeros(H), np.zeros(H), np.full((H, len(ps)), rc.INT32_MIN, np.int32),
                  np.full((H, len(ps)), np.nan))
    table = want.oracle.decompress_table(want.precision)
    for h in np.unique(u >> 16):
        d = want.dense(h)
        ref = want.oracle.process_histogram(d, ps, want.precision)
        r = rc.Reference(rc.sparse(d), table)
        red.counts[h] = np.uint64(r.count)
        red.pkeys[h], red.pvals[h] = ref["pkeys"], ref["pvals"]
        red.sums[h] = float(r.sum)
        red.avgs[h] = rc.avg_of(float(r.sum), r)
    return red, Sparse(offsets, keys.copy(), c.copy(), want.counters.copy())


@pytest.fixture(scope="module")
def two_intervals(oracle):
    cfg = S.Config(100, 40, 64, **TINY)
    pools, intervals = S.gen(S.SEEDS[1], cfg, oracle)
    wants = [S.interval_want(oracle, cfg, pools, iv) for iv in intervals]
    i = next(k for k in range(1, len(wants)) if wants[k].sparse()[0].size and wants[k - 1].sparse()[0].size
             and wants[k].counters.any())
    return wants[i - 1], wants[i]


def clone(want):
    w = S.Want(want.oracle, want.H, want.C, want.precision)
    w.parts, w.counters, w.dropped = list(want.parts), want.counters.copy(), want.dropped
    return w


def perturbations(prev, want):
    """(name, (Reduced, Sparse), dropped) of one wrong snapshot each."""
    red, sp = snapshot_of(want)
    out = []
    j = int(np.argmax(sp.counts))
    for d in (1, -1):
        s = copy.deepcopy(sp)
        s.counts[j] = np.uint64(int(s.counts[j]) + d)
        out.append(("bucket %+d" % d, (red, s), want.dropped))
    # one count moved to the neighbouring key of the same histogram (the wrong snapshot is what such a Want holds)
    u, c = want.sparse()
    moved = clone(want)
    moved.parts.append((np.array([u[0], u[0] + 1 if (u[0] & 0xFFFF) < 0xFFFF else u[0] - 1]),
                        np.array([2 ** 64 - 1, 1], np.uint64)))
    out.append(("count moved to the next key", snapshot_of(moved), want.dropped))
    # one count of the previous interval carried into this one
    pu, _ = prev.sparse()
    carried = clone(want)
    carried.parts.append((pu[-1:], np.array([1], np.uint64)))
    out.append(("count carried over", snapshot_of(carried), want.dropped))
    s = copy.deepcopy(sp)
    k = int(np.flatnonzero(want.counters)[0])
    s.counter_deltas[k] = np.uint64((int(s.counter_deltas[k]) + 2 ** 32) % 2 ** 64)
    out.append(("counter + 2^32", (red, s), want.dropped))
    out.append(("dropped + 1", (red, sp), want.dropped + 1))
    out.append(("dropped - 1", (red, sp), want.dropped - 1))
    r = copy.deepcopy(red)
    h = int(u[0] >> 16)
    r.pvals[h, 1] = np.nextafter(r.pvals[h, 1], np.inf)
    out.append(("percentile value 1 ulp", (r, sp), want.dropped))
    return out


def test_check_passes_on_the_model(two_intervals):
    prev, want = two_intervals
    S.check(FakeEngine(want.dropped), want, "model", dropped_before=0, snap=snapshot_of(want), every=True)


@pytest.mark.parametrize("which", range(8))
def test_check_catches_one_wrong_count(two_intervals, which):
    prev, want = two_intervals
    name, snap, dropped = perturbations(prev, want)[which]
    with pytest.raises(AssertionError):
        S.check(FakeEngine(dropped), want, name, dropped_before=0, snap=snap, every=True)
