"""Small end-to-end pass over every kernel, meant to run under compute-sanitizer (racecheck / memcheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loghisto_b200 as lh

PS = [0.0, 0.5, 0.99, 1.0]


class View:
    """n 8-byte elements at a device address, as a __cuda_array_interface__ object (an item of ingest_batch)."""
    def __init__(self, ptr, n, typestr="<f8"):
        self.n = n
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


n = 300_001
total = 0
with lh.Engine(device=0, max_histograms=64, max_counters=64) as e:
    d = e.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED)
    ids = e.gen_ids_u16(0, n, 64, lh.DEFAULT_SEED)
    amt = e.gen_stream(lh.STREAM_AMOUNTS, n, lh.DEFAULT_SEED)
    ns = e.gen_stream(lh.STREAM_TIMER_NS, n, lh.DEFAULT_SEED)
    for vi, name in enumerate(e.k1_variants()):        # every K1 shape
        if name.startswith("probe"):
            continue
        e.tune("k1", vi)
        e.ingest_f64(1, d.offset(1), n - 1)
        total += n - 1
    e.tune("keyed_mode", 1)                             # L2-atomic kernel
    e.ingest_keyed_f64_u16(ids, d, n); total += n
    e.ingest_keyed_i64ns_u16(ids, ns, n); total += n
    e.tune("keyed_mode", 2); e.tune("kp_chunk", 65536)  # write-combining owner kernel, every tile shape, several chunks
    for spt in (6, 4, 3, 8):
        e.tune("wc_spt", spt)
        e.ingest_keyed_f64_u16(ids, d, n); total += n
    e.ingest_keyed_pair_u16(ids, d, n, ids, ns, n); total += 2 * n   # float64 + int64 segments in one launch
    e.tune("keyed_mode", 0)
    items = [(i % 64, View(d.offset(i * 700), 700 + 3 * i)) for i in range(300)]   # batch kernel, pieces across items
    items += [(5, View(ns.offset(1), 20_000, "<i8")), (6, View(d.offset(3), 9_000))]       # int64 ns, misaligned starts
    e.ingest_batch(items); total += sum(v.n for _, v in items)
    e.counter_add_u16(ids, amt, n)                      # vector + scalar counter kernels
    e.counter_add_u16(ids.offset(1), amt.offset(1), n - 1)
    e.snapshot_begin()
    h = e.snapshot_reduce_async(PS)
    sp = e.snapshot_export()
    e.snapshot_end()
    red = e.snapshot_result(h)
    assert int(red.counts.sum()) == total, (int(red.counts.sum()), total)
    # the export reduced again from the sparse form: more segments than one scratch batch, out-of-window keys
    offsets = list(sp.offsets) + [int(sp.offsets[-1])] * 300
    rs = e.reduce_sparse(offsets, sp.keys, sp.counts, PS + [-0.0])
    assert int(rs.counts.sum()) == total
with lh.Engine(device=0, max_histograms=4, max_counters=4) as e:    # few histograms: shared-memory privatised keyed kernel
    d = e.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED)
    ids = e.gen_ids_u16(0, n, 4, lh.DEFAULT_SEED)
    e.ingest_keyed_f64_u16(ids, d, n)
    red, sp2 = e.snapshot(PS)
    assert int(red.counts.sum()) == n
with lh.Engine(device=0, max_histograms=64, max_counters=64) as e:  # mapped (record-scope) keyed and counter calls
    d = e.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED)
    ns = e.gen_stream(lh.STREAM_TIMER_NS, n, lh.DEFAULT_SEED)
    amt = e.gen_stream(lh.STREAM_AMOUNTS, n, lh.DEFAULT_SEED)
    ids = e.gen_ids_u16(0, n, 64, lh.DEFAULT_SEED)
    m = [(i * 7) % 64 for i in range(62)] + [0xFFFFFFFF]       # ids 62 unbound, 63 past the map
    e.ingest_keyed_mapped_u16(m, ids, d, 0, n)                  # vector body
    e.ingest_keyed_mapped_u16(m, ids.offset(1), ns.offset(1), 1, n - 1)   # scalar kernel only
    e.ingest_keyed_mapped_u16(m[:8], ids, d, 0, n)              # shared-memory privatised kernel, most samples dropped
    e.tune("keyed_mode", 2); e.tune("kp_chunk", 65536)
    e.ingest_keyed_mapped_u16(m, ids, d, 0, n)                  # write-combining owner kernel
    e.tune("keyed_mode", 0)
    e.counter_add_mapped_u16(m, ids, amt, n)
    e.counter_add_mapped_u16(m, ids.offset(1), amt.offset(1), n - 1)
    red, _ = e.snapshot(PS)
    assert int(red.counts.sum()) + e.stats()["dropped"] > 0
with lh.Engine(device=0, max_histograms=4, max_counters=4) as e:    # graph recorder: batch ingest into its rows, drains
    d = e.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED)
    with e.graph_recorder([2, 3, 0xFFFFFFFF], [1]) as g:      # local row 2 unbound: dropped and counted
        g.ingest([(0, View(d.ptr, n)), (1, View(d.offset(1), 5_000)), (2, View(d.offset(2), 700))], stream=0)
        red, _ = e.snapshot(PS)                          # collection drain: window and full rows, one unbound row
        assert int(red.counts[2]) == n and int(red.counts[3]) == 5_000
        g.ingest([(1, View(d.ptr, 3_000))], stream=0)
        g.close(stream=0)                                # final drain
    red, _ = e.snapshot(PS)
    assert int(red.counts[3]) == 3_000
with lh.Engine(device=0, max_histograms=4, max_counters=2) as e:    # device subscription: publish (staged too), read
    d = e.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED)
    e.ingest_f64(1, d, n)
    e.snapshot_begin()
    e.snapshot_reduce_async(PS)
    with e.board(4, 2) as b:
        b.publish([1, 0xFFFFFFFF, 0, 3], [1, 0xFFFFFFFF], [7, 8])
        e.snapshot_end()
        e.sync()
        v = b.read(stream=0)
        e.sync()
        assert int(v["count"][0].item()) == n and int(v["collection"].item()) == 1
with lh.Engine(device=0, max_histograms=1, max_counters=1) as e:     # device gauges: a read split over two launches
    import ctypes as C
    import numpy as np
    from loghisto_b200 import _lib as L
    g = e.upload(np.arange(1025, dtype=np.float64))
    srcs = (L.lh_gauge_src * 1025)(*[L.lh_gauge_src(g.offset(i), L.LH_GAUGE_F64, 0) for i in range(1025)])
    vals = np.zeros(1025)
    e._check(e.lib.lh_gauges_read(e.h, srcs, 1025, vals.ctypes.data))
    assert (vals == np.arange(1025)).all()
# two contexts on one device: the peer all-reduce kernel
engs = [lh.Engine(device=0, max_histograms=3, max_counters=2) for _ in range(2)]
handles = b"".join(x.comm_export() for x in engs)
for r, x in enumerate(engs):
    x.comm_import(r, 2, handles)
for r, x in enumerate(engs):
    dd = x.gen_stream(lh.STREAM_S, n, lh.DEFAULT_SEED, start=r * n)
    x.ingest_f64(1, dd, n)
for x in engs:
    x.snapshot_begin(); x.snapshot_allreduce()
for x in engs:
    red = x.snapshot_reduce(PS); x.snapshot_end()
    assert int(red.counts[1]) == 2 * n
for x in engs:
    x.close()
print("sanitize pass ok:", total, "samples,", int(sp.offsets[-1]), "non-empty buckets")
