"""The dispatch restatement in tests/_ingest_routes.py (no GPU): its constants, hand-checked points of the prediction,
and the promises of its case builders."""
import numpy as np
import pytest

import _ingest_routes as R

SMS = 132     # H100 SXM


def test_parsed_constants():
    c = R.CONST
    assert c["K2_SMEM_COUNTERS"] == 8192
    assert c["KS_SMEM_BYTES"] == 196608
    assert c["KS_MAX_PASSES"] == 4
    assert c["kSmemBudget"] == 227 * 1024
    assert c["WC_MAX_PARTS"] == 160
    assert c["WC_ROW_EXTRA"] == 64 + 8
    assert c["WC_RARE_CAP"] == 8192
    assert c["WC_ROW_CAPS"] == (256, 192, 128)
    assert c["K1_SMALLER"] == (5, 0, 2, 3)
    names = [v["name"] for v in c["K1_VARIANTS"]]
    assert names == ["bulk2_w16_s4_32768_b1_sign1", "bulk2_w16_s3_65536_b1_sign1", "bulk2_w8_s4_16384_b2_sign1",
                     "ldg_t512_u2_b2", "probe_read_only_t512_u4", "bulk2_w16_s4_32768_b1_sign0",
                     "bulk2_w16_s3_65536_b1_sign0"]
    assert [v["smem_fixed"] for v in c["K1_VARIANTS"]] == [131136, 196656, 65600, 0, 0, 131136, 196656]


def test_prec_derivations():
    assert [R.window(p) for p in (1, 2, 50, 100, 200, 250)] == [45, 88, 2184, 4368, 8735, 10918]
    assert R.a_int(1) == 0 and R.a_int(2) == 1 and R.a_int(100) == 69
    assert R.ks_ids_per_pass(100) == 11


def test_small_kernel_edge():
    """At precision 100 a pass privatises 11 windows and 4 passes are allowed: H = 44 is the last H of the small
    kernel; H = 34 (3.1 passes) is well inside it."""
    assert R.small_edge(100) == 44
    for H, kernel in ((34, R.SMALL), (44, R.SMALL), (45, R.VEC)):
        assert R.keyed_route(H, 1_200_003, 100, SMS).kernel == kernel, H
    assert R.keyed_route(34, 1_200_003, 100, SMS).passes == 4
    assert R.keyed_route(45, 1 << 22, 100, SMS).kernel == R.WC          # big batch: write-combining instead
    assert R.keyed_route(44, 1 << 22, 100, SMS, keyed_mode=1).kernel == R.VEC
    assert R.keyed_route(44, 4 * 4095, 100, SMS).kernel != R.SMALL       # fewer than 4096 vector groups


def test_wc_geometry_points():
    r = R.keyed_route(1024, 1 << 22, 100, SMS)
    assert r.kernel == R.WC and r.wc.row_cap == 256 and r.wc.P == 132 and r.wc.ids_per == 8
    caps, hmax = R.wc_h_by_row_cap(100, SMS, hi=4096)
    assert (caps[256][-1], caps[192][0], caps[192][-1], caps[128][0], hmax) == (1056, 1057, 1188, 1189, 1320)
    assert R.keyed_route(1321, 1 << 22, 100, SMS).kernel == R.VEC
    assert R.keyed_route(1024, 1 << 22, 100, SMS, k1_reserve_sms=1).wc.P == 131
    assert R.wc_geometry(1024, 100, SMS, SMS - 7) is None                # fewer than 8 owners
    assert R.wc_geometry(100, 100, SMS, SMS - 8)[0] == 8
    # small batches take the L2-atomic kernel unless the write-combining one is forced
    assert R.keyed_route(1024, (1 << 22) - 4, 100, SMS).kernel == R.VEC
    assert R.keyed_route(1024, 1 << 16, 100, SMS, keyed_mode=2).kernel == R.WC
    # the row_cap 192 / 128 shapes flush sooner
    f = {cap: R.keyed_route(H, 1 << 22, 100, SMS).wc.flush_tiles for cap, H in ((256, 1000), (192, 1100), (128, 1300))}
    assert f[256] > f[192] > f[128] >= 1


def test_alignment_routes():
    # values 8 bytes past a 32-byte boundary: a scalar head of 3; u32 ids then need their own 16-byte alignment
    assert R.keyed_route(5, 100_000, 100, SMS, id_bytes=4, vals_addr=8, ids_addr=0).kernel == R.SCALAR
    r = R.keyed_route(5, 100_000, 100, SMS, id_bytes=4, vals_addr=8, ids_addr=4)
    assert r.kernel == R.SMALL and r.head == 3
    assert R.keyed_route(5, 3, 100, SMS).kernel == R.SCALAR
    assert R.keyed_route(5, 0, 100, SMS, previous=R.VEC).kernel == R.VEC


def test_pair_route():
    assert R.pair_route(1024, 1 << 21, 1 << 21, 100, SMS).kernel == R.WC      # the two segments together reach 2^22
    assert R.pair_route(1024, 1 << 21, 0, 100, SMS).kernel == R.VEC
    assert R.pair_route(44, 1 << 22, 1 << 22, 100, SMS).kernel == R.SMALL
    assert R.pair_route(1024, 1 << 22, 1 << 22, 100, SMS, keyed_mode=1).kernel == R.VEC
    # the owner windows are uint32 for a whole launch: a fused pair takes at most 2^32 - 1 samples
    assert R.CONST["WC_MAX_LAUNCH"] == 2 ** 32 - 1
    fused = R.pair_route(1024, 2 ** 31, 2 ** 31 - 1, 100, SMS)
    assert fused.kernel == R.WC and fused.wc.taken + fused.wc.taken2 > 2 ** 32 - 4096 and "apart" not in fused.extra
    apart = R.pair_route(1024, 2 ** 31, 2 ** 31, 100, SMS)
    assert apart.kernel == R.WC and apart.extra["apart"] and apart.wc.taken2 == 0
    assert R.pair_route(1024, 2 ** 20, 2 ** 32, 100, SMS).extra["apart"]


def test_keyed_pieces():
    """A call of more than 2^32 - 1 samples on the write-combining route goes out in pieces of at most 2^32 - 1, each
    routed at its own address: 2^32 - 1 is odd, so the pieces after the first start 24, 16 and 8 bytes past a 32-byte
    boundary and take scalar heads of 1, 2 and 3 samples."""
    n = 3 * (2 ** 32 - 1) + 5
    pieces = R.keyed_pieces(32, n, 100, SMS, k1_reserve_sms=SMS - 32, keyed_mode=2)
    assert [m for m, _ in pieces] == [2 ** 32 - 1] * 3 + [5]
    assert [r.kernel for _, r in pieces] == [R.WC] * 3 + [R.SCALAR]
    assert [r.head for _, r in pieces] == [0, 1, 2, 3]
    assert [R.keyed_launches(m, r) for m, r in pieces] == [2, 3, 3, 1]


def test_counter_routes():
    assert R.counter_route(8192, 100_000).kernel == R.COUNTER_SMEM
    assert R.counter_route(8193, 100_000).kernel == R.COUNTER_GLOBAL
    assert R.counter_route(8192, 100_003).extra["launches"] == 2                       # vector body + tail
    assert R.counter_route(8192, 100_004, amounts_addr=8, ids_addr=2).extra["launches"] == 3   # head + body + tail
    assert R.counter_route(8192, 100_004, amounts_addr=8, ids_addr=4, id_bytes=4).extra["launches"] == 3   # head + body + tail
    assert R.counter_route(8192, 100_003, amounts_addr=8, ids_addr=0, id_bytes=4).extra["launches"] == 1
    assert R.counter_route(8192, 16_000).extra["launches"] == 1                       # < 4096 groups: scalar only


def test_hot_window_plan():
    """The guard drains before 2^32 - 2^30 pending samples and never lets one launch take the window past 2^32 - 1."""
    cap = 1_500_000_000
    plan = R.hot_window_plan([cap, cap, 300_000_000, cap, cap, cap])
    assert plan == [[cap], [cap], [300_000_000], ["fold", cap], [cap], [2 ** 32 - 1 - 2 * cap, "fold", 3 * cap - 2 ** 32 + 1]]
    assert sum(x for ev in plan for x in ev if x != "fold") > 2 ** 32


def test_k1_substitution_table():
    """Which code runs under each K1 variant name: the two 3 x 64 KiB-ring variants give way to the 4 x 32 KiB-ring
    kernel with the same arithmetic from precision 103 on; nothing else is ever substituted."""
    assert R.k1_substitution_precisions() == {1: 103, 6: 103}
    for p in (1, 102):
        assert [code for _, code, _ in R.k1_variants(p)] == list(range(7))
    for p in (103, 146, 147, 250):
        assert [code for _, code, _ in R.k1_variants(p)] == [0, 5, 2, 3, 4, 5, 5]
    assert all(smem <= R.CONST["kSmemBudget"] for p in range(1, 251) for _, _, smem in R.k1_variants(p))


def test_exact_route_batch_overflows_the_rare_queue(oracle):
    n = (1 << 22) + 3
    vals = R.exact_route_values(oracle, n, 7)
    ex = R.definitely_exact(vals)
    assert ex.mean() > 0.85
    for reserve in (0, 1):
        wc = R.keyed_route(300, n, 100, SMS, k1_reserve_sms=reserve).wc
        counts = R.wc_slice_counts(ex, wc)
        assert counts.shape == (1, SMS - reserve)
        assert (counts > R.CONST["WC_RARE_CAP"]).sum() > counts.size // 2
    # and the values are what the name says: negatives, |v| >= 2^63, +-Inf and NaNs with payloads all occur
    bits = vals.view(np.uint64)
    nan = np.isnan(vals)
    assert (vals < 0).any() and (np.abs(vals[np.isfinite(vals)]) >= 2.0 ** 63).any() and np.isinf(vals).sum() > 0
    assert np.unique(bits[nan] & np.uint64((1 << 52) - 1)).size > 1000 and (bits[nan] >> np.uint64(63)).any()


@pytest.mark.parametrize("H,reserve", [(1024, 0), (1000, 1), (100, "sm-8")])
def test_one_owner_case_overflows_buffer_and_sub_queues(oracle, H, reserve):
    """The one-owner GPU case: every writer's buffer for the owner overflows in every flush interval, and at P = 132
    and 131 every writer offers the owner's sub-queue more records per chunk than its `cap`."""
    import test_gpu_ingest_routes as T
    vals = T.samples(oracle, 100)[0]
    tune, want, ids = T.one_owner_case(SMS, H, reserve)
    wc = want.wc
    assert want.kernel == R.WC and (ids % wc.P == 3).all() and (ids < H).all()
    sure = ~R.definitely_exact(vals[:wc.taken])              # records the owner receives, up to a few flagged ones
    per_tile = sure.reshape(-1, wc.tile).sum(axis=1)
    assert per_tile.min() >= 2 * wc.row_cap                 # the buffer overflows whatever the fast path flags
    queued, spilled = R.wc_owner_queue(sure, wc)
    if wc.P > 8:
        assert (wc.flush_tiles, wc.slice_tiles) == (1, 2) and wc.cap < 2 * wc.row_cap
        full = queued == wc.cap                              # writers whose slice holds two tiles
        assert full.sum() >= (wc.nchunks - 1) * wc.P and (spilled[full] > 0).all()
    else:
        assert wc.cap > wc.slice_tiles * wc.row_cap and spilled.sum() == 0


def test_owner_queue_model():
    """wc_owner_queue against hand-worked cases: 2 tiles per writer, 1 tile between flushes, row_cap 256, cap 320."""
    wc = R.WcShape(P=2, ids_per=1, row_cap=256, smem=0, flush_tiles=1, slice_tiles=2, nchunks=2, cap=320, tile=1000,
                   taken=8000)
    q, s = R.wc_owner_queue(np.ones(8000, bool), wc)
    # per chunk and writer: 2 flushes of 4 full lines each; 5 lines fit the queue, 3 go the exact route
    assert (q == 320).all() and (s == 192).all()
    mask = np.zeros(8000, bool)
    mask[:100] = True                                        # writer 0, chunk 0, first tile: 100 records
    q, s = R.wc_owner_queue(mask, wc)
    assert q[0, 0] == 64 and q[1, 0] == 36 and s.sum() == 0  # one line at the flush, the remainder at the very end


def test_same_residue_ids():
    for H, P in ((1024, 132), (1000, 131), (100, 8)):
        ids = R.same_residue_ids(1 << 16, H, P, 3, 1)
        assert (ids < H).all() and (ids % P == 3).all()
        assert np.unique(ids).size == len(range(3, H, P)) > 1


def test_high_ids():
    bad = R.high_ids(300, 5)
    assert list(bad) == [65541, 2 ** 31, 2 ** 32 - 1]
    assert (bad.astype(np.uint16) == np.array([5, 0, 65535], np.uint16)).all()     # what a 16-bit truncation would see
    ids = R.with_bad_ids(np.zeros(10, np.uint32), bad, 4)
    assert list(ids) == [65541, 0, 0, 0, 2 ** 31, 0, 0, 0, 2 ** 32 - 1, 0]


def test_gpu_cases_cover_every_route():
    """The GPU boundary cases reach every keyed route, at every precision they run at."""
    import test_gpu_ingest_routes as T
    for precision in (50, 100, 200):
        seen = set()
        for reserve in (0, 1, SMS - 8):
            ragged = 0
            for label, H in T.boundary_cases(precision, SMS, reserve):
                r = R.keyed_route(H, T.N, precision, SMS, k1_reserve_sms=reserve)
                seen.add(r.kernel)
                if label.startswith("row_cap_"):
                    assert r.wc.row_cap == int(label[8:]) and H % r.wc.P, (precision, reserve, label, H)
                    ragged += 1
            assert ragged, (precision, reserve)       # some write-combining case has H that P does not divide
        assert seen == {R.SMALL, R.WC, R.VEC}, precision
