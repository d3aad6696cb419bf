"""Every uint32 count on the ingest path, driven past 2^31 (and, summed over one call, past 2^32) samples.

Several ingest kernels count into uint32 cells (K1's per-CTA sub-histogram, the per-CTA lh::BlockRecorder table of the
batch and graph-recorder kernels, the owner windows of the write-combining keyed kernel, lh::BlockHistogram and
lh::BlockRecorder in a caller's kernel) before they add them to the uint64 rows.  Each is exact only because the host
bounds how many samples one launch, or one CTA, may put into it.  Here every one of those cells gets close to its bound
in one launch, so a missing split, a narrowing cast or a sign extension in a flush shows as a wrong bucket.

Inputs of 2^33 to 2^37 samples are aliased device memory: one physical allocation of GRANULE bytes, filled once with a
pattern of period L, mapped again and again over a reserved virtual range (the CUDA virtual memory management driver
API).  Element i of such an array is pattern[(offset + i) % L], so the exact result of n samples is
q * oracle(one period) + oracle(first r samples of the period), n = q * L + r, with the period rotated to the offset.

Each case checks every bucket of the touched rows, the reduced counts and percentiles against oracle.process_histogram,
the dropped tally, and the number of kernel launches the host's per-launch bound implies."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import _ingest_routes as R

pytestmark = pytest.mark.gpu

SEED = 0x2_0032
PS = [0.0, 0.5, 0.99, 1.0]
PREC = 100                     # the oracle's keyed ingest is at precision 100
L = 1 << 18                    # period of every pattern, in samples
SPARSE = 4096                  # one special value (and one dropped id) per SPARSE samples of a period
GRANULE = 32 << 20             # bytes of the physical allocation behind each aliased array
U32_MAX = (1 << 32) - 1
SMEM_PER_SM = 228 * 1024       # H100: shared memory of one SM, of which each resident CTA takes 1 KiB more
MAX_THREADS_PER_SM = 2048


def _batch_constants():
    k = R._src("lh_kernels.cuh")
    return {"threads": R._int_expr(k, r"constexpr int BI_THREADS = ([^;]+);", {}),
            "entries": R._int_expr(k, r"constexpr uint32_t BI_TABLE_ENTRIES = ([^;]+);", {}),
            "items": R._int_expr(k, r"constexpr int BI_MAX_ITEMS = ([^;]+);", {}),
            "k1_min": R._int_expr(R._src("lh_api.cu"), r"constexpr size_t kBatchK1Min = ([^;]+);", {})}


BI = _batch_constants()


def ctas_per_sm(threads: int, smem: int) -> int:
    """The most CTAs of `threads` threads and `smem` bytes of dynamic shared memory one SM can hold, by threads and
    shared memory (registers can only lower it)."""
    return max(1, min(MAX_THREADS_PER_SM // threads, SMEM_PER_SM // (smem + 1024)))


def k1_launches(n: int, grid: int) -> int:
    """launch_single: pieces of at most min(2^36, grid << 31) samples."""
    per = min(1 << 36, grid << 31)
    return -(-n // per)


def batch_cap(grid_max: int) -> int:
    return min(1 << 36, grid_max << 31)


def batch_launches(items, grid_max: int, k1_grid: int) -> int:
    """launch_batch over items [(n, kind)]: K1 for float64 items of at least kBatchK1Min samples, the rest packed into
    launches of k_ingest_batch of at most BI_MAX_ITEMS segments and batch_cap samples."""
    cap, launches, k, total = batch_cap(grid_max), 0, 0, 0
    for n, kind in items:
        if kind == "f64" and n >= BI["k1_min"]:
            launches += k1_launches(n, k1_grid)
            continue
        while n:
            if k == BI["items"] or total == cap:
                launches, k, total = launches + 1, 0, 0
            m = min(n, cap - total)
            total, k, n = total + m, k + 1, n - m
    return launches + (1 if k else 0)


# ------------------------------------------------------------------------------------------------ aliased arrays
class _Location(C.Structure):
    _fields_ = [("type", C.c_int), ("id", C.c_int)]


class _AllocFlags(C.Structure):
    _fields_ = [("compressionType", C.c_ubyte), ("gpuDirectRDMACapable", C.c_ubyte), ("usage", C.c_ushort),
                ("reserved", C.c_ubyte * 4)]


class _AllocationProp(C.Structure):          # CUmemAllocationProp_v1
    _fields_ = [("type", C.c_int), ("requestedHandleTypes", C.c_int), ("location", _Location),
                ("win32HandleMetaData", C.c_void_p), ("allocFlags", _AllocFlags)]


class _AccessDesc(C.Structure):              # CUmemAccessDesc_v1
    _fields_ = [("location", _Location), ("flags", C.c_int)]


_CU_MEM_ALLOCATION_TYPE_PINNED, _CU_MEM_LOCATION_TYPE_DEVICE, _CU_MEM_ACCESS_FLAGS_PROT_READWRITE = 1, 1, 3


class _Driver:
    def __init__(self):
        assert C.sizeof(_AllocationProp) == 32 and C.sizeof(_AccessDesc) == 12
        cu = C.CDLL("libcuda.so.1")
        u64, sz, vp = C.c_uint64, C.c_size_t, C.c_void_p
        sigs = {"cuMemAddressReserve": [C.POINTER(u64), sz, sz, u64, C.c_ulonglong],
                "cuMemAddressFree": [u64, sz],
                "cuMemCreate": [C.POINTER(u64), sz, C.POINTER(_AllocationProp), C.c_ulonglong],
                "cuMemRelease": [u64],
                "cuMemMap": [u64, sz, sz, u64, C.c_ulonglong],
                "cuMemUnmap": [u64, sz],
                "cuMemSetAccess": [u64, sz, C.POINTER(_AccessDesc), sz],
                "cuMemGetAllocationGranularity": [C.POINTER(sz), C.POINTER(_AllocationProp), C.c_int],
                "cuMemcpyHtoD_v2": [u64, vp, sz]}
        for name, args in sigs.items():
            f = getattr(cu, name)
            f.argtypes, f.restype = args, C.c_int
            setattr(self, name, f)
        self.prop = _AllocationProp()
        self.prop.type = _CU_MEM_ALLOCATION_TYPE_PINNED
        self.prop.location = _Location(_CU_MEM_LOCATION_TYPE_DEVICE, 0)
        self.access = _AccessDesc(_Location(_CU_MEM_LOCATION_TYPE_DEVICE, 0), _CU_MEM_ACCESS_FLAGS_PROT_READWRITE)

    def check(self, rc, what):
        assert rc == 0, "%s failed: CUresult %d" % (what, rc)


_PEAK = {"used": 0}


@pytest.fixture(scope="module")
def drv():
    import torch
    torch.zeros(1, device="cuda:0")                 # the primary context, current on this thread
    d = _Driver()
    gran = C.c_size_t()
    d.check(d.cuMemGetAllocationGranularity(C.byref(gran), C.byref(d.prop), 0), "cuMemGetAllocationGranularity")
    assert gran.value and GRANULE % gran.value == 0, gran.value
    free0, total = torch.cuda.mem_get_info(0)
    yield d
    print("\npeak device memory above the start of the module while aliased arrays were mapped: %.1f MiB "
          "(%.1f MiB in use at its start)" % (_PEAK["used"] / 2 ** 20, (total - free0) / 2 ** 20))


@contextlib.contextmanager
def aliased(drv, pattern: np.ndarray, n: int, offset: int = 0):
    """Device address of an n-element array whose element i is pattern[(offset + i) % pattern.size]: one physical
    allocation of GRANULE bytes holding the pattern repeated, mapped over and over across a reserved range.  Everything
    is unmapped and released on exit, after the device has finished."""
    import torch
    item = pattern.dtype.itemsize
    assert GRANULE % (pattern.size * item) == 0
    size = -(-(offset + n) * item // GRANULE) * GRANULE
    base, handle = C.c_uint64(0), C.c_uint64(0)
    reserved = created = False
    mapped = 0
    try:
        drv.check(drv.cuMemAddressReserve(C.byref(base), size, GRANULE, 0, 0), "cuMemAddressReserve of %d GiB" % (size >> 30))
        reserved = True
        drv.check(drv.cuMemCreate(C.byref(handle), GRANULE, C.byref(drv.prop), 0), "cuMemCreate")
        created = True
        for off in range(0, size, GRANULE):
            drv.check(drv.cuMemMap(base.value + off, GRANULE, 0, handle.value, 0), "cuMemMap")
            mapped += 1
        drv.check(drv.cuMemSetAccess(base.value, size, C.byref(drv.access), 1), "cuMemSetAccess")
        host = np.ascontiguousarray(np.tile(pattern, GRANULE // (pattern.size * item)))
        drv.check(drv.cuMemcpyHtoD_v2(base.value, host.ctypes.data, GRANULE), "cuMemcpyHtoD")
        free, total = torch.cuda.mem_get_info(0)
        _PEAK["used"] = max(_PEAK["used"], total - free)
        yield base.value + offset * item
    finally:
        torch.cuda.synchronize()
        for i in range(mapped):
            drv.check(drv.cuMemUnmap(base.value + i * GRANULE, GRANULE), "cuMemUnmap")
        if created:
            drv.check(drv.cuMemRelease(handle.value), "cuMemRelease")
        if reserved:
            drv.check(drv.cuMemAddressFree(base.value, size), "cuMemAddressFree")


class DevArray:
    """n elements at a raw device address, as a __cuda_array_interface__ object."""

    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


# ------------------------------------------------------------------------------------------------------ patterns
def special_values(oracle) -> np.ndarray:
    """Samples the fast paths must not bin as the common value: negatives, values past the window, NaNs, +-Inf, zeros,
    the smallest subnormal, and bucket thresholds and their predecessors (one ulp below)."""
    T = R.thresholds(oracle, PREC, R.window(PREC) - 1).view(np.float64)
    t = T[[5, 400, 1500, 2900, 3600, 4300]]
    return np.concatenate([[-1000.0, -1.5, -(2.0 ** 70), 2.0 ** 63, 2.0 ** 64, 1e300, np.nan, -np.nan,
                            np.uint64(0x7FF0000000000123).view(np.float64), np.inf, -np.inf, 0.0, -0.0, 5e-324],
                           t, np.nextafter(t, 0.0)])


NS_SPECIALS = np.array([-1, -1000, 0, 1, np.iinfo(np.int64).min, np.iinfo(np.int64).max, (1 << 53) + 1, 10 ** 12,
                        -(10 ** 15), 999, 1001], np.int64)


def sprinkle(base: np.ndarray, specials: np.ndarray, seed: int) -> np.ndarray:
    """`base` with L // SPARSE of its positions, chosen at random, replaced by the specials in turn."""
    rng = np.random.default_rng(seed)
    out = base.copy()
    pos = rng.choice(base.size, base.size // SPARSE, replace=False)
    out[pos] = specials[np.arange(pos.size) % specials.size]
    return out


def value_pattern(oracle, v: float, seed: int) -> np.ndarray:
    return sprinkle(np.full(L, v, np.float64), special_values(oracle), seed)


def ns_pattern(ns: int, seed: int) -> np.ndarray:
    return sprinkle(np.full(L, ns, np.int64), NS_SPECIALS, seed)


def id_pattern(base: np.ndarray, bad, dtype, seed: int) -> np.ndarray:
    """ids `base` (one period) with a sprinkle of ids >= H, which must be dropped and counted."""
    return sprinkle(base.astype(np.uint32), np.asarray(bad, np.uint32), seed).astype(dtype)


def periodic(n: int, offset: int, hist_of, *patterns):
    """hist_of(*arrays) over n samples starting `offset` into the periodic patterns: q * hist(period) + hist(head of
    the period), q, r = divmod(n, L), each pattern rotated to start at `offset`."""
    q, r = divmod(n, L)
    rot = [np.roll(p, -offset) for p in patterns]
    return hist_of(*rot) * np.uint64(q) + hist_of(*[p[:r] for p in rot])


# ---------------------------------------------------------------------------------------------------- checking
@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def check(e, oracle, H, want: dict, dropped: int, before: dict, launches=None, allowed=None, what=""):
    """One collection: the rows in `want` ({row: dense uint64[65536]}) bucket for bucket, every other row empty, the
    reduced counts, percentile keys and values bit for bit against oracle.process_histogram, the dropped tally since
    `before`, then `launches` (the kernel launches of the ingest call) against the set the host's bounds allow."""
    red, sp = e.snapshot(PS)
    e.sync()
    st = e.stats()
    offs = sp.offsets.astype(np.int64)
    empty = [h for h in range(H) if h not in want and offs[h + 1] != offs[h]]
    assert not empty, (what, "rows written that should be empty", empty[:5])
    for h, w in want.items():
        got = np.zeros(65536, np.uint64)
        got[sp.keys[offs[h]:offs[h + 1]].view(np.uint16)] = sp.counts[offs[h]:offs[h + 1]]
        bad = np.nonzero(got != w)[0]
        assert bad.size == 0, (what, h, [(int(k), int(got[k]), int(w[k]), int(w[k]) - int(got[k])) for k in bad[:5]])
        ref = oracle.process_histogram(w, PS, PREC)
        assert int(red.counts[h]) == ref["total"] == int(w.sum()), (what, h)
        assert (red.pkeys[h] == ref["pkeys"]).all(), (what, h, red.pkeys[h], ref["pkeys"])
        assert (red.pvals[h].view(np.uint64) == ref["pvals"].view(np.uint64)).all(), (what, h)
    others = np.ones(H, bool)
    others[list(want)] = False
    assert (red.counts[others] == 0).all(), what
    assert st["dropped"] - before["dropped"] == dropped, (what, st["dropped"] - before["dropped"], dropped)
    if allowed is not None:
        assert launches in allowed, (what, launches, sorted(allowed))


def dense(hist):
    return {h: hist[h] for h in range(hist.shape[0]) if hist[h].any()}


# ----------------------------------------------------------------------------------------------------------- K1
K1_COUNTING = [i for i, v in enumerate(R.CONST["K1_VARIANTS"]) if not v["probe"]]


@pytest.mark.parametrize("variant", K1_COUNTING)
def test_k1_sub_histograms_near_2_31(lh, oracle, drv, sms, variant):
    """K1 on one SM (k1_reserve_sms = sm_count - 1), so that grid << 31 bounds a launch: n = 2^33 + 2^20 + 3 samples
    from 8 bytes past a 32-byte boundary.  One SM holds one or two CTAs of any K1 variant (shared memory, or registers
    for the 512-thread kernel), so without the split some CTA cell would pass 2^32; with it, each hot cell reaches about
    2^31 per launch."""
    n = (1 << 33) + (1 << 20) + 3
    pat = value_pattern(oracle, 4.2e5, SEED ^ variant)
    want = periodic(n, 1, lambda v: oracle.ingest(v), pat)
    assert want.max() > 1 << 32
    H, hid = 2, 1
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, aliased(drv, pat, n, 1) as d_v:
        assert d_v % 32 == 8
        e.tune("k1", variant)
        e.tune("k1_reserve_sms", sms - 1)
        before = e.stats()
        e.ingest_f64(hid, d_v, n)
        launches = e.stats()["kernel_launches"] - before["kernel_launches"]
        check(e, oracle, H, {hid: want}, 0, before, launches, {k1_launches(n, g) for g in (1, 2)}, ("k1", variant))


# -------------------------------------------------------------------------------------------------- keyed (WC)
KEYED_H = 32
KEYED_N = (1 << 37) + (1 << 27) + 12_345


def wc_launches(n, sms, *, id_bytes, k1_reserve_sms, vals_addr=0, ids_addr=0):
    """Kernel launches of one keyed call routed to the write-combining kernel, from the route of every piece."""
    pieces = R.keyed_pieces(KEYED_H, n, PREC, sms, id_bytes=id_bytes, vals_addr=vals_addr, ids_addr=ids_addr,
                            k1_reserve_sms=k1_reserve_sms, keyed_mode=2)
    assert all(r.kernel == R.WC for _, r in pieces), pieces
    assert all(m <= R.CONST["WC_MAX_LAUNCH"] for m, _ in pieces)
    return len(pieces), sum(R.keyed_launches(m, r) for m, r in pieces)


@pytest.mark.parametrize("variant", ["f64_u16", "f64_u32", "i64ns_u16", "mapped_u16"])
def test_keyed_wc_owner_cells_past_2_32(lh, oracle, drv, sms, variant):
    """The write-combining kernel with P = 32 owners (k1_reserve_sms = sm_count - 32, keyed_mode 2), H = 32, ids i % 32:
    every owner holds one id, whose hot cell gets more than 2^32 samples over the call.  The owner windows are uint32
    and flushed once per launch, so the call must go out in pieces of at most 2^32 - 1 samples."""
    assert sms >= 40
    reserve = sms - 32
    H = KEYED_H
    id_dtype, bad = (np.uint32, R.high_ids(H, 7)) if variant == "f64_u32" else (np.uint16, [H, 65535])
    ids = id_pattern(np.arange(L) % H, bad, id_dtype, SEED + 1)
    if variant == "i64ns_u16":
        vals = ns_pattern(1000, SEED + 2)
        hist_of = lambda i, v: oracle.ingest_keyed_i64(i[i < H], v[i < H], H)
    else:
        vals = value_pattern(oracle, 1000.0, SEED + 2)
        hist_of = lambda i, v: oracle.ingest_keyed(i[i < H], v[i < H], H)
    n = KEYED_N
    want = periodic(n, 0, hist_of, ids, vals)
    dropped = int(periodic(n, 0, lambda i: np.array([(i >= H).sum()], np.uint64), ids)[0])
    assert want.max() > 1 << 32 and dropped > 0
    rows = np.arange(H)
    E = H
    if variant == "mapped_u16":                  # 32 local ids onto scattered rows of a larger context
        E = 1000
        rows = np.random.default_rng(SEED).choice(E, H, replace=False)
    pieces, launches = wc_launches(n, sms, id_bytes=np.dtype(id_dtype).itemsize, k1_reserve_sms=reserve)
    from loghisto_b200 import _lib
    assert pieces >= 33
    with lh.Engine(device=0, max_histograms=E, max_counters=1, precision=PREC) as e, \
            aliased(drv, ids, n) as d_i, aliased(drv, vals, n) as d_v:
        e.tune("k1_reserve_sms", reserve)
        e.tune("keyed_mode", 2)
        before = e.stats()
        if variant == "mapped_u16":
            e.ingest_keyed_mapped_u16([int(r) for r in rows], d_i, d_v, _lib.LH_VALUES_F64, n)
        else:
            getattr(e, "ingest_keyed_" + variant)(d_i, d_v, n)
        got = e.stats()["kernel_launches"] - before["kernel_launches"]
        assert e.keyed_kernel_name() == R.WC
        check(e, oracle, E, {int(rows[h]): want[h] for h in range(H)}, dropped, before, got, {launches}, ("keyed", variant))


def test_keyed_pair_owner_cells_past_2_32(lh, oracle, drv, sms):
    """lh_ingest_keyed_pair_u16 with n_f64 = n_ns = 2^36 + delta, the same ids for both and values 1000.0 and 1000 ns
    (one bucket): the hot cell of every owner gets more than 2^32 samples of the two arrays together.  One fused
    write-combining launch would wrap it; the pair must go apart, each array in pieces of at most 2^32 - 1."""
    assert sms >= 40
    reserve = sms - 32
    H = KEYED_H
    n = (1 << 36) + (1 << 26) + 777
    ids = id_pattern(np.arange(L) % H, [H, 65535], np.uint16, SEED + 3)
    vals = value_pattern(oracle, 1000.0, SEED + 4)
    ns = ns_pattern(1000, SEED + 5)
    assert oracle.compress(1000.0) == oracle.compress(float(1000))
    want = periodic(n, 0, lambda i, v: oracle.ingest_keyed(i[i < H], v[i < H], H), ids, vals) + \
        periodic(n, 0, lambda i, v: oracle.ingest_keyed_i64(i[i < H], v[i < H], H), ids, ns)
    dropped = 2 * int(periodic(n, 0, lambda i: np.array([(i >= H).sum()], np.uint64), ids)[0])
    assert want.max() > 1 << 32
    route = R.pair_route(H, n, n, PREC, sms, k1_reserve_sms=reserve, keyed_mode=2)
    assert route.extra.get("apart") and route.kernel == R.WC
    launches = 2 * wc_launches(n, sms, id_bytes=2, k1_reserve_sms=reserve)[1]
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, \
            aliased(drv, ids, n) as d_i, aliased(drv, vals, n) as d_v, aliased(drv, ns, n) as d_n:
        e.tune("k1_reserve_sms", reserve)
        e.tune("keyed_mode", 2)
        before = e.stats()
        e.ingest_keyed_pair_u16(d_i, d_v, n, d_i, d_n, n)
        got = e.stats()["kernel_launches"] - before["kernel_launches"]
        assert e.keyed_kernel_name() == R.WC
        check(e, oracle, H, dense(want), dropped, before, got, {launches}, "pair")


# ------------------------------------------------------------------------------------- batch and graph recorder
def batch_grid_max(sms):
    """batch_grid_max at k1_reserve_sms = sm_count - 1: the CTAs of k_ingest_batch one SM holds (its launch bounds ask
    for two, and its table leaves room for no more)."""
    g = ctas_per_sm(BI["threads"], 12 * BI["entries"])
    assert g == 2, g
    return g


def test_batch_table_slots_near_2_31(lh, oracle, drv, sms):
    """lh_ingest_batch on one SM: short float64 items, one int64 item of 2 * batch_cap + delta samples and a float64
    item for K1.  Every launch of k_ingest_batch carries batch_cap = grid << 31 samples, so each CTA's table slot of the
    hot bucket reaches about 2^31 before its one flush."""
    H = 4
    grid = batch_grid_max(sms)
    cap = batch_cap(grid)
    vals = value_pattern(oracle, 4.2e5, SEED + 6)
    ns = ns_pattern(123_456_789, SEED + 7)
    n_big, n_k1 = 2 * cap + (1 << 20) + 5, BI["k1_min"] + 9
    shorts = [(0, 1, 1000), (0, 3, 4097), (3, 5, 77), (3, 0, 60_000)]        # (histogram, offset, n) of float64 items
    items = [("f64", hid, off, m) for hid, off, m in shorts[:2]] + [("ns", 1, 0, n_big), ("f64", 2, 1, n_k1)] + \
        [("f64", hid, off, m) for hid, off, m in shorts[2:]]
    want = np.zeros((H, 65536), np.uint64)
    for kind, hid, off, m in items:
        if kind == "ns":
            want[hid] += periodic(m, off, lambda v: oracle.ingest_keyed_i64(np.zeros(v.size, np.uint32), v, 1)[0], ns)
        else:
            want[hid] += periodic(m, off, lambda v: oracle.ingest(v), vals)
    assert want[1].max() > 1 << 32
    k1_grid_bound = {k1_launches(n_k1, g) for g in range(1, 5)}
    assert k1_grid_bound == {1}
    launches = batch_launches([(m, kind) for kind, _, _, m in items], grid, 1)
    assert launches == 4, launches
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, \
            aliased(drv, vals, n_k1 + 8) as d_v, aliased(drv, ns, n_big) as d_n:
        e.tune("k1_reserve_sms", sms - 1)
        arrays = []
        for kind, hid, off, m in items:
            if kind == "ns":
                arrays.append((hid, DevArray(d_n + 8 * off, m, "<i8")))
            else:
                arrays.append((hid, DevArray(d_v + 8 * off, m, "<f8")))
        before = e.stats()
        e.ingest_batch(arrays)
        got = e.stats()["kernel_launches"] - before["kernel_launches"]
        check(e, oracle, H, dense(want), 0, before, got, {launches}, "batch")


def test_graph_recorder_keyed_table_slots_near_2_31(lh, oracle, drv, sms):
    """k_ingest_keyed_graph on one SM: 2 * batch_cap + delta keyed samples, almost all into local id 0, captured once
    into a CUDA graph and replayed 1 then 2 times, one collection after each: every collection == R x the want, and
    each replay's CTAs fill one table slot to about 2^31."""
    import torch
    H, k = 6, 3
    hmap = [5, 0, 2]
    grid = batch_grid_max(sms)
    n = 2 * batch_cap(grid) + (1 << 20) + 11
    ids = id_pattern(np.where(np.arange(L) % 997 == 0, 1, np.where(np.arange(L) % 1009 == 0, 2, 0)), [k, 65535],
                     np.uint16, SEED + 8)
    vals = value_pattern(oracle, 7.5e3, SEED + 9)
    local = periodic(n, 0, lambda i, v: oracle.ingest_keyed(i[i < k], v[i < k], k), ids, vals)
    dropped = int(periodic(n, 0, lambda i: np.array([(i >= k).sum()], np.uint64), ids)[0])
    want = {hmap[i]: local[i] for i in range(k)}
    assert local.max() > 1 << 32
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, \
            aliased(drv, ids, n) as d_i, aliased(drv, vals, n) as d_v:
        e.tune("k1_reserve_sms", sms - 1)
        with e.graph_recorder(hmap) as gr:
            before = e.stats()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.Stream()):
                gr.keyed(DevArray(d_i, n, "<u2"), DevArray(d_v, n, "<f8"))
            torch.cuda.synchronize()
            captured = e.stats()["kernel_launches"] - before["kernel_launches"]
            assert captured == -(-n // batch_cap(grid)) == 3, captured
            for reps in (1, 2):
                before = e.stats()
                for _ in range(reps):
                    g.replay()
                torch.cuda.synchronize()
                check(e, oracle, H, {h: w * np.uint64(reps) for h, w in want.items()}, reps * dropped, before,
                      what=("graph", reps))
            del g


# --------------------------------------------------------------------------------------------- device API edges
@pytest.fixture(scope="module")
def clients():
    from loghisto_b200 import _lib, build
    rp, vp, sz, u32 = C.POINTER(_lib.lh_recorder), C.c_void_p, C.c_size_t, C.c_uint32
    for path in (build.CLIENT_LIB, build.BLOCK_CLIENT_LIB):
        assert os.path.exists(path), "build() did not produce " + path
    dev, blk = C.CDLL(build.CLIENT_LIB), C.CDLL(build.BLOCK_CLIENT_LIB)
    dev.lhc_block.argtypes = [rp, vp, vp, sz, sz, vp]
    blk.brc_record.argtypes = [rp, vp, vp, sz, sz, u32, C.c_int, vp]
    dev.lhc_set_device.argtypes = blk.brc_set_device.argtypes = [C.c_int]
    for f in (dev.lhc_block, blk.brc_record, dev.lhc_set_device, blk.brc_set_device):
        f.restype = C.c_int
    assert dev.lhc_set_device(0) == 0 and blk.brc_set_device(0) == 0
    return dev, blk


def test_block_histogram_flushes_of_2_32_minus_1(lh, oracle, drv, clients):
    """lh::BlockHistogram at its contract's edge: 2 CTAs, each with a chunk of 2 * (2^32 - 1) samples, flushing after
    each half, so every flush carries exactly 2^32 - 1 adds, almost all in one cell."""
    dev, _ = clients
    chunk = 2 * U32_MAX
    n = 2 * chunk
    H = 3
    vals = value_pattern(oracle, 3.3e4, SEED + 10)
    block_ids = np.array([2, 0], np.uint32)
    want = {int(block_ids[b]): periodic(chunk, (b * chunk) % L, lambda v: oracle.ingest(v), vals) for b in range(2)}
    assert all(w.max() > 2 * (1 << 31) and int(w.sum()) == chunk for w in want.values())
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, aliased(drv, vals, n) as d_v:
        d_b = e.upload(block_ids)
        before = e.stats()
        with e.recording() as rec:
            assert dev.lhc_block(C.byref(rec), d_b.ptr, d_v, n, chunk, e.ingest_stream) == 0
        check(e, oracle, H, want, 0, before, what="BlockHistogram")


def test_block_recorder_flush_of_2_32_minus_1(lh, oracle, drv, clients):
    """lh::BlockRecorder (64 slots, no mid-chunk flush) at its contract's edge: 2 CTAs of 2^32 - 1 records each, so the
    one flush of each CTA carries 2^32 - 1 counts, almost all in one slot."""
    _, blk = clients
    chunk = U32_MAX
    n = 2 * chunk
    H = 4
    ids = id_pattern(np.where(np.arange(L) % 499 == 0, 3, 1), [H, 65536 + 1, U32_MAX], np.uint32, SEED + 11)
    vals = value_pattern(oracle, 2.5e2, SEED + 12)
    local = periodic(n, 0, lambda i, v: oracle.ingest_keyed(i[i < H], v[i < H], H), ids, vals)
    dropped = int(periodic(n, 0, lambda i: np.array([(i >= H).sum()], np.uint64), ids)[0])
    assert local.max() > 1 << 32 and dropped > 0
    with lh.Engine(device=0, max_histograms=H, max_counters=1, precision=PREC) as e, \
            aliased(drv, ids, n) as d_i, aliased(drv, vals, n) as d_v:
        before = e.stats()
        with e.recording() as rec:
            assert blk.brc_record(C.byref(rec), d_i, d_v, n, chunk, 64, 0, e.ingest_stream) == 0
        check(e, oracle, H, dense(local), dropped, before, what="BlockRecorder")
