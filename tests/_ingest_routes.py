"""The host's ingest dispatch (loghisto_b200/csrc/lh_api.cu) restated in Python, plus builders of batches with known
properties.

`keyed_route` / `pair_route` / `counter_route` / `k1_variants` return what the library should run for a configuration:
the kernel, and for the write-combining kernel the launch shape (P, ids per owner, owner-buffer records `row_cap`,
`flush_tiles`, `slice_tiles`, chunks and the per-(owner, writer) sub-queue `cap`).  The constants they use are read
from the CUDA sources, so a change to any of them changes the prediction (or fails the parse) instead of silently
leaving a test on the wrong side of a boundary.  Nothing here needs a GPU.
"""
from __future__ import annotations

import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "loghisto_b200", "csrc")
_LN2 = 0.6931471805599453094172321


def _src(name: str) -> str:
    with open(os.path.join(_CSRC, name)) as f:
        return f.read()


def _int_expr(text: str, pattern: str, env: dict) -> int:
    m = re.search(pattern, text)
    if not m:
        raise AssertionError("dispatch constant not found in the CUDA sources: " + pattern)
    expr = m.group(1)
    if not re.fullmatch(r"[\w\s*+()]+", expr):
        raise AssertionError("unexpected form of a dispatch constant: " + expr)
    return int(eval(expr, {"__builtins__": {}}, dict(env)))


def _parse_constants() -> dict:
    k, a = _src("lh_kernels.cuh"), _src("lh_api.cu")
    c = {}
    c["K2_SMEM_COUNTERS"] = _int_expr(k, r"constexpr int K2_SMEM_COUNTERS = ([^;]+);", c)
    c["KS_SMEM_BYTES"] = _int_expr(k, r"constexpr int KS_SMEM_BYTES = ([^;]+);", c)
    c["KS_THREADS"] = _int_expr(k, r"constexpr int KS_THREADS = ([^;]+);", c)
    c["WC_MAX_PARTS"] = _int_expr(k, r"constexpr int WC_MAX_PARTS = ([^;]+);", c)
    c["WC_LINE"] = _int_expr(k, r"constexpr int WC_LINE = ([^;]+);", c)
    c["WC_ROW_EXTRA"] = _int_expr(k, r"constexpr int WC_ROW_EXTRA = ([^;]+);", c)
    c["WC_RARE_CAP"] = _int_expr(k, r"constexpr uint32_t WC_RARE_CAP = ([^;]+);", c)
    c["KS_MAX_PASSES"] = _int_expr(a, r"constexpr uint32_t KS_MAX_PASSES = ([^;]+);", c)
    c["kSmemBudget"] = _int_expr(a, r"constexpr size_t kSmemBudget = ([^;]+);", c)
    c["kDefaultK1Variant"] = _int_expr(a, r"constexpr int kDefaultK1Variant = ([^;]+);", c)
    m = re.search(r"constexpr size_t kWcMaxLaunch = 0x([0-9A-Fa-f]+)u;", a)
    if not m:
        raise AssertionError("dispatch constant not found in the CUDA sources: kWcMaxLaunch")
    c["WC_MAX_LAUNCH"] = int(m.group(1), 16)
    # the owner-buffer sizes launch_keyed_wc_spt tries, largest first
    m = re.search(r"for \(uint32_t cap_try : \{([^}]*)\}\)", a)
    c["WC_ROW_CAPS"] = tuple(int(x.strip().rstrip("u")) for x in m.group(1).split(","))
    # the K1 variant table and the substitution order of lh_create
    body = re.search(r"K1Variant g_k1_variants\[\] = \{(.*?)\n\};", a, re.S).group(1)
    variants = []
    for line in body.splitlines():
        line = line.split("//")[0].strip()
        if not line:
            continue
        if line.startswith("BULK_VARIANT("):
            w, s, b, mb, f = (int(x) for x in re.match(r"BULK_VARIANT\(([^)]*)\)", line).group(1).split(","))
            variants.append({"name": "bulk2_w%d_s%d_%d_b%d_sign%d" % (w, s, b, mb, f), "smem_fixed": s * b + s * 16,
                             "probe": False})
        elif line.startswith("LDG_VARIANT("):
            t, u, mb = (int(x) for x in re.match(r"LDG_VARIANT\(([^)]*)\)", line).group(1).split(","))
            variants.append({"name": "ldg_t%d_u%d_b%d" % (t, u, mb), "smem_fixed": 0, "probe": False})
        elif line.startswith("{"):
            name = re.match(r'\{\s*"([^"]+)"', line).group(1)
            variants.append({"name": name, "smem_fixed": 0, "probe": "launch_probe" in line})
        else:
            raise AssertionError("unrecognised K1 variant entry: " + line)
    c["K1_VARIANTS"] = variants
    m = re.search(r"static const int smaller\[\] = \{([^}]*)\};", a)
    c["K1_SMALLER"] = tuple(int(x) for x in m.group(1).split(","))
    # WcShape: shape code -> threads, samples per thread
    m = re.search(r"THREADS = SPT == 4 \? (\d+) : SPT == 6 \? (\d+) : SPT == 3 \? (\d+) : (\d+);", k)
    t4, t6, t3, t8 = (int(x) for x in m.groups())
    m = re.search(r"PER = SPT == 8 \? (\d+) : (\d+);", k)
    per8, per = int(m.group(1)), int(m.group(2))
    c["WC_SHAPES"] = {4: (t4, per), 6: (t6, per), 3: (t3, per), 8: (t8, per8)}
    return c


CONST = _parse_constants()

# keyed_kernel_name() of each route
SMALL, WC, VEC, SCALAR = "k_ingest_keyed_small", "k_ingest_keyed_wc", "k_ingest_keyed_vec", "k_ingest_keyed"
COUNTER_SMEM, COUNTER_GLOBAL = "k_counter_add_smem", "k_counter_add"

# the library's tuning defaults (lh_ctx)
DEFAULTS = dict(keyed_mode=0, k1_reserve_sms=0, kp_chunk=256 << 20, wc_spt=6, wc_flush=24576)


def window(precision: int) -> int:
    """Prec.win: cells of one histogram's positive window (make_prec)."""
    return int(math.floor(precision * 63.0 * _LN2 + 0.5)) + 1


def a_int(precision: int) -> int:
    return int(math.floor(precision * _LN2))


def ks_ids_per_pass(precision: int) -> int:
    return max(1, CONST["KS_SMEM_BYTES"] // (window(precision) * 4))


def small_passes(H: int, precision: int) -> int:
    per = ks_ids_per_pass(precision)
    return (H + per - 1) // per


@dataclass
class WcShape:
    P: int
    ids_per: int
    row_cap: int
    smem: int
    flush_tiles: int = 0
    slice_tiles: int = 0
    nchunks: int = 0
    cap: int = 0
    tile: int = 0
    taken: int = 0          # samples the launch bins (whole tiles); the rest goes to the scalar kernel
    taken2: int = 0         # ... of the int64 segment of a fused pair launch


def wc_geometry(H: int, precision: int, sm_count: int, k1_reserve_sms: int = 0):
    """(P, ids_per, row_cap, smem) of the write-combining kernel, or None when it cannot hold these histograms."""
    P = min(sm_count - k1_reserve_sms, CONST["WC_MAX_PARTS"])
    if P < 8:
        return None
    win = window(precision)
    ids_per = (H + P - 1) // P
    hist_bytes = ((ids_per * win + 3) & ~3) * 4
    for cap_try in CONST["WC_ROW_CAPS"]:
        smem = hist_bytes + 2 * CONST["WC_MAX_PARTS"] * 4 + (P + 1) * (cap_try + CONST["WC_ROW_EXTRA"]) * 2
        if smem <= CONST["kSmemBudget"]:
            break
    else:
        return None
    if ids_per * win > 65535:
        return None
    return P, ids_per, cap_try, smem


def wc_launch(H: int, precision: int, sm_count: int, n_samples: int, n2: int = 0, *, k1_reserve_sms=0, keyed_mode=0,
              kp_chunk=DEFAULTS["kp_chunk"], wc_spt=DEFAULTS["wc_spt"], wc_flush=DEFAULTS["wc_flush"]):
    """launch_keyed_wc_spt for n_samples vector-body samples (and n2 int64 samples of a fused pair, a second segment):
    a WcShape, or None when it declines.  Each segment is cut to whole tiles on its own."""
    geo = wc_geometry(H, precision, sm_count, k1_reserve_sms)
    if geo is None or n_samples + n2 == 0:
        return None
    P, ids_per, row_cap, smem = geo
    if keyed_mode != 2 and n_samples + n2 < (1 << 22):
        return None
    threads, per = CONST["WC_SHAPES"].get(wc_spt, CONST["WC_SHAPES"][8])
    tile = threads * per
    taken, taken2 = n_samples // tile * tile, n2 // tile * tile
    if taken + taken2 == 0:
        return None
    slice_max = max(1, (kp_chunk + P * tile - 1) // (P * tile))
    tiles_all = (taken + taken2) // tile
    nchunks = (tiles_all + slice_max * P - 1) // (slice_max * P)
    slice_tiles = max(1, (tiles_all + nchunks * P - 1) // (nchunks * P))
    expect = slice_max * tile // P
    line = CONST["WC_LINE"]
    cap = ((expect * 5 // 4 + 3 * line + line - 1) // line) * line
    room = row_cap - 63.0
    m_max = ((-3.5 + math.sqrt(3.5 * 3.5 + 4.0 * room)) / 2.0) ** 2
    flush_samples = min(wc_flush, int(m_max * P))
    flush_tiles = max(1, flush_samples // tile)
    return WcShape(P, ids_per, row_cap, smem, flush_tiles, slice_tiles, nchunks, cap, tile, taken, taken2)


@dataclass
class Route:
    kernel: str                       # what keyed_kernel_name() reports after the call
    vec_samples: int = 0              # samples of the aligned vector body
    head: int = 0                     # samples of the scalar head
    passes: int = 0                   # k_ingest_keyed_small passes
    wc: WcShape | None = None
    extra: dict = field(default_factory=dict)


def keyed_route(H: int, n: int, precision: int, sm_count: int, *, id_bytes=2, vals_addr=0, ids_addr=0,
                previous: str = "", **tune) -> Route:
    """launch_keyed for one call whose hot window starts drained (the call is not split by the fold guard).
    vals_addr / ids_addr: the pointers modulo 32 (device allocations are 256-byte aligned)."""
    t = dict(DEFAULTS, **tune)
    head = min(n, ((32 - (vals_addr & 31)) & 31) // 8)
    vec_ok = ((ids_addr + head * id_bytes) & (4 * id_bytes - 1)) == 0
    n4 = (n - head) // 4 if vec_ok else 0
    if not vec_ok:
        head = 0
    if n4 == 0:
        return Route(SCALAR if n else previous, 0, head)
    passes = small_passes(H, precision)
    if passes <= CONST["KS_MAX_PASSES"] and t["keyed_mode"] == 0 and n4 >= 4096:
        return Route(SMALL, n4 * 4, head, passes=passes)
    if t["keyed_mode"] != 1:
        wc = wc_launch(H, precision, sm_count, n4 * 4, k1_reserve_sms=t["k1_reserve_sms"], keyed_mode=t["keyed_mode"],
                       kp_chunk=t["kp_chunk"], wc_spt=t["wc_spt"], wc_flush=t["wc_flush"])
        if wc is not None:
            return Route(WC, n4 * 4, head, wc=wc)
    return Route(VEC, n4 * 4, head)


def pair_route(H: int, n_f: int, n_ns: int, precision: int, sm_count: int, **tune) -> Route:
    """launch_keyed_pair with 32-byte aligned values and ids: one write-combining launch for both segments when it is
    eligible and they hold at most WC_MAX_LAUNCH samples together, else two keyed ingests (the route of the last one,
    `extra["apart"]` set; an array of more than WC_MAX_LAUNCH samples that of its first piece)."""
    t = dict(DEFAULTS, **tune)
    small = small_passes(H, precision) <= 4 and t["keyed_mode"] == 0
    if n_f and n_ns and t["keyed_mode"] != 1 and not small and n_f + n_ns <= CONST["WC_MAX_LAUNCH"]:
        wc = wc_launch(H, precision, sm_count, n_f, n_ns, k1_reserve_sms=t["k1_reserve_sms"],
                       keyed_mode=t["keyed_mode"], kp_chunk=t["kp_chunk"], wc_spt=t["wc_spt"], wc_flush=t["wc_flush"])
        if wc is not None:
            return Route(WC, n_f + n_ns, 0, wc=wc)
    r = Route("")
    for m in (n_f, n_ns):
        if m:
            r = keyed_route(H, min(m, CONST["WC_MAX_LAUNCH"]), precision, sm_count, previous=r.kernel, **tune)
    if n_f or n_ns:
        r.extra["apart"] = True
    return r


def keyed_pieces(H: int, n: int, precision: int, sm_count: int, *, id_bytes=2, vals_addr=0, ids_addr=0, **tune):
    """launch_keyed for one call whose hot window starts drained and takes nothing (every piece goes to the
    write-combining or the scalar kernel): [(samples, Route)] of its pieces, each at most WC_MAX_LAUNCH samples and
    routed at its own address."""
    out, done = [], 0
    while done < n:
        m = min(n - done, CONST["WC_MAX_LAUNCH"])
        r = keyed_route(H, m, precision, sm_count, id_bytes=id_bytes, vals_addr=(vals_addr + 8 * done) & 31,
                        ids_addr=(ids_addr + id_bytes * done) & 31, **tune)
        assert r.kernel in (WC, SCALAR), r
        out.append((m, r))
        done += m
    return out


def keyed_launches(m: int, r: Route) -> int:
    """Kernel launches of one piece of m samples on route r (write-combining or scalar): the scalar head, the body,
    the ragged tail past the body's whole tiles."""
    if r.kernel == SCALAR:
        return 1 if m else 0
    return (1 if r.head else 0) + 1 + (1 if m - r.head - r.wc.taken else 0)


def counter_route(C: int, n: int, *, id_bytes=2, amounts_addr=0, ids_addr=0) -> Route:
    """launch_counter: the kernel of the body and the number of launches (`extra["launches"]`)."""
    if n == 0:
        return Route("", extra={"launches": 0})
    if C > CONST["K2_SMEM_COUNTERS"]:
        return Route(COUNTER_GLOBAL, extra={"launches": 1})
    head = min(n, ((32 - (amounts_addr & 31)) & 31) // 8)
    vec_ok = ((ids_addr + head * id_bytes) & (4 * id_bytes - 1)) == 0 and (amounts_addr & 7) == 0
    n4 = (n - head) // 4 if vec_ok else 0
    if n4 < 4096:
        head, n4 = 0, 0
    tail = n - head - n4 * 4
    launches = (1 if head else 0) + (1 if n4 else 0) + (1 if tail else 0)
    return Route(COUNTER_SMEM, n4 * 4, head, extra={"launches": launches, "vec": n4 > 0})


def hot_window_plan(calls, cap=0xFFFFFFFF, margin=1 << 30):
    """launch_keyed's fold guard over a sequence of call sizes (all samples counted into the hot window): for every
    call, the list of ("fold" | piece size) events in order."""
    pending, plan = 0, []
    for n in calls:
        ev, done = [], 0
        while done < n:
            if pending >= cap - margin:
                ev.append("fold")
                pending = 0
            m = min(n - done, cap - pending)
            ev.append(m)
            pending += m
            done += m
        plan.append(ev)
    return plan


def k1_variants(precision: int):
    """lh_create's K1 table at this precision: [(name, index of the code that runs, smem)] per variant slot."""
    budget, win = CONST["kSmemBudget"], window(precision)
    hist = (2 * win + 8) * 4
    out = []
    for i, v in enumerate(CONST["K1_VARIANTS"]):
        if v["probe"]:
            out.append((v["name"], i, 0))
            continue
        code, smem = i, v["smem_fixed"] + hist
        if smem > budget:
            for j in CONST["K1_SMALLER"]:
                if CONST["K1_VARIANTS"][j]["smem_fixed"] + hist <= budget:
                    code, smem = j, CONST["K1_VARIANTS"][j]["smem_fixed"] + hist
                    break
        out.append((v["name"], code, smem))
    return out


def k1_substitution_precisions(lo=1, hi=250):
    """{variant index: first precision at which another variant's code runs under its name}."""
    first = {}
    for p in range(lo, hi + 1):
        for i, (_, code, _) in enumerate(k1_variants(p)):
            if code != i and i not in first:
                first[i] = p
    return first


# ---------------------------------------------------------------------------------------------------- route search
def small_edge(precision: int) -> int:
    """Largest H that k_ingest_keyed_small takes (H + 1 does not)."""
    return CONST["KS_MAX_PASSES"] * ks_ids_per_pass(precision)


def wc_h_by_row_cap(precision: int, sm_count: int, k1_reserve_sms: int = 0, lo: int = 1, hi: int = 65536):
    """{row_cap: [H, ...]} of the H in [lo, hi) the write-combining kernel accepts, and the largest such H."""
    out, hmax = {}, None
    for H in range(lo, hi):
        g = wc_geometry(H, precision, sm_count, k1_reserve_sms)
        if g is not None:
            out.setdefault(g[2], []).append(H)
            hmax = H
    return out, hmax


# --------------------------------------------------------------------------------------------------- case builders
def exact_route_values(oracle, n: int, seed: int) -> np.ndarray:
    """n float64 values every one of which the fast paths must hand to the exact route: negatives, |v| >= 2^63, +-Inf,
    NaNs with payloads (both signs), and the inputs inside the +-2^-12 band around bucket boundaries."""
    rng = np.random.default_rng(seed)
    neg = -oracle.gen_stream(oracle.STREAM_U, n, seed) - 1e-300
    big = np.ldexp(1.0 + rng.random(n), rng.integers(63, 1023, n))
    big[::2] *= -1
    nan_bits = np.uint64(0x7FF0000000000000) | rng.integers(1, 1 << 52, n, dtype=np.uint64)
    nan_bits[::3] |= np.uint64(1 << 63)
    nans = nan_bits.view(np.float64)
    infs = np.where(rng.random(n) < 0.5, np.inf, -np.inf)
    kinds = rng.integers(0, 10, n)
    out = np.where(kinds < 4, neg, np.where(kinds < 6, big, np.where(kinds < 8, nans, infs)))
    band = epsilon_band_values(oracle, 100)
    m = min(band.size, n // 8)
    out[:m] = band[:m]
    return np.ascontiguousarray(out, dtype=np.float64)


def definitely_exact(vals: np.ndarray) -> np.ndarray:
    """Samples no fast path can bin: negative (sign bit set), non-finite, or |v| >= 2^63."""
    bits = vals.view(np.uint64)
    return ((bits >> np.uint64(63)) == 1) | ~np.isfinite(vals) | (np.abs(vals) >= 2.0 ** 63)


def epsilon_band_values(oracle, precision: int = 100) -> np.ndarray:
    """Inputs just inside and just outside the +-2^-12 band around every bucket boundary of the window, both signs
    (the inputs of test_ingest_at_the_edge_of_the_epsilon_band)."""
    T = thresholds(oracle, precision, window(precision) - 1).view(np.float64)
    T = T[T > 0.02]
    eps = 2.0 ** -12
    vals = []
    for mult in (0.6, 0.9, 1.1, 1.5, 3.0):
        dv = (1.0 + T) * (mult * eps) / precision
        vals += [T + dv, T - dv, -(T + dv), -(T - dv)]
    return np.concatenate(vals)


def thresholds(oracle, precision: int, kmax: int) -> np.ndarray:
    """T[k] = smallest positive double (as bits) whose un-wrapped bucket is >= k, for k = 1..kmax."""
    ks = np.arange(1, kmax + 1, dtype=np.int64)
    lo = np.zeros(ks.size, dtype=np.uint64)
    hi = np.full(ks.size, 0x7FEFFFFFFFFFFFFF, dtype=np.uint64)

    def pre_wrap(bits):
        v = bits.view(np.float64)
        k16 = oracle.compress_many(v, precision).astype(np.int64) & 0xFFFF
        approx = np.floor(precision * np.log1p(v) + 0.5)
        wraps = np.round((approx - k16) / 65536.0)
        return k16 + wraps.astype(np.int64) * 65536
    for _ in range(64):
        mid = lo + (hi - lo) // np.uint64(2)
        ge = pre_wrap(mid) >= ks
        hi = np.where(ge, mid, hi)
        lo = np.where(ge, lo, mid)
    return hi


def wc_slice_counts(mask: np.ndarray, wc: WcShape) -> np.ndarray:
    """[chunk][CTA] number of True samples of `mask` (over the launch's taken samples) in each CTA's slice."""
    tiles = wc.taken // wc.tile
    per_tile = mask[:wc.taken].reshape(tiles, wc.tile).sum(axis=1)
    chunk_tiles = wc.slice_tiles * wc.P
    out = np.zeros((wc.nchunks, wc.P), dtype=np.int64)
    for c in range(wc.nchunks):
        for p in range(wc.P):
            a = c * chunk_tiles + p * wc.slice_tiles
            out[c, p] = per_tile[a:min(a + wc.slice_tiles, tiles)].sum() if a < tiles else 0
    return out


def wc_owner_queue(owner_mask: np.ndarray, wc: WcShape):
    """One owner's side of a write-combining launch: what every writer tries to move into its sub-queue of that owner.

    owner_mask marks the samples (of the launch's taken samples) whose record goes to the owner.  Every writer bins its
    slice tile by tile into its shared-memory buffer for the owner (records past row_cap take the exact route at once);
    every flush_tiles tiles (the count runs on across chunks) the full 64-record lines go to the sub-queue, which holds
    `cap` records per chunk; the last chunk also sends the partly filled line.  Returns [chunk][writer] arrays of the
    records that fit the sub-queue and of those that did not (and take the exact route through wc_spill)."""
    line = CONST["WC_LINE"]
    tiles = wc.taken // wc.tile
    per_tile = owner_mask[:wc.taken].reshape(tiles, wc.tile).sum(axis=1)
    chunk_tiles = wc.slice_tiles * wc.P
    queued = np.zeros((wc.nchunks, wc.P), dtype=np.int64)
    spilled = np.zeros((wc.nchunks, wc.P), dtype=np.int64)
    for p in range(wc.P):
        since, fill = 0, 0
        for c in range(wc.nchunks):
            off, spill = 0, 0
            a = c * chunk_tiles + p * wc.slice_tiles
            for t in range(a, min(a + wc.slice_tiles, tiles)):
                fill = min(fill + int(per_tile[t]), wc.row_cap)
                since += 1
                if since == wc.flush_tiles:
                    since = 0
                    for _ in range(fill // line):
                        if off + line <= wc.cap:
                            off += line
                        else:
                            spill += line
                    fill %= line
            if c + 1 == wc.nchunks:
                while fill:
                    nrec = min(line, fill)
                    if off + line <= wc.cap:
                        off += nrec
                    else:
                        spill += nrec
                    fill -= nrec
            queued[c, p], spilled[c, p] = off, spill
    return queued, spilled


def same_residue_ids(n: int, H: int, P: int, r: int, seed: int) -> np.ndarray:
    """n ids, all below H and all congruent to r modulo P (so one write-combining owner receives every record), spread
    over every such id."""
    pool = np.arange(r, H, P, dtype=np.uint32)
    rng = np.random.default_rng(seed)
    return pool[rng.integers(0, pool.size, n)]


def high_ids(H: int, k: int):
    """u32 ids that must be dropped: 65536 + k (k a valid id: a 16-bit truncation would count it into k), 2^31 and
    2^32 - 1."""
    assert 0 <= k < H <= 65536
    return np.array([65536 + k, 1 << 31, 0xFFFFFFFF], dtype=np.uint32)


def with_bad_ids(ids: np.ndarray, bad: np.ndarray, every: int) -> np.ndarray:
    """ids with ids[i] replaced by bad[(i // every) % len(bad)] at every `every`-th position."""
    out = np.array(ids, dtype=np.uint32, copy=True)
    pos = np.arange(0, out.size, every)
    out[pos] = bad[np.arange(pos.size) % bad.size]
    return out
