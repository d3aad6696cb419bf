// lh_kernels.cuh -- sm_90a (H100) kernels of the loghisto hot path.
//
//   K1   k_ingest_single_*  one histogram, float64 stream -> bucket counts
//                           (compress + Histogram increment, metrics.go:273-295, 316-322)
//          _bulk  : cp.async.bulk (TMA 1-D, UBLKCP) into a shared-memory ring guarded by mbarriers, one producer
//                   warp + N consumer warps, pairwise FP32 bucket arithmetic: the shipped default
//          _ldg   : 2 x 128-bit ld.global.nc loads per 4 samples, software-pipelined in registers, scalar fast_candidate() (first version;
//                   kept as the second, independently written evaluator the parity tests run against the oracle)
//        both privatise the histogram in shared memory (uint32 sub-histograms, ATOMS.POPC.INC) and flush once per
//        CTA with one global 64-bit atomic per non-empty bucket.  _bulk also comes in a 4-byte form (float32 / int32)
//        and a 16-bit form (float16 / bfloat16, a key table from k_fill_key16 instead of the log) for lh_ingest_arrays.
//   K1k  k_ingest_keyed_small   (id,value) pairs, as many ids per pass as fit privatised in shared memory (HBM-bound)
//        k_ingest_keyed_vec     any number of ids: one L2 RED per sample into a compact, replicated uint32 window
//        k_ingest_keyed_wc      owner-partitioned, write-combining cooperative kernel (many histograms)
//        k_ingest_keyed         scalar fallback for ragged / misaligned pieces;  k_fold_hot drains the window
//   K2   k_counter_add{_smem}   (id,amount) pairs -> counters[id]        (metrics.go:251-269)
//   K3   k_reduce               per histogram: count, sum, avg, percentiles (processHistograms + percentile,
//                               metrics.go:336-418)
//   K4   k_scan_nnz, k_export   sparse (key,count) lists (RawMetricSet.Histograms);  k_merge_sparse is the inverse
//   K5   k_peer_allreduce       multi-GPU: sums the live window of every peer's frozen arrays over NVLink peer
//                               mappings (SURVEY.md section 8e) -- no library collective
//        k_rows_pack, k_rows_unpack   job-wide rows to and from a payload the caller all-reduces (any transport)
//   K6   k_scatter_segments, k_sparse_epilogue   caller-supplied sparse histograms -> scratch rows -> K3
//                               (lh_reduce_sparse_host)
//   k_ingest_batch          many device arrays under many ids (lh_ingest_batch, lh_graph_recorder_ingest)
//   k_ingest_arrays         every element of device arrays of any gauge dtype -> the frozen interval (distribution
//                           gauges, lh_snapshot_ingest_arrays), or with streaming loads the short items of
//                           lh_ingest_arrays / lh_graph_recorder_ingest_arrays
//   k_ingest_keyed_graph    (id,value) pairs into a graph recorder's rows (lh_graph_recorder_ingest_keyed_*)
//   k_graph_drain           graph recorders' rows -> the interval being frozen (lh_snapshot_begin)
//   k_raw_publish, k_raw_publish_window, k_raw_percentiles, k_raw_ranks   running bucket counts of a snapshot (or of
//                           the last `window` of them) -> raw device subscription rows, and exact percentile / rank
//                           queries over them (lh_snapshot_publish_raw, lh_raw_*)
//   misc k_clear_touched, k_fill_decompress, k_fill_key16, k_compress_probe, k_fastpath_margin, k_fastpath_certify, k_stream_probe,
//        k_gen_stream, k_gen_ids_u16
//
// Per-histogram flags (uint32[H], one array per bucket buffer): 0 = untouched since the buffer was cleared,
// 1 = counts inside the fast window only, 3 = some count outside it.  Every kernel that adds into the uint64
// arrays raises them; the snapshot kernels (reduce, export, clear, all-reduce) scan only what they cover.
#pragma once
#include "../../include/loghisto_b200.h"
#include <type_traits>
#include "lh_device.cuh"

namespace lh {

// ---------------------------------------------------------------- helpers
// Streaming loads: read-once data, keep it out of L1 and first in line for L2 eviction.
// sm_90 has no 256-bit global loads and accepts an L2 eviction priority on loads only through a cache-policy
// operand, so one 32-byte group is two 128-bit loads (LDG.E.128) carrying an evict_first policy.
struct f64x4 { double a, b, c, d; };
__device__ __forceinline__ uint64_t policy_evict_first() {   // not volatile: the compiler hoists it out of loops
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void ldg_stream_u64x4(const void *p, unsigned long long (&r)[4]) {
    const uint64_t pol = policy_evict_first();
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;"
                 : "=l"(r[0]), "=l"(r[1]) : "l"(p), "l"(pol));
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;"
                 : "=l"(r[2]), "=l"(r[3]) : "l"((const char *)p + 16), "l"(pol));
}
__device__ __forceinline__ f64x4 ldg_stream_f64x4(const void *p) {
    unsigned long long u[4];
    ldg_stream_u64x4(p, u);
    f64x4 r;
    r.a = __longlong_as_double((long long)u[0]); r.b = __longlong_as_double((long long)u[1]);
    r.c = __longlong_as_double((long long)u[2]); r.d = __longlong_as_double((long long)u[3]);
    return r;
}
__device__ __forceinline__ f64x4 ldg_stream_f64x2x2(const void *p) {   // two 128-bit loads (comparison variant)
    f64x4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(r.a), "=d"(r.b) : "l"(p));
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(r.c), "=d"(r.d) : "l"((const char *)p + 16));
    return r;
}
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "LH_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra LH_DONE_%=;\n\t"
        "bra LH_WAIT_%=;\n\t"
        "LH_DONE_%=:\n\t}"
        ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar,
                                         uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void red_add_u32_keep(unsigned int *addr, unsigned int v, uint64_t policy) {
    asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(addr), "r"(v), "l"(policy) : "memory");
}

// Up to three scalar stragglers on either side of the vector body (misaligned head, ragged tail).
__device__ __forceinline__ void bucket_stragglers(const double *p, int n, const Prec &pc,
                                                  unsigned long long *__restrict__ counts, uint32_t *flag) {
    for (int i = 0; i < n; i++) add_bucket_global(counts, flag, key16_of(p[i], pc), 1ull, pc.win);
}

// ------------------------------------------------------------------- K1/ldg
// First version, kept as a second evaluator: scalar fast_candidate() per sample, 32-byte groups double-buffered in
// registers.  vals32: 32-byte aligned, nvec 32-byte vectors (4 samples each).
template <int NS>
__device__ __forceinline__ void bucket_samples(const double (&v)[NS], uint32_t *hist, const Prec &pc,
                                               unsigned long long *__restrict__ counts, uint32_t *flag) {
    uint32_t idx[NS];
    bool slow[NS];
    bool any = false;
#pragma unroll
    for (int i = 0; i < NS; i++) { fast_candidate(v[i], pc, idx[i], slow[i]); any |= slow[i]; }
    if (__any_sync(0xFFFFFFFFu, any)) {
#pragma unroll
        for (int i = 0; i < NS; i++) {
            if (slow[i]) {
                const uint32_t key = exact_key16(v[i], pc.precision);
                uint32_t slot = key16_to_slot(key, pc.win);
                if (slot == 0xFFFFFFFFu) { add_bucket_global(counts, flag, key, 1ull, pc.win); slot = 2u * pc.win; }
                idx[i] = slot;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < NS; i++) atomicAdd(&hist[idx[i]], 1u);
}

template <int THREADS, int UNROLL, int MINB>
__global__ void __launch_bounds__(THREADS, MINB)
k_ingest_single_ldg(const double *__restrict__ vals32, size_t nvec, const double *head, int nhead,
                    const double *tail, int ntail, unsigned long long *__restrict__ counts, uint32_t *flag, Prec pc) {
    extern __shared__ __align__(16) uint32_t s_hist[];
    for (uint32_t i = threadIdx.x; i < subhist_words(pc.win); i += THREADS) s_hist[i] = 0;
    __syncthreads();
    const char *base = reinterpret_cast<const char *>(vals32);

    constexpr size_t TILE = (size_t)THREADS * UNROLL;   // 32-byte vectors per tile
    const size_t ntiles = nvec / TILE;
    f64x4 cur[UNROLL], nxt[UNROLL];
    size_t tile = blockIdx.x;
    if (tile < ntiles) {
#pragma unroll
        for (int u = 0; u < UNROLL; u++) cur[u] = ldg_stream_f64x4(base + (tile * TILE + (size_t)u * THREADS + threadIdx.x) * 32);
    }
    while (tile < ntiles) {
        const size_t nt = tile + gridDim.x;
        if (nt < ntiles) {
#pragma unroll
            for (int u = 0; u < UNROLL; u++) nxt[u] = ldg_stream_f64x4(base + (nt * TILE + (size_t)u * THREADS + threadIdx.x) * 32);
        }
        double v[4 * UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) { v[4 * u] = cur[u].a; v[4 * u + 1] = cur[u].b; v[4 * u + 2] = cur[u].c; v[4 * u + 3] = cur[u].d; }
        bucket_samples<4 * UNROLL>(v, s_hist, pc, counts, flag);
#pragma unroll
        for (int u = 0; u < UNROLL; u++) cur[u] = nxt[u];
        tile = nt;
    }
    // partial last tile + stragglers: one CTA, bounds-checked (rare, < TILE vectors)
    if (blockIdx.x == ntiles % gridDim.x) {
        for (size_t j = ntiles * TILE * 4 + threadIdx.x; j < nvec * 4; j += THREADS)
            atomicAdd(&s_hist[fixup_slot(vals32[j], pc, counts, flag)], 1u);
        if (threadIdx.x == 0) { bucket_stragglers(head, nhead, pc, counts, flag); bucket_stragglers(tail, ntail, pc, counts, flag); }
    }
    __syncthreads();
    flush_subhist(s_hist, threadIdx.x, THREADS, counts, flag, pc.win);
}

// ------------------------------------------------------- pairwise FP32 bucket arithmetic
// Same algorithm as fast_candidate() with the per-sample instruction count cut so that the kernel stays HBM-bound
// under sustained load:
//   * samples are processed in pairs, each FP32 op written with an explicit rounding (__fmaf_rn / __fadd_rn) so the
//     compiler neither contracts nor reorders them;
//   * (float)e comes from one I2FP and the -1023 bias rides in the FMA addend (Prec::kb);
//   * ONE flag per sample: estimate too close to a bucket boundary, OR x = 1+|v| outside the window
//     (x's high word >= 0x43E00000: |v| >= 2^63, Inf, NaN);
//   * the sign of v is folded into the slot (negative values land in [win, 2*win)) instead of being flagged, so a
//     stream with many negative durations (readme.md:43) stays on the fast path;
//   * the shared-memory byte offset is built as eb*a4 + (rounded bits << 2) + const: one IMAD and one LEA.
// Extra estimate error vs fast_candidate(): the float constant -1023*c2, at most half an ulp of a float below 1024:
// <= 1.53e-5 bucket units at precision 100 (|1023*c2| = 321.9), <= 3.1e-5 at any precision.  Certified worst case of
// this form over every input and precision 1..250: 6.69e-5 (fast_candidate: 4.61e-5), eps at least 5.2 times that
// (lh_fastpath_certify).
// FOLD_SIGN = false: positive-only layout (rows of `win` slots); negative samples are flagged instead.
// SHIFT = 2: byte offsets into a uint32 sub-histogram; SHIFT = 0: slot indices.
// est[i]: the FP32 part of sample i's estimate, precision*ln(1+|v|) ~= (eb - 1023) * a_int + est (as fast_candidate's w;
// k_fastpath_certify reads it, the kernels use the form without it).
template <int NS, bool FOLD_SIGN, int SHIFT = 2>
__device__ __forceinline__ void bucket_offsets_v2(const double (&v)[NS], const Prec &pc, uint32_t one_bits,
                                                  uint32_t (&off)[NS], bool (&flag)[NS], float (&est)[NS]) {
    static_assert(NS % 2 == 0, "pairs");
    constexpr float MAGIC = 12582912.0f;
    const uint32_t negoff = pc.win << SHIFT;
    const uint32_t am = SHIFT ? pc.a4 : pc.a_int, cm = SHIFT ? pc.coff : pc.coff0;
#pragma unroll
    for (int i = 0; i < NS; i += 2) {
        const double x0 = __dadd_rn(1.0, fabs(v[i])), x1 = __dadd_rn(1.0, fabs(v[i + 1]));
        const uint32_t h0 = (uint32_t)__double2hiint(x0), h1 = (uint32_t)__double2hiint(x1);
        const uint32_t t0 = __funnelshift_l((uint32_t)__double2loint(x0), h0, 3);
        const uint32_t t1 = __funnelshift_l((uint32_t)__double2loint(x1), h1, 3);
        uint32_t m0, m1;
        asm("lop3.b32 %0, %1, 0x007FFFFF, %2, 0xEA;" : "=r"(m0) : "r"(t0), "r"(one_bits));   // (t & mask) | 1.0f
        asm("lop3.b32 %0, %1, 0x007FFFFF, %2, 0xEA;" : "=r"(m1) : "r"(t1), "r"(one_bits));
        float2 lg;
        asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(lg.x) : "f"(__uint_as_float(m0)));
        asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(lg.y) : "f"(__uint_as_float(m1)));
        const uint32_t e0 = h0 >> 20, e1 = h1 >> 20;                    // 1023 + e
        const float2 ef = make_float2(__uint2float_rn(e0), __uint2float_rn(e1));
        const float2 a = make_float2(__fmaf_rn(ef.x, pc.c2, pc.kb), __fmaf_rn(ef.y, pc.c2, pc.kb));
        const float2 w = make_float2(__fmaf_rn(lg.x, pc.c1, a.x), __fmaf_rn(lg.y, pc.c1, a.y));
        est[i] = w.x; est[i + 1] = w.y;
        const float2 r = make_float2(__fadd_rn(w.x, MAGIC), __fadd_rn(w.y, MAGIC));
        const float2 s = make_float2(__fadd_rn(r.x, -MAGIC), __fadd_rn(r.y, -MAGIC));
        const float2 d = make_float2(__fmaf_rn(s.x, -1.0f, w.x), __fmaf_rn(s.y, -1.0f, w.y));   // w - s, one rounding
        if (FOLD_SIGN) {
            flag[i] = (fabsf(d.x) > pc.thresh) | (h0 >= 0x43E00000u);
            flag[i + 1] = (fabsf(d.y) > pc.thresh) | (h1 >= 0x43E00000u);
            const uint32_t n0 = (uint32_t)__double2hiint(v[i]) >> 31, n1 = (uint32_t)__double2hiint(v[i + 1]) >> 31;
            off[i] = e0 * am + (__float_as_uint(r.x) << SHIFT) + (n0 * negoff + cm);
            off[i + 1] = e1 * am + (__float_as_uint(r.y) << SHIFT) + (n1 * negoff + cm);
        } else {
            // v's high word >= 0x43E00000 unsigned: |v| >= 2^63, Inf, NaN and every negative value
            flag[i] = (fabsf(d.x) > pc.thresh) | ((uint32_t)__double2hiint(v[i]) >= 0x43E00000u);
            flag[i + 1] = (fabsf(d.y) > pc.thresh) | ((uint32_t)__double2hiint(v[i + 1]) >= 0x43E00000u);
            off[i] = e0 * am + (__float_as_uint(r.x) << SHIFT) + cm;
            off[i + 1] = e1 * am + (__float_as_uint(r.y) << SHIFT) + cm;
        }
    }
}
template <int NS, bool FOLD_SIGN, int SHIFT = 2>
__device__ __forceinline__ void bucket_offsets_v2(const double (&v)[NS], const Prec &pc, uint32_t one_bits,
                                                  uint32_t (&off)[NS], bool (&flag)[NS]) {
    float est[NS];
    bucket_offsets_v2<NS, FOLD_SIGN, SHIFT>(v, pc, one_bits, off, flag, est);
}

template <int NS, bool FOLD_SIGN>
__device__ __forceinline__ void bucket_samples_v2(const double (&v)[NS], uint32_t *hist, const Prec &pc, uint32_t one_bits,
                                                  unsigned long long *__restrict__ counts, uint32_t *gflag) {
    uint32_t off[NS];
    bool flag[NS];
    bucket_offsets_v2<NS, FOLD_SIGN>(v, pc, one_bits, off, flag);
    bool any = false;
#pragma unroll
    for (int i = 0; i < NS; i++) any |= flag[i];
    if (__any_sync(0xFFFFFFFFu, any)) {
        // only the sample positions some lane flagged are re-derived (a warp-uniform branch per position)
#pragma unroll
        for (int i = 0; i < NS; i++)
            if (__any_sync(0xFFFFFFFFu, flag[i])) {
                if (flag[i]) off[i] = fixup_slot(v[i], pc, counts, gflag) * 4u;
            }
    }
#pragma unroll
    for (int i = 0; i < NS; i++) atomicAdd(reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(hist) + off[i]), 1u);
}

// --------------------------------------------------------------- read probe
// Diagnostic only (a K1 "variant" that produces NO counts): the same streaming loads as K1/ldg with the
// bucket arithmetic replaced by an XOR fold, to separate memory-side from SM-side limits.
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS, 2)
k_stream_probe(const double *__restrict__ vals32, size_t nvec, const double *, int, const double *, int,
               unsigned long long *__restrict__ counts, uint32_t *, Prec) {
    const char *base = reinterpret_cast<const char *>(vals32);
    constexpr size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    unsigned long long acc = 0;
    for (size_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        f64x4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) v[u] = ldg_stream_f64x4(base + (tile * TILE + (size_t)u * THREADS + threadIdx.x) * 32);
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
            acc ^= f64_as_u64(v[u].a) ^ f64_as_u64(v[u].b) ^ f64_as_u64(v[u].c) ^ f64_as_u64(v[u].d);
    }
    if (acc == 0x123456789ABCDEFull) counts[65535] = acc;   // never true in practice; keeps the loads alive
}

// ------------------------------------------------------------------ K1/bulk
// Producer warp streams STAGE_BYTES tiles into a STAGES-deep shared ring with
// cp.async.bulk; CW consumer warps bucket them.  Tiles are dealt round-robin.
// FOLD_SIGN: negative samples stay on the fast path (their slot is offset by `win`) at the price of two more integer
// instructions per sample; without it they are flagged and re-derived in the fix-up.
// Cv: the element type and its conversion to float64 (K1F64 below, the float64 kernel; K1F32 / K1I32 and K1F16 /
// K1BF16 after the gauge conversions, lh_ingest_arrays).  The producer and the ring move bytes whatever the element;
// vals32 is 32-byte aligned and holds nvec32 32-byte groups, head / tail the (at most 32 / sizeof(T) - 1) elements on
// either side.  4-byte elements are converted exactly and binned with bucket_offsets_v2 like float64 ones.  16-bit
// elements (Cv::kTable) skip the arithmetic: `keys` is the dtype's 32768-entry table of k_fill_key16, copied into
// shared memory ahead of the sub-histogram, giving each magnitude's window slot (the sign adds `win`), or 0xFFFF for a
// key outside the window, which goes through fixup_slot.
struct K1F64 { using T = double; static constexpr bool kTable = false; };
template <int CW, int STAGES, int STAGE_BYTES, int MINB, bool FOLD_SIGN, typename Cv = K1F64>
__global__ void __launch_bounds__((CW + 1) * 32, MINB)
k_ingest_single_bulk(const typename Cv::T *__restrict__ vals32, size_t nvec32, const typename Cv::T *head, int nhead,
                     const typename Cv::T *tail, int ntail, unsigned long long *__restrict__ counts, uint32_t *flag, Prec pc,
                     const uint16_t *keys = nullptr) {
    using T = typename Cv::T;
    constexpr bool F64 = std::is_same<T, double>::value;
    constexpr int SPV = 16 / (int)sizeof(T);          // samples per 16-byte vector
    const double2 *vals16 = reinterpret_cast<const double2 *>(vals32);
    const size_t nvec = nvec32 * 2;   // 16-byte vectors
    constexpr int CT = CW * 32;                       // consumer threads
    constexpr int STAGE_VEC = STAGE_BYTES / 16;
    constexpr int PER_THREAD = STAGE_VEC / CT;        // 16-byte vectors per consumer thread per stage
    static_assert(STAGE_VEC % CT == 0, "stage must divide evenly over consumer threads");
    extern __shared__ __align__(128) unsigned char s_raw[];
    double2 *s_data = reinterpret_cast<double2 *>(s_raw);
    uint64_t *full = reinterpret_cast<uint64_t *>(s_raw + (size_t)STAGES * STAGE_BYTES);
    uint64_t *empty = full + STAGES;
    uint16_t *s_keys = reinterpret_cast<uint16_t *>(empty + STAGES);   // Cv::kTable only
    uint32_t *s_hist = reinterpret_cast<uint32_t *>(empty + STAGES) + (Cv::kTable ? 16384 : 0);

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    for (uint32_t i = tid; i < subhist_words(pc.win); i += (CW + 1) * 32) s_hist[i] = 0;
    if constexpr (Cv::kTable) {
        for (uint32_t i = tid; i < 4096u; i += (CW + 1) * 32)
            reinterpret_cast<uint4 *>(s_keys)[i] = __ldg(reinterpret_cast<const uint4 *>(keys) + i);
    }
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const size_t ntiles = (nvec + STAGE_VEC - 1) / STAGE_VEC;
    if (warp == CW) {
        // ===== producer =====
        if ((tid & 31) == 0) {
            const uint64_t pol = policy_evict_first();
            uint32_t it = 0;
            for (size_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, it++) {
                const int s = it % STAGES;
                mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                size_t first = tile * (size_t)STAGE_VEC;
                size_t rem = nvec - first;
                uint32_t bytes = (uint32_t)((rem < (size_t)STAGE_VEC ? rem : (size_t)STAGE_VEC) * 16);
                mbar_expect_tx(&full[s], bytes);
                bulk_g2s(s_data + (size_t)s * STAGE_VEC, vals16 + first, bytes, &full[s], pol);
            }
        }
    } else {
        // ===== consumers =====
        uint32_t one_bits;
        asm volatile("mov.b32 %0, 0x3F800000;" : "=r"(one_bits));   // opaque to constant folding: keeps LOP3 at one instruction
        uint32_t it = 0;
        for (size_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, it++) {
            const int s = it % STAGES;
            mbar_wait(&full[s], (it / STAGES) & 1);
            const double2 *st = s_data + (size_t)s * STAGE_VEC;
            size_t first = tile * (size_t)STAGE_VEC;
            size_t rem = nvec - first;
            if (rem >= (size_t)STAGE_VEC) {
                if constexpr (F64) {
                    double v[2 * PER_THREAD];
#pragma unroll
                    for (int u = 0; u < PER_THREAD; u++) {
                        double2 d = st[u * CT + tid];
                        v[2 * u] = d.x; v[2 * u + 1] = d.y;
                    }
                    __syncwarp();
                    if ((tid & 31) == 0) mbar_arrive(&empty[s]);   // registers hold the data: release early
#pragma unroll
                    for (int q = 0; q < 2 * PER_THREAD; q += 4) {
                        const double v4[4] = {v[q], v[q + 1], v[q + 2], v[q + 3]};
                        bucket_samples_v2<4, FOLD_SIGN>(v4, s_hist, pc, one_bits, counts, flag);
                    }
                } else {
                    uint32_t w[4 * PER_THREAD];
#pragma unroll
                    for (int u = 0; u < PER_THREAD; u++) {
                        const uint4 d = reinterpret_cast<const uint4 *>(st)[u * CT + tid];
                        w[4 * u] = d.x; w[4 * u + 1] = d.y; w[4 * u + 2] = d.z; w[4 * u + 3] = d.w;
                    }
                    __syncwarp();
                    if ((tid & 31) == 0) mbar_arrive(&empty[s]);
                    if constexpr (Cv::kTable) {
#pragma unroll
                        for (int q = 0; q < 4 * PER_THREAD; q++) {
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const uint32_t x = h ? w[q] >> 16 : w[q] & 0xFFFFu;
                                uint32_t slot = s_keys[x & 0x7FFFu];
                                if (slot == 0xFFFFu) slot = fixup_slot(Cv::f64((unsigned short)x), pc, counts, flag);
                                else slot += (x >> 15) * pc.win;
                                atomicAdd(&s_hist[slot], 1u);
                            }
                        }
                    } else {
#pragma unroll
                        for (int q = 0; q < 4 * PER_THREAD; q += 4) {
                            const double v4[4] = {Cv::f64(w[q]), Cv::f64(w[q + 1]), Cv::f64(w[q + 2]), Cv::f64(w[q + 3])};
                            bucket_samples_v2<4, FOLD_SIGN>(v4, s_hist, pc, one_bits, counts, flag);
                        }
                    }
                }
            } else {
                if constexpr (F64) {
                    for (int j = tid; j < (int)rem; j += CT) {
                        double2 d = st[j];
                        atomicAdd(&s_hist[fixup_slot(d.x, pc, counts, flag)], 1u);
                        atomicAdd(&s_hist[fixup_slot(d.y, pc, counts, flag)], 1u);
                    }
                } else {
                    const T *e = reinterpret_cast<const T *>(st);
                    for (int j = tid; j < (int)rem * SPV; j += CT) atomicAdd(&s_hist[fixup_slot(Cv::f64(e[j]), pc, counts, flag)], 1u);
                }
                __syncwarp();
                if ((tid & 31) == 0) mbar_arrive(&empty[s]);
            }
        }
        if (blockIdx.x == 0 && tid == 0) {
            if constexpr (F64) {
                bucket_stragglers(head, nhead, pc, counts, flag); bucket_stragglers(tail, ntail, pc, counts, flag);
            } else {
                for (int i = 0; i < nhead; i++) add_bucket_global(counts, flag, key16_of(Cv::f64(head[i]), pc), 1ull, pc.win);
                for (int i = 0; i < ntail; i++) add_bucket_global(counts, flag, key16_of(Cv::f64(tail[i]), pc), 1ull, pc.win);
            }
        }
    }
    __syncthreads();
    flush_subhist(s_hist, tid, (CW + 1) * 32, counts, flag, pc.win);
}

// --------------------------------------------------------------------- K1k
// (id,value) pairs.  1024 histograms x ~4.4K live buckets cannot be privatised
// in one CTA's shared memory.  The general fallback keeps the cells in L2: a compact uint32 "hot window"
// [H][2*win] (36 MB at H = 1024, vs 512 MB for the dense uint64 arrays)
// updated with no-return atomics that carry an L2 evict_last policy, while the
// sample stream is read once with evict_first loads so it does not push
// the cells out of the 50 MB L2.  Keys outside the window go straight to the
// uint64 array.  k_fold_hot drains the window into the uint64 buckets at every
// snapshot (and before any cell could reach 2^32).
template <typename T> __device__ __forceinline__ double sample_to_f64(T v);
template <> __device__ __forceinline__ double sample_to_f64<double>(double v) { return v; }
// float64(duration.Nanoseconds()): CVTSQ2SD, round-to-nearest-even
template <> __device__ __forceinline__ double sample_to_f64<long long>(long long v) { return __ll2double_rn(v); }

struct KeyedOut {
    unsigned int *hot;                 // [replicas][H][2*win] uint32
    unsigned long long *buckets;       // [H][65536]
    uint32_t *flags;                   // [H]
    unsigned long long *dropped;
    uint32_t H;
};

// Id-map policies of the keyed and counter kernels (their last template parameter, passed by value as their last
// argument).  IdIdentity: an id is a row (the raw calls).  IdMap: ids are local to a record scope; local id l < k means
// row row[l], and an id >= k or a row of LH_GRAPH_UNBOUND drops the sample (counted).  Binning and privatisation stay in
// local-id space; the map is read only where a row address is formed.  The kernels read it through a view, MapRows,
// over the parameter block (indexed loads from the constant bank; the parameter is not __grid_constant__, which would
// change how the other by-value parameters are loaded) or over a copy in shared memory; IdIdentity is its own view and
// compiles to the unmapped code.
constexpr uint32_t LH_MAP_MAX = 4096;          // entries of an IdMap (16 KiB of the parameter block)
struct IdIdentity {
    __device__ __forceinline__ uint32_t bound(uint32_t H) const { return H; }
    __device__ __forceinline__ bool lookup(uint32_t id, uint32_t H, uint32_t &) const { return id < H; }   // row = id
    __device__ __forceinline__ uint32_t row(uint32_t id) const { return id; }
    __device__ __forceinline__ bool drops(uint32_t id, uint32_t C) const { return id >= C; }
};
struct IdMap {
    uint32_t k;
    uint32_t any_unbound;            // some row[l] is unbound: the counter kernels check every op
    uint32_t row[LH_MAP_MAX];
};
struct MapRows {
    const uint32_t *rows;
    uint32_t k;
    bool any_unbound;
    __device__ __forceinline__ uint32_t bound(uint32_t) const { return k; }
    // a counter op under local id l is dropped (the op count of an unbound row is not known at the flush)
    __device__ __forceinline__ bool drops(uint32_t l, uint32_t) const { return l >= k || (any_unbound && rows[l] == 0xFFFFFFFFu); }
    // local id l -> its row in r (r may alias l); false: drop the sample
    __device__ __forceinline__ bool lookup(uint32_t l, uint32_t, uint32_t &r) const {
        if (l >= k) return false;
        const uint32_t x = rows[l];
        r = x;
        return x != 0xFFFFFFFFu;
    }
    __device__ __forceinline__ uint32_t row(uint32_t l) const { return rows[l]; }   // l < k; may be unbound
};
template <typename Map> constexpr bool kMapped = !std::is_same<Map, IdIdentity>::value;
// the map as read from the parameter block (flushes and rare paths)
__device__ __forceinline__ IdIdentity map_view(const IdIdentity &) { return {}; }
__device__ __forceinline__ MapRows map_view(const IdMap &m) { return MapRows{m.row, m.k, m.any_unbound != 0}; }
// the map copied into shared memory `s` (k words) by the whole CTA, for kernels that look up every sample
__device__ __forceinline__ IdIdentity map_to_smem(const IdIdentity &, uint32_t *) { return {}; }
__device__ __forceinline__ MapRows map_to_smem(const IdMap &m, uint32_t *s) {
    for (uint32_t i = threadIdx.x; i < m.k; i += blockDim.x) s[i] = m.row[i];
    __syncthreads();
    return MapRows{s, m.k, m.any_unbound != 0};
}
// the dynamic shared memory map_to_smem needs (host side, for the launch)
inline size_t map_smem_bytes(const IdIdentity &) { return 0; }
inline size_t map_smem_bytes(const IdMap &m) { return (size_t)m.k * 4; }

template <typename ValT, typename V = IdIdentity>
__device__ __forceinline__ void keyed_one(uint32_t id, ValT raw, const Prec &pc, const KeyedOut &o, unsigned int *hot, uint64_t pol,
                                          const V &m = {}) {
    if (!m.lookup(id, o.H, id)) { atomicAdd(o.dropped, 1ull); return; }
    double v = sample_to_f64<ValT>(raw);
    uint32_t idx; bool slow;
    fast_candidate(v, pc, idx, slow);
    if (slow) {
        uint32_t key = exact_key16(v, pc.precision);
        idx = key16_to_slot(key, pc.win);
        if (idx == 0xFFFFFFFFu) { add_bucket_global(o.buckets + (size_t)id * 65536u, o.flags + id, key, 1ull, pc.win); return; }
    }
    red_add_u32_keep(&hot[(size_t)id * (2u * pc.win) + idx], 1u, pol);
}
// The same sample straight into the uint64 arrays (one 64-bit atomic + the histogram's flag): for the few samples
// that reach the scalar kernel (ragged heads / tails) and the rare paths of the write-combining kernel, so that those
// launches leave nothing in the uint32 hot window for the snapshot to fold.
template <typename ValT, typename V = IdIdentity>
__device__ __forceinline__ void keyed_one_direct(uint32_t id, ValT raw, const Prec &pc, const KeyedOut &o, const V &m = {}) {
    if constexpr (kMapped<V>) {
        if (!m.lookup(id, o.H, id)) { atomicAdd(o.dropped, 1ull); return; }
    } else {
        if (id >= o.H) { atomicAdd(o.dropped, 1ull); return; }   // (written out: through lookup() the value load moves)
    }
    add_bucket_global(o.buckets + (size_t)id * 65536u, o.flags + id, key16_of(sample_to_f64<ValT>(raw), pc), 1ull, pc.win);
}

// Out-of-line form for kernels whose common path must stay small (the write-combining kernel calls it for the
// ~0.05 % of samples its fast path does not cover).
template <typename ValT>
__device__ __noinline__ void keyed_one_slow(uint32_t id, unsigned long long raw, Prec pc, KeyedOut o) {
    ValT r;
    memcpy(&r, &raw, 8);
    keyed_one_direct<ValT>(id, r, pc, o);
}
// Mapped: the row is resolved here, so that the map (in the parameter block) is only read inline.
template <typename ValT, typename V>
__device__ __forceinline__ void keyed_one_slow_v(uint32_t id, unsigned long long raw, const Prec &pc, const KeyedOut &o, const V &m) {
    if constexpr (kMapped<V>) {
        if (!m.lookup(id, o.H, id)) { atomicAdd(o.dropped, 1ull); return; }
    }
    keyed_one_slow<ValT>(id, raw, pc, o);
}

__device__ __forceinline__ void load_vals4(const void *vals, size_t g, unsigned long long (&raw)[4]) {
    ldg_stream_u64x4(reinterpret_cast<const char *>(vals) + g * 32, raw);
}

// ids of one 4-sample group, kept PACKED while they wait in registers (unpacking right after the load would make the
// prefetch wait for its own data)
template <typename IdT> struct IdPack;
template <> struct IdPack<unsigned short> {
    unsigned int lo, hi;
    __device__ __forceinline__ void load(const unsigned short *ids, size_t g) {
        asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(lo), "=r"(hi) : "l"(reinterpret_cast<const char *>(ids) + g * 8));
    }
    __device__ __forceinline__ uint32_t get(int j) const { const unsigned int w = j < 2 ? lo : hi; return (j & 1) ? (w >> 16) : (w & 0xFFFFu); }
};
template <> struct IdPack<unsigned int> {
    unsigned int w[4];
    __device__ __forceinline__ void load(const unsigned int *ids, size_t g) {
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                     : "l"(reinterpret_cast<const char *>(ids) + g * 16));
    }
    __device__ __forceinline__ uint32_t get(int j) const { return w[j]; }
};

// Vector body: every thread takes 4 consecutive pairs (two 128-bit value loads, one 64/128-bit id load).
// vals must be 32-byte aligned and ids 4*sizeof(IdT)-aligned; n4 = number of 4-sample groups.
// `hot` holds `replicas` copies of the window ([replicas][H][2*win]); CTA b updates copy b % replicas, which
// divides the same-address pressure on hot cells (clustered, latency-like data) by the replica count while every
// copy stays L2-resident.  k_fold_hot sums the copies.
// Mapped: the map is copied into dynamic shared memory (k words) and the sample goes to its row's window.
template <typename IdT, typename ValT, int THREADS, typename Map = IdIdentity>
__global__ void __launch_bounds__(THREADS)
k_ingest_keyed_vec(const IdT *__restrict__ ids, const ValT *__restrict__ vals, size_t n4, uint32_t replicas, KeyedOut o, Prec pc,
                   const Map map) {
    extern __shared__ uint32_t kv_map[];
    const auto mv = map_to_smem(map, kv_map);
    unsigned int *hot = o.hot + (size_t)(blockIdx.x % replicas) * o.H * (2u * pc.win);
    const uint64_t pol = policy_evict_last();
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t g = (size_t)blockIdx.x * THREADS + threadIdx.x; g < n4; g += stride) {
        unsigned long long raw[4];
        IdPack<IdT> idp;
        load_vals4(vals, g, raw);
        idp.load(ids, g);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            ValT r;
            memcpy(&r, &raw[j], 8);
            keyed_one<ValT>(idp.get(j), r, pc, o, hot, pol, mv);
        }
    }
}

// Scalar version for ragged heads/tails and misaligned inputs.  Mapped: as k_ingest_keyed_vec.
template <typename IdT, typename ValT, int THREADS, typename Map = IdIdentity>
__global__ void __launch_bounds__(THREADS)
k_ingest_keyed(const IdT *__restrict__ ids, const ValT *__restrict__ vals, size_t n, KeyedOut o, Prec pc,
               const Map map) {
    extern __shared__ uint32_t ks_map[];
    const auto mv = map_to_smem(map, ks_map);
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += stride)
        keyed_one_direct<ValT>((uint32_t)ids[i], vals[i], pc, o, mv);
}

// ------------------------------------------------------------------ K1k/small
// Keyed ingest when only a few histograms are configured: all their windows (uint32[ids][2*win]) are privatised
// per CTA in shared memory, exactly like K1, so the kernel is HBM-bound (10 B/sample) instead of L2-atomic-bound.
// Same pairwise FP32 bucket arithmetic as K1 but with positive-only rows (uint32[ids][win]) so that twice as many
// histograms fit; the ONE flag per sample also covers id >= H, and flagged samples (boundary-close estimates,
// negatives, |v| >= 2^63, NaN/Inf, bad ids) take the L2 route of keyed_one().  Windows are added into the uint32
// hot window at the end.
constexpr int KS_THREADS = 1024;
constexpr int KS_SMEM_BYTES = 196608;        // shared memory the windows of one pass may take (11 ids at precision 100)

template <typename IdT, typename ValT, typename Map = IdIdentity>
__global__ void __launch_bounds__(KS_THREADS, 1)
k_ingest_keyed_small(const IdT *__restrict__ ids, const ValT *__restrict__ vals, size_t n4,
                     uint32_t id_lo, uint32_t id_cnt, KeyedOut o, Prec pc, const Map map) {
    // This launch owns ids [id_lo, id_lo + id_cnt); with more histograms than fit, the host
    // runs one pass per id sub-range over the same batch.  Samples of other valid ids are skipped; ids >= H are
    // dropped (and counted) by the pass that starts at id 0.  Mapped: ids, passes and windows are local (H is k); the
    // flush adds a window to its row, or counts an unbound row's total as dropped.
    const auto mv = map_view(map);
    extern __shared__ __align__(16) uint32_t ks_hist[];          // [id_cnt][win] + trash word
    const uint32_t row = pc.win;
    const uint32_t words = id_cnt * row;
    for (uint32_t i = threadIdx.x; i <= words; i += KS_THREADS) ks_hist[i] = 0;
    __syncthreads();
    const uint64_t pol = policy_evict_last();
    uint32_t one_bits;
    asm volatile("mov.b32 %0, 0x3F800000;" : "=r"(one_bits));
    const uint32_t trash_off = words * 4u;

    // The loop bound is warp-uniform (base index of the CTA's row of groups); lanes past the end are predicated
    // off, because the fix-up below votes with the full warp mask.
    const size_t stride = (size_t)gridDim.x * KS_THREADS;
    size_t base = (size_t)blockIdx.x * KS_THREADS;
    unsigned long long cur[4] = {0, 0, 0, 0}, nxt[4] = {0, 0, 0, 0};
    IdPack<IdT> cur_id{}, nxt_id{};
    if (base + threadIdx.x < n4) { load_vals4(vals, base + threadIdx.x, cur); cur_id.load(ids, base + threadIdx.x); }
    for (; base < n4; base += stride) {
        const bool valid = base + threadIdx.x < n4;
        const size_t gn = base + stride + threadIdx.x;
        if (gn < n4) { load_vals4(vals, gn, nxt); nxt_id.load(ids, gn); }
        double v[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { ValT r; memcpy(&r, &cur[i], 8); v[i] = sample_to_f64<ValT>(r); }
        uint32_t off[4];
        bool flag[4];
        bucket_offsets_v2<4, false>(v, pc, one_bits, off, flag);
        bool any = false;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t l = cur_id.get(i) - id_lo;                              // local id (wraps when below id_lo)
            const bool mine = valid & (l < id_cnt);
            const bool bad = valid & (cur_id.get(i) >= mv.bound(o.H)) & (id_lo == 0);
            flag[i] = (mine & flag[i]) | bad;
            off[i] = mine ? off[i] + l * (row * 4u) : trash_off;
            any |= flag[i];
        }
        if (__any_sync(0xFFFFFFFFu, any)) {
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (!flag[i]) continue;
                ValT rv;
                memcpy(&rv, &cur[i], 8);
                // uncertain samples of a valid id could stay in shared memory; the L2 route is exact too
                // and keeps this path trivial (it handles ~0.05 % of the samples)
                keyed_one<ValT>(cur_id.get(i), rv, pc, o, o.hot, pol, mv);
                off[i] = trash_off;
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) atomicAdd(reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(ks_hist) + off[i]), 1u);
#pragma unroll
        for (int i = 0; i < 4; i++) cur[i] = nxt[i];
        cur_id = nxt_id;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < words; i += KS_THREADS) {
        const uint32_t c = ks_hist[i];
        if (!c) continue;
        const uint32_t lid = i / row, slot = i - lid * row;
        const uint32_t r = mv.row(id_lo + lid);
        if (kMapped<Map> && r == 0xFFFFFFFFu) atomicAdd(o.dropped, (unsigned long long)c);
        else atomicAdd(&o.hot[(size_t)r * (2u * pc.win) + slot], c);
    }
}

// ------------------------------------------------------------------- K1k/wc
// Many histograms (H x window does not fit one CTA's shared memory): gets the keyed path past the L2 atomic
// rate (one RED sector per sample, ~0.25 x HBM roofline) by routing every sample to the SM that OWNS its histogram.
// One persistent cooperative CTA per SM; CTA p owns the ids {p, p+P, p+2P, ...} and keeps their positive windows
// (uint32[ids_per][win]) in shared memory for the whole launch.  The stream is processed in chunks; per chunk
//   phase A  every CTA ("writer") bins its slice: bucket index via the pairwise FP32 fast path, one 16-bit record
//            (lid*win + slot) per sample appended to a per-owner WRITE-COMBINING buffer in shared memory -- the
//            position comes from one returning shared atomic on the owner's fill counter (tools/ubench.cu: a
//            warp-wide shared atomic on spread addresses costs a fraction of MATCH.ANY or ballot ranking).  After each tile of WC_TILE samples the full 128-byte lines are copied to the
//            (owner, writer) sub-queue in global memory (L2-resident) with 128-bit stores and the remainder (< 64
//            records) moves to the front of the buffer.  Every (owner, writer) pair has its own region, so the
//            append offsets live in shared memory and no global atomic is needed;
//   barrier  grid-wide (one per chunk; sub-queues are double-buffered by chunk parity);
//   phase B  every owner drains its P sub-queues (L2 hits) into its shared-memory windows (ATOMS.POPC.INC).
// Samples the window does not cover (negative, |v| >= 2^63, NaN/Inf, estimates within eps of a bucket boundary),
// ids >= H, and records that do not fit their buffer or sub-queue (heavily skewed ids) take the exact L2-atomic
// route of keyed_one().  At the end each CTA adds its windows straight into the uint64 bucket arrays: nothing goes
// through the uint32 hot window, so these launches add nothing to the host's tally of it (hot_pending).
constexpr int WC_MAX_PARTS = 160;             // owners = CTAs (one per SM)
constexpr int WC_LINE = 64;                   // records per line (128 B)

template <int SPT> struct WcShape {           // shape code -> threads x samples per thread and tile (registers per thread):
                                              // 6: 896 x 4 (72, default), 4: 1024 x 4 (64), 3: 768 x 4 (80), 8: 512 x 8 (128);
                                              // 640 x 4 and 512 x 4 were 3 - 10 % slower, and a register pipeline three tiles
                                              // deep (640 x 4, 96 registers) gained nothing over the L2 prefetch below
    static constexpr int THREADS = SPT == 4 ? 1024 : SPT == 6 ? 896 : SPT == 3 ? 768 : 512;
    static constexpr int PER = SPT == 8 ? 8 : 4;               // samples per thread per tile
    static constexpr int TILE = THREADS * PER;
};
// An owner's shared-memory buffer holds row_cap records (WcParams; 256 when it fits, else 192 or 128): < WC_LINE carried
// over from the last flush + its share of the samples binned between two flushes + ~3.5 sigma of the binomial; a record
// that does not fit takes the exact route.  Storage per owner = row_cap + one spill line (the remainder copy reads a
// whole line) + 8 records of padding so that the 128-bit accesses of the flush are bank-conflict free.
constexpr int WC_ROW_EXTRA = WC_LINE + 8;

struct WcParams {
    const void *ids;                 // IdT[n], 4*sizeof(IdT)-aligned
    const void *vals;                // ValT[n], 32-byte aligned
    size_t n;                        // multiple of the tile size (the host sends the ragged tail to k_ingest_keyed)
    const void *ids2;                // optional second segment of the same launch (ValT = double only): int64 nanosecond
    const void *vals2;               //   values (TimerToken.Stop(), metrics.go:242-246), converted with (double) like Go's
    size_t n2;                       //   float64(duration.Nanoseconds()); multiple of the tile size, 0 = none
    uint32_t ids_per;                // ceil(H / P)
    uint32_t cap;                    // records per (owner, writer) sub-queue per parity, multiple of WC_LINE
    uint32_t slice_tiles;            // tiles per CTA per chunk
    uint32_t inv_p;                  // floor(2^32 / P) + 1: id / P == __umulhi(id, inv_p) for id < 65536
    uint32_t flush_tiles;            // tiles binned between two flushes of the owner buffers
    uint32_t pf_tiles;               // the tile this many tiles past the one being loaded is asked of L2 (0 = off)
    uint32_t row_cap;                // records an owner's shared-memory buffer holds (multiple of 64; the host takes what fits)
    uint32_t row_stride;             // row_cap + one spill line + 8 records of padding (bank-conflict-free 128-bit flush)
    unsigned short *queues;          // [2][P owners][P writers][cap]
    unsigned int *q_cnt;             // [2][P owners][P writers]
    unsigned int *barrier;           // grid barrier counter, zeroed by the host before the launch
    uint4 *rare;                     // [P][WC_RARE_CAP] samples set aside for the exact path: {raw lo, raw hi, id, -}
    KeyedOut o;
};
constexpr uint32_t WC_RARE_CAP = 8192;       // per CTA and chunk; beyond that a rare sample is resolved on the spot

__device__ __forceinline__ void grid_barrier(unsigned int *bar, unsigned int target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(bar, 1u);
        unsigned int v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
        } while (v < target);
    }
    __syncthreads();
}

// a record that could not be queued: add it to its bucket directly (exact, one L2 atomic; positive rows: slot == key)
template <typename V = IdIdentity>
__device__ __forceinline__ void wc_spill(uint32_t rec, uint32_t owner, uint32_t P, const Prec &pc, const KeyedOut &o, const V &m = {}) {
    const uint32_t lid = rec / pc.win, slot = rec - lid * pc.win, id = m.row(lid * P + owner);
    if (kMapped<V> && id == 0xFFFFFFFFu) { atomicAdd(o.dropped, 1ull); return; }
    add_bucket_global(o.buckets + (size_t)id * 65536u, o.flags + id, slot, 1ull, pc.win);
}

// Mapped (non-PAIR only): ids are local, owners hold ceil(k / P) windows (ids_per) and o.H's bound is k; the map is read
// by the spills, the rare path and the final flush, which counts an unbound row's window total as dropped.
// Bound: the owners' windows are uint32 cells, zeroed at the start and flushed once at the end of the launch, so one
// launch takes at most 2^32 - 1 samples, n + n2 together (kWcMaxLaunch; launch_keyed and plan_keyed keep to it).
template <typename IdT, typename ValT, int SPT, bool PAIR = false, typename Map = IdIdentity>   // PAIR: a second, int64 segment follows the float64 one
__global__ void __launch_bounds__(WcShape<SPT>::THREADS, 1)
k_ingest_keyed_wc(WcParams prm, Prec pc, const Map map) {
    static_assert(!PAIR || std::is_same<ValT, double>::value, "the int64 segment rides on the float64 instantiation");
    static_assert(!PAIR || !kMapped<Map>, "pairs are not mapped");
    const auto mv = map_view(map);
    using S = WcShape<SPT>;
    constexpr int WC_THREADS = S::THREADS;
    constexpr int GROUPS = S::PER / 4;
    extern __shared__ __align__(16) unsigned char wc_smem[];
    const uint32_t P = gridDim.x, p = blockIdx.x, tid = threadIdx.x;
    unsigned int *s_hist = reinterpret_cast<unsigned int *>(wc_smem);                       // [ids_per][win]
    const uint32_t hist_words = prm.ids_per * pc.win;
    unsigned int *s_fill = s_hist + ((hist_words + 3u) & ~3u);                              // records in each owner's buffer
    unsigned int *s_off = s_fill + WC_MAX_PARTS;                                            // records appended to my sub-queues this chunk; phase B: record counts
    unsigned short *s_buf = reinterpret_cast<unsigned short *>(s_off + WC_MAX_PARTS);       // [P + 1][STRIDE], row P = trash
    uint32_t fill_addr = smem_u32(s_fill);
    const uint32_t hist_addr = smem_u32(s_hist);
    asm volatile("mov.b32 %0, %0;" : "+r"(fill_addr));          // keep it in a register: recomputing it costs 7 instructions per tile
    const uint32_t buf_addr = fill_addr + 2u * WC_MAX_PARTS * 4u;
    unsigned int *s_rare = s_fill + (WC_MAX_PARTS - 1);                                     // samples set aside this chunk (slot P..158 of s_fill are free)
    uint4 *rareq = prm.rare + (size_t)p * WC_RARE_CAP;
    uint32_t negP = 0u - P;
    asm volatile("mov.b32 %0, %0;" : "+r"(negP));

    for (uint32_t i = tid; i < hist_words; i += WC_THREADS) s_hist[i] = 0;
    if (tid < WC_MAX_PARTS) { s_fill[tid] = 0; s_off[tid] = 0; }
    uint32_t one_bits;
    asm volatile("mov.b32 %0, 0x3F800000;" : "=r"(one_bits));
    __syncthreads();

    const size_t tiles_seg0 = prm.n / S::TILE;                   // the host passes whole tiles only
    const size_t tiles_total = tiles_seg0 + (PAIR ? prm.n2 / S::TILE : 0);    // tiles [tiles_seg0, tiles_total) are the int64 segment
    const size_t chunk_tiles = (size_t)prm.slice_tiles * P;
    const size_t nchunks = (tiles_total + chunk_tiles - 1) / chunk_tiles;
    const IdT *ids = reinterpret_cast<const IdT *>(prm.ids);
    const unsigned int cap = prm.cap;
    const uint32_t row_cap = prm.row_cap, row_stride = prm.row_stride;


    unsigned long long cur[GROUPS][4], nxt[GROUPS][4];
    IdPack<IdT> cur_id[GROUPS], nxt_id[GROUPS];
    uint32_t since_flush = 0;
    // tile `tile` = TILE consecutive samples; thread tid takes the 4-sample groups tid, tid + THREADS, ... of it.  The
    // pointers below walk the CTA's slice one tile at a time (no 64-bit multiplies inside the loop).
    const char *vptr = nullptr;                  // this thread's first 32-byte value group of the current tile
    const IdT *iptr = nullptr;                   // ... and its 4 ids
    // The register pipeline is one tile deep and the first use of a tile (DADD) is the kernel's hottest stall site: the
    // loads come back late.  A steady L2 prefetch of the tile AFTER the one being loaded turns that load into an L2 hit.
    const size_t pf_v = (size_t)prm.pf_tiles * S::TILE * 8, pf_i = (size_t)prm.pf_tiles * S::TILE;
    auto load_tile = [&](const char *vp, const IdT *ip, unsigned long long (&raw)[GROUPS][4], IdPack<IdT> (&idp)[GROUPS]) {
#pragma unroll
        for (int g = 0; g < GROUPS; g++) {
            load_vals4(vp, (size_t)g * WC_THREADS, raw[g]);
            idp[g].load(ip, (size_t)g * WC_THREADS);
        }
    };

    for (size_t c = 0; c < nchunks; c++) {
        const size_t par = c & 1;
        unsigned short *qset = prm.queues + par * (size_t)P * P * cap;      // [owner][writer][cap]
        unsigned int *cset = prm.q_cnt + par * (size_t)P * P;              // [owner][writer]
        const bool last_chunk = c + 1 == nchunks;
        // ---------------- phase A: bin my slice of chunk c (I am writer p)
        const size_t tile0 = c * chunk_tiles + (size_t)p * prm.slice_tiles;
        const uint32_t ntile_all = tile0 >= tiles_total ? 0u : (uint32_t)min((size_t)prm.slice_tiles, tiles_total - tile0);   // uniform per CTA
        // one tile: bin the 4-sample groups held in (raw, idp), then flush when due.  Two register sets alternate (A is
        // being binned while B's loads are in flight and vice versa), so no register copies between tiles.
        auto bin_tile = [&](unsigned long long (&raw)[GROUPS][4], IdPack<IdT> (&idp)[GROUPS], const bool as_i64) {
            if constexpr (PAIR) {
                if (as_i64) {                    // tile of the int64 segment (warp-uniform): from here on the bits are a float64
#pragma unroll
                    for (int g = 0; g < GROUPS; g++)
#pragma unroll
                        for (int j = 0; j < 4; j++) raw[g][j] = (unsigned long long)__double_as_longlong(__ll2double_rn((long long)raw[g][j]));
                }
            }
#pragma unroll
            for (int g = 0; g < GROUPS; g++) {
                double v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) { ValT r; memcpy(&r, &raw[g][j], 8); v[j] = sample_to_f64<ValT>(r); }
                uint32_t idx[4];
                bool flag[4];
                bucket_offsets_v2<4, false, 0>(v, pc, one_bits, idx, flag);      // slot indices (positive-only rows)
                bool any = false;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t id = idp[g].get(j);
                    const uint32_t lid = __umulhi(id, prm.inv_p), owner = lid * negP + id;   // id / P, id % P
                    const uint32_t rec = lid * pc.win + idx[j];
                    const bool rare = flag[j] | (id >= mv.bound(prm.o.H));
                    // branch-free append: rare samples draw from a trash counter (a predicated atomic makes ptxas branch and spill)
                    const uint32_t oe = rare ? P : owner;
                    uint32_t pos;
                    asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(pos) : "r"(fill_addr + oe * 4u) : "memory");
                    flag[j] = rare | (pos >= row_cap);                            // buffer full (skewed ids): exact route as well
                    if (!flag[j])                                                          // one predicated store, no branch
                        asm volatile("st.shared.u16 [%0], %1;" ::"r"(buf_addr + (oe * row_stride + pos) * 2u), "h"((unsigned short)rec) : "memory");
                    any |= flag[j];
                }
                if (__any_sync(0xFFFFFFFFu, any)) {
                    // set the sample aside: the exact path (FP64 log, ~1K cycles) is run for all of them together at the end of
                    // the chunk, every lane busy, instead of stalling this warp lane by lane in the middle of the stream
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (flag[j]) {
                            const unsigned int at = atomicAdd(s_rare, 1u);
                            if (at < WC_RARE_CAP) rareq[at] = make_uint4((unsigned int)raw[g][j], (unsigned int)(raw[g][j] >> 32), idp[g].get(j), 0u);
                            else keyed_one_slow_v<ValT>(idp[g].get(j), raw[g][j], pc, prm.o, mv);
                        }
                }
            }
            // ---- flush every prm.flush_tiles tiles.  Four lanes (4 x 32 B = one 128-byte line) serve one owner, so the
            //      8 x 32 = 256 lane groups of the CTA cover all owners in ONE pass: an owner's full lines go to my sub-queue
            //      of that owner as coalesced 128-byte stores, the remainder (< 64 records) moves to the front.  No barrier
            //      is needed between tiles that do not flush: appends are atomic.
            if (++since_flush == prm.flush_tiles) {
                since_flush = 0;
                __syncthreads();
                constexpr uint32_t GROUPS_PER_WARP = 8;
                const uint32_t sub = (tid & 31) >> 2, k4 = (tid & 3) * 2;
                for (uint32_t base = (tid >> 5) * GROUPS_PER_WARP; base < P; base += (WC_THREADS / 32) * GROUPS_PER_WARP) {   // warp-uniform trip count
                    const uint32_t o = base + sub;
                    const bool act = o < P;
                    unsigned int n = 0, nfull = 0, off0 = 0;
                    uint4 keep0 = make_uint4(0, 0, 0, 0), keep1 = keep0;
                    uint4 *src = reinterpret_cast<uint4 *>(s_buf + (act ? o : 0) * row_stride);
                    if (act) {
                        n = min(s_fill[o], row_cap);
                        nfull = n / WC_LINE;
                        off0 = s_off[o];
                        unsigned short *qbase = qset + ((size_t)o * P + p) * cap;
                        keep0 = src[nfull * 8 + k4];                                       // the line that holds the remainder
                        keep1 = src[nfull * 8 + k4 + 1];
                        for (unsigned int l = 0; l < nfull; l++) {
                            if (off0 + WC_LINE <= cap) {
                                uint4 *dst = reinterpret_cast<uint4 *>(qbase + off0);
                                const uint4 a0 = src[l * 8 + k4], a1 = src[l * 8 + k4 + 1];
                                dst[k4] = a0;
                                dst[k4 + 1] = a1;
                                off0 += WC_LINE;
                            } else if (k4 == 0) {                                          // sub-queue full: these records go the L2 route
                                const unsigned short *r = s_buf + o * row_stride + l * WC_LINE;
                                for (unsigned int k = 0; k < (unsigned int)WC_LINE; k++) wc_spill(r[k], o, P, pc, prm.o, mv);
                            }
                        }
                    }
                    __syncwarp();
                    if (act) {
                        if (nfull) { src[k4] = keep0; src[k4 + 1] = keep1; }
                        if (k4 == 0) { s_off[o] = off0; s_fill[o] = n - nfull * WC_LINE; }
                    }
                }
                __syncthreads();
            }
        };
        // the slice may straddle the two segments: part 0 = its float64 tiles, part 1 = its int64 tiles
        for (int part = 0; part < (PAIR ? 2 : 1); part++) {
            const size_t lo = part == 0 ? tile0 : max(tile0, tiles_seg0);
            const size_t hi = part == 0 ? min(tile0 + ntile_all, tiles_seg0) : tile0 + ntile_all;
            if (hi <= lo) continue;
            const uint32_t ntile = (uint32_t)(hi - lo);
            const bool as_i64 = part == 1;
            const size_t first = (part == 0 ? lo : lo - tiles_seg0) * S::TILE + (size_t)tid * 4;     // sample index inside the segment
            vptr = reinterpret_cast<const char *>(part == 0 ? prm.vals : prm.vals2) + first * 8;
            iptr = (part == 0 ? ids : reinterpret_cast<const IdT *>(prm.ids2)) + first;
            load_tile(vptr, iptr, cur, cur_id);
            auto prefetch_ahead = [&](uint32_t tile_loaded) {       // tile_loaded: index (in this part) of the tile vptr points to
                if (prm.pf_tiles && tile_loaded + prm.pf_tiles < ntile) {
#pragma unroll
                    for (int g = 0; g < GROUPS; g++) {
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(vptr + pf_v + (size_t)g * WC_THREADS * 32));
                        if ((tid & 3) == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(iptr + pf_i + (size_t)g * WC_THREADS * 4));
                    }
                }
            };
            for (uint32_t t = 0; t < ntile; t += 2) {
                vptr += (size_t)S::TILE * 8;                 // -> tile t + 1
                iptr += S::TILE;
                if (t + 1 < ntile) load_tile(vptr, iptr, nxt, nxt_id);
                prefetch_ahead(t + 1);
                bin_tile(cur, cur_id, as_i64);
                if (t + 1 >= ntile) break;
                vptr += (size_t)S::TILE * 8;                 // -> tile t + 2
                iptr += S::TILE;
                if (t + 2 < ntile) load_tile(vptr, iptr, cur, cur_id);
                prefetch_ahead(t + 2);
                bin_tile(nxt, nxt_id, as_i64);
            }
        }
        __syncthreads();    // every append of this chunk's tiles is in the buffers
        {   // the samples set aside: exact path, all threads at once
            const unsigned int nr = min(*s_rare, WC_RARE_CAP);
            for (unsigned int i = tid; i < nr; i += WC_THREADS) {
                const uint4 e = rareq[i];
                ValT r;
                const unsigned long long raw = ((unsigned long long)e.y << 32) | e.x;
                memcpy(&r, &raw, 8);
                keyed_one_direct<ValT>(e.z, r, pc, prm.o, mv);
            }
            __syncthreads();
            if (tid == 0) *s_rare = 0;
        }
        if (last_chunk) {   // everything still waiting in the buffers goes out, the last line of each owner partially filled
            if (tid < P) {
                const uint32_t o = tid;
                const unsigned int n = min(s_fill[o], row_cap);
                unsigned int off0 = s_off[o];
                const uint4 *src = reinterpret_cast<const uint4 *>(s_buf + o * row_stride);
                for (unsigned int l = 0; l * WC_LINE < n; l++) {
                    const unsigned int nrec = min((unsigned int)WC_LINE, n - l * WC_LINE);
                    if (off0 + WC_LINE <= cap) {
                        uint4 *dst = reinterpret_cast<uint4 *>(qset + ((size_t)o * P + p) * cap + off0);
#pragma unroll
                        for (int k = 0; k < 8; k++) dst[k] = src[l * 8 + k];
                        off0 += nrec;
                    } else {
                        const unsigned short *r = s_buf + o * row_stride + l * WC_LINE;
                        for (unsigned int k = 0; k < nrec; k++) wc_spill(r[k], o, P, pc, prm.o, mv);
                    }
                }
                s_off[o] = off0;
                s_fill[o] = 0;
            }
            __syncthreads();
        }
        // publish my P record counts (zero for owners I sent nothing to), then the grid-wide barrier
        if (tid < P) { cset[(size_t)tid * P + p] = s_off[tid]; }
        grid_barrier(prm.barrier, (unsigned int)((c + 1) * (size_t)P));
        // ---------------- phase B: drain the P sub-queues I own.  The record counts go to shared memory first; then the
        // P * vq 16-byte vectors of my region are dealt to the threads as ONE flat index space (vector v belongs to
        // writer v / vq), so every thread has several independent L2 loads in flight instead of a count -> data chain.
        if (tid < P) s_off[tid] = __ldcg(&cset[(size_t)p * P + tid]);
        __syncthreads();
        {
            // warp w drains the sub-queues of writers w, w + NW, ...: the record counts are already in shared memory, so the
            // 16-byte vector loads of a sub-queue are independent (a lane has several in flight) and no index is wasted
            const unsigned short *qmine = qset + (size_t)p * P * cap;
            const uint32_t lane = tid & 31;
#define LH_WC_INC2(word)                                                                                              \
            asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(hist_addr + (((word) << 2) & 0x3FFFCu)) : "memory");     \
            asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(hist_addr + (((word) >> 14) & 0x3FFFCu)) : "memory");
            for (uint32_t w = tid >> 5; w < P; w += WC_THREADS / 32) {
                const unsigned int cnt = s_off[w];
                const unsigned short *q = qmine + (size_t)w * cap;
                const uint4 *qv = reinterpret_cast<const uint4 *>(q);
                const unsigned int nv = cnt >> 3;
#pragma unroll 2
                for (unsigned int i = lane; i < nv; i += 32) {
                    const uint4 v4 = __ldcg(qv + i);
                    LH_WC_INC2(v4.x) LH_WC_INC2(v4.y) LH_WC_INC2(v4.z) LH_WC_INC2(v4.w)
                }
                const unsigned int r0 = nv * 8u + lane;                                    // the < 8 records after the last full vector
                if (r0 < cnt) asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(hist_addr + (unsigned int)__ldcg(q + r0) * 4u) : "memory");
            }
#undef LH_WC_INC2
        }
        __syncthreads();
        if (tid < P) s_off[tid] = 0;
        // no grid barrier here: the next chunk writes the other parity; this parity is rewritten only after the
        // next grid barrier, which every CTA reaches after finishing this drain
    }
    __syncthreads();
    // ---------------- flush my windows straight into the uint64 bucket arrays (positive rows: slot == key) and raise the
    // flags of the histograms that received counts; nothing of the common path goes through the uint32 hot window
    for (uint32_t lid = 0; lid < prm.ids_per; lid++) {
        if (lid * P + p >= mv.bound(prm.o.H)) break;
        const uint32_t id = mv.row(lid * P + p);
        if (kMapped<Map> && id == 0xFFFFFFFFu) {
            unsigned long long lost = 0;
            for (uint32_t slot = tid; slot < pc.win; slot += WC_THREADS) lost += s_hist[lid * pc.win + slot];
            if (lost) atomicAdd(prm.o.dropped, lost);
            continue;
        }
        int any = 0;
        for (uint32_t slot = tid; slot < pc.win; slot += WC_THREADS) {
            const unsigned int cnt = s_hist[lid * pc.win + slot];
            if (cnt) { atomicAdd(&prm.o.buckets[(size_t)id * 65536u + slot], (unsigned long long)cnt); any = 1; }
        }
        any = __syncthreads_or(any);
        if (any && tid == 0) mark(&prm.o.flags[id], 1u);
    }
}

// Drain the hot window into the uint64 buckets.  atomicExch/atomicAdd so that ingest on other
// streams may keep running against the same buffer.
__global__ void k_fold_hot(unsigned int *__restrict__ hot, unsigned long long *__restrict__ buckets, uint32_t *__restrict__ flags,
                           size_t cells, uint32_t replicas, uint32_t win) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const uint32_t row = 2u * win;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += stride) {
        unsigned long long sum = 0;
        for (uint32_t r = 0; r < replicas; r++) {
            unsigned int *cell = hot + (size_t)r * cells + i;
            if (*cell) sum += atomicExch(cell, 0u);
        }
        if (sum) {
            size_t h = i / row;
            uint32_t slot = (uint32_t)(i - h * row);
            atomicAdd(&buckets[h * 65536u + slot_to_key16(slot, win)], sum);
            mark(&flags[h], 1u);
        }
    }
}

// ---------------------------------------------------------------------- K2
// Counter(name, amount): counters[id] += amount (wrapping uint64).  Up to
// K2_SMEM_COUNTERS ids are privatised per CTA as lo/hi uint32 halves in shared
// memory: one returning shared atomic on the low half, a second one on the
// high half only when the amount has high bits or the low half carried.
constexpr int K2_SMEM_COUNTERS = 8192;

// Mapped (k_counter_add_smem{,_vec}): C is the number of local ids; the map follows the 2C halves in shared memory, an
// op is dropped per op when its local id is >= C or unbound, and the flush adds counter i into its row.
// The steps both kernels share: s_cnt is [C] low halves, [C] high halves, then the map.
template <int THREADS, typename Map>
__device__ __forceinline__ auto counter_smem_init(unsigned int *s_cnt, uint32_t C, const Map &map) {
    for (uint32_t i = threadIdx.x; i < 2 * C; i += THREADS) s_cnt[i] = 0;
    const auto mv = map_to_smem(map, s_cnt + 2 * C);
    __syncthreads();
    return mv;
}
template <typename MV>
__device__ __forceinline__ void counter_smem_add(unsigned int *s_cnt, uint32_t C, uint32_t id, unsigned long long amt,
                                                 unsigned long long *dropped, const MV &mv) {
    if (mv.drops(id, C)) { atomicAdd(dropped, 1ull); return; }
    unsigned int a_lo = (unsigned int)amt, a_hi = (unsigned int)(amt >> 32);
    unsigned int old = atomicAdd(&s_cnt[id], a_lo);
    a_hi += (old + a_lo < old) ? 1u : 0u;        // carry out of the low half
    if (a_hi) atomicAdd(&s_cnt[C + id], a_hi);
}
template <int THREADS, typename MV>
__device__ __forceinline__ void counter_smem_flush(const unsigned int *s_cnt, uint32_t C, unsigned long long *counters, const MV &mv) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < C; i += THREADS) {
        unsigned long long v = ((unsigned long long)s_cnt[C + i] << 32) | s_cnt[i];
        if (v) atomicAdd(&counters[mv.row(i)], v);            // v == 0 for an unbound row: its ops were dropped
    }
}

template <typename IdT, int THREADS, typename Map = IdIdentity>
__global__ void __launch_bounds__(THREADS)
k_counter_add_smem(const IdT *__restrict__ ids, const unsigned long long *__restrict__ amounts, size_t n,
                   unsigned long long *__restrict__ counters, uint32_t C,
                   unsigned long long *__restrict__ dropped, const Map map) {
    extern __shared__ unsigned int s_cnt[];
    const auto mv = counter_smem_init<THREADS>(s_cnt, C, map);
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += stride)
        counter_smem_add(s_cnt, C, (uint32_t)ids[i], amounts[i], dropped, mv);
    counter_smem_flush<THREADS>(s_cnt, C, counters, mv);
}

// Vector body: 4 consecutive (id, amount) pairs per thread and iteration (two 128-bit amount loads, one 64/128-bit id
// load), the next group prefetched while the current one is added.  amounts 32-byte aligned, ids 4*sizeof(IdT)-aligned.
template <typename IdT, int THREADS, typename Map = IdIdentity>
__global__ void __launch_bounds__(THREADS)
k_counter_add_smem_vec(const IdT *__restrict__ ids, const unsigned long long *__restrict__ amounts, size_t n4,
                       unsigned long long *__restrict__ counters, uint32_t C, unsigned long long *__restrict__ dropped,
                       const Map map) {
    extern __shared__ unsigned int s_cnt[];
    const auto mv = counter_smem_init<THREADS>(s_cnt, C, map);
    const size_t stride = (size_t)gridDim.x * THREADS;
    size_t g = (size_t)blockIdx.x * THREADS + threadIdx.x;
    unsigned long long cur[4], nxt[4];
    IdPack<IdT> cid, nid;
    if (g < n4) { load_vals4(amounts, g, cur); cid.load(ids, g); }
    for (; g < n4; g += stride) {
        const size_t gn = g + stride;
        if (gn < n4) { load_vals4(amounts, gn, nxt); nid.load(ids, gn); }
#pragma unroll
        for (int j = 0; j < 4; j++) counter_smem_add(s_cnt, C, cid.get(j), cur[j], dropped, mv);
#pragma unroll
        for (int j = 0; j < 4; j++) cur[j] = nxt[j];
        cid = nid;
    }
    counter_smem_flush<THREADS>(s_cnt, C, counters, mv);
}

template <typename IdT, int THREADS>
__global__ void __launch_bounds__(THREADS)
k_counter_add(const IdT *__restrict__ ids, const unsigned long long *__restrict__ amounts, size_t n,
              unsigned long long *__restrict__ counters, uint32_t C,
              unsigned long long *__restrict__ dropped) {
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += stride) {
        uint32_t id = (uint32_t)ids[i];
        if (id < C) atomicAdd(&counters[id], amounts[i]);
        else atomicAdd(dropped, 1ull);
    }
}

// ------------------------------------------------------------------- merge
// Adds sparse (histogram id, int16 key, uint64 count) triples -- the wire format lh_snapshot_export produces --
// into the bucket arrays: merging snapshots from other hosts / GPUs is the same commutative uint64 sum.
__global__ void k_merge_sparse(const uint32_t *__restrict__ ids, const short *__restrict__ keys,
                               const unsigned long long *__restrict__ counts, size_t n, uint32_t H,
                               unsigned long long *__restrict__ buckets, uint32_t *__restrict__ flags,
                               unsigned long long *__restrict__ dropped, uint32_t win) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t id = ids[i];
        if (id >= H) { atomicAdd(dropped, 1ull); continue; }
        add_bucket_global(buckets + (size_t)id * 65536u, flags + id, (uint32_t)(int)keys[i] & 0xFFFFu, counts[i], win);
    }
}

// ---------------------------------------------------------------------- K3
// One CTA per histogram, 32 warps.  Warp w owns the 2048 consecutive keys
// [-32768 + 2048 w, +2047] (ascending key == ascending value, the order
// percentile() sorts into, metrics.go:409) and reads them as 64 coalesced
// 256-byte rows.  Pass 1: per-warp count / sum / non-empty totals, then a scan
// over the 32 warp totals.  Pass 2: the warp whose range contains a
// percentile's crossing walks its rows again (L2 hits) with a warp prefix sum
// and applies the reference's rule float64(sofar)/float64(total) >= p
// (metrics.go:413) to non-empty buckets only.
// The histogram's flag prunes the scan: untouched histograms are answered without reading a bucket, and when
// every count lies in the fast window only the (at most 6) warps that overlap it read anything.
constexpr int K3_THREADS = 1024;
constexpr int K3_WARP_KEYS = 2048;

__device__ __forceinline__ bool warp_scans(int key0, uint32_t level, uint32_t win) {
    if (level & 2u) return true;
    return key0 <= (int)win - 1 && key0 + K3_WARP_KEYS - 1 >= -((int)win - 1);
}

__device__ __forceinline__ void reduce_dense(uint32_t level, const unsigned long long *__restrict__ buckets, const uint32_t *__restrict__ flags, uint32_t win,
         const double *__restrict__ decomp,
         const double *__restrict__ ps, int np, unsigned long long *__restrict__ out_count,
         double *__restrict__ out_sum, double *__restrict__ out_avg, int *__restrict__ out_pkeys,
         double *__restrict__ out_pvals, uint32_t *__restrict__ out_nnz) {
    __shared__ unsigned long long s_cnt[32];    // per-warp totals, then exclusive prefix
    __shared__ unsigned long long s_tot[32];    // per-warp totals (kept)
    __shared__ double s_sum[32];
    __shared__ unsigned int s_nnz[32];
    __shared__ int s_owner[LH_MAX_PCT];
    __shared__ unsigned long long s_total;
    const int h = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const unsigned long long *hb = buckets + (size_t)h * 65536u;
    const int key0 = -32768 + warp * K3_WARP_KEYS;
    const bool scans = warp_scans(key0, level, win);

    unsigned long long mine = 0;
    double msum = 0.0;
    unsigned int nnz = 0;
    unsigned int high = 0;   // OR of the counts' high words: 64 counts below 2^58 cannot pass 2^64
    if (scans) {
#pragma unroll 16
        for (int r = 0; r < K3_WARP_KEYS / 32; r++) {      // 16 independent 256-byte rows in flight per warp
            unsigned int slot = (unsigned int)(key0 + r * 32 + lane) & 0xFFFFu;
            unsigned long long c = hb[slot];
            high |= (unsigned int)(c >> 32);
            if (c) { mine += c; msum += decomp[slot] * (double)c; nnz++; }
        }
    }
    // an addition of the count reduction or scan passed 2^64 (the exact total is >= 2^64).  A lane with a count of
    // 2^58 or more adds its cells again with a check per addition; the reduction and the scan below check each step.
    int wrap = 0;
    if (high >> 26) {
        unsigned long long again = 0;
        for (int r = 0; r < K3_WARP_KEYS / 32; r++) {
            const unsigned long long c = hb[(unsigned int)(key0 + r * 32 + lane) & 0xFFFFu];
            again += c;
            wrap |= again < c;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, mine, o);
        mine += y;
        wrap |= mine < y;
        msum += __shfl_xor_sync(0xFFFFFFFFu, msum, o);
        nnz += __shfl_xor_sync(0xFFFFFFFFu, nnz, o);
    }
    if (lane == 0) { s_cnt[warp] = mine; s_tot[warp] = mine; s_sum[warp] = msum; s_nnz[warp] = nnz; }
    if (t < LH_MAX_PCT) s_owner[t] = 0x7FFFFFFF;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = s_cnt[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
            if (lane >= o) { wi += y; wrap |= wi < y; }
        }
        s_cnt[lane] = wi - w;
        if (lane == 31) s_total = wi;
        double ts = s_sum[lane];
        unsigned int tn = s_nnz[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ts += __shfl_xor_sync(0xFFFFFFFFu, ts, o);
            tn += __shfl_xor_sync(0xFFFFFFFFu, tn, o);
        }
        if (lane == 0) { s_sum[0] = ts; s_nnz[0] = tn; }
    }
    const bool wrapped = __syncthreads_or(wrap);
    const unsigned long long total = s_total;
    const double ftotal = (double)total;
    if (wrapped) {
        // Go's uint64 running count wrapped: a crossing inside a warp need not survive to the warp's end, so every
        // scanning warp applies the rule to each of its non-empty cells (running counts mod 2^64, as Go's) and the
        // block keeps the smallest key per percentile.
        if (scans) {
            unsigned long long sofar = s_cnt[warp];
            unsigned int pending = np == 32 ? 0xFFFFFFFFu : (1u << np) - 1u;
            for (int r = 0; r < K3_WARP_KEYS / 32 && pending; r++) {
                const int key = key0 + r * 32 + lane;
                const unsigned long long c = hb[(unsigned int)key & 0xFFFFu];
                unsigned long long incl = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                    if (lane >= o) incl += y;
                }
                const double frac = __ddiv_rn((double)(sofar + incl), ftotal);
                for (int j = 0; j < np; j++) {
                    if (!(pending >> j & 1u)) continue;
                    const unsigned int hit = __ballot_sync(0xFFFFFFFFu, c != 0 && frac >= ps[j]);
                    if (hit) {
                        if (lane == __ffs(hit) - 1) atomicMin(&s_owner[j], key);
                        pending &= ~(1u << j);
                    }
                }
                sofar += __shfl_sync(0xFFFFFFFFu, incl, 31);
            }
        }
        __syncthreads();
        if (t < np && s_owner[t] != 0x7FFFFFFF) {
            out_pkeys[(size_t)h * np + t] = s_owner[t];
            out_pvals[(size_t)h * np + t] = decomp[(unsigned int)s_owner[t] & 0xFFFFu];
        }
    } else {
        // owner of percentile j = first non-empty warp whose inclusive prefix satisfies the rule
        if (lane == 0 && s_tot[warp]) {
            const unsigned long long end_incl = s_cnt[warp] + s_tot[warp];
            for (int j = 0; j < np; j++)
                if (__ddiv_rn((double)end_incl, ftotal) >= ps[j]) atomicMin(&s_owner[j], warp);
        }
        __syncthreads();
        unsigned int pending = 0;
        for (int j = 0; j < np; j++) if (s_owner[j] == warp) pending |= 1u << j;
        if (pending) {
            unsigned long long sofar = s_cnt[warp];
            for (int r = 0; r < K3_WARP_KEYS / 32 && pending; r++) {
                int key = key0 + r * 32 + lane;
                unsigned long long c = hb[(unsigned int)key & 0xFFFFu];
                unsigned long long incl = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                    if (lane >= o) incl += y;
                }
                const double frac = __ddiv_rn((double)(sofar + incl), ftotal);
                for (int j = 0; j < np; j++) {
                    if (!(pending >> j & 1u)) continue;
                    unsigned int hit = __ballot_sync(0xFFFFFFFFu, c != 0 && frac >= ps[j]);
                    if (hit) {
                        if (lane == __ffs(hit) - 1) {
                            out_pkeys[(size_t)h * np + j] = key;
                            out_pvals[(size_t)h * np + j] = decomp[(unsigned int)key & 0xFFFFu];
                        }
                        pending &= ~(1u << j);
                    }
                }
                sofar += __shfl_sync(0xFFFFFFFFu, incl, 31);
            }
        }
    }
    if (t == 0) {
        for (int j = 0; j < np; j++)
            if (s_owner[j] == 0x7FFFFFFF) {   // percentile() error (no bucket satisfies the rule): key omitted by the caller
                out_pkeys[(size_t)h * np + j] = (int)0x80000000;
                out_pvals[(size_t)h * np + j] = __longlong_as_double(0x7FF8000000000000ll);
            }
        out_count[h] = total;
        out_sum[h] = s_sum[0];
        out_avg[h] = __ddiv_rn(s_sum[0], ftotal);    // metrics.go:356 (NaN when empty)
        out_nnz[h] = s_nnz[0];
    }
}

// percentile_threshold (the integer form of the reference's percentile rule) lives in the public device header,
// where lh::raw_percentile shares it.

// One CTA per histogram.  Untouched histograms are answered without reading a bucket.  A histogram whose counts all
// lie in the fast window (flag 1; the normal case) is reduced from shared memory: its 2*win-1 cells are loaded once
// (ascending key order == ascending value order, metrics.go:409), count / sum / non-empty totals come from a block
// reduction, an in-place block scan turns the cells into running counts, and every percentile is one binary search
// for its integer threshold -- no per-bucket FP64 division, no serial walk.  Histograms with out-of-window keys
// (wrapped int16 keys, NaN / Inf -> 0 ...) take the dense path over all 65 536 keys.
__global__ void __launch_bounds__(K3_THREADS)
k_reduce(const unsigned long long *__restrict__ buckets, const uint32_t *__restrict__ flags, uint32_t win,
         const double *__restrict__ decomp,
         const double *__restrict__ ps, int np, unsigned long long *__restrict__ out_count,
         double *__restrict__ out_sum, double *__restrict__ out_avg, int *__restrict__ out_pkeys,
         double *__restrict__ out_pvals, uint32_t *__restrict__ out_nnz, uint32_t smem_cells) {
    extern __shared__ __align__(16) unsigned long long k3_cells[];      // [2*win-1] when the window path is enabled
    const int h = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t level = flags[h];
    if (level == 0) {   // untouched this interval: the caller reports the histogram as absent
        if (t == 0) {
            out_count[h] = 0; out_sum[h] = 0.0; out_avg[h] = __longlong_as_double(0x7FF8000000000000ll); out_nnz[h] = 0;
            for (int j = 0; j < np; j++) {
                out_pkeys[(size_t)h * np + j] = (int)0x80000000;
                out_pvals[(size_t)h * np + j] = __longlong_as_double(0x7FF8000000000000ll);
            }
        }
        return;
    }
    const uint32_t n = 2u * win - 1u;
    if ((level & 2u) || smem_cells < n) {
        reduce_dense(level, buckets, flags, win, decomp, ps, np, out_count, out_sum, out_avg, out_pkeys, out_pvals, out_nnz);
        return;
    }
    __shared__ unsigned long long s_c[32];
    __shared__ double s_s[32];
    __shared__ unsigned int s_n[32];
    __shared__ unsigned long long s_total;
    const unsigned long long *hb = buckets + (size_t)h * 65536u;
    // cell i of the window holds key i - (win-1)
    constexpr int PER = 32;                                       // contiguous cells per thread in the scan (PER * 1024 >= n up to win = 16384)
    unsigned long long mine = 0;
    double msum = 0.0;
    unsigned int nnz = 0;
    unsigned int high = 0;                                        // OR of the counts' high words
    for (uint32_t i = t; i < n; i += K3_THREADS) {
        const unsigned int slot = (unsigned int)((int)i - (int)(win - 1u)) & 0xFFFFu;
        const unsigned long long c = hb[slot];
        k3_cells[i] = c;
        high |= (unsigned int)(c >> 32);
        if (c) { mine += c; msum += decomp[slot] * (double)c; nnz++; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mine += __shfl_xor_sync(0xFFFFFFFFu, mine, o);
        msum += __shfl_xor_sync(0xFFFFFFFFu, msum, o);
        nnz += __shfl_xor_sync(0xFFFFFFFFu, nnz, o);
    }
    if (lane == 0) { s_c[warp] = mine; s_s[warp] = msum; s_n[warp] = nnz; }
    // at most 2^15 cells below 2^49 each cannot sum to 2^64: only a window holding a count of 2^49 or more checks its
    // scan for a running count that passes 2^64
    const int big = __syncthreads_or(high >> 17);
    if (warp == 0) {
        unsigned long long c = s_c[lane];
        double sm = s_s[lane];
        unsigned int nz = s_n[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
            sm += __shfl_xor_sync(0xFFFFFFFFu, sm, o);
            nz += __shfl_xor_sync(0xFFFFFFFFu, nz, o);
        }
        if (lane == 0) {
            s_total = c;
            out_count[h] = c;
            out_sum[h] = sm;
            out_avg[h] = __ddiv_rn(sm, (double)c);                // metrics.go:356
            out_nnz[h] = nz;
        }
    }
    // in-place inclusive scan of the cells: thread t owns cells [t*per, (t+1)*per)
    const uint32_t per = (n + K3_THREADS - 1) / K3_THREADS;
    const uint32_t first = t * per, last = min(first + per, n);
    unsigned long long local = 0;
    for (uint32_t i = first; i < last; i++) local += k3_cells[i];
    unsigned long long incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += y;
    }
    __syncthreads();                                              // s_c was read by warp 0 above
    if (lane == 31) s_c[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = s_c[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
            if (lane >= o) wi += y;
        }
        s_c[lane] = wi - w;                                       // exclusive prefix of the warp totals
    }
    __syncthreads();
    unsigned long long run = s_c[warp] + incl - local;
    int wrap = 0;                                                 // a step of the running count passed 2^64
    if (big) {
        for (uint32_t i = first; i < last; i++) { const unsigned long long c = k3_cells[i]; run += c; k3_cells[i] = run; wrap |= run < c; }
    } else {
        for (uint32_t i = first; i < last; i++) { run += k3_cells[i]; k3_cells[i] = run; }
    }
    if (__syncthreads_or(wrap)) {
        // Go's uint64 running count wrapped (the counts sum to 2^64 or more): it is no longer monotone and the total
        // may be 0, so apply the rule literally.  Cell i is non-empty iff its running count differs from cell i-1's;
        // percentile j is the first non-empty cell with float64(run) / float64(total) >= p (x / 0.0 = +Inf, 0 / 0.0 =
        // NaN), the minimum over the threads' first hits in their own cells.
        if (t < LH_MAX_PCT) s_c[t] = ~0ull;
        __syncthreads();
        const double ftotal = (double)s_total;
        for (int j = 0; j < np; j++) {
            const double p = ps[j];
            unsigned int hit = 0xFFFFFFFFu;
            unsigned long long prev = first && first < last ? k3_cells[first - 1] : 0ull;
            for (uint32_t i = first; i < last; i++) {
                const unsigned long long r = k3_cells[i];
                if (r != prev && __ddiv_rn((double)r, ftotal) >= p) { hit = i; break; }
                prev = r;
            }
            hit = __reduce_min_sync(0xFFFFFFFFu, hit);
            if (lane == 0 && hit != 0xFFFFFFFFu) atomicMin(&s_c[j], (unsigned long long)hit);
        }
        __syncthreads();
        if (t < np) {
            int key = (int)0x80000000;
            double val = __longlong_as_double(0x7FF8000000000000ll);
            if (s_c[t] != ~0ull) {
                key = (int)s_c[t] - (int)(win - 1u);
                val = decomp[(unsigned int)key & 0xFFFFu];
            }
            out_pkeys[(size_t)h * np + t] = key;
            out_pvals[(size_t)h * np + t] = val;
        }
        return;
    }
    (void)PER;
    // one thread per percentile: integer threshold, then the first cell whose running count reaches it.  Without a
    // wrap the running counts are exact and monotone, and a total of 0 means no non-empty cell.
    if (t < np) {
        const unsigned long long total = s_total;
        unsigned long long T;
        int key = (int)0x80000000;
        double val = __longlong_as_double(0x7FF8000000000000ll);
        if (total && percentile_threshold(ps[t], total, &T)) {
            if (T == 0) T = 1;                                    // p <= 0: the smallest non-empty bucket
            uint32_t lo = 0, hi = n - 1;                          // k3_cells[n-1] == total >= T
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (k3_cells[mid] >= T) hi = mid; else lo = mid + 1; }
            key = (int)lo - (int)(win - 1u);
            val = decomp[(unsigned int)key & 0xFFFFu];
        }
        out_pkeys[(size_t)h * np + t] = key;
        out_pvals[(size_t)h * np + t] = val;
    }
}

// ---------------------------------------------------------------------- K4
// offsets[h] = exclusive prefix of nnz (computed by k_scan_nnz); entries are
// written in ascending key order.
__global__ void k_scan_nnz(const uint32_t *__restrict__ nnz, uint32_t H, uint32_t *__restrict__ offsets) {
    // single CTA, H is small (<= a few thousand): serial per-chunk scan is fine
    __shared__ uint32_t s_part[1024];
    const int t = threadIdx.x;
    const uint32_t per = (H + 1023u) / 1024u;
    uint32_t a = 0;
    for (uint32_t i = 0; i < per; i++) { uint32_t idx = t * per + i; if (idx < H) a += nnz[idx]; }
    s_part[t] = a;
    __syncthreads();
    if (t == 0) { uint32_t run = 0; for (int i = 0; i < 1024; i++) { uint32_t x = s_part[i]; s_part[i] = run; run += x; } offsets[H] = run; }
    __syncthreads();
    uint32_t run = s_part[t];
    for (uint32_t i = 0; i < per; i++) { uint32_t idx = t * per + i; if (idx < H) { offsets[idx] = run; run += nnz[idx]; } }
}

__global__ void __launch_bounds__(K3_THREADS)
k_export(const unsigned long long *__restrict__ buckets, const uint32_t *__restrict__ flags, uint32_t win,
         const uint32_t *__restrict__ offsets, short *__restrict__ out_keys, unsigned long long *__restrict__ out_counts) {
    __shared__ unsigned int s_warp[32];
    const int h = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t level = flags[h];
    if (level == 0) return;
    const unsigned long long *hb = buckets + (size_t)h * 65536u;
    const int key0 = -32768 + warp * K3_WARP_KEYS;
    const bool scans = warp_scans(key0, level, win);
    unsigned int nnz = 0;
    if (scans) {
#pragma unroll 4
        for (int r = 0; r < K3_WARP_KEYS / 32; r++)
            nnz += __popc(__ballot_sync(0xFFFFFFFFu, hb[(unsigned int)(key0 + r * 32 + lane) & 0xFFFFu] != 0));
    }
    if (lane == 0) s_warp[warp] = nnz;     // every lane holds the warp total
    __syncthreads();
    if (warp == 0) {
        unsigned int w = s_warp[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { unsigned int y = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += y; }
        s_warp[lane] = wi - w;
    }
    __syncthreads();
    if (!nnz) return;
    unsigned int pos = offsets[h] + s_warp[warp];
    for (int r = 0; r < K3_WARP_KEYS / 32; r++) {
        int key = key0 + r * 32 + lane;
        unsigned long long c = hb[(unsigned int)key & 0xFFFFu];
        unsigned int m = __ballot_sync(0xFFFFFFFFu, c != 0);
        if (c) {
            unsigned int p = pos + __popc(m & ((1u << lane) - 1u));
            out_keys[p] = (short)key;
            out_counts[p] = c;
        }
        pos += __popc(m);
    }
}

// Zero what an interval wrote: per touched histogram its window cells (all 65536 when it holds out-of-window
// counts), then its flag.  Replaces a memset of the whole uint64[H][65536] array (512 MiB at H = 1024).
// Window cell i of 2*win-1: i < win -> key i; otherwise key -(i - win + 1), i.e. index 65536 - (i - win + 1).
__device__ __forceinline__ uint32_t window_cell(uint32_t i, uint32_t win) { return i < win ? i : 65536u - (i - win + 1u); }

__global__ void __launch_bounds__(256)
k_clear_touched(unsigned long long *__restrict__ buckets, uint32_t *__restrict__ flags, uint32_t win) {
    const uint32_t h = blockIdx.x;
    const uint32_t level = flags[h];
    if (level == 0) return;
    unsigned long long *hb = buckets + (size_t)h * 65536u;
    if (level & 2u) {
        for (uint32_t i = threadIdx.x; i < 65536u; i += 256) hb[i] = 0ull;
    } else {
        for (uint32_t i = threadIdx.x; i < 2u * win - 1u; i += 256) hb[window_cell(i, win)] = 0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) flags[h] = 0;
}

// ---------------------------------------------------------------------- K6
// processHistograms over caller-supplied sparse histograms (lh_reduce_sparse_host), in batches of at most
// K6_BATCH segments: k_scatter_segments adds a batch into scratch rows 0..nb-1 (flags raised as by every other
// writer), K3 reduces the rows unchanged, k_sparse_epilogue restores what the dense rows cannot tell (a key that
// is present with a merged count of 0), k_clear_touched zeroes the rows for the next batch.
constexpr int K6_BATCH = 256;            // scratch rows: 256 x 512 KiB = 128 MiB

// Entries [offsets[0], offsets[nb]) - base of the call's keys / counts; segment r of the batch goes to row r.
// One thread per entry (a segment can hold the concatenated exports of many hosts); each entry finds its segment by
// binary search over the batch's offsets in shared memory, then one 64-bit global RED per entry.
__global__ void __launch_bounds__(256)
k_scatter_segments(const uint32_t *__restrict__ offsets, uint32_t nb, uint32_t base, const short *__restrict__ keys,
                   const unsigned long long *__restrict__ counts, unsigned long long *__restrict__ rows,
                   uint32_t *__restrict__ flags, uint32_t win) {
    __shared__ uint32_t s_off[K6_BATCH + 1];
    for (uint32_t i = threadIdx.x; i <= nb; i += blockDim.x) s_off[i] = offsets[i] - base;
    __syncthreads();
    const size_t end = s_off[nb], stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = s_off[0] + (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < end; e += stride) {
        uint32_t lo = 0, hi = nb - 1;              // last segment starting at or before e (empty ones share its offset)
        while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (s_off[mid] <= e) lo = mid; else hi = mid - 1; }
        add_bucket_global(rows + (size_t)lo * 65536u, flags + lo, (uint32_t)(int)keys[e] & 0xFFFFu, counts[e], win);
    }
}

// One CTA per segment of the batch, after K3 and before the clear.  Go's map keeps a key whose counts summed to 0
// (metrics.go:342-347), the dense row does not, and two answers depend on it:
//   * p <= 0 with total > 0 (the uint64 total, which wraps at 2^64): percentile() returns the first entry in value
//     order whatever its count (float64(0)/float64(total) >= p), i.e. the smallest key present; K3 gives the smallest
//     non-empty one;
//   * decompress(key) = +-Inf with count 0 (precision <= 46, the ends of the key range): Inf * 0 makes the sum and
//     the average NaN; K3 skips empty cells.
// out_* point at the batch's first result.
__global__ void __launch_bounds__(256)
k_sparse_epilogue(const uint32_t *__restrict__ offsets, uint32_t base, const short *__restrict__ keys,
                  const unsigned long long *__restrict__ rows, const double *__restrict__ decomp,
                  const double *__restrict__ ps, int np, const unsigned long long *__restrict__ out_count,
                  double *__restrict__ out_sum, double *__restrict__ out_avg, int *__restrict__ out_pkeys,
                  double *__restrict__ out_pvals) {
    __shared__ int s_min[8];
    __shared__ int s_infzero[8];
    const uint32_t s = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const unsigned long long *row = rows + (size_t)s * 65536u;
    const uint32_t a = offsets[s] - base, b = offsets[s + 1] - base;
    int kmin = 0x7FFFFFFF, infzero = 0;
    for (uint32_t e = a + t; e < b; e += 256) {
        const int k = keys[e];
        const uint32_t slot = (uint32_t)k & 0xFFFFu;
        kmin = min(kmin, k);
        if (isinf(decomp[slot]) && row[slot] == 0ull) infzero = 1;
    }
    kmin = __reduce_min_sync(0xFFFFFFFFu, kmin);
    infzero = __reduce_or_sync(0xFFFFFFFFu, (unsigned)infzero);
    if (lane == 0) { s_min[warp] = kmin; s_infzero[warp] = infzero; }
    __syncthreads();
    if (t != 0) return;
    for (int w = 1; w < 8; w++) { kmin = min(kmin, s_min[w]); infzero |= s_infzero[w]; }
    if (infzero) {
        out_sum[s] = __longlong_as_double(0x7FF8000000000000ll);
        out_avg[s] = __longlong_as_double(0x7FF8000000000000ll);
    }
    // total 0: the segment is empty (every percentile an error) or its counts wrapped to 0 (sums of 2^64, 2^65 ...).
    // Then a key before the first non-empty one has running count 0 and ratio 0/0.0 = NaN, which fails every p, so
    // p <= 0 picks the first non-empty key (ratio x/0.0 = +Inf): K3's answer stands either way.
    if (out_count[s] == 0ull) return;
    for (int j = 0; j < np; j++)
        if (ps[j] <= 0.0) {                           // false for NaN
            out_pkeys[(size_t)s * np + j] = kmin;
            out_pvals[(size_t)s * np + j] = decomp[(uint32_t)kmin & 0xFFFFu];
        }
}

// ---------------------------------------------------------------------- K5
// Multi-GPU snapshot: one small kernel per rank sums, for every histogram some rank touched, the window cells of
// ALL ranks' frozen arrays (peer-mapped device memory: direct NVLink loads, no staging copy, no library
// collective) into this rank's `out` arrays, so every rank ends with the global histogram (the "tiny all-reduce of
// the ~4K-entry bucket arrays").  uint64 sums are associative: bit-identical to a single-GPU run.
// Protocol (comm block = uint64[32] per rank, slot r written only by rank r):
//   arrive[r]  rank r's frozen arrays for snapshot `seq` are complete      (pushed into every peer's block)
//   depart[r]  rank r has finished reading this rank's arrays for `seq`    (pushed when its last CTA is done)
// The kernel ends only after every peer departed, so the caller may clear its frozen arrays right after it.
// token = seq*2 + frozen buffer index: ranks must take their snapshots in lock-step (same count, same order).
static_assert(LH_MAX_RANKS == 16, "comm block layout assumes 16 ranks");
constexpr int K5_THREADS = 1024;
constexpr int K5_CHUNK = 2 * K5_THREADS;     // cells per work item (one-shot form)
constexpr int K5_DEEP = 9;                   // cells per thread and pass of the two-shot form: 9 x 1024 covers the 8 735-cell window of precision 100

struct PeerParams {
    uint32_t rank, world, H, C, win, do_counters, frozen, pad;
    unsigned long long seq;
    unsigned long long timeout_ns;
    const unsigned long long *buckets[LH_MAX_RANKS];     // every rank's FROZEN uint64[H][65536] (own rank: local pointer)
    const uint32_t *flags[LH_MAX_RANKS];
    const unsigned long long *counters[LH_MAX_RANKS];
    unsigned long long *comm[LH_MAX_RANKS];               // every rank's comm block
    unsigned long long *out_buckets;                      // this rank's reduced arrays (zero outside what is written)
    unsigned long long *out_peer[LH_MAX_RANKS];           // every rank's reduced bucket array (own rank: out_buckets)
    uint32_t two_shot;                                    // 1: each rank sums 1/world of the cells and pushes the sums to every rank
    uint32_t arrive_only;                                 // 1: announce + wait for every peer, nothing else (one small CTA ahead of a wide launch)
    uint32_t *out_flags;
    unsigned long long *out_counters;
    unsigned int *block_counter;                          // local, zero between launches
    unsigned int *status;                                 // local: 1 = a peer never arrived, 2 = buffer parity mismatch
    unsigned long long *cells;                            // local: cells summed by this launch (zeroed by the host)
};

__device__ __forceinline__ unsigned long long ld_sys_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// Bulk reads of a peer's frozen arrays: ordinary L2-only loads (ld.global.cg), which a warp coalesces into 128-byte
// requests - strong system-scope loads went out as one small NVLink request per lane (35 MB took 0.7 - 3 ms).  They are
// ordered after the acquire of the peer's arrival token, and L1 (which could hold the same addresses from two
// snapshots ago) is bypassed; peer memory is not cached in the local L2.
__device__ __forceinline__ unsigned long long ld_peer_u64(const unsigned long long *p) { return __ldcg(p); }
__device__ __forceinline__ uint32_t ld_sys_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// spin until slot >= token (tokens grow with the snapshot sequence); false on timeout
__device__ __forceinline__ bool wait_token(const unsigned long long *slot, unsigned long long token, unsigned long long timeout_ns,
                                           unsigned long long *seen) {
    const unsigned long long t0 = global_timer_ns();
    unsigned int spins = 0;
    for (;;) {
        const unsigned long long v = ld_acquire_sys_u64(slot);
        if ((v >> 1) >= (token >> 1)) { *seen = v; return true; }
        if ((++spins & 1023u) == 0 && global_timer_ns() - t0 > timeout_ns) return false;
    }
}

// Row policy of K5 (its last template parameter and argument).  RowIdentity: row h of every rank sums into row h
// (lh_snapshot_allreduce).  RowMap: job-wide rows g < n_rows (lh_snapshot_allreduce_rows): rank r contributes its
// frozen row hist[r * n_rows + g], or nothing for LH_ROW_ABSENT; counters alike over n_counter_rows.  Everything the
// kernel iterates (flag OR, sums, two-shot ownership, pushes) is over g, and the reduced arrays are indexed by g on
// every rank.  The maps live in device memory (up to 16 x 4 096 entries: too large for the parameter block).
struct RowIdentity {};
struct RowMap {
    const uint32_t *hist;          // [world][n_rows]
    const uint32_t *ctr;           // [world][n_counter_rows]
    uint32_t n_rows, n_counter_rows;
    uint32_t frozen_mask;          // bit r: the buffer rank r froze (announced in its token)
};
constexpr uint32_t K5_ROW_ABSENT = 0xFFFFFFFFu;

// Step 3 of K5 over job-wide rows: the identity form's sums with every row address taken through the maps.  ok false
// (a peer did not arrive, or froze another half than announced): this rank alone, through its own map.
__device__ __forceinline__ void k5_sum_mapped(const PeerParams &p, const RowMap &m, bool ok, unsigned char *s_level,
                                              unsigned long long *s_cells) {
    const uint32_t t = threadIdx.x;
    const uint32_t r0 = ok ? 0u : p.rank, r1 = ok ? p.world : p.rank + 1u;
    const bool push = ok && p.two_shot;
    const uint32_t wcells = 2u * p.win - 1u;
    const uint32_t n = m.n_rows;
    constexpr uint32_t PER_H = 65536u / K5_CHUNK;
    const uint32_t chunks_w = (wcells + K5_CHUNK - 1) / K5_CHUNK;
    unsigned long long cells = 0;
    for (uint32_t g = t; g < n; g += K5_THREADS) {
        uint32_t lv = 0;
        for (uint32_t r = r0; r < r1; r++) {
            const uint32_t h = __ldg(m.hist + (size_t)r * n + g);
            if (h != K5_ROW_ABSENT) lv |= ld_sys_u32(p.flags[r] + h);
        }
        s_level[g] = (unsigned char)lv;
        if (blockIdx.x == 0 && lv) { p.out_flags[g] = lv; cells += (lv & 2u) ? 65536u : wcells; }
    }
    if (blockIdx.x == 0 && cells) atomicAdd(s_cells, cells);
    __syncthreads();
    if (ok && blockIdx.x == 0 && t == 0) *p.cells = *s_cells;
    if (!push) {
        const size_t nitems = (size_t)n * PER_H;
        for (size_t item = blockIdx.x; item < nitems; item += gridDim.x) {
            const uint32_t g = (uint32_t)(item / PER_H), chunk = (uint32_t)(item % PER_H);
            const uint32_t level = s_level[g];
            if (level == 0) continue;
            const bool dense = (level & 2u) != 0;
            if (!dense && chunk >= chunks_w) continue;
            const uint32_t ncell = dense ? 65536u : wcells;
            constexpr int K = K5_CHUNK / K5_THREADS;
#pragma unroll
            for (int k = 0; k < K; k++) {
                const uint32_t i = chunk * K5_CHUNK + k * K5_THREADS + t;
                if (i >= ncell) continue;
                const uint32_t c = dense ? i : window_cell(i, p.win);
                unsigned long long sum = 0;
                for (uint32_t r = r0; r < r1; r++) {
                    const uint32_t h = __ldg(m.hist + (size_t)r * n + g);
                    if (h != K5_ROW_ABSENT) sum += ld_peer_u64(p.buckets[r] + (size_t)h * 65536u + c);
                }
                if (sum) p.out_buckets[(size_t)g * 65536u + c] = sum;
            }
        }
    } else {
        // two-shot: a rank owns the rows g = rank (mod world); as the identity form, K5_DEEP cells x world loads in
        // flight per thread
        for (uint32_t g = p.rank + blockIdx.x * p.world; g < n; g += gridDim.x * p.world) {
            const uint32_t level = s_level[g];
            if (level == 0) continue;
            const bool dense = (level & 2u) != 0;
            const uint32_t ncell = dense ? 65536u : wcells;
            for (uint32_t base = 0; base < ncell; base += K5_DEEP * K5_THREADS) {
                uint32_t cell[K5_DEEP];                  // cell index inside a row
                unsigned long long sum[K5_DEEP];
#pragma unroll
                for (int k = 0; k < K5_DEEP; k++) {
                    const uint32_t i = base + k * K5_THREADS + t;
                    cell[k] = i < ncell ? (dense ? i : window_cell(i, p.win)) : 0xFFFFFFFFu;
                    sum[k] = 0;
                }
#pragma unroll 4
                for (uint32_t r = 0; r < p.world; r++) {
                    const uint32_t h = __ldg(m.hist + (size_t)r * n + g);
                    if (h == K5_ROW_ABSENT) continue;
                    const unsigned long long *src = p.buckets[r] + (size_t)h * 65536u;
#pragma unroll
                    for (int k = 0; k < K5_DEEP; k++)
                        if (cell[k] != 0xFFFFFFFFu) sum[k] += ld_peer_u64(src + cell[k]);
                }
#pragma unroll
                for (int k = 0; k < K5_DEEP; k++) {
                    if (cell[k] == 0xFFFFFFFFu || sum[k] == 0) continue;
                    for (uint32_t r = 0; r < p.world; r++) p.out_peer[r][(size_t)g * 65536u + cell[k]] = sum[k];
                }
            }
        }
    }
    if (p.do_counters && blockIdx.x == 0) {
        const uint32_t nc = m.n_counter_rows;
        for (uint32_t i = t; i < p.C; i += K5_THREADS) {
            unsigned long long sum = 0;
            if (i < nc)
                for (uint32_t r = r0; r < r1; r++) {
                    const uint32_t c = __ldg(m.ctr + (size_t)r * nc + i);
                    if (c != K5_ROW_ABSENT) sum += ld_sys_u64(p.counters[r] + c);
                }
            p.out_counters[i] = sum;
        }
    }
    if (push) __threadfence_system();
}

// The body of both K5 kernels.  They are separate __global__ functions, not one template: a template kernel takes the
// module's largest dynamic shared-memory alignment, which moved the identity form's s_level.
template <typename Rows>
__device__ __forceinline__ void k5_body(PeerParams p, Rows rows, unsigned char *s_level) {
    __shared__ unsigned long long s_cells;
    const uint32_t t = threadIdx.x;
    const unsigned long long token = p.seq * 2ull + p.frozen;
    unsigned long long *mine = p.comm[p.rank];
    // 1. announce: my frozen arrays were completed by earlier kernels on this stream
    if (blockIdx.x == 0 && t < p.world && t != p.rank) {
        __threadfence_system();
        st_release_sys_u64(p.comm[t] + p.rank, token);
    }
    // 2. wait until every peer announced the same snapshot
    if (t < p.world && t != p.rank) {
        unsigned long long seen = 0;
        if (!wait_token(mine + t, token, p.timeout_ns, &seen)) atomicMax(p.status, 1u);
        else if constexpr (std::is_same<Rows, RowMap>::value) {
            if ((seen >> 1) == p.seq && (seen & 1ull) != ((rows.frozen_mask >> t) & 1u)) atomicMax(p.status, 2u);
        } else if ((seen >> 1) == p.seq && (seen & 1ull) != p.frozen) atomicMax(p.status, 2u);
    }
    if (p.arrive_only) return;
    if (t == 0) s_cells = 0;
    __syncthreads();
    const bool ok = ld_sys_u32(p.status) == 0;
    if constexpr (std::is_same<Rows, RowMap>::value) {
        k5_sum_mapped(p, rows, ok, s_level, &s_cells);
    } else
    // 3. sum.  Work item = (histogram, chunk of K5_CHUNK cells); the set of cells follows the OR of all ranks' flags.
    //    one-shot (small payload): every rank sums every item into its own array - one NVLink round trip.
    //    two-shot (large payload): the rank that owns an item sums it and pushes the sum into every rank's array, so a
    //    rank moves 2 * (world - 1) / world of the payload over NVLink instead of (world - 1) times the payload.
    //    When a peer did not arrive or froze the other buffer (status != 0), the one-shot form runs over this rank
    //    alone: its reduced arrays get its own frozen cells, flags and counters, and nothing goes to a peer's arrays.
    {
        const uint32_t r0 = ok ? 0u : p.rank, r1 = ok ? p.world : p.rank + 1u;
        const bool push = ok && p.two_shot;
        const uint32_t wcells = 2u * p.win - 1u;
        constexpr uint32_t PER_H = 65536u / K5_CHUNK;         // items are indexed as if every histogram were dense
        const uint32_t chunks_w = (wcells + K5_CHUNK - 1) / K5_CHUNK;
        unsigned long long cells = 0;
        for (uint32_t h = t; h < p.H; h += K5_THREADS) {
            uint32_t lv = 0;
            for (uint32_t r = r0; r < r1; r++) lv |= ld_sys_u32(p.flags[r] + h);
            s_level[h] = (unsigned char)lv;
            if (blockIdx.x == 0 && lv) { p.out_flags[h] = lv; cells += (lv & 2u) ? 65536u : wcells; }
        }
        if (blockIdx.x == 0 && cells) atomicAdd(&s_cells, cells);
        __syncthreads();
        if (ok && blockIdx.x == 0 && t == 0) *p.cells = s_cells;      // nothing was read from a peer otherwise
        if (!push) {
            const size_t nitems = (size_t)p.H * PER_H;
            for (size_t item = blockIdx.x; item < nitems; item += gridDim.x) {
                const uint32_t h = (uint32_t)(item / PER_H), chunk = (uint32_t)(item % PER_H);
                const uint32_t level = s_level[h];
                if (level == 0) continue;
                const bool dense = (level & 2u) != 0;
                if (!dense && chunk >= chunks_w) continue;
                const uint32_t ncell = dense ? 65536u : wcells;
                constexpr int K = K5_CHUNK / K5_THREADS;
#pragma unroll
                for (int k = 0; k < K; k++) {
                    const uint32_t i = chunk * K5_CHUNK + k * K5_THREADS + t;
                    if (i >= ncell) continue;
                    const size_t cell = (size_t)h * 65536u + (dense ? i : window_cell(i, p.win));
                    unsigned long long sum = 0;
                    for (uint32_t r = r0; r < r1; r++) sum += ld_peer_u64(p.buckets[r] + cell);
                    if (sum) p.out_buckets[cell] = sum;
                }
            }
        } else {
            // two-shot: a rank owns the histograms h = rank (mod world); a CTA takes one owned histogram at a time and every
            // thread keeps K5_DEEP cells x world loads in flight (a few CTAs on the SMs the ingest kernel leaves free must
            // cover the NVLink latency-bandwidth product on their own)
            for (uint32_t h = p.rank + blockIdx.x * p.world; h < p.H; h += gridDim.x * p.world) {
                const uint32_t level = s_level[h];
                if (level == 0) continue;
                const bool dense = (level & 2u) != 0;
                const uint32_t ncell = dense ? 65536u : wcells;
                for (uint32_t base = 0; base < ncell; base += K5_DEEP * K5_THREADS) {
                    // all loads of a pass before its first store: K5_DEEP cells x world ranks, independent, as many in flight
                    // per thread as the 64 registers allow (one CTA per SM)
                    uint32_t cell[K5_DEEP];                  // cell index inside the [H][65536] array (H <= 65535: fits 32 bits)
                    unsigned long long sum[K5_DEEP];
#pragma unroll
                    for (int k = 0; k < K5_DEEP; k++) {
                        const uint32_t i = base + k * K5_THREADS + t;
                        cell[k] = i < ncell ? h * 65536u + (dense ? i : window_cell(i, p.win)) : 0xFFFFFFFFu;
                        sum[k] = 0;
                    }
#pragma unroll 4
                    for (uint32_t r = 0; r < p.world; r++) {
                        const unsigned long long *src = p.buckets[r];
#pragma unroll
                        for (int k = 0; k < K5_DEEP; k++)
                            if (cell[k] != 0xFFFFFFFFu) sum[k] += ld_peer_u64(src + cell[k]);
                    }
#pragma unroll
                    for (int k = 0; k < K5_DEEP; k++) {
                        if (cell[k] == 0xFFFFFFFFu || sum[k] == 0) continue;
                        for (uint32_t r = 0; r < p.world; r++) p.out_peer[r][cell[k]] = sum[k];
                    }
                }
            }
        }
        if (p.do_counters && blockIdx.x == 0) {
            for (uint32_t i = t; i < p.C; i += K5_THREADS) {
                unsigned long long sum = 0;
                for (uint32_t r = r0; r < r1; r++) sum += ld_sys_u64(p.counters[r] + i);
                p.out_counters[i] = sum;
            }
        }
        if (push) __threadfence_system();                    // my pushes are performed before this CTA checks out
    }
    // 4. depart: the last CTA of this rank tells every peer it has finished reading them and that the sums it pushed
    //    are visible (every CTA fences at system scope before it checks out), then waits for the same from every peer
    __syncthreads();
    __shared__ bool s_last;
    if (t == 0) {
        __threadfence_system();
        s_last = atomicAdd(p.block_counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    if (t == 0) *p.block_counter = 0;
    if (t < p.world && t != p.rank) {
        __threadfence_system();
        st_release_sys_u64(p.comm[t] + LH_MAX_RANKS + p.rank, token);
        unsigned long long seen = 0;
        if (!wait_token(mine + LH_MAX_RANKS + t, token, p.timeout_ns, &seen)) atomicMax(p.status, 1u);
    }
}

__global__ void __launch_bounds__(K5_THREADS, 1)
k_peer_allreduce(PeerParams p) {
    extern __shared__ unsigned char s_level[];               // [H]: OR over ranks of the histogram's flag
    k5_body(p, RowIdentity{}, s_level);
}

__global__ void __launch_bounds__(K5_THREADS, 1)
k_peer_allreduce_rows(PeerParams p, RowMap rows) {
    extern __shared__ unsigned char s_level[];               // [n_rows]: OR over ranks of the row's flag
    k5_body(p, rows, s_level);
}

// ------------------------------------------------ job-wide rows through the caller's all-reduce (lh_snapshot_*_rows)
// A payload every rank lays out alike, so that an element-wise uint64 sum over ranks (any transport: gloo, NCCL, MPI)
// is the job-wide interval.  Row g of level 1 (every rank's counts inside the fast window) is its 2*win-1 window cells,
// indices [0, win) then [65536-(win-1), 65536); level 3 is all 65536 cells in index order; level 0 is nothing.  The
// counter rows follow.  k_rows_pack gathers this rank's frozen rows into it, k_rows_unpack writes a payload into the
// reduced arrays at row g.  Work item = (row, chunk of ROWS_CHUNK payload words); every access is 16 bytes wide except
// a segment's first and last word when they are unpaired.
constexpr int ROWS_THREADS = 256;
constexpr uint32_t ROWS_CHUNK = 8u * ROWS_THREADS;               // payload words per work item: 4 pairs per thread
constexpr uint32_t ROWS_PER_ROW = 65536u / ROWS_CHUNK;          // work items per row (a window row uses the first few)

struct RowsEntry {                  // 16 bytes per job-wide row, in the device table
    uint32_t row;                   // this rank's frozen row (pack), or K5_ROW_ABSENT
    uint32_t level;                 // 0, 1 or 3: the agreed level
    unsigned long long off;         // payload word of the row's first cell
};

// dst[0, n) = src[0, n) (src NULL: zeros), one CTA.  Stores are 16-byte aligned pairs after at most one scalar head;
// a source of the other parity is read as the aligned pairs around it (the pair before its first word and after its
// last lie in the same 16-byte granule as a word of the segment, so they are inside the allocation).
__device__ __forceinline__ void rows_copy(unsigned long long *dst, const unsigned long long *src, uint32_t n) {
    const uint32_t t = threadIdx.x;
    const uint32_t head = min(n, (uint32_t)(((uintptr_t)dst >> 3) & 1u));
    if (t == 0 && head) dst[0] = src ? __ldg(src) : 0ull;
    dst += head; n -= head;
    if (src) src += head;
    const uint32_t np = n >> 1;
    ulonglong2 *d2 = reinterpret_cast<ulonglong2 *>(dst);
    if (!src) {
        for (uint32_t k = t; k < np; k += ROWS_THREADS) d2[k] = make_ulonglong2(0ull, 0ull);
    } else if ((((uintptr_t)src >> 3) & 1u) == 0) {
        const ulonglong2 *s2 = reinterpret_cast<const ulonglong2 *>(src);
        for (uint32_t k = t; k < np; k += ROWS_THREADS) d2[k] = __ldg(s2 + k);
    } else {
        const ulonglong2 *s2 = reinterpret_cast<const ulonglong2 *>(src - 1);
        for (uint32_t k = t; k < np; k += ROWS_THREADS) {
            const ulonglong2 a = __ldg(s2 + k), b = __ldg(s2 + k + 1);
            d2[k] = make_ulonglong2(a.y, b.x);
        }
    }
    if (t == 0 && (n & 1u)) dst[n - 1] = src ? __ldg(src + n - 1) : 0ull;
}

// The payload words [j0, j1) of a row at level `level` and where they sit in its 65536 cells: calls
// f(first payload word, first cell, words) for each run of consecutive cells (one or two per work item).
template <typename F>
__device__ __forceinline__ void rows_runs(uint32_t level, uint32_t chunk, uint32_t win, F f) {
    const uint32_t len = (level & 2u) ? 65536u : 2u * win - 1u;
    const uint32_t j0 = chunk * ROWS_CHUNK, j1 = min(len, j0 + ROWS_CHUNK);
    if (j0 >= j1) return;
    if (level & 2u) { f(j0, j0, j1 - j0); return; }
    if (j0 < win) f(j0, j0, min(j1, win) - j0);
    if (j1 > win) {
        const uint32_t a = max(j0, win);
        f(a, a + 65537u - 2u * win, j1 - a);        // payload word win is cell 65536 - (win - 1)
    }
}

__global__ void __launch_bounds__(ROWS_THREADS)
k_rows_pack(const RowsEntry *__restrict__ table, uint32_t n_rows, uint32_t win,
            const unsigned long long *__restrict__ buckets, const uint32_t *__restrict__ ctr_rows, uint32_t n_counter_rows,
            const unsigned long long *__restrict__ counters, unsigned long long ctr_off,
            unsigned long long *__restrict__ payload) {
    for (uint32_t i = blockIdx.x * ROWS_THREADS + threadIdx.x; i < n_counter_rows; i += gridDim.x * ROWS_THREADS) {
        const uint32_t c = __ldg(ctr_rows + i);
        payload[ctr_off + i] = c == K5_ROW_ABSENT ? 0ull : __ldg(counters + c);
    }
    const size_t items = (size_t)n_rows * ROWS_PER_ROW;
    for (size_t item = blockIdx.x; item < items; item += gridDim.x) {
        const RowsEntry e = table[item / ROWS_PER_ROW];
        if (e.level == 0) continue;
        const unsigned long long *src = e.row == K5_ROW_ABSENT ? nullptr : buckets + (size_t)e.row * 65536u;
        rows_runs(e.level, (uint32_t)(item % ROWS_PER_ROW), win, [&](uint32_t j, uint32_t cell, uint32_t n) {
            rows_copy(payload + e.off + j, src ? src + cell : nullptr, n);
        });
    }
}

// Row g < n_rows: cells from the payload, flag = level; counters below n_counter_rows from the payload, the rest 0.
// The reduced arrays are zero outside flagged rows (lh_snapshot_end clears them by their flags), so nothing else moves.
__global__ void __launch_bounds__(ROWS_THREADS)
k_rows_unpack(const RowsEntry *__restrict__ table, uint32_t n_rows, uint32_t win,
              const unsigned long long *__restrict__ payload, uint32_t n_counter_rows, uint32_t C,
              unsigned long long ctr_off, unsigned long long *__restrict__ out_buckets, uint32_t *__restrict__ out_flags,
              unsigned long long *__restrict__ out_counters) {
    const uint32_t tid = blockIdx.x * ROWS_THREADS + threadIdx.x, nthreads = gridDim.x * ROWS_THREADS;
    for (uint32_t g = tid; g < n_rows; g += nthreads) out_flags[g] = table[g].level;
    for (uint32_t i = tid; i < C; i += nthreads) out_counters[i] = i < n_counter_rows ? __ldg(payload + ctr_off + i) : 0ull;
    const size_t items = (size_t)n_rows * ROWS_PER_ROW;
    for (size_t item = blockIdx.x; item < items; item += gridDim.x) {
        const uint32_t g = (uint32_t)(item / ROWS_PER_ROW);
        const RowsEntry e = table[g];
        if (e.level == 0) continue;
        unsigned long long *dst = out_buckets + (size_t)g * 65536u;
        rows_runs(e.level, (uint32_t)(item % ROWS_PER_ROW), win, [&](uint32_t j, uint32_t cell, uint32_t n) {
            rows_copy(dst + cell, payload + e.off + j, n);
        });
    }
}

// ----------------------------------------------------------- batch ingest (lh_ingest_batch)
// Many short device arrays, each under its own histogram id, in one launch.  The item table travels in the parameter
// block (no copy, no allocation): descriptors plus prefix offsets of their lengths.  The concatenation of the items is
// cut into pieces of BI_PIECE samples, dealt round-robin to the CTAs; a piece may span several items.  Every CTA counts
// into one lh::BlockRecorder combining table over the interval's rows and flushes it once, so a sample costs shared
// atomics wherever the CTA's distinct (id, bucket) pairs fit the table, and the table's direct path otherwise: the
// count is exact whatever the fill.  The host bounds the samples of a launch so that no CTA counts more than 2^31 of
// them (the table's counts are uint32).
constexpr int BI_THREADS = 512;
constexpr uint32_t BI_TABLE_ENTRIES = 8192;  // 96 KB of combining table: two CTAs per SM
constexpr uint32_t BI_PIECE = 2048;          // samples per piece: 4 per thread
constexpr int BI_MAX_ITEMS = 1024;           // items per launch: 24 B each in the parameter block

struct BatchSeg {
    const unsigned long long *vals;          // 8-byte samples (float64 or int64 ns)
    uint32_t id;
    uint32_t kind;                           // LH_VALUES_*
};
struct BatchParams {
    lh_recorder rec;                         // the interval's rows, built by the library (no scope)
    uint32_t n_items;
    uint32_t pad;
    unsigned long long start[BI_MAX_ITEMS + 1];   // prefix offsets of the items' lengths
    BatchSeg seg[BI_MAX_ITEMS];
};

__global__ void __launch_bounds__(BI_THREADS, 2)
k_ingest_batch(const __grid_constant__ BatchParams p) {
    extern __shared__ __align__(16) unsigned char bi_smem[];
    BlockRecorder br(p.rec, bi_smem, BI_TABLE_ENTRIES);
    br.init();
    const unsigned long long total = p.start[p.n_items];
    const unsigned long long pieces = (total + BI_PIECE - 1) / BI_PIECE;
    for (unsigned long long pc = blockIdx.x; pc < pieces; pc += gridDim.x) {
        unsigned long long lo = pc * BI_PIECE;
        const unsigned long long hi = min(lo + BI_PIECE, total);
        // the item holding sample lo: the last one whose start is <= lo (uniform over the CTA)
        uint32_t a = 0, b = p.n_items - 1;
        while (a < b) {
            const uint32_t m = (a + b + 1) / 2;
            if (p.start[m] <= lo) a = m; else b = m - 1;
        }
        // every thread walks the piece's samples across item boundaries (its item index only grows), so the loads of a
        // piece are in flight together however short the items are
        uint32_t it = a;
        for (unsigned long long g0 = lo + threadIdx.x; g0 < hi; g0 += 2 * BI_THREADS) {
            unsigned long long raw[2];
            uint32_t id[2];
            bool ns[2];
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const unsigned long long g = g0 + k * BI_THREADS;
                raw[k] = 0ull; id[k] = 0u; ns[k] = false;
                if (g < hi) {
                    while (p.start[it + 1] <= g) ++it;
                    id[k] = p.seg[it].id;
                    ns[k] = p.seg[it].kind == LH_VALUES_I64NS;
                    raw[k] = __ldcs(p.seg[it].vals + (g - p.start[it]));
                }
            }
#pragma unroll
            for (int k = 0; k < 2; k++)
                if (g0 + k * BI_THREADS < hi)
                    br.record(id[k], ns[k] ? __ll2double_rn((long long)raw[k]) : __longlong_as_double((long long)raw[k]));
        }
    }
    br.flush();
}

// ----------------------------------------------------------- captured keyed ingest (lh_graph_recorder_ingest_keyed_*)
// (id, value) pairs into a graph recorder's rows, ids local.  The keyed kernels above cannot be captured (the hot window
// needs a host-tallied fold, the write-combining kernel cross-launch scratch and events), so this one counts like
// k_ingest_batch instead: every CTA through one lh::BlockRecorder over the recorder, flushed once, with the id taken per
// sample; an id >= max_histograms is dropped and counted by the recorder.  Samples [0, nhead) and [nhead + 4 n4, n) go
// one per thread (all of them when the id and value alignments do not line up); the vector body in between takes
// 4 samples per thread and iteration (two 16-byte value loads, one IdPack id load), the next group loaded while the
// current one is counted.  vals + nhead is 32-byte aligned and ids + nhead 4*sizeof(IdT)-aligned.  The host bounds a
// launch as it bounds k_ingest_batch's, so no CTA counts more than 2^31 samples.
template <typename IdT>
__global__ void __launch_bounds__(BI_THREADS, 2)
k_ingest_keyed_graph(const __grid_constant__ lh_recorder rec, const IdT *__restrict__ ids,
                     const unsigned long long *__restrict__ vals, size_t nhead, size_t n4, size_t n, bool ns) {
    extern __shared__ __align__(16) unsigned char kg_smem[];
    BlockRecorder br(rec, kg_smem, BI_TABLE_ENTRIES);
    br.init();
    auto value = [ns](unsigned long long raw) { return ns ? __ll2double_rn((long long)raw) : __longlong_as_double((long long)raw); };
    const size_t stride = (size_t)gridDim.x * BI_THREADS;
    const size_t t0 = (size_t)blockIdx.x * BI_THREADS + threadIdx.x;
    for (size_t i = t0; i < nhead; i += stride) br.record((uint32_t)ids[i], value(__ldcs(vals + i)));
    const IdT *bid = ids + nhead;
    const unsigned long long *bv = vals + nhead;
    size_t g = t0;
    unsigned long long cur[4], nxt[4];
    IdPack<IdT> cid, nid;
    if (g < n4) { load_vals4(bv, g, cur); cid.load(bid, g); }
    for (; g < n4; g += stride) {
        const size_t gn = g + stride;
        if (gn < n4) { load_vals4(bv, gn, nxt); nid.load(bid, gn); }
#pragma unroll
        for (int j = 0; j < 4; j++) br.record(cid.get(j), value(cur[j]));
#pragma unroll
        for (int j = 0; j < 4; j++) cur[j] = nxt[j];
        cid = nid;
    }
    for (size_t i = nhead + 4 * n4 + t0; i < n; i += stride) br.record((uint32_t)ids[i], value(__ldcs(vals + i)));
    br.flush();
}

// ----------------------------------------------------------- graph recorder drain (lh_graph_recorder_*)
// Moves the counts of graph-owned rows into an interval's rows.  One CTA per entry of the table, which travels in the
// parameter block: a histogram row (src, src_flag, target id) or a counter (src, no flag, target id).  A row whose flag
// is 0 is skipped; otherwise its window (every cell when flag & 2) is read with 16-byte loads through L2, and every
// non-zero cell is taken with an atomic exchange to 0 and added to the target row with add_bucket_global, which raises
// the target flag for the key as every writer does.  Unbound targets (LH_GRAPH_UNBOUND) add the total to `dropped`.
//
// Exactness while replays keep recording into the source rows: a replay's add and the drain's exchange are atomics on
// the same cell, so every add is taken by exactly one exchange, this one or a later drain's; nothing is lost or counted
// twice.  Source flags are never cleared: a writer adds to the cell before it raises the flag, but another SM may see
// the flag first or the cell first.  A drain that reads a stale flag (0, or 1 where an out-of-window cell was just
// written) or a stale zero cell skips counts that a later drain will find, since the flag stays raised; it never takes
// a count twice.  The cost is one scan per touched row per drain, bounded by the rows the recorders declare.
constexpr int DR_THREADS = 256;
constexpr int DR_MAX_ENTRIES = 1024;         // entries per launch: 24 B each in the parameter block

struct DrainEntry {
    unsigned long long *src;                 // row [65536], or one counter
    uint32_t *src_flag;                      // nullptr for a counter
    uint32_t target;                         // histogram / counter id of the interval, or LH_GRAPH_UNBOUND
    uint32_t pad;
};
struct DrainParams {
    unsigned long long *buckets;             // the interval's rows [H][65536]
    uint32_t *flags;                         // [H]
    unsigned long long *counters;            // [C]
    unsigned long long *dropped;
    uint32_t win;
    uint32_t n;
    DrainEntry e[DR_MAX_ENTRIES];
};

__device__ __forceinline__ ulonglong2 ld_cg_u64x2(const unsigned long long *p) {
    ulonglong2 r;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(r.x), "=l"(r.y) : "l"(p) : "memory");
    return r;
}

__global__ void __launch_bounds__(DR_THREADS)
k_graph_drain(const __grid_constant__ DrainParams p) {
    const DrainEntry &e = p.e[blockIdx.x];
    const bool unbound = e.target == LH_GRAPH_UNBOUND;
    unsigned long long lost = 0;
    if (!e.src_flag) {
        if (threadIdx.x == 0 && *reinterpret_cast<volatile unsigned long long *>(e.src)) {
            const unsigned long long c = atomicExch(e.src, 0ull);
            if (unbound) lost = c;
            else if (c) atomicAdd(p.counters + e.target, c);
        }
    } else {
        const uint32_t level = *reinterpret_cast<volatile uint32_t *>(e.src_flag);
        if (level == 0) return;
        unsigned long long *row = unbound ? nullptr : p.buckets + (size_t)e.target * 65536u;
        uint32_t *flag = unbound ? nullptr : p.flags + e.target;
        auto take = [&](uint32_t key) {
            const unsigned long long c = atomicExch(e.src + key, 0ull);
            if (!c) return;
            if (unbound) lost += c;
            else add_bucket_global(row, flag, key, c, p.win);
        };
        // cell pairs to scan: all 32768, or the pairs holding keys [0, win) and [65536 - win + 1, 65536)
        const uint32_t lo_pairs = (level & 2u) ? 32768u : (p.win + 1u) / 2u;
        const uint32_t hi_first = (level & 2u) ? 32768u : (65536u - p.win + 1u) / 2u;
        const uint32_t n_pairs = lo_pairs + (32768u - hi_first);
        for (uint32_t j = threadIdx.x; j < n_pairs; j += DR_THREADS) {
            const uint32_t pair = j < lo_pairs ? j : hi_first + (j - lo_pairs);
            const ulonglong2 v = ld_cg_u64x2(e.src + 2u * pair);
            if (v.x) take(2u * pair);
            if (v.y) take(2u * pair + 1u);
        }
    }
    if (lost) atomicAdd(p.dropped, lost);
}

// ----------------------------------------------------------- device subscriptions (lh_board_*, lh_snapshot_publish)
// k_board_publish writes one collection's rows into a board (layout and row semantics: include/loghisto_b200.h), one
// CTA, under a seqlock whose word is the board's first uint64:
//   1. thread 0 makes the word odd, fence.acq_rel.gpu, __syncthreads;
//   2. every thread gathers rows from the result slot of the reduction (count / sum / avg / pvals / pkeys at the
//      res_layout offsets for that reduction's np; the percentiles from its d_ps) and the counter deltas of the
//      snapshot view, and writes them with strong relaxed stores;
//   3. __threadfence, __syncthreads;
//   4. thread 0 writes the publish count and makes the word even with st.release.gpu.
// A reader (k_board_read, lh::read_histogram / read_counter) loads the word with ld.acquire.gpu and retries while it
// is odd, loads the rows with strong relaxed loads, then fence.acq_rel.gpu and the word again, and retries if it
// changed.  A reader that saw a row store of this publish synchronises with step 1's fence, so its second load of the
// word sees the odd value or a later one and the read is retried; a reader that saw the even word of step 4 sees every
// row store before it.
//
// Termination: the writer waits on nothing -- no lock, no flag, no other kernel -- so once its CTA is resident it
// finishes in a bounded number of steps, and the word is odd only while it is resident.  A reader therefore spins only
// while a resident writer runs, whatever else occupies the GPU.  That is why the whole odd window lies inside one
// kernel: an id table too large for one parameter block is first copied into the board's table area by k_board_stage
// launches, which do not touch the word.
constexpr int BP_THREADS = 512;
constexpr int BP_MAX_ENTRIES = 1536;         // entries per launch: 16 B each in the parameter block

struct BoardEntry {
    uint32_t row;                            // < k: histogram row; else counter row (row - k)
    uint32_t id;                             // histogram / counter id of the snapshot, or LH_GRAPH_UNBOUND
    unsigned long long total;                // counter rows: the caller's total
};
struct BoardParams {
    char *board;                             // header, k histogram rows, kc counter rows
    BoardEntry *table;                       // entries staged by k_board_stage, [n_staged]
    const unsigned long long *count;         // the reduction's result slot
    const double *sum, *avg, *pvals;
    const int *pkeys;
    const double *ps;                        // its percentiles [np]
    const unsigned long long *counters;      // counter deltas of the snapshot view
    uint32_t np, k;
    uint32_t n_staged, n;                    // entries in `table`, then in e[]
    BoardEntry e[BP_MAX_ENTRIES];
    const uint32_t *nnz;                     // the reduction's non-empty bucket counts: presence (a count can wrap to 0)
};

__global__ void __launch_bounds__(BP_THREADS)
k_board_stage(const __grid_constant__ BoardParams p) {
    for (uint32_t i = threadIdx.x; i < p.n; i += BP_THREADS) p.table[p.n_staged + i] = p.e[i];
}

__global__ void __launch_bounds__(BP_THREADS)
k_board_publish(const __grid_constant__ BoardParams p) {
    unsigned long long *seq = reinterpret_cast<unsigned long long *>(p.board);
    const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
    if (t == 0) {
        board::st_relaxed(seq, board::ld_relaxed(seq) + 1ull);   // odd: the previous publish ended (stream order)
        board::fence_acq_rel();
    }
    __syncthreads();
    const double qnan = __longlong_as_double(0x7FF8000000000000ll);
    char *hdr = p.board;
    if (t < LH_MAX_PERCENTILES)
        board::st_relaxed(hdr + offsetof(lh_board_header, percentiles) + 8 * t,
                          (unsigned long long)__double_as_longlong(t < p.np ? p.ps[t] : qnan));
    if (t == 0) board::st_relaxed_u32(hdr + offsetof(lh_board_header, np), p.np);
    const uint32_t total = p.n_staged + p.n;
    auto entry = [&](uint32_t i) { return i < p.n_staged ? p.table[i] : p.e[i - p.n_staged]; };
    // histogram rows: one warp each, lane j writes percentile slot j
    for (uint32_t i = warp; i < total; i += BP_THREADS / 32) {
        const BoardEntry e = entry(i);
        if (e.row >= p.k) continue;
        char *r = p.board + sizeof(lh_board_header) + (size_t)e.row * sizeof(lh_board_hist_row);
        const bool bound = e.id != LH_GRAPH_UNBOUND;
        int key = (int)0x80000000;
        double val = qnan;
        if (bound && lane < p.np) {
            key = p.pkeys[(size_t)e.id * p.np + lane];
            val = p.pvals[(size_t)e.id * p.np + lane];
        }
        board::st_relaxed(r + offsetof(lh_board_hist_row, pvals) + 8 * lane, (unsigned long long)__double_as_longlong(val));
        board::st_relaxed_u32(r + offsetof(lh_board_hist_row, pkeys) + 4 * lane, (uint32_t)key);
        if (lane == 0) {
            const unsigned long long c = bound ? p.count[e.id] : 0ull;
            board::st_relaxed(r + offsetof(lh_board_hist_row, count), c);
            board::st_relaxed(r + offsetof(lh_board_hist_row, sum), (unsigned long long)__double_as_longlong(bound ? p.sum[e.id] : 0.0));
            board::st_relaxed(r + offsetof(lh_board_hist_row, avg), (unsigned long long)__double_as_longlong(bound ? p.avg[e.id] : qnan));
            board::st_relaxed_u32(r + offsetof(lh_board_hist_row, present), bound && p.nnz[e.id] != 0u);
        }
    }
    // counter rows: one thread each
    char *crows = p.board + sizeof(lh_board_header) + (size_t)p.k * sizeof(lh_board_hist_row);
    for (uint32_t i = t; i < total; i += BP_THREADS) {
        const BoardEntry e = entry(i);
        if (e.row < p.k) continue;
        char *r = crows + (size_t)(e.row - p.k) * sizeof(lh_board_counter_row);
        const bool bound = e.id != LH_GRAPH_UNBOUND;
        board::st_relaxed(r + offsetof(lh_board_counter_row, rate), bound ? p.counters[e.id] : 0ull);
        board::st_relaxed(r + offsetof(lh_board_counter_row, total), e.total);
        board::st_relaxed_u32(r + offsetof(lh_board_counter_row, present), bound ? 1u : 0u);
    }
    __threadfence();
    __syncthreads();
    if (t == 0) {
        const unsigned long long s = board::ld_relaxed(seq) + 1ull;   // even
        board::st_relaxed(hdr + offsetof(lh_board_header, publishes), s >> 1);
        board::st_release(seq, s);
    }
}

// Copies a consistent image of a board (`words` uint64) to `out`, one CTA: the seqlock read of k_board_publish's
// comment over the whole board, each thread fencing its own loads before thread 0 re-reads the word.  A torn copy is
// overwritten by the retry; the image's word is the even value it was read under.
constexpr int BR_THREADS = 512;

__global__ void __launch_bounds__(BR_THREADS)
k_board_read(const unsigned long long *__restrict__ board, unsigned long long *__restrict__ out, uint32_t words) {
    __shared__ unsigned long long s_seq;
    __shared__ int s_ok;
    const uint32_t t = threadIdx.x;
    for (;;) {
        if (t == 0) {
            unsigned long long s;
            while ((s = board::ld_acquire(board)) & 1ull) __nanosleep(64);
            s_seq = s;
        }
        __syncthreads();
        const unsigned long long s = s_seq;
        for (uint32_t i = t + 1; i < words; i += BR_THREADS) out[i] = board::ld_relaxed(board + i);
        board::fence_acq_rel();
        __syncthreads();
        if (t == 0) s_ok = board::ld_relaxed(board) == s;
        __syncthreads();
        if (s_ok) {
            if (t == 0) out[0] = s;
            return;
        }
    }
}

// ----------------------------------------------------------- device gauges (lh_gauges_read)
// One thread per gauge.  Each value is read with one naturally aligned ld.relaxed.gpu (a strong load: never torn
// against a strong store of the same size, and served from L2, never from a stale L1 line), then converted to float64
// as Go's float64(x) does: exact widening for f32 (and f16 / bf16 through f32) and s32, cvt.rn for s64 / u64.  The
// table comes by value in the parameter block; the values go to host-mapped pinned memory.
constexpr int GR_THREADS = 128;
constexpr int GR_MAX_ENTRIES = 1024;         // entries per launch: 16 B each in the parameter block

struct GaugeEntry {
    const void *p;
    uint32_t dtype;                          // LH_GAUGE_*, checked on the host
    uint32_t reserved;
};
struct GaugeParams {
    double *out;                             // [n], device view of mapped pinned memory
    uint32_t n, reserved;
    GaugeEntry e[GR_MAX_ENTRIES];
};

namespace gauge {
__device__ __forceinline__ unsigned long long ld64(const void *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.b64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld32(const void *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned short ld16(const void *p) {
    unsigned short v;
    asm volatile("ld.relaxed.gpu.b16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double f32(float x) {   // exact, subnormals kept (no .ftz)
    double d;
    asm("cvt.f64.f32 %0, %1;" : "=d"(d) : "f"(x));
    return d;
}
// Go's float64(x) of the raw bits of one element: exact widening for f32 (and f16 / bf16 through f32) and s32, cvt.rn
// (round to nearest even) for s64 / u64.  The one definition of the conversion: every kernel that takes LH_GAUGE_*
// elements (k_gauge_read, k_ingest_arrays, the narrow forms of K1 and the key table of k_fill_key16) converts here.
__device__ __forceinline__ double from_f32(uint32_t b) { return f32(__uint_as_float(b)); }
__device__ __forceinline__ double from_f16(unsigned short b) {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(b));
    return f32(f);
}
__device__ __forceinline__ double from_bf16(unsigned short b) { return f32(__uint_as_float((uint32_t)b << 16)); }
__device__ __forceinline__ double from_i64(unsigned long long b) {
    double v;
    asm("cvt.rn.f64.s64 %0, %1;" : "=d"(v) : "l"(b));
    return v;
}
__device__ __forceinline__ double from_i32(uint32_t b) {
    double v;
    asm("cvt.rn.f64.s32 %0, %1;" : "=d"(v) : "r"(b));
    return v;
}
__device__ __forceinline__ double from_u64(unsigned long long b) {
    double v;
    asm("cvt.rn.f64.u64 %0, %1;" : "=d"(v) : "l"(b));
    return v;
}
// Load policies of load(): Relaxed, one strong load (a device gauge or a distribution read outside stream order, never
// torn against an aligned store); Streaming, read-once stream-ordered data (lh_ingest_arrays), ld.global.cs as
// k_ingest_batch loads its samples.
struct Relaxed {
    static __device__ __forceinline__ unsigned long long ld64(const void *p) { return gauge::ld64(p); }
    static __device__ __forceinline__ uint32_t ld32(const void *p) { return gauge::ld32(p); }
    static __device__ __forceinline__ unsigned short ld16(const void *p) { return gauge::ld16(p); }
};
struct Streaming {
    static __device__ __forceinline__ unsigned long long ld64(const void *p) { return __ldcs((const unsigned long long *)p); }
    static __device__ __forceinline__ uint32_t ld32(const void *p) { return __ldcs((const unsigned int *)p); }
    static __device__ __forceinline__ unsigned short ld16(const void *p) { return __ldcs((const unsigned short *)p); }
};
// The value at p of dtype LH_GAUGE_* (checked on the host) as Go's float64(x): one load of its width under policy Ld,
// then the conversion.
template <typename Ld = Relaxed>
__device__ __forceinline__ double load(const void *p, uint32_t dtype) {
    double v;
    switch (dtype) {
    case LH_GAUGE_F64: v = __longlong_as_double((long long)Ld::ld64(p)); break;
    case LH_GAUGE_F32: v = from_f32(Ld::ld32(p)); break;
    case LH_GAUGE_F16: v = from_f16(Ld::ld16(p)); break;
    case LH_GAUGE_BF16: v = from_bf16(Ld::ld16(p)); break;
    case LH_GAUGE_I64: v = from_i64(Ld::ld64(p)); break;
    case LH_GAUGE_I32: v = from_i32(Ld::ld32(p)); break;
    default: v = from_u64(Ld::ld64(p)); break;   // LH_GAUGE_U64
    }
    return v;
}
// log2 of the element size of dtype LH_GAUGE_*: one nibble per dtype, F64 in the lowest (8 4 2 2 8 4 8 bytes)
__device__ __forceinline__ uint32_t shift(uint32_t dtype) { return (0x3231123u >> (4u * dtype)) & 15u; }
}  // namespace gauge

__global__ void __launch_bounds__(GR_THREADS)
k_gauge_read(const __grid_constant__ GaugeParams p) {
    const uint32_t i = blockIdx.x * GR_THREADS + threadIdx.x;
    if (i >= p.n) return;
    const GaugeEntry e = p.e[i];
    p.out[i] = gauge::load(e.p, e.dtype);
}

// ----------------------------------------------------------- narrow forms of K1 (lh_ingest_arrays)
// The element converters of k_ingest_single_bulk for long arrays of 4-byte and 16-bit samples: T is the raw element,
// f64 the gauge conversion of its bits.
struct K1F32 { using T = uint32_t; static constexpr bool kTable = false;
               static __device__ __forceinline__ double f64(uint32_t b) { return gauge::from_f32(b); } };
struct K1I32 { using T = uint32_t; static constexpr bool kTable = false;
               static __device__ __forceinline__ double f64(uint32_t b) { return gauge::from_i32(b); } };
struct K1F16 { using T = unsigned short; static constexpr bool kTable = true;
               static __device__ __forceinline__ double f64(unsigned short b) { return gauge::from_f16(b); } };
struct K1BF16 { using T = unsigned short; static constexpr bool kTable = true;
                static __device__ __forceinline__ double f64(unsigned short b) { return gauge::from_bf16(b); } };

// The key tables of the 16-bit form, built once per context: table[0] for float16, table[1] for bfloat16, entry m
// (magnitude bits, x & 0x7FFF) the window slot of exact_key16(float64(m)), 0xFFFF when that key has no slot below win.
// compress(-v) = -compress(v) and key16_to_slot puts key -k at slot win + k, so a sample with the sign bit set takes
// the entry plus win (slot win is key 0, as is slot 0).  Inf and NaN take the entry of whatever key exact_key16 gives.
__global__ void k_fill_key16(uint16_t *__restrict__ table, double precision, uint32_t win) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 65536u) return;
    const unsigned short m = (unsigned short)(i & 0x7FFFu);
    const double v = (i >> 15) ? gauge::from_bf16(m) : gauge::from_f16(m);
    const uint32_t slot = key16_to_slot(exact_key16(v, precision), win);
    table[i] = slot < win ? (uint16_t)slot : (uint16_t)0xFFFFu;
}

// ----------------------------------------------------------- distribution gauges (lh_snapshot_ingest_arrays)
// Every element of many device arrays, each of dtype LH_GAUGE_* under its own histogram id, into the frozen interval's
// rows.  The work is k_ingest_batch's: the item table travels in the parameter block, the items' concatenation is cut
// into BI_PIECE-sample pieces dealt round-robin to the CTAs, each thread walks its piece across item boundaries, and
// every CTA counts through one lh::BlockRecorder of BI_TABLE_ENTRIES entries, flushed once.  Only the sample load
// differs: an element is read as a device gauge is (gauge::load), so a value written by one aligned store is never
// torn.  The host bounds a launch's samples as it bounds k_ingest_batch's (no CTA counts more than 2^31 of them).
// Ld = gauge::Streaming is the short-item route of lh_ingest_arrays / lh_graph_recorder_ingest_arrays: the same walk
// over stream-ordered arrays with streaming loads, into the active interval's or a graph recorder's rows.
struct ArraySeg {
    const void *vals;                        // dtype-aligned, the whole item inside one allocation (checked on the host)
    uint32_t id;
    uint32_t dtype;                          // LH_GAUGE_*
};
struct ArrayParams {
    lh_recorder rec;                         // the frozen interval's rows
    uint32_t n_items;
    uint32_t pad;
    unsigned long long start[BI_MAX_ITEMS + 1];   // prefix offsets of the items' lengths
    ArraySeg seg[BI_MAX_ITEMS];
};

template <typename Ld>
__global__ void __launch_bounds__(BI_THREADS, 2)
k_ingest_arrays(const __grid_constant__ ArrayParams p) {
    extern __shared__ __align__(16) unsigned char ia_smem[];
    BlockRecorder br(p.rec, ia_smem, BI_TABLE_ENTRIES);
    br.init();
    const unsigned long long total = p.start[p.n_items];
    const unsigned long long pieces = (total + BI_PIECE - 1) / BI_PIECE;
    for (unsigned long long pc = blockIdx.x; pc < pieces; pc += gridDim.x) {
        const unsigned long long lo = pc * BI_PIECE;
        const unsigned long long hi = min(lo + BI_PIECE, total);
        uint32_t a = 0, b = p.n_items - 1;   // the item holding sample lo (uniform over the CTA)
        while (a < b) {
            const uint32_t m = (a + b + 1) / 2;
            if (p.start[m] <= lo) a = m; else b = m - 1;
        }
        uint32_t it = a;
        for (unsigned long long g0 = lo + threadIdx.x; g0 < hi; g0 += 2 * BI_THREADS) {
            double v[2];
            uint32_t id[2];
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const unsigned long long g = g0 + k * BI_THREADS;
                v[k] = 0.0; id[k] = 0u;
                if (g < hi) {
                    while (p.start[it + 1] <= g) ++it;
                    const ArraySeg s = p.seg[it];
                    id[k] = s.id;
                    v[k] = gauge::load<Ld>((const char *)s.vals + ((g - p.start[it]) << gauge::shift(s.dtype)), s.dtype);
                }
            }
#pragma unroll
            for (int k = 0; k < 2; k++)
                if (g0 + k * BI_THREADS < hi) br.record(id[k], v[k]);
        }
    }
    br.flush();
}

// ----------------------------------------------------------- raw device subscriptions (lh_raw_*, lh_snapshot_publish_raw)
// k_raw_publish writes the running bucket counts of one collection into a raw board (layout: include/loghisto_b200.h),
// one CTA per row, each row under its own seqlock whose word is the row header's first uint64:
//   1. thread 0 makes the word odd, fence.acq_rel.gpu, __syncthreads;
//   2. the row's id picks its source row of the snapshot view and that row's flag picks the cells: none (flag 0 or
//      unbound: an empty row), the 2*win-1 keys of the fast window (flag 1), or all 65 536 keys (flag & 2).  The cells
//      are loaded in ascending key order in chunks of RP_CHUNK, block-scanned with the running total of the chunks
//      before as carry (the window of precision 250 is 43 669 cells, more than shared memory holds at once), and
//      written with strong relaxed stores to cell key + 32768 of the row;
//   3. thread 0 writes total and the key range into the header (key_hi + LH_RAW_KEY_WRAPPED when a running count
//      passed 2^64, seen as a step whose sum is below its addend), __threadfence, __syncthreads;
//   4. thread 0 writes the publish count and makes the word even with st.release.gpu.
// Readers (include/loghisto_b200_device.cuh: lh::raw_percentile / raw_rank / raw_bucket_count, which k_raw_percentiles
// and k_raw_ranks call) load the word with ld.acquire.gpu and retry while it is odd, load the header and the cells they
// need with strong relaxed loads, then fence.acq_rel.gpu and the word again, and retry if it changed.  A reader that
// saw a store of this publish synchronises with step 1's fence, so its second load of the word sees the odd value or a
// later one and it retries; a reader that saw step 4's even word sees every store before it.  Cells outside the header's
// range are never read (they read as 0 below it and total above it), so a dense row published earlier leaves nothing a
// later window-only publish of the row has to clear.
//
// Termination: the CTA that writes a row waits on nothing -- no lock, no flag, no other CTA or kernel -- so once it is
// resident it finishes in a bounded number of steps, and the row's word is odd only while that CTA is resident.  A
// reader therefore spins only while a resident writer runs, whatever else occupies the GPU (CTAs of the same launch
// that have not started yet leave their rows' words even).  An id table too large for one parameter block is first
// copied into the board's table area by k_raw_stage launches, which touch no word.
constexpr int RP_THREADS = 512;
constexpr int RP_PER = 8;                        // contiguous cells per thread in the scan
constexpr int RP_CHUNK = RP_THREADS * RP_PER;    // cells per chunk
constexpr int RP_MAX_IDS = 4096;                 // ids per launch: 4 B each in the parameter block

// shared-memory index of chunk cell i: one pad word per 8 cells, so that the scan's per-thread runs of 8 hit distinct
// banks
__device__ __forceinline__ uint32_t rp_slot(uint32_t i) { return i + (i >> 3); }

struct RawPublishParams {
    char *rows;                              // k lh_raw_row_header
    unsigned long long *cells;               // k rows of uint64[65536]
    uint32_t *table;                         // ids staged by k_raw_stage, [n_staged]
    const unsigned long long *buckets;       // the snapshot view's rows and flags
    const uint32_t *flags;
    uint32_t win;
    uint32_t n_staged, n;                    // ids in `table`, then in ids[]
    // window boards only (k_raw_publish_window; see below)
    unsigned long long *sums;                // k rows of uint64[65536], by uint16 key: the window's per-key sums
    unsigned long long *slots;               // k * window rows of uint64[65536], by uint16 key: row r's slot j at r * window + j
    uint32_t *nlevel;                        // [k][2]: slots of row r at level 1, at level 2
    uint8_t *levels;                         // [k][window]: level of each slot (0 empty, 1 window keys, 2 all keys)
    uint32_t window, slot;                   // slots per row; the slot (the oldest) this publish replaces
    uint32_t ids[RP_MAX_IDS];
};

// the id of `row` (staged or in the parameter block), and the level of its source row: 0 none (unbound or untouched),
// 1 the fast window's keys, 2 all keys.  rp_range gives a level's key range (lo > hi: empty).
__device__ __forceinline__ uint32_t rp_id(const RawPublishParams &p, uint32_t row) {
    return row < p.n_staged ? p.table[row] : p.ids[row - p.n_staged];
}
__device__ __forceinline__ uint32_t rp_level(const RawPublishParams &p, uint32_t id) {
    const uint32_t f = id == LH_GRAPH_UNBOUND ? 0u : p.flags[id];
    return f == 0u ? 0u : (f & 2u) ? 2u : 1u;
}
__device__ __forceinline__ void rp_range(uint32_t level, uint32_t win, int &lo, int &hi) {
    lo = level == 2u ? -32768 : level == 1u ? -(int)(win - 1u) : 0;
    hi = level == 2u ? 32767 : level == 1u ? (int)(win - 1u) : -1;
}

// The chunked running-count scan of one row, by the whole CTA: keys [lo, hi] of src (indexed by uint16 key, as the
// snapshot's rows) are loaded in ascending key order in chunks of RP_CHUNK, block-scanned with the running total of
// the chunks before as carry, and written with strong relaxed stores to cells key + 32768 of dst.  Returns the running
// count after key hi (0 for lo > hi); wrap becomes nonzero in the threads that saw a running count pass 2^64.  Every
// thread must call it; it ends with a __syncthreads.
__device__ __forceinline__ unsigned long long rp_scan_row(const unsigned long long *src, int lo, int hi,
                                                          unsigned long long *dst, unsigned long long *s_cells,
                                                          unsigned long long *s_warp, int &wrap) {
    const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
    unsigned long long carry = 0;
    if (lo > hi) return carry;
    const uint32_t n = (uint32_t)(hi - lo + 1);
    dst += (uint32_t)(lo + 32768);
    for (uint32_t c0 = 0; c0 < n; c0 += RP_CHUNK) {
#pragma unroll
        for (int j = 0; j < RP_PER; j++) {                    // coalesced: chunk cell i is key lo + c0 + i
            const uint32_t i = (uint32_t)j * RP_THREADS + t;
            s_cells[rp_slot(i)] = c0 + i < n ? src[(uint32_t)(lo + (int)(c0 + i)) & 0xFFFFu] : 0ull;
        }
        __syncthreads();
        unsigned long long v[RP_PER], local = 0;
#pragma unroll
        for (int j = 0; j < RP_PER; j++) { v[j] = s_cells[rp_slot(t * RP_PER + j)]; local += v[j]; }
        unsigned long long incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= (uint32_t)o) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const unsigned long long w = lane < RP_THREADS / 32 ? s_warp[lane] : 0ull;
            unsigned long long wi = w;
#pragma unroll
            for (int o = 1; o < RP_THREADS / 32; o <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
                if (lane >= (uint32_t)o) wi += y;
            }
            if (lane < RP_THREADS / 32) s_warp[lane] = wi - w;   // exclusive prefix of the warp totals
        }
        __syncthreads();
        unsigned long long run = carry + s_warp[warp] + incl - local;
#pragma unroll
        for (int j = 0; j < RP_PER; j++) { run += v[j]; wrap |= run < v[j]; s_cells[rp_slot(t * RP_PER + j)] = run; }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < RP_PER; j++) {
            const uint32_t i = (uint32_t)j * RP_THREADS + t;
            if (c0 + i < n) board::st_relaxed(dst + c0 + i, s_cells[rp_slot(i)]);
        }
        carry = s_cells[rp_slot(RP_CHUNK - 1)];                // the running count after this chunk
        __syncthreads();                                      // before the next chunk overwrites s_cells / s_warp
    }
    return carry;
}

// Steps 1 and 3-4 of the seqlock sequence above, around the body of a publish.
__device__ __forceinline__ void rp_open(char *h) {
    if (threadIdx.x == 0) {
        unsigned long long *seq = reinterpret_cast<unsigned long long *>(h);
        board::st_relaxed(seq, board::ld_relaxed(seq) + 1ull);   // odd: the previous publish ended (stream order)
        board::fence_acq_rel();
    }
    __syncthreads();
}
__device__ __forceinline__ void rp_close(char *h, unsigned long long total, int lo, int hi, int wrap) {
    if (__syncthreads_or(wrap)) hi += LH_RAW_KEY_WRAPPED;          // readers fall back to Go's literal rule
    if (threadIdx.x == 0) {
        board::st_relaxed(h + offsetof(lh_raw_row_header, total), total);
        board::st_relaxed(h + offsetof(lh_raw_row_header, key_lo),
                          (unsigned long long)(uint32_t)lo | (unsigned long long)(uint32_t)hi << 32);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long *seq = reinterpret_cast<unsigned long long *>(h);
        const unsigned long long s = board::ld_relaxed(seq) + 1ull;   // even
        board::st_relaxed(h + offsetof(lh_raw_row_header, publishes), s >> 1);
        board::st_release(seq, s);
    }
}

__global__ void __launch_bounds__(RP_THREADS)
k_raw_stage(const __grid_constant__ RawPublishParams p) {
    for (uint32_t i = threadIdx.x; i < p.n; i += RP_THREADS) p.table[p.n_staged + i] = p.ids[i];
}

__global__ void __launch_bounds__(RP_THREADS)
k_raw_publish(const __grid_constant__ RawPublishParams p) {
    __shared__ unsigned long long s_cells[RP_CHUNK + RP_CHUNK / 8];
    __shared__ unsigned long long s_warp[RP_THREADS / 32];
    const uint32_t row = blockIdx.x;
    const uint32_t id = rp_id(p, row);
    const uint32_t level = rp_level(p, id);
    char *h = p.rows + (size_t)row * sizeof(lh_raw_row_header);
    rp_open(h);
    int lo, hi;
    rp_range(level, p.win, lo, hi);
    int wrap = 0;                                                 // a running count passed 2^64
    const unsigned long long total = rp_scan_row(p.buckets + (size_t)(level ? id : 0u) * 65536u, lo, hi,
                                                 p.cells + (size_t)row * 65536u, s_cells, s_warp, wrap);
    rp_close(h, total, lo, hi, wrap);
}

// k_raw_publish_window publishes into a board of `window` > 1 publishes per row (lh_raw_board_create_window): row r
// answers for the per-key sums, mod 2^64, of its last `window` entering intervals.  Per row the board keeps a dense sum
// row and `window` slots, each holding one entering interval's counts and its level (0 empty, 1 window keys, 2 all
// keys), with the number of slots at levels 1 and 2.  The sum's key range is that of the widest level among the slots;
// a slot's cells are read only inside its own level's range, and the sum's cells outside its range are 0 (below).
// One CTA per row, inside the row's seqlock exactly as k_raw_publish (steps 1 and 3-4 above), and, like it, waiting on
// nothing; all the row's bookkeeping is touched only by the CTA that writes the row, and two publishes of a board are
// ordered by the stream.  In step 2:
//   a. the entering interval is the row's source row as in k_raw_publish, at level lin; it replaces slot p.slot, at
//      level lout; the sum's level before is lsum, after it lnew (from the slot counts);
//   b. over the keys of max(lsum, lin): sum += in - out (in, out read as 0 outside their own ranges), and the slot takes
//      in over lin's range.  A key outside lnew's range then holds 0 mod 2^64: every slot left is 0 there;
//   c. __syncthreads (the CTA's own stores of the sum row are visible to it), then the chunked scan of the sum row over
//      lnew's range, whose wrap rule therefore follows the window's own running counts.
constexpr int RW_PER = 4;                        // keys per thread in flight in step b

__global__ void __launch_bounds__(RP_THREADS)
k_raw_publish_window(const __grid_constant__ RawPublishParams p) {
    __shared__ unsigned long long s_cells[RP_CHUNK + RP_CHUNK / 8];
    __shared__ unsigned long long s_warp[RP_THREADS / 32];
    const uint32_t row = blockIdx.x, t = threadIdx.x;
    const uint32_t id = rp_id(p, row);
    const uint32_t lin = rp_level(p, id);
    char *h = p.rows + (size_t)row * sizeof(lh_raw_row_header);
    rp_open(h);
    uint8_t *lv = p.levels + (size_t)row * p.window + p.slot;
    uint32_t *cnt = p.nlevel + (size_t)row * 2u;
    const uint32_t lout = *lv, n1 = cnt[0], n2 = cnt[1];
    const uint32_t m1 = n1 - (lout == 1u) + (lin == 1u), m2 = n2 - (lout == 2u) + (lin == 2u);
    const uint32_t lsum = n2 ? 2u : n1 ? 1u : 0u, lnew = m2 ? 2u : m1 ? 1u : 0u;
    __syncthreads();                                              // every thread has read the bookkeeping
    if (t == 0) { *lv = (uint8_t)lin; cnt[0] = m1; cnt[1] = m2; }
    int ilo, ihi, olo, ohi, ulo, uhi;
    rp_range(lin, p.win, ilo, ihi);
    rp_range(lout, p.win, olo, ohi);
    rp_range(lsum > lin ? lsum : lin, p.win, ulo, uhi);
    const unsigned long long *src = p.buckets + (size_t)(lin ? id : 0u) * 65536u;
    unsigned long long *sum = p.sums + (size_t)row * 65536u;
    unsigned long long *slot = p.slots + ((size_t)row * p.window + p.slot) * 65536u;
    if (ulo <= uhi) {
        const uint32_t n = (uint32_t)(uhi - ulo + 1);
        for (uint32_t c0 = 0; c0 < n; c0 += RP_THREADS * RW_PER) {
            unsigned long long in[RW_PER], out[RW_PER], s[RW_PER];
#pragma unroll
            for (int j = 0; j < RW_PER; j++) {                    // every load of the group before any store
                const uint32_t i = c0 + (uint32_t)j * RP_THREADS + t;
                const int key = ulo + (int)i;
                const uint32_t k16 = (uint32_t)key & 0xFFFFu;
                const bool live = i < n;
                in[j] = live && key >= ilo && key <= ihi ? src[k16] : 0ull;
                out[j] = live && key >= olo && key <= ohi ? slot[k16] : 0ull;
                s[j] = live ? sum[k16] : 0ull;
            }
#pragma unroll
            for (int j = 0; j < RW_PER; j++) {
                const uint32_t i = c0 + (uint32_t)j * RP_THREADS + t;
                const int key = ulo + (int)i;
                const uint32_t k16 = (uint32_t)key & 0xFFFFu;
                if (i < n) {
                    sum[k16] = s[j] + in[j] - out[j];
                    if (key >= ilo && key <= ihi) slot[k16] = in[j];
                }
            }
        }
    }
    __syncthreads();
    int lo, hi;
    rp_range(lnew, p.win, lo, hi);
    int wrap = 0;
    const unsigned long long total = rp_scan_row(sum, lo, hi, p.cells + (size_t)row * 65536u, s_cells, s_warp, wrap);
    rp_close(h, total, lo, hi, wrap);
}

// One thread per query; the answers are the device API's (one definition of the read).  rows == nullptr: the grid
// form, query i is row i / m with input i % m.
constexpr int RQ_THREADS = 256;

__global__ void __launch_bounds__(RQ_THREADS)
k_raw_percentiles(const lh_raw_board b, const uint32_t *__restrict__ rows, const double *__restrict__ ps, uint32_t n,
                  uint32_t m, int32_t *__restrict__ keys, double *__restrict__ vals, unsigned long long *__restrict__ publish) {
    const uint32_t i = blockIdx.x * RQ_THREADS + threadIdx.x;
    if (i >= n) return;
    int32_t key;
    double val;
    publish[i] = raw_percentile(b, rows ? rows[i] : i / m, ps[rows ? i : i % m], &key, &val);
    keys[i] = key;
    vals[i] = val;
}

__global__ void __launch_bounds__(RQ_THREADS)
k_raw_ranks(const lh_raw_board b, const uint32_t *__restrict__ rows, const double *__restrict__ values, uint32_t n,
            uint32_t m, unsigned long long *__restrict__ ranks, unsigned long long *__restrict__ totals,
            unsigned long long *__restrict__ publish) {
    const uint32_t i = blockIdx.x * RQ_THREADS + threadIdx.x;
    if (i >= n) return;
    uint64_t rank, total;
    publish[i] = raw_rank(b, rows ? rows[i] : i / m, values[rows ? i : i % m], &rank, &total);
    ranks[i] = rank;
    if (rows) totals[i] = total;
    else if (i % m == 0) totals[i / m] = total;
}

// ----------------------------------------------------------- GPU timers (lh_gpu_timer_*)
// One thread each: their cost is the launch, not the body.  The start writes %globaltimer into the token's slot; the
// stop records float64(now - start) into one histogram row through the same bucket function and row writer every
// device caller uses (what lh::record_ns does, without the warp combining a single thread cannot use).  A slot that
// holds kTimerNeverStarted (a graph recorder's mark before its first start) records nothing and counts 1 in `dropped`.
constexpr unsigned long long kTimerNeverStarted = ~0ull;
__global__ void k_gpu_timer_mark(unsigned long long *__restrict__ slot) { *slot = globaltimer_ns(); }

__global__ void k_gpu_timer_stop(const unsigned long long *__restrict__ slot, unsigned long long *__restrict__ row,
                                 uint32_t *flag, long long *out, unsigned long long *dropped, Prec pc) {
    const unsigned long long start = *slot;
    if (start == kTimerNeverStarted) { atomicAdd(dropped, 1ull); return; }
    const long long ns = (long long)(globaltimer_ns() - start);
    add_bucket_global(row, flag, key16_of(__ll2double_rn(ns), pc), 1ull, pc.win);
    if (out) *out = ns;
}

// ----------------------------------------------------------- probes / tables
__global__ void k_fill_decompress(double *__restrict__ table, double precision) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 65536) table[i] = go_decompress((int)(short)i, precision);
}

__global__ void k_compress_probe(const double *__restrict__ v, size_t n, short *__restrict__ out, int mode, Prec pc) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (short)(mode == 1 ? exact_key16(v[i], pc.precision) : key16_of(v[i], pc));
}

// max | estimate - precision*ln(x) | over samples inside the fast window, for both estimators that ship:
//   [0] fast_candidate()      (k_ingest_keyed*, probes, ragged tails)
//   [2] bucket_offsets_v2()   (pairwise FP32 form with the -1023*c2 constant folded into the FMA; K1, keyed_small, keyed_wc)
// plus [1] the tally of samples fast_candidate() sends to the exact path.
__global__ void k_fastpath_margin(const double *__restrict__ v, size_t n, unsigned long long *__restrict__ out, Prec pc) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double x = __dadd_rn(1.0, fabs(v[i]));
    uint32_t hi = (uint32_t)__double2hiint(x), lo = (uint32_t)__double2loint(x);
    uint32_t idx; bool slow;
    fast_candidate(v[i], pc, idx, slow);
    if (slow) atomicAdd(&out[1], 1ull);
    if (hi >= 0x43E00000u) return;
    uint32_t t = __funnelshift_l(lo, hi, 3);
    float m = __uint_as_float((t & 0x007FFFFFu) | 0x3F800000u);
    float lg;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(lg) : "f"(m));
    uint32_t eb = hi >> 20;
    const double truth = pc.precision * log(x);
    const double base = (double)(int)(eb - 1023u) * (double)pc.a_int;
    {   // estimator 1
        float ef = __fadd_rn(__uint_as_float(0x4B000000u | eb), -(8388608.0f + 1023.0f));
        float w = __fmaf_rn(lg, pc.c1, __fmul_rn(ef, pc.c2));
        atomicMax(&out[0], (unsigned long long)__double_as_longlong(fabs(base + (double)w - truth)));
    }
    {   // estimator 2 (same constants as bucket_offsets_v2)
        float a = __fmaf_rn(__uint2float_rn(eb), pc.c2, pc.kb);
        float w = __fmaf_rn(lg, pc.c1, a);
        atomicMax(&out[2], (unsigned long long)__double_as_longlong(fabs(base + (double)w - truth)));
    }
}

// Exhaustive certification of the fast path at one precision (lh_fastpath_certify; one launch per precision).
// The forms' outputs depend on v only through its sign and the cell of x = 1+|v|: the biased exponent eb and the top
// 23 mantissa bits t.  Every cell with eb in 1023..1086 (x in [1, 2^64)) is visited with v = X_lo - 1 and -v, X_lo
// the cell's smallest double, through the inline functions the kernels call with the arguments they pass:
//   form 0  fast_candidate()                  (key16_of, the keyed vec / scalar kernels, K1 ldg, the fix-ups, device API)
//   form 1  bucket_offsets_v2<4, true, 2>     (K1 bulk, sign folded into the slot)
//   form 2  bucket_offsets_v2<4, false, 2>    (K1 bulk, negatives flagged; k_ingest_keyed_small)
//   form 3  bucket_offsets_v2<4, false, 0>    (k_ingest_keyed_wc)
// and each output is decoded as the kernels decode it (slot -> key16).  The reference is FP64 log at both ends of the
// cell, L_lo = P ln X_lo and L_hi = P ln X_hi (X_hi the next cell's X_lo); ln is monotone, so [L_lo, L_hi] holds
// P ln x for every double of the cell.  Per form, as FC_* words of out[form * FC_FIELDS]:
//   samples            samples inside the window: x < 2^63, and v >= 0 for the positive-only forms 2 and 3
//   flagged            ... of them handed to the exact path
//   wrong              unflagged, but [L_lo, L_hi] not inside (key - 0.5 + 2^-30, key + 0.5 - 2^-30): some double of
//                      the cell could get another key than Go's (FP64 log errs by far less than 2^-30 bucket units)
//   out_of_range       unflagged with a slot outside the sub-histogram ([0, 2 win), [0, win) for forms 2 and 3): a
//                      shared-memory write past the window
//   unflagged_outside  a sample outside the window (x >= 2^63; a negative one for forms 2 and 3) left unflagged
//   over_flagged       flagged although [L_lo, L_hi] lies farther than eps + (this sample's estimate error) + 2^-20
//                      from every half-integer: a flag the eps band does not explain
//   input_mismatch     fl(1 + |v|) != X_lo (the same count for every form)
//   max_err            max |estimate - L| at both ends over every sample with x < 2^63 (double bits)
//   min_margin         min distance of an unflagged interval from a bucket boundary, floored at 0 (double bits)
constexpr int FC_FORMS = 4;
constexpr int FC_FIELDS = 9;
constexpr int FC_SAMPLES = 0, FC_FLAGGED = 1, FC_WRONG = 2, FC_OUT_OF_RANGE = 3, FC_UNFLAGGED_OUTSIDE = 4,
              FC_OVER_FLAGGED = 5, FC_INPUT_MISMATCH = 6, FC_MAX_ERR = 7, FC_MIN_MARGIN = 8;
constexpr int FC_THREADS = 256;
constexpr uint32_t FC_CELL_BITS = 29;        // 64 exponents x 2^23 mantissa prefixes
constexpr uint32_t FC_RUN = 64;              // consecutive cells per thread and run: one FP64 log per cell

struct FcAcc {
    uint32_t n[FC_INPUT_MISMATCH];           // FC_SAMPLES .. FC_OVER_FLAGGED
    double max_err, min_margin;
};

// One sample of one form.  slot = the sub-histogram slot the form produced (0xFFFFFFFF: not a slot), nslots = the
// sub-histogram's length, pos_only = positive-only layout (slot == key), w = the FP32 part of the estimate.
__device__ __forceinline__ void fc_account(FcAcc &a, bool flag, uint32_t slot, uint32_t nslots, bool pos_only, bool neg,
                                           uint32_t eb, float w, double L_lo, double L_hi, double eps, const Prec &pc) {
    const double E = (double)((int)eb - 1023) * (double)pc.a_int + (double)w;
    const double err = fmax(fabs(E - L_lo), fabs(E - L_hi));
    const bool in_range = eb < 1086u;                    // x < 2^63
    if (in_range) a.max_err = fmax(a.max_err, err);
    if (!in_range || (pos_only && neg)) {
        if (!flag) a.n[FC_UNFLAGGED_OUTSIDE]++;
        return;
    }
    a.n[FC_SAMPLES]++;
    if (flag) {
        a.n[FC_FLAGGED]++;
        // distance of [L_lo, L_hi] from the nearest half-integer (the interval is far shorter than one bucket)
        const double h0 = floor(L_lo) + 0.5, h1 = floor(L_hi) + 0.5;
        const double dist = fmin(fmax(0.0, fmax(L_lo - h0, h0 - L_hi)), fmax(0.0, fmax(L_lo - h1, h1 - L_hi)));
        if (dist > eps + err + 0x1p-20) a.n[FC_OVER_FLAGGED]++;
        return;
    }
    if (slot >= nslots) { a.n[FC_OUT_OF_RANGE]++; return; }
    const uint32_t key16 = pos_only ? slot : slot_to_key16(slot, pc.win);
    const double key = (double)(short)key16, mag = neg ? -key : key;
    const double margin = fmin(L_lo - (mag - 0.5), (mag + 0.5) - L_hi);
    if (!(margin > 0x1p-30)) a.n[FC_WRONG]++;
    a.min_margin = fmin(a.min_margin, fmax(margin, 0.0));
}

__global__ void __launch_bounds__(FC_THREADS)
k_fastpath_certify(unsigned long long *__restrict__ out, Prec pc) {
    __shared__ unsigned long long s_red[FC_FORMS][FC_FIELDS];
    for (int i = threadIdx.x; i < FC_FORMS * FC_FIELDS; i += FC_THREADS) {
        const int f = i % FC_FIELDS;
        s_red[i / FC_FIELDS][f] = f == FC_MIN_MARGIN ? 0x7FF0000000000000ull : 0ull;   // +Inf: the identity of min
    }
    __syncthreads();
    uint32_t one_bits;
    asm volatile("mov.b32 %0, 0x3F800000;" : "=r"(one_bits));
    const double eps = 0.5 - (double)pc.thresh;
    FcAcc acc[FC_FORMS];
#pragma unroll
    for (int f = 0; f < FC_FORMS; f++) {
#pragma unroll
        for (int i = 0; i < FC_INPUT_MISMATCH; i++) acc[f].n[i] = 0;
        acc[f].max_err = 0.0;
        acc[f].min_margin = __longlong_as_double(0x7FF0000000000000ll);
    }
    uint32_t mismatch = 0;
    const uint64_t one = 0x3FF0000000000000ull;          // X_lo of cell c: bits one + (c << 29)
    const uint32_t nruns = (1u << FC_CELL_BITS) / FC_RUN;
    for (uint32_t run = blockIdx.x * FC_THREADS + threadIdx.x; run < nruns; run += gridDim.x * FC_THREADS) {
        const uint64_t c0 = (uint64_t)run * FC_RUN;
        const uint32_t eb = 1023u + (uint32_t)(c0 >> 23);                  // a run never crosses an exponent
        double L_prev = pc.precision * log(u64_as_f64(one + (c0 << 29)));
        for (uint32_t j = 0; j < FC_RUN; j += 2) {                         // two cells: the forms take 4 samples
            const uint64_t c = c0 + j;
            const double X0 = u64_as_f64(one + (c << 29)), X1 = u64_as_f64(one + ((c + 1) << 29));
            const double L[3] = {L_prev, pc.precision * log(X1), pc.precision * log(u64_as_f64(one + ((c + 2) << 29)))};
            L_prev = L[2];
            const double v0 = __dsub_rn(X0, 1.0), v1 = __dsub_rn(X1, 1.0);
            const double v[4] = {v0, -v0, v1, -v1};
            mismatch += 2u * ((__dadd_rn(1.0, v0) != X0) + (__dadd_rn(1.0, v1) != X1));
            {   // form 0
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    uint32_t idx; bool slow; float w;
                    fast_candidate(v[s], pc, idx, slow, w);
                    fc_account(acc[0], slow, idx, 2u * pc.win, false, s & 1, eb, w, L[s >> 1], L[(s >> 1) + 1], eps, pc);
                }
            }
            uint32_t off[4]; bool flag[4]; float est[4];
            bucket_offsets_v2<4, true, 2>(v, pc, one_bits, off, flag, est);
#pragma unroll
            for (int s = 0; s < 4; s++)
                fc_account(acc[1], flag[s], (off[s] & 3u) ? 0xFFFFFFFFu : off[s] >> 2, 2u * pc.win, false, s & 1, eb, est[s],
                           L[s >> 1], L[(s >> 1) + 1], eps, pc);
            bucket_offsets_v2<4, false, 2>(v, pc, one_bits, off, flag, est);
#pragma unroll
            for (int s = 0; s < 4; s++)
                fc_account(acc[2], flag[s], (off[s] & 3u) ? 0xFFFFFFFFu : off[s] >> 2, pc.win, true, s & 1, eb, est[s],
                           L[s >> 1], L[(s >> 1) + 1], eps, pc);
            bucket_offsets_v2<4, false, 0>(v, pc, one_bits, off, flag, est);
#pragma unroll
            for (int s = 0; s < 4; s++)
                fc_account(acc[3], flag[s], off[s], pc.win, true, s & 1, eb, est[s], L[s >> 1], L[(s >> 1) + 1], eps, pc);
        }
    }
    // warp, then CTA, then one global atomic per word and CTA
#pragma unroll
    for (int f = 0; f < FC_FORMS; f++) {
        unsigned long long w[FC_FIELDS];
#pragma unroll
        for (int i = 0; i < FC_INPUT_MISMATCH; i++) w[i] = acc[f].n[i];
        w[FC_INPUT_MISMATCH] = mismatch;
        double mx = acc[f].max_err, mn = acc[f].min_margin;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
#pragma unroll
            for (int i = 0; i <= FC_INPUT_MISMATCH; i++) w[i] += __shfl_xor_sync(0xFFFFFFFFu, w[i], o);
            mx = fmax(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
            mn = fmin(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o));
        }
        if ((threadIdx.x & 31) == 0) {
#pragma unroll
            for (int i = 0; i <= FC_INPUT_MISMATCH; i++) atomicAdd(&s_red[f][i], w[i]);
            atomicMax(&s_red[f][FC_MAX_ERR], (unsigned long long)__double_as_longlong(mx));    // both >= 0: bits order
            atomicMin(&s_red[f][FC_MIN_MARGIN], (unsigned long long)__double_as_longlong(mn));
        }
    }
    __syncthreads();
    if (threadIdx.x < FC_FORMS * FC_FIELDS) {
        const int f = threadIdx.x / FC_FIELDS, i = threadIdx.x % FC_FIELDS;
        const unsigned long long x = s_red[f][i];
        unsigned long long *dst = out + f * FC_FIELDS + i;
        if (i == FC_MAX_ERR) atomicMax(dst, x);
        else if (i == FC_MIN_MARGIN) atomicMin(dst, x);
        else if (x) atomicAdd(dst, x);
    }
}

// ---------------------------------------------------------- synthetic streams
__device__ __constant__ unsigned char c_streamL_exp[16] = {17, 18, 18, 19, 19, 19, 20, 20, 20, 20, 21, 21, 21, 22, 22, 23};

__device__ __forceinline__ uint64_t stream_bits(int kind, uint64_t seed, uint64_t i) {
    uint64_t u = splitmix64(seed + i);
    uint64_t mant = u & 0x000FFFFFFFFFFFFFull;
    switch (kind) {
    case 0: return ((uint64_t)(1023 + (u >> 52) % 63) << 52) | mant;
    case 1: return ((uint64_t)(1023 + c_streamL_exp[(u >> 52) & 15]) << 52) | mant;
    case 2: {
        uint32_t sel = (uint32_t)(u >> 52) & 0xFFFu;
        if (sel < 41) return 0x8000000000000000ull | ((uint64_t)(1023 + (u >> 40) % 63) << 52) | mant;
        if (sel < 60) return splitmix64(u);
        if (sel < 80) return ((u >> 11) & 0x8000000000000000ull) | ((uint64_t)(1023 - 10 + (u >> 40) % 12) << 52) | mant;
        if (sel < 90) return ((u >> 13) & 0x8000000000000000ull) | ((uint64_t)(1023 + 63 + (u >> 40) % 961) << 52) | mant;
        return ((uint64_t)(1023 + (u >> 40) % 63) << 52) | mant;
    }
    case 3: return 0x40F86A0000000000ull;
    case 4:
        if (u >> 63) return 0x40F86A0000000000ull;
        return ((uint64_t)(1023 + c_streamL_exp[(u >> 52) & 15]) << 52) | mant;
    case 6: {   // timer durations as int64 nanoseconds: the L stream truncated toward zero
        double d = u64_as_f64(((uint64_t)(1023 + c_streamL_exp[(u >> 52) & 15]) << 52) | mant);
        return (uint64_t)__double2ll_rz(d);
    }
    case 7: return 1 + (u >> 60);   // counter amounts 1..16
    case 8: return ((u >> 11) & 0x8000000000000000ull) | ((uint64_t)(1023 + (u >> 52) % 63) << 52) | mant;   // N: stream U, random sign
    default: return u;
    }
}

__global__ void k_gen_stream(int kind, uint64_t seed, uint64_t start, size_t n, double *__restrict__ out) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = u64_as_f64(stream_bits(kind, seed, start + i));
}

__global__ void k_gen_ids_u16(int kind, uint64_t seed, uint64_t start, size_t n, uint32_t H,
                              unsigned short *__restrict__ out) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint64_t u = splitmix64((seed ^ 0xA5A5A5A5DEADBEEFull) + start + i);
        uint32_t a = (uint32_t)((u & 0xFFFFFFFFu) % H), b = (uint32_t)((u >> 32) % H);
        out[i] = (unsigned short)(kind == 0 ? a : (a < b ? a : b));
    }
}

}  // namespace lh
