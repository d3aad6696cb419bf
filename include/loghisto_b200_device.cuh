// loghisto_b200_device.cuh -- device API of the loghisto engine: record Histogram, Timer and Counter samples from
// inside CUDA kernels, with the same bucket arithmetic the library's ingest kernels use (this header IS that
// arithmetic: the library includes it, so there is one definition of the bucket function).
//
//   lh::record(rec, id, v)        Histogram(name, v)          metrics.go:273-295 (compress, metrics.go:316-322)
//   lh::record_ns(rec, id, ns)    TimerToken.Stop()           metrics.go:242-246  value = float64(ns)
//   lh::count(rec, id, amount)    Counter(name, amount)       metrics.go:251-269  wrapping uint64 add
//   lh::start_timer(id) / lh::stop(rec, token)
//                                 StartTimer(name) / Stop()   metrics.go:232-246  durations on the GPU's clock
//   lh::BlockHistogram            one CTA feeding one histogram through a shared-memory sub-histogram
//   lh::BlockRecorder             one CTA feeding any number of histograms through a shared-memory combining table
//   lh::read_histogram / lh::read_counter
//                                 the latest collection's processed metrics of a name, from a device subscription
//                                 board (lh_board, MetricSystem::NewDeviceSubscription)   metrics.go:218, 508-525
//   lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count
//                                 exact percentile, rank and bucket queries over the latest collection's bucket counts
//                                 of a name, from a raw device subscription board (lh_raw_board,
//                                 MetricSystem::NewRawDeviceSubscription)                 metrics.go:203-215, 508-525
//
// `rec` is an lh_recorder (include/loghisto_b200.h) obtained from lh_record_begin on the host and passed to the kernel
// by value.  Kernels that use it must be enqueued on the recorder's stream between lh_record_begin and lh_record_end;
// the snapshot that takes the interval waits for lh_record_end.  A MetricSystem (loghisto_b200/host/metric_system.h)
// hands out recorders and ids by name through MetricSystem::BeginRecording.  Records go straight into the uint64 bucket rows of the
// active interval, so they are visible to lh_snapshot_reduce / _export exactly like samples of the ingest calls.
//
// Every function here has internal or inline linkage: the header may be included by several translation units of one
// program, with or without -rdc=true.  Needs sm_70 or later (__match_any_sync); the library itself targets sm_90a.
// tests/test_device_api_builds_cpu.py compiles it warning-free under C++14 / 17 / 20 for compute_70 PTX, sm_80, sm_90 and
// sm_90a and device-links two -rdc=true units; tests/test_gpu_device_api_builds.py runs one client built with the
// library's flags, --use_fast_math, -G, -maxrregcount=32, -rdc=true and as compute_90 / compute_70 PTX against the oracle.
//
// Bucket arithmetic -- two evaluators of compress() (reference metrics.go:316-322; `precision` is metrics.go:40-43,
// 100 by default and configurable through lh_config.precision):
//
//   exact_key16()   evaluates Go's math.Log algorithm (src/math/log.go, the
//                   FreeBSD e_log.c port; identical op tree to log_amd64.s) in
//                   FP64 with one IEEE rounding per operation (__dadd_rn /
//                   __dmul_rn / __ddiv_rn never contract to FMA), then Go's
//                   precision*L+0.5 and the amd64 CVTTSD2SL + low-16-bit truncation.
//                   IEEE-754 guarantees these are the same bits the Go code
//                   produces on amd64 (GOAMD64=v1).
//
//   fast_candidate() a ~14-instruction FP32 estimate of precision*ln(1+|v|) whose
//                   error is bounded by Prec::eps bucket units.  It returns
//                   the bucket whenever the estimate is farther than
//                   eps from a bucket boundary and flags the sample
//                   for exact_key16() otherwise (~0.05 % of samples at precision 100).
//
// The result of the pair is therefore exactly exact_key16() for every input;
// the fast path only decides how much work it takes to get there.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "loghisto_b200.h"

namespace lh {

// Everything that depends on `precision`, derived once on the host (make_prec in lh_api.cu) and passed to the
// kernels by value (constant bank).
//   precision * ln(x) = a_int * e + [ c2 * e + c1 * log2(m) ],   x = m * 2^e,  c1 = precision * ln 2,
//   a_int = floor(c1), c2 = c1 - a_int: the integer part is exact integer arithmetic, the bracket (< 64 + c1)
//   is evaluated in FP32.
// Fast window: keys 0..win-1 cover every x = 1+|v| < 2^63 (win = floor(precision*ln(2^63) + 0.5) + 1; 4368 at 100).
// Shared-memory sub-histograms hold [0,win) for v >= 0 and [win, 2*win) for v < 0.
//
// Error budget of the estimate, in bucket units, at precision P (derivation in DESIGN.md):
//   lg2.approx on [1,2): 2^-22 abs          * c1     = 1.7e-5 * P/100
//   mantissa truncated to 23 bits: 2^-23 rel * P      = 1.2e-5 * P/100
//   three FP32 roundings at magnitude < 64 + c1       = 1.2e-5 (P <= 100) .. 2.3e-5 (P <= 250)
//   constant representation                            = 0.6e-5 * P/100
// eps = 2^-12 * max(1, P/100).  The realised error is certified for every input at every precision 1..250 on the
// device (lh_fastpath_certify visits every (exponent, 23-bit mantissa prefix) cell of 1+|v|; tests/
// test_gpu_fastpath_exhaustive.py), measured on an H100 SXM 80 GB (700 W limit; MUFU.LG2 is what sets the error):
//   fast_candidate()                          max error 4.61e-5 (P = 239), smallest eps / max error 11.7 (P = 141)
//   bucket_offsets_v2() (all three layouts)   max error 6.69e-5 (P = 213), smallest eps / max error  5.2 (P = 85)
// and no unflagged cell lies closer than 2.0e-4 bucket units to a boundary.
struct Prec {
    double precision;   // as a float64, the factor Go multiplies by
    float c1;           // precision * ln2
    float c2;           // c1 - a_int
    float kb;           // -1023 * c2 (folds the exponent bias into the FMA of the packed form)
    float thresh;       // 0.5 - eps
    uint32_t a_int;     // floor(c1)
    uint32_t win;       // fast-window length
    uint32_t coff;      // byte-offset constant of the packed form: 0 - 1023*a_int*4 - (0x4B400000 << 2)
    uint32_t a4;        // a_int * 4
    uint32_t coff0;     // slot-index constant of the packed form: 0 - 1023*a_int - 0x4B400000
    uint32_t pad0;
};
static_assert(sizeof(Prec) == sizeof(((lh_recorder *)0)->prec), "lh_recorder.prec must hold an lh::Prec");

__device__ __forceinline__ double u64_as_f64(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t f64_as_u64(double d) { return (uint64_t)__double_as_longlong(d); }

// Go's math.Log for finite x >= 1 (compress only ever passes 1+|v|).
__device__ __forceinline__ double go_log_ge1(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01;
    const double Ln2Lo = 1.90821492927058770002e-10;
    const double L1 = 6.666666666666735130e-01;
    const double L2 = 3.999999999940941908e-01;
    const double L3 = 2.857142874366239149e-01;
    const double L4 = 2.222219843214978396e-01;
    const double L5 = 1.818357216161805012e-01;
    const double L6 = 1.531383769920937332e-01;
    const double L7 = 1.479819860511658591e-01;
    const double HalfSqrt2 = 7.07106781186547524401e-01;

    uint64_t xb = f64_as_u64(x);
    int ki = (int)(xb >> 52) - 1022;                                   // Frexp exponent
    double f1 = u64_as_f64((xb & 0x000FFFFFFFFFFFFFull) | 0x3FE0000000000000ull);  // in [0.5,1)
    if (f1 < HalfSqrt2) { f1 = __dmul_rn(f1, 2.0); ki--; }
    double f = __dadd_rn(f1, -1.0);
    double k = (double)ki;

    double s = __ddiv_rn(f, __dadd_rn(2.0, f));
    double s2 = __dmul_rn(s, s);
    double s4 = __dmul_rn(s2, s2);
    double t1 = __dmul_rn(s2, __dadd_rn(L1, __dmul_rn(s4, __dadd_rn(L3, __dmul_rn(s4, __dadd_rn(L5, __dmul_rn(s4, L7)))))));
    double t2 = __dmul_rn(s4, __dadd_rn(L2, __dmul_rn(s4, __dadd_rn(L4, __dmul_rn(s4, L6)))));
    double R = __dadd_rn(t1, t2);
    double hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
    // k*Ln2Hi - ((hfsq - (s*(hfsq+R) + k*Ln2Lo)) - f)
    double a = __dadd_rn(__dmul_rn(s, __dadd_rn(hfsq, R)), __dmul_rn(k, Ln2Lo));
    double b = __dsub_rn(__dsub_rn(hfsq, a), f);
    return __dsub_rn(__dmul_rn(k, Ln2Hi), b);
}

// compress(), bit-exact.  Returns (uint16)key zero-extended.  Out of line (it is the rare path of every caller) but
// inline in the C++ sense, so that every translation unit may carry its copy.
inline __device__ __noinline__ uint32_t exact_key16(double v, double precision) {
    double x = __dadd_rn(1.0, fabs(v));
    uint32_t key;
    if ((f64_as_u64(x) >> 52) >= 0x7FFull) {
        key = 0;  // log(+Inf)=+Inf, log(NaN)=NaN -> CVTTSD2SL indefinite 0x80000000 -> low 16 bits 0
    } else {
        double t = __dadd_rn(__dmul_rn(precision, go_log_ge1(x)), 0.5);   // 0.5 <= t < 709.8*precision + 1 < 2^31
        key = (uint32_t)__double2int_rz(t) & 0xFFFFu;                     // CVTTSD2SL, then int16 truncation
    }
    if (v < 0.0) key = (0u - key) & 0xFFFFu;                              // -1 * i, int16 wrap
    return key;
}

// Fast estimate.  On return:
//   idx  = sub-histogram slot (valid when !slow): key for v >= 0, win + key for v < 0
//   slow = the sample needs exact_key16()
//   w    = the FP32 part of the estimate: precision*ln(1+|v|) ~= (eb - 1023) * a_int + w, eb the biased exponent of
//          1+|v| (lh_fastpath_certify measures the error of this sum for every input)
__device__ __forceinline__ void fast_candidate(double v, const Prec &pc, uint32_t &idx, bool &slow, float &w) {
    double x = __dadd_rn(1.0, fabs(v));          // exactly Go's 1.0+math.Abs(value)
    uint32_t hi = (uint32_t)__double2hiint(x);
    uint32_t lo = (uint32_t)__double2loint(x);
    uint32_t t = __funnelshift_l(lo, hi, 3);     // top 23 mantissa bits of x in t[22:0]
    float m = __uint_as_float((t & 0x007FFFFFu) | 0x3F800000u);
    float lg;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(lg) : "f"(m));
    uint32_t eb = hi >> 20;                      // 1023 + e (sign bit is 0: x >= 1)
    float ef = __fadd_rn(__uint_as_float(0x4B000000u | eb), -(8388608.0f + 1023.0f));  // (float)e, exact
    w = __fmaf_rn(lg, pc.c1, __fmul_rn(ef, pc.c2));
    float r = __fadd_rn(w, 12582912.0f);         // 1.5*2^23: low mantissa bits = rn(w)
    float d = __fadd_rn(w, -__fadd_rn(r, -12582912.0f));
    uint32_t k = (eb - 1023u) * pc.a_int + (__float_as_uint(r) - 0x4B400000u);
    // x >= 2^63, Inf and NaN (hi >= 0x43E00000) leave the window: exact path.
    slow = (fabsf(d) > pc.thresh) | (hi >= 0x43E00000u);
    uint32_t neg = (uint32_t)__double2hiint(v) >> 31;
    idx = k + neg * pc.win;
}
__device__ __forceinline__ void fast_candidate(double v, const Prec &pc, uint32_t &idx, bool &slow) {
    float w;
    fast_candidate(v, pc, idx, slow, w);
}

// Map an exact (uint16)key to a sub-histogram slot, or 0xFFFFFFFF if outside the window.
__device__ __forceinline__ uint32_t key16_to_slot(uint32_t key16, uint32_t win) {
    if (key16 < win) return key16;
    uint32_t nk = 65536u - key16;                // |key| for negative keys
    if (nk < win) return win + nk;
    return 0xFFFFFFFFu;
}
// Inverse: slot -> (uint16)key.  Slot win (negative zero) folds onto key 0.
__device__ __forceinline__ uint32_t slot_to_key16(uint32_t slot, uint32_t win) {
    return slot < win ? slot : ((65536u - (slot - win)) & 0xFFFFu);
}
// Is (uint16)key inside the window the snapshot kernels scan when a histogram has no out-of-window counts?
__device__ __forceinline__ bool key16_in_window(uint32_t key16, uint32_t win) {
    return key16 < win || key16 > 65536u - win;
}

// (uint16)key for any input, via the fast path when possible.
__device__ __forceinline__ uint32_t key16_of(double v, const Prec &pc) {
    uint32_t idx; bool slow;
    fast_candidate(v, pc, idx, slow);
    if (slow) return exact_key16(v, pc.precision);
    return slot_to_key16(idx, pc.win);
}

// ---------------------------------------------------------------- flags
// Per-histogram flags (uint32[H], one array per bucket buffer): 0 = untouched since the buffer was cleared,
// 1 = counts inside the fast window only, 3 = some count outside it.  Every writer of the uint64 rows raises them;
// the snapshot kernels (reduce, export, clear, all-reduce) scan only what they cover.
// Plain read first: the flag is almost always already set, and same-address atomics from every thread would
// serialise in L2.
__device__ __forceinline__ void mark(uint32_t *flag, uint32_t level) {
    if ((*reinterpret_cast<volatile uint32_t *>(flag) & level) != level) atomicOr(flag, level);
}
// One count (or c of them) straight into the uint64 row of a histogram, raising its flag.
__device__ __forceinline__ void add_bucket_global(unsigned long long *__restrict__ row, uint32_t *flag, uint32_t key16,
                                                  unsigned long long c, uint32_t win) {
    atomicAdd(&row[key16], c);
    mark(flag, key16_in_window(key16, win) ? 1u : 3u);
}

// Shared sub-histogram of one histogram: [0, 2*win) slots + one trash slot that is never flushed (samples
// outside the window are counted straight into the global array and redirected there so that the shared atomic
// stays unconditional).
__host__ __device__ __forceinline__ uint32_t subhist_words(uint32_t win) { return 2u * win + 8u; }

// Flush: one 64-bit global atomic per non-empty slot, then one flag update per CTA.
__device__ __forceinline__ void flush_subhist(const uint32_t *hist, int tid, int nthreads,
                                              unsigned long long *__restrict__ counts, uint32_t *flag, uint32_t win) {
    int any = 0;
    for (uint32_t slot = tid; slot < 2u * win; slot += nthreads) {
        const uint32_t c = hist[slot];
        if (c) { atomicAdd(&counts[slot_to_key16(slot, win)], (unsigned long long)c); any = 1; }
    }
    any = __syncthreads_or(any);
    if (any && tid == 0) mark(flag, 1u);
}

// Exact slot of one sample for the fix-up paths; out-of-window keys are counted globally and sent to the trash slot.
__device__ __forceinline__ uint32_t fixup_slot(double v, const Prec &pc, unsigned long long *__restrict__ counts,
                                               uint32_t *flag) {
    const uint32_t key = key16_of(v, pc);
    uint32_t slot = key16_to_slot(key, pc.win);
    if (slot == 0xFFFFFFFFu) { add_bucket_global(counts, flag, key, 1ull, pc.win); slot = 2u * pc.win; }
    return slot;
}

// ================================================================ recording from CUDA code
// The recorder's precision block, as the library filled it (lh_record_begin copies the context's Prec into it).
__device__ __forceinline__ const Prec &recorder_prec(const lh_recorder &rec) {
    return *reinterpret_cast<const Prec *>(rec.prec);
}
__device__ __forceinline__ unsigned long long *recorder_row(const lh_recorder &rec, uint32_t id) {
    return reinterpret_cast<unsigned long long *>(rec.d_buckets) + (size_t)id * LH_KEYS_PER_HISTOGRAM;
}
__device__ __forceinline__ unsigned long long *recorder_dropped(const lh_recorder &rec) {
    return reinterpret_cast<unsigned long long *>(rec.d_dropped);
}
__device__ __forceinline__ uint32_t lane_id() {
    uint32_t l;
    asm("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}

// One sample of histogram `id` whose (uint16)key is already known: the body of record() after the bucket function.
// The lanes of a warp that arrive together are combined: lanes with the same (id, key) elect one leader, which adds
// their number with one 64-bit atomic.  An id >= max_histograms is dropped and counted in lh_stats.dropped.
__device__ __forceinline__ void record_key16(const lh_recorder &rec, uint32_t id, uint32_t key) {
    const bool ok = id < rec.max_histograms;
    const unsigned long long tag = ok ? ((unsigned long long)id << 16) | key : ~0ull;   // every dropped lane combines
    const uint32_t active = __activemask();
    const uint32_t peers = __match_any_sync(active, tag);
    if (lane_id() != (uint32_t)(__ffs(peers) - 1)) return;
    const unsigned long long c = (unsigned long long)__popc(peers);
    if (!ok) { atomicAdd(recorder_dropped(rec), c); return; }
    add_bucket_global(recorder_row(rec, id), rec.d_flags + id, key, c, recorder_prec(rec).win);
}

// Histogram(name, v): one sample of histogram `id`.  Callable from any thread under any divergence; lanes of a warp
// with the same (id, bucket) are combined as record_key16 describes.
__device__ __forceinline__ void record(const lh_recorder &rec, uint32_t id, double v) {
    record_key16(rec, id, key16_of(v, recorder_prec(rec)));
}

// TimerToken.Stop(): the value is float64(duration.Nanoseconds()), round-to-nearest-even as Go's CVTSQ2SD.
__device__ __forceinline__ void record_ns(const lh_recorder &rec, uint32_t id, long long ns) {
    record(rec, id, __ll2double_rn(ns));
}

// StartTimer(name) / TimerToken.Stop() (metrics.go:232-246) measured on the device.  The clock is %globaltimer, the
// GPU's nanosecond timer: it is NOT the host's steady_clock, and the timers of two GPUs are not synchronised, so a token
// is stopped on the GPU that started it.  A token is plain data: it may be written to memory and stopped by another
// thread or by a later kernel on the same GPU (queueing time between a producer and a consumer kernel).
// start_timer needs no recorder and may run before the scope opens; stop records, so it runs inside a scope.
struct TimerToken {
    uint64_t start_ns;
    uint32_t id;
    uint32_t pad;
};
static_assert(sizeof(TimerToken) == 16, "lh::TimerToken is 16 bytes of plain data");

__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ TimerToken start_timer(uint32_t id) {
    TimerToken t;
    t.start_ns = globaltimer_ns();
    t.id = id;
    t.pad = 0;
    return t;
}

// Records float64(now - start) under the token's id, as record_ns does, and returns the duration in ns (Go's Stop
// returns the time.Duration it recorded).
__device__ __forceinline__ long long stop(const lh_recorder &rec, const TimerToken &t) {
    const long long ns = (long long)(globaltimer_ns() - t.start_ns);
    record_ns(rec, t.id, ns);
    return ns;
}

// Counter(name, amount): one wrapping 64-bit add into the interval's counter delta.  An id >= max_counters is
// dropped and counted.
__device__ __forceinline__ void count(const lh_recorder &rec, uint32_t id, uint64_t amount) {
    if (id >= rec.max_counters) { atomicAdd(recorder_dropped(rec), 1ull); return; }
    atomicAdd(reinterpret_cast<unsigned long long *>(rec.d_counters) + id, (unsigned long long)amount);
}

__device__ __forceinline__ uint32_t block_thread_rank() {
    return threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
}
__device__ __forceinline__ uint32_t block_thread_count() { return blockDim.x * blockDim.y * blockDim.z; }

// One CTA feeding one histogram: samples are counted in a uint32 sub-histogram in shared memory (the arithmetic of
// the library's single-histogram kernel) and flushed into the histogram's row with one 64-bit atomic per non-empty
// bucket.  The caller provides rec.block_smem_bytes of shared memory (usually the kernel's dynamic shared memory).
//
//   __shared__ / extern __shared__ ... smem;
//   lh::BlockHistogram bh(rec, smem);
//   bh.init(id);            // every thread of the CTA
//   ... bh.add(v) ...       // any thread, any number of times
//   bh.flush();             // every thread of the CTA; init is not needed again before further adds
//
// Contract: at most 2^32 - 1 adds per CTA between two flushes (the shared cells are uint32).  When `id` is out of
// range every add is dropped and counted instead.
class BlockHistogram {
  public:
    __device__ __forceinline__ BlockHistogram(const lh_recorder &rec, void *smem)
        : rec_(rec), hist_(reinterpret_cast<uint32_t *>(smem)) {}

    // Binds histogram `id` and zeroes the sub-histogram.  The id is needed now: adds whose bucket lies outside the
    // shared window go straight into the histogram's row.
    __device__ __forceinline__ void init(uint32_t id) {
        ok_ = id < rec_.max_histograms;
        row_ = ok_ ? recorder_row(rec_, id) : nullptr;
        flag_ = ok_ ? rec_.d_flags + id : nullptr;
        const uint32_t words = subhist_words(recorder_prec(rec_).win);
        for (uint32_t i = block_thread_rank(); i < words; i += block_thread_count()) hist_[i] = 0;
        __syncthreads();
    }

    __device__ __forceinline__ void add(double v) {
        if (!ok_) {
            const uint32_t active = __activemask();
            if (lane_id() == (uint32_t)(__ffs(active) - 1)) atomicAdd(recorder_dropped(rec_), (unsigned long long)__popc(active));
            return;
        }
        const Prec &pc = recorder_prec(rec_);
        uint32_t idx; bool slow;
        fast_candidate(v, pc, idx, slow);
        if (slow) idx = fixup_slot(v, pc, row_, flag_);
        atomicAdd(&hist_[idx], 1u);
    }

    // Adds the sub-histogram into the row and zeroes it for the next adds.
    __device__ __forceinline__ void flush() {
        const uint32_t win = recorder_prec(rec_).win;
        __syncthreads();
        if (ok_) flush_subhist(hist_, (int)block_thread_rank(), (int)block_thread_count(), row_, flag_, win);
        else __syncthreads();
        for (uint32_t i = block_thread_rank(); i < 2u * win; i += block_thread_count()) hist_[i] = 0;
        __syncthreads();
    }

  private:
    const lh_recorder &rec_;
    uint32_t *hist_;
    unsigned long long *row_ = nullptr;
    uint32_t *flag_ = nullptr;
    bool ok_ = false;
};

// Any number of histograms from one CTA: a write-combining table in shared memory, keyed by the exact (id, bucket) of
// each sample and flushed into the interval's rows with one 64-bit atomic per occupied slot.  Where the CTA's distinct
// (id, bucket) pairs fit the table, a sample costs shared-memory atomics only (lh::record costs one global atomic per
// distinct (id, bucket) per warp call).  The caller provides BlockRecorder::smem_bytes(entries) bytes of shared memory,
// 8-byte aligned (usually the kernel's dynamic shared memory).
//
//   extern __shared__ __align__(16) unsigned char smem[];
//   lh::BlockRecorder br(rec, smem, entries);
//   br.init();                        // every thread of the CTA
//   ... br.record(id, v) ...          // Histogram(name, v): any thread, any id, any divergence
//   ... br.record_ns(id, ns) ...      // TimerToken.Stop(): float64(ns), as lh::record_ns
//   ... ns = br.stop(token) ...       // lh::stop through the table; returns the duration
//   br.flush();                       // every thread of the CTA; the table is empty afterwards and takes more records
//
// Table: `entries` rounded down to a power of two slots (no table below kMinEntries: every sample takes the direct
// path), each a 64-bit tag ((id << 16 | key) + 1; 0 = empty) and a uint32 count, 12 B per slot, tags first.  A sample
// probes at most kProbes consecutive slots from a multiplicative hash of its tag: a slot holding its tag is a hit, an
// empty one is claimed with one 64-bit shared CAS (which may find the same tag, claimed by another lane: a hit too),
// and a hit adds 1 to the slot's count.  A sample that finds neither goes straight into the row (record_key16, the
// path of lh::record).  So every sample lands on key16_of(v) of its id however full the table is; only the speed
// depends on it.  An id >= max_histograms is dropped and counted in lh_stats.dropped as by lh::record, and never
// enters the table.
//
// Contract: at most 2^32 - 1 records per CTA between two flushes (the counts are uint32).  The table lives only as long
// as the CTA: records after its last flush are lost, so every CTA ends with flush().  Above 48 KB of dynamic shared
// memory the kernel needs cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), as for
// BlockHistogram.
class BlockRecorder {
  public:
    static constexpr uint32_t kMinEntries = 32;
    static constexpr uint32_t kProbes = 8;      // slots a sample probes before it takes the direct path

    // Slots of a table asked for `entries`: the largest power of two <= entries, or 0 below kMinEntries.
    __host__ __device__ static constexpr uint32_t table_entries(uint32_t entries) {
        if (entries < kMinEntries) return 0;
        uint32_t p = kMinEntries;
        while (p <= entries / 2) p *= 2;
        return p;
    }
    // Shared memory for a table asked for `entries` (a table that fits a CTA has at most 2^14 slots).
    __host__ __device__ static constexpr uint32_t smem_bytes(uint32_t entries) { return 12u * table_entries(entries); }

    __device__ __forceinline__ BlockRecorder(const lh_recorder &rec, void *smem, uint32_t entries)
        : rec_(rec), n_(table_entries(entries)), tags_(reinterpret_cast<unsigned long long *>(smem)),
          counts_(reinterpret_cast<uint32_t *>(tags_ + n_)) {}

    // Empties the table.
    __device__ __forceinline__ void init() {
        for (uint32_t i = block_thread_rank(); i < n_; i += block_thread_count()) { tags_[i] = 0ull; counts_[i] = 0u; }
        __syncthreads();
    }

    __device__ __forceinline__ void record(uint32_t id, double v) {
        const uint32_t key = key16_of(v, recorder_prec(rec_));
        if (id < rec_.max_histograms && insert((((unsigned long long)id << 16) | key) + 1ull)) return;
        record_key16(rec_, id, key);
    }

    __device__ __forceinline__ void record_ns(uint32_t id, long long ns) { record(id, __ll2double_rn(ns)); }

    __device__ __forceinline__ long long stop(const TimerToken &t) {
        const long long ns = (long long)(globaltimer_ns() - t.start_ns);
        record_ns(t.id, ns);
        return ns;
    }

    // Adds every occupied slot's count into its row (raising the histogram's flag as every writer does) and empties
    // the table for the next records.
    __device__ __forceinline__ void flush() {
        const uint32_t win = recorder_prec(rec_).win;
        __syncthreads();
        for (uint32_t i = block_thread_rank(); i < n_; i += block_thread_count()) {
            const unsigned long long t = tags_[i];
            if (t) {
                const uint32_t id = (uint32_t)((t - 1ull) >> 16);
                add_bucket_global(recorder_row(rec_, id), rec_.d_flags + id, (uint32_t)(t - 1ull) & 0xFFFFu, counts_[i], win);
                tags_[i] = 0ull;
                counts_[i] = 0u;
            }
        }
        __syncthreads();
    }

  private:
    // true when the sample was counted in the table
    __device__ __forceinline__ bool insert(unsigned long long tag) {
        if (n_ == 0) return false;
        uint32_t s = (uint32_t)((tag * 0x9E3779B97F4A7C15ull) >> 32);
        for (uint32_t p = 0; p < kProbes; ++p, ++s) {
            const uint32_t i = s & (n_ - 1u);
            unsigned long long t = *reinterpret_cast<volatile unsigned long long *>(&tags_[i]);
            if (t == 0ull) t = atomicCAS(&tags_[i], 0ull, tag);
            if (t == 0ull || t == tag) { atomicAdd(&counts_[i], 1u); return true; }
        }
        return false;
    }

    const lh_recorder &rec_;
    uint32_t n_;
    unsigned long long *tags_;
    uint32_t *counts_;
};

// ================================================================ reading a device subscription (lh_board)
// A board (lh_board_create) holds the processed metrics of the latest collection that published into it: what the
// reference hands SubscribeToProcessedMetrics subscribers (metrics.go:508-525), for kernels and CUDA-graph replays.
//
//   lh::HistogramStats s;
//   if (lh::read_histogram(board, row, &s) && s.present && s.np > 2) clip = s.pvals[2];   // e.g. the p99 label
//
// Each read is a seqlock-consistent copy of one row: the sequence word is loaded with ld.acquire.gpu and retried while
// odd (a publish is writing), the row with strong relaxed loads, which go to L2 (a plain load could hit an L1 line that
// a persistent kernel cached before the latest publish), then fence.acq_rel.gpu and the word again: a changed word
// means the row may mix two publishes, and the read is retried.  A publish is one CTA that never waits on anything, so
// the retry loop ends as soon as it has run.  The value returned is the publish number the row belongs to (the number
// of publishes into the board so far), 0 if nothing has been published yet.  A kernel must not wait for the next
// publish: collections run on the host, which may never run another.
namespace board {
__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed(const void *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const void *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(void *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u32(void *p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

__device__ __forceinline__ char *hist_row(const lh_board &b, uint32_t row) {
    return (char *)b.d_board + sizeof(lh_board_header) + (size_t)row * sizeof(lh_board_hist_row);
}
__device__ __forceinline__ char *counter_row(const lh_board &b, uint32_t row) {
    return (char *)b.d_board + sizeof(lh_board_header) + (size_t)b.k * sizeof(lh_board_hist_row) +
           (size_t)row * sizeof(lh_board_counter_row);
}
// the even sequence word a consistent read starts from
__device__ __forceinline__ unsigned long long begin_read(const lh_board &b) {
    for (;;) {
        const unsigned long long s = ld_acquire((const unsigned long long *)b.d_board);
        if (!(s & 1ull)) return s;
        __nanosleep(64);
    }
}
// true when nothing was published while the loads before it ran
__device__ __forceinline__ bool end_read(const lh_board &b, unsigned long long s) {
    fence_acq_rel();
    return ld_relaxed(b.d_board) == s;
}
}  // namespace board

struct HistogramStats {          // one histogram row of the latest publish (lh_board_hist_row)
    uint64_t count;              // the name's _count (as uint64)
    double sum, avg;             // _sum, _avg
    bool present;                // the name was in that collection's Histograms: a non-empty bucket (count != 0 unless
                                 // the uint64 count wrapped to 0)
    uint32_t np;                 // percentile labels of that collection
    double pvals[LH_MAX_PERCENTILES];    // value of label j, j < np; NaN where pkeys[j] is INT32_MIN (label omitted)
    int32_t pkeys[LH_MAX_PERCENTILES];   // bucket key of label j
};
struct CounterStats {            // one counter row of the latest publish (lh_board_counter_row)
    uint64_t rate;               // the name's _rate: the interval delta
    uint64_t total;              // its running total (Counters[name]) as the publisher passed it
    bool present;                // the name was in that collection's Rates
};

// A consistent copy of histogram row `row` (< b.k) of board b; returns its publish number (0: nothing published yet,
// or row out of range: *out is then all zero).
__device__ __forceinline__ uint64_t read_histogram(const lh_board &b, uint32_t row, HistogramStats *out) {
    if (row >= b.k) { *out = HistogramStats{}; return 0; }
    const char *r = board::hist_row(b, row);
    for (;;) {
        const unsigned long long s = board::begin_read(b);
        out->np = board::ld_relaxed_u32((const char *)b.d_board + offsetof(lh_board_header, np));
        out->count = board::ld_relaxed(r + offsetof(lh_board_hist_row, count));
        out->sum = __longlong_as_double((long long)board::ld_relaxed(r + offsetof(lh_board_hist_row, sum)));
        out->avg = __longlong_as_double((long long)board::ld_relaxed(r + offsetof(lh_board_hist_row, avg)));
        out->present = board::ld_relaxed_u32(r + offsetof(lh_board_hist_row, present)) != 0;
#pragma unroll 8
        for (int j = 0; j < LH_MAX_PERCENTILES; j++)
            out->pvals[j] = __longlong_as_double((long long)board::ld_relaxed(r + offsetof(lh_board_hist_row, pvals) + 8 * j));
#pragma unroll 8
        for (int j = 0; j < LH_MAX_PERCENTILES; j += 2) {
            const unsigned long long two = board::ld_relaxed(r + offsetof(lh_board_hist_row, pkeys) + 4 * j);
            out->pkeys[j] = (int32_t)(uint32_t)two;
            out->pkeys[j + 1] = (int32_t)(uint32_t)(two >> 32);
        }
        if (board::end_read(b, s)) return s >> 1;
    }
}

// A consistent copy of counter row `row` (< b.kc) of board b; returns its publish number as read_histogram does.
__device__ __forceinline__ uint64_t read_counter(const lh_board &b, uint32_t row, CounterStats *out) {
    if (row >= b.kc) { *out = CounterStats{}; return 0; }
    const char *r = board::counter_row(b, row);
    for (;;) {
        const unsigned long long s = board::begin_read(b);
        out->rate = board::ld_relaxed(r + offsetof(lh_board_counter_row, rate));
        out->total = board::ld_relaxed(r + offsetof(lh_board_counter_row, total));
        out->present = board::ld_relaxed_u32(r + offsetof(lh_board_counter_row, present)) != 0;
        if (board::end_read(b, s)) return s >> 1;
    }
}

// ================================================================ querying a raw device subscription (lh_raw_board)
// A raw board (lh_raw_board_create) holds, per row, the running bucket counts of one histogram of the latest
// collection that published into it: the buckets the reference hands SubscribeToRawMetrics subscribers
// (metrics.go:508-525), for kernels and CUDA-graph replays.  Three exact queries, each one seqlock read of one row:
//
//   int32_t key; double v;
//   lh::raw_percentile(raw, row, p, &key, &v);        // p read at run time: the same (key, value) K3 gives for p
//   uint64_t below, total;
//   lh::raw_rank(raw, row, budget, &below, &total);   // samples in buckets at or below budget's bucket
//
// A read is the protocol of lh::read_histogram applied to the row's own sequence word: ld.acquire.gpu of the word
// (retried while odd), the header and the cells the query needs with strong relaxed loads, fence.acq_rel.gpu, and the
// word again; a changed word retries the query.  A row is written by one CTA of k_raw_publish that waits on nothing,
// so the retry loop ends as soon as that CTA has run.  Each query returns the publish number its answer comes from
// (0 before the first publish, or for a row >= b.k, which answers as an empty row).  A kernel must not wait for the
// next publish: collections run on the host, which may never run another.

// Smallest s in [0, total] with float64(s)/float64(total) >= p -- the reference's rule (metrics.go:413) turned into an
// integer threshold on the running count: the quotient is monotone in s, so "first non-empty bucket whose running count
// satisfies the rule" == "first non-empty bucket whose running count reaches T".  Returns false when no s in
// [0, total] satisfies the rule (p > 1 or NaN).  That settles percentile() only while the running counts are exact:
// once Go's uint64 running count wraps (counts summing to 2^64 or more) it is not monotone, can exceed the wrapped
// total (ratios above 1, so p > 1 may answer) and the total may be 0 (ratios +Inf, or NaN at 0), and callers apply the
// rule to every non-empty bucket instead.
__device__ __forceinline__ bool percentile_threshold(double p, unsigned long long total, unsigned long long *T) {
    const double ft = (double)total;
    if (!(__ddiv_rn(ft, ft) >= p)) return false;                 // even s = total fails (p > 1, NaN)
    auto ok = [&](unsigned long long s) { return __ddiv_rn((double)s, ft) >= p; };
    unsigned long long s = 0;
    if (p > 0.0) {
        const double est = ceil(p * ft);
        s = est >= ft ? total : (unsigned long long)est;
    }
    int steps = 0;
    while (s > 0 && ok(s - 1) && steps < 8) { s--; steps++; }
    while (!ok(s) && steps < 16) { s++; steps++; }
    if (steps >= 8 && (!ok(s) || (s > 0 && ok(s - 1)))) {        // long plateaus of float64(s) (totals beyond 2^53): bisection
        unsigned long long lo = 0, hi = total;                  // ok(hi) holds
        while (lo < hi) { const unsigned long long mid = lo + (hi - lo) / 2; if (ok(mid)) hi = mid; else lo = mid + 1; }
        s = lo;
    }
    *T = s;
    return true;
}

namespace raw {
__device__ __forceinline__ const char *header(const lh_raw_board &b, uint32_t row) {
    return (const char *)b.d_rows + (size_t)row * sizeof(lh_raw_row_header);
}
// cell key + 32768 of the row: running count at key
__device__ __forceinline__ const char *cells(const lh_raw_board &b, uint32_t row) {
    return (const char *)b.d_rows + LH_RAW_CELLS_OFFSET(b.k) + (size_t)row * (65536u * 8u);
}
__device__ __forceinline__ unsigned long long begin_read(const char *h) {
    for (;;) {
        const unsigned long long s = board::ld_acquire((const unsigned long long *)h);
        if (!(s & 1ull)) return s;
        __nanosleep(64);
    }
}
__device__ __forceinline__ bool end_read(const char *h, unsigned long long s) {
    board::fence_acq_rel();
    return board::ld_relaxed(h) == s;
}
struct Range {
    unsigned long long total;
    int lo, hi;                  // written keys; lo > hi: empty
    bool wrapped;                // a running count passed 2^64 (key_hi was stored + LH_RAW_KEY_WRAPPED)
};
__device__ __forceinline__ Range range(const char *h) {
    const unsigned long long two = board::ld_relaxed(h + offsetof(lh_raw_row_header, key_lo));
    const int hi = (int)(uint32_t)(two >> 32);
    const bool wrapped = hi > 32767;
    return Range{board::ld_relaxed(h + offsetof(lh_raw_row_header, total)), (int)(uint32_t)two,
                 wrapped ? hi - LH_RAW_KEY_WRAPPED : hi, wrapped};
}
// running count at key: 0 below the written range, total above it
__device__ __forceinline__ unsigned long long running(const char *c, const Range &r, int key) {
    if (key < r.lo) return 0ull;
    if (key > r.hi) return r.total;
    return board::ld_relaxed(c + (size_t)(key + 32768) * 8u);
}
}  // namespace raw

// (key, value) of percentile p of row `row`: bit for bit what lh_snapshot_reduce reports for the row's histogram with
// that p.  INT32_MIN / NaN where no bucket satisfies the rule (p > 1 unless the running counts wrapped, NaN, an empty
// row); p <= 0 gives the smallest non-empty key.  A row whose running counts wrapped is answered by a linear scan of
// its written keys.
__device__ __forceinline__ uint64_t raw_percentile(const lh_raw_board &b, uint32_t row, double p, int32_t *key, double *val) {
    *key = (int32_t)0x80000000;
    *val = __longlong_as_double(0x7FF8000000000000ll);
    if (row >= b.k) return 0;
    const char *h = raw::header(b, row), *c = raw::cells(b, row);
    for (;;) {
        const unsigned long long s = raw::begin_read(h);
        const raw::Range r = raw::range(h);
        unsigned long long T;
        bool found = false;
        int lo = r.lo, hi = r.hi;
        if (r.wrapped) {                                          // Go's rule on each non-empty bucket, in key order
            const double ft = (double)r.total;
            unsigned long long prev = 0;
            for (int k = lo; k <= hi; k++) {
                const unsigned long long run = board::ld_relaxed(c + (size_t)(k + 32768) * 8u);
                if (run != prev && __ddiv_rn((double)run, ft) >= p) { lo = k; found = true; break; }
                prev = run;
            }
        } else if (r.total && lo <= hi && percentile_threshold(p, r.total, &T)) {
            if (T == 0) T = 1;                                    // p <= 0: the smallest non-empty bucket
            while (lo < hi) {                                     // running(hi) == total >= T
                const int mid = lo + ((hi - lo) >> 1);
                if (board::ld_relaxed(c + (size_t)(mid + 32768) * 8u) >= T) hi = mid; else lo = mid + 1;
            }
            found = true;
        }
        if (raw::end_read(h, s)) {
            if (found) {
                *key = lo;
                *val = b.d_decomp[(uint32_t)lo & 0xFFFFu];
            }
            return s >> 1;
        }
    }
}

// Samples of row `row` whose bucket key is <= the key lh::record gives v (NaN and +-Inf: key 0), and the row's total.
__device__ __forceinline__ uint64_t raw_rank(const lh_raw_board &b, uint32_t row, double v, uint64_t *rank, uint64_t *total) {
    *rank = 0;
    *total = 0;
    if (row >= b.k) return 0;
    const int key = (int)(int16_t)(uint16_t)key16_of(v, *reinterpret_cast<const Prec *>(b.prec));
    const char *h = raw::header(b, row), *c = raw::cells(b, row);
    for (;;) {
        const unsigned long long s = raw::begin_read(h);
        const raw::Range r = raw::range(h);
        const unsigned long long n = raw::running(c, r, key);
        if (raw::end_read(h, s)) {
            *rank = n;
            *total = r.total;
            return s >> 1;
        }
    }
}

// Samples of row `row` in bucket `key` (0 for a key with none, or outside int16).
__device__ __forceinline__ uint64_t raw_bucket_count(const lh_raw_board &b, uint32_t row, int32_t key, uint64_t *count) {
    *count = 0;
    if (row >= b.k) return 0;
    const char *h = raw::header(b, row), *c = raw::cells(b, row);
    for (;;) {
        const unsigned long long s = raw::begin_read(h);
        const raw::Range r = raw::range(h);
        const unsigned long long n = key < -32768 || key > 32767 ? 0ull
                                   : raw::running(c, r, key) - raw::running(c, r, key - 1);
        if (raw::end_read(h, s)) {
            *count = n;
            return s >> 1;
        }
    }
}

// ================================================================ writing a device gauge (lh_gauges_read)
// A device gauge (MetricSystem::RegisterDeviceGauge) is a scalar in device memory that every collection reads with one
// naturally aligned strong load (ld.relaxed.gpu).  The PTX memory model promises an untorn read only against a strong
// store of the same size, which is what lh::set_gauge issues (st.relaxed.gpu):
//
//   lh::set_gauge(d_loss, loss);     // T = double, float, __half, __nv_bfloat16, int64_t, int32_t or uint64_t
//
// Plain aligned stores of one value -- what torch's fill_ / copy_ kernels emit -- are single instructions of the same
// width on sm_90 and are read whole in practice (tests/test_gpu_device_gauges.py checks both), but only set_gauge is
// covered by the memory model.  T must be one of the seven gauge types, matching the dtype registered for p.
namespace gauge_store {
template <int N> struct bits;
template <> struct bits<2> { typedef unsigned short type; };
template <> struct bits<4> { typedef unsigned int type; };
template <> struct bits<8> { typedef unsigned long long type; };
__device__ __forceinline__ void st(void *p, unsigned short u) {
    asm volatile("st.relaxed.gpu.b16 [%0], %1;" :: "l"(p), "h"(u) : "memory");
}
__device__ __forceinline__ void st(void *p, unsigned int u) {
    asm volatile("st.relaxed.gpu.b32 [%0], %1;" :: "l"(p), "r"(u) : "memory");
}
__device__ __forceinline__ void st(void *p, unsigned long long u) {
    asm volatile("st.relaxed.gpu.b64 [%0], %1;" :: "l"(p), "l"(u) : "memory");
}
}  // namespace gauge_store

template <typename T>
__device__ __forceinline__ void set_gauge(T *p, T v) {
    static_assert(sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "a gauge is a 2-, 4- or 8-byte scalar");
    typename gauge_store::bits<(int)sizeof(T)>::type u;
    __builtin_memcpy(&u, &v, sizeof u);
    gauge_store::st(p, u);
}

}  // namespace lh
