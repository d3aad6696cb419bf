/*
 * loghisto_oracle.c -- CPU restatement of the spacejam/loghisto hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, the smoke()
 * entry in __graft_entry__.py and bench.py's cpu_baseline / --impl reference
 * legs may load it.  The product (loghisto_b200/) never links or calls it.
 *
 * What it restates (all citations are <file>:<line> in the reference repository):
 *   compress            metrics.go:316-322   (precision = 100, metrics.go:40-43)
 *   decompress          metrics.go:326-332
 *   Histogram ingest    metrics.go:273-295   (dense uint64[65536] indexed by (uint16)key)
 *   Counter ingest      metrics.go:251-269
 *   processHistograms   metrics.go:336-387   (count / sum / avg / percentiles / agg store)
 *   percentile          metrics.go:406-418
 *   collectRawMetrics   metrics.go:420-479   (interval-delta semantics)
 *   processMetrics      metrics.go:483-506
 *   reaper _agg_*       metrics.go:590-608
 *
 * Arithmetic that lives OUTSIDE the reference tree (Go standard library, not
 * vendored, no go.mod; .travis.yml:3-5 pins only "Go 1.4 and tip"):
 *   math.Log  -- src/math/log.go (port of FreeBSD e_log.c).  On amd64 the Go
 *                tree also carries log_amd64.s; it evaluates the very same
 *                expression tree with scalar SSE2 ops (one rounding per op, no
 *                FMA), so for x >= 1 (the only inputs compress() produces) the
 *                two are bit-identical.  Restated here op-for-op.
 *   math.Exp  -- on amd64 Go uses exp_amd64.s (Shibata/SLEEF-style: reduce by
 *                ln2, scale by 1/16, degree-8 Taylor for e^x-1, four
 *                (x+2)*x squarings).  Restated as lho_go_exp(); the pure-Go
 *                src/math/exp.go (FreeBSD e_exp.c) is lho_go_exp_purego().
 *                The 15 full-precision decompress() outputs printed by real Go
 *                runs (readme.md:35-43, print_benchmark.go:34-39) pin which
 *                one the reference used; see tests/test_oracle_kat.py.
 *   float64 -> int16 conversion on amd64: CVTTSD2SL then keep the low 16 bits
 *                (out-of-range / NaN -> 0x80000000 -> 0).
 *   float64 -> uint64 (metrics.go:374): CVTTSD2SQ for x < 2^63 (negative
 *                values wrap two's-complement), subtract-2^63 path above.
 *
 * Reference platform for every parity claim: amd64, GOAMD64=v1 (no FMA
 * contraction), so this file MUST be compiled with -ffp-contract=off and
 * without -ffast-math (see oracle/Makefile).
 */
#define _GNU_SOURCE
#include <math.h>
#include <pthread.h>
#include <semaphore.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#if defined(__FAST_MATH__)
#error "the oracle must not be built with -ffast-math"
#endif

#define LHO_EXPORT __attribute__((visibility("default")))

static inline double bits_to_f64(uint64_t b) { double d; memcpy(&d, &b, 8); return d; }
static inline uint64_t f64_to_bits(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }

/* ------------------------------------------------------------------ */
/* math.Frexp (src/math/frexp.go): frac in [0.5,1), x = frac * 2^exp.   */
static double go_frexp(double f, int *e) {
    if (f == 0 || isinf(f) || isnan(f)) { *e = 0; return f; }
    int ex = 0;
    if (fabs(f) < 2.2250738585072014e-308) { /* normalize subnormal */
        f *= 4503599627370496.0; /* 2^52 */
        ex = -52;
    }
    uint64_t x = f64_to_bits(f);
    ex += (int)((x >> 52) & 0x7FF) - 1022;
    x &= ~((uint64_t)0x7FF << 52);
    x |= (uint64_t)1022 << 52;
    *e = ex;
    return bits_to_f64(x);
}

/* math.Log, src/math/log.go (== log_amd64.s for normal inputs). */
LHO_EXPORT double lho_go_log(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01; /* 3fe62e42 fee00000 */
    const double Ln2Lo = 1.90821492927058770002e-10; /* 3dea39ef 35793c76 */
    const double L1 = 6.666666666666735130e-01;      /* 3FE55555 55555593 */
    const double L2 = 3.999999999940941908e-01;      /* 3FD99999 9997FA04 */
    const double L3 = 2.857142874366239149e-01;      /* 3FD24924 94229359 */
    const double L4 = 2.222219843214978396e-01;      /* 3FCC71C5 1D8E78AF */
    const double L5 = 1.818357216161805012e-01;      /* 3FC74664 96CB03DE */
    const double L6 = 1.531383769920937332e-01;      /* 3FC39A09 D078C69F */
    const double L7 = 1.479819860511658591e-01;      /* 3FC2F112 DF3E5244 */
    const double HalfSqrt2 = 7.07106781186547524401e-01;

    if (isnan(x) || (isinf(x) && x > 0)) return x;
    if (x < 0) return NAN;
    if (x == 0) return -INFINITY;

    int ki;
    double f1 = go_frexp(x, &ki);
    if (f1 < HalfSqrt2) { f1 *= 2; ki--; }
    double f = f1 - 1;
    double k = (double)ki;

    double s = f / (2 + f);
    double s2 = s * s;
    double s4 = s2 * s2;
    double t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)));
    double t2 = s4 * (L2 + s4 * (L4 + s4 * L6));
    double R = t1 + t2;
    double hfsq = 0.5 * f * f;
    return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f);
}

/* math.Ldexp restricted to what exp needs (normal results + over/underflow). */
static double go_ldexp(double frac, int e) { return ldexp(frac, e); }

/* math.Exp, pure Go (src/math/exp.go, FreeBSD e_exp.c). */
LHO_EXPORT double lho_go_exp_purego(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01;
    const double Ln2Lo = 1.90821492927058770002e-10;
    const double Log2e = 1.44269504088896338700e+00;
    const double Overflow = 7.09782712893383973096e+02;
    const double Underflow = -7.45133219101941108420e+02;
    const double NearZero = 1.0 / (double)(1 << 28);
    const double P1 = 1.66666666666666657415e-01;
    const double P2 = -2.77777777770155933842e-03;
    const double P3 = 6.61375632143793436117e-05;
    const double P4 = -1.65339022054652515390e-06;
    const double P5 = 4.13813679705723846039e-08;

    if (isnan(x) || (isinf(x) && x > 0)) return x;
    if (isinf(x)) return 0;
    if (x > Overflow) return INFINITY;
    if (x < Underflow) return 0;
    if (-NearZero < x && x < NearZero) return 1 + x;

    int k = 0;
    if (x < 0) k = (int)(Log2e * x - 0.5);
    else if (x > 0) k = (int)(Log2e * x + 0.5);
    double hi = x - (double)k * Ln2Hi;
    double lo = (double)k * Ln2Lo;

    double r = hi - lo;
    double t = r * r;
    double c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
    double y = 1 - ((lo - (r * c) / (2 - c)) - hi);
    return go_ldexp(y, k);
}

/* math.Exp as amd64 Go computes it (src/math/exp_amd64.s, non-FMA path). */
LHO_EXPORT double lho_go_exp(double x) {
    const double LOG2E = 1.4426950408889634073599246810018920;
    const double LN2U = 0.69314718055966295651160180568695068359375;
    const double LN2L = 0.28235290563031577122588448175013436025525412068e-12;
    const double T1 = 0.5;
    const double T2 = 1.6666666666666666667e-1;
    const double T3 = 4.1666666666666666667e-2;
    const double T4 = 8.3333333333333333333e-3;
    const double T5 = 1.3888888888888888889e-3;
    const double T6 = 1.9841269841269841270e-4;
    const double T7 = 2.4801587301587301587e-5;

    if (isnan(x)) return x;
    if (isinf(x)) return x > 0 ? x : 0.0;
    if (x > 7.09782712893384e+02) return INFINITY;

    double q = LOG2E * x;
    /* CVTSD2SL: round to nearest even under the default MXCSR. */
    long e = lrint(q);
    double ef = (double)e;
    double r = x - ef * LN2U;
    r = r - ef * LN2L;
    r = r * 0.0625;
    double p = T7;
    p = p * r + T6;
    p = p * r + T5;
    p = p * r + T4;
    p = p * r + T3;
    p = p * r + T2;
    p = p * r + T1;
    p = p * r + 1.0;
    r = r * p;          /* e^r - 1 */
    r = r * (r + 2.0);  /* four squarings undo the /16 */
    r = r * (r + 2.0);
    r = r * (r + 2.0);
    r = r * (r + 2.0);
    r = r + 1.0;
    long be = e + 0x3FF;
    if (be <= 0) return 0.0;
    if (be >= 0x7FF) return INFINITY;
    return r * bits_to_f64((uint64_t)be << 52);
}

/* amd64 float64 -> int32 (CVTTSD2SL): truncation, "integer indefinite" on NaN/overflow. */
static inline int32_t amd64_cvttsd2sl(double t) {
    if (!(t > -2147483649.0 && t < 2147483648.0)) return (int32_t)0x80000000u;
    return (int32_t)t;
}

/* compress, metrics.go:316-322, with the package constant `precision` (metrics.go:40-43, 100 in the reference)
 * as a parameter: i := int16(precision*math.Log(1.0+math.Abs(value)) + 0.5). */
LHO_EXPORT int16_t lho_compress_p(double value, double precision) {
    double t = precision * lho_go_log(1.0 + fabs(value)) + 0.5;
    int16_t i = (int16_t)(uint16_t)(uint32_t)amd64_cvttsd2sl(t);
    if (value < 0) return (int16_t)(uint16_t)(0u - (uint16_t)i); /* -1*i, wraps */
    return i;
}
LHO_EXPORT int16_t lho_compress(double value) { return lho_compress_p(value, 100.0); }

/* decompress, metrics.go:326-332: math.Exp(math.Abs(float64(compressedValue))/precision) - 1. */
LHO_EXPORT double lho_decompress_p(int16_t k, double precision) {
    double f = lho_go_exp(fabs((double)k) / precision) - 1.0;
    if (k < 0) return -1.0 * f;
    return f;
}
LHO_EXPORT double lho_decompress(int16_t k) { return lho_decompress_p(k, 100.0); }

LHO_EXPORT double lho_decompress_purego(int16_t k) {
    double f = lho_go_exp_purego(fabs((double)k) / 100.0) - 1.0;
    if (k < 0) return -1.0 * f;
    return f;
}

/* amd64 float64 -> uint64 as the Go compiler lowers it (metrics.go:374). */
LHO_EXPORT uint64_t lho_go_f64_to_u64(double x) {
    if (x < 9223372036854775808.0) {
        if (!(x > -9223372036854777856.0)) return 0x8000000000000000ull; /* indefinite */
        return (uint64_t)(int64_t)x;
    }
    if (!(x < 18446744073709551616.0)) return 0; /* indefinite ^ sign bit */
    return (uint64_t)(int64_t)(x - 9223372036854775808.0) ^ 0x8000000000000000ull;
}

/* ------------------------------------------------------------------ */
/* Dense ingest: counts[(uint16)key] += 1.  metrics.go:273-295 minus maps. */
LHO_EXPORT void lho_ingest(const double *v, size_t n, uint64_t *counts65536) {
    for (size_t i = 0; i < n; i++) counts65536[(uint16_t)lho_compress(v[i])]++;
}

LHO_EXPORT void lho_compress_many(const double *v, size_t n, int16_t *out) {
    for (size_t i = 0; i < n; i++) out[i] = lho_compress(v[i]);
}
LHO_EXPORT void lho_compress_many_p(const double *v, size_t n, int16_t *out, double precision) {
    for (size_t i = 0; i < n; i++) out[i] = lho_compress_p(v[i], precision);
}
LHO_EXPORT void lho_ingest_p(const double *v, size_t n, uint64_t *counts65536, double precision) {
    for (size_t i = 0; i < n; i++) counts65536[(uint16_t)lho_compress_p(v[i], precision)]++;
}

LHO_EXPORT void lho_ingest_keyed(const uint32_t *ids, const double *v, size_t n,
                                 uint64_t *counts /* [H][65536] */) {
    for (size_t i = 0; i < n; i++)
        counts[(size_t)ids[i] * 65536u + (uint16_t)lho_compress(v[i])]++;
}

LHO_EXPORT void lho_ingest_keyed_u16(const uint16_t *ids, const double *v, size_t n,
                                     uint64_t *counts /* [H][65536] */) {
    for (size_t i = 0; i < n; i++)
        counts[(size_t)ids[i] * 65536u + (uint16_t)lho_compress(v[i])]++;
}

/* Timer samples: Histogram(name, float64(duration.Nanoseconds())), metrics.go:242-246. */
LHO_EXPORT void lho_ingest_keyed_i64(const uint32_t *ids, const int64_t *ns, size_t n,
                                     uint64_t *counts) {
    for (size_t i = 0; i < n; i++)
        counts[(size_t)ids[i] * 65536u + (uint16_t)lho_compress((double)ns[i])]++;
}

/* Counter(name, amount), metrics.go:251-269: wrapping uint64 add. */
LHO_EXPORT void lho_counter_add(const uint32_t *ids, const uint64_t *amounts, size_t n,
                                uint64_t *counters) {
    for (size_t i = 0; i < n; i++) counters[ids[i]] += amounts[i];
}

/*
 * processHistograms + percentile (metrics.go:336-356, 378-385, 406-418) on one
 * dense histogram.  Go iterates its map in random order; the oracle visits
 * non-empty buckets in ascending key order (== ascending decompressed value,
 * which is also the order percentile() sorts into), so `sum` matches the
 * reference only up to FP64 re-association (tests use 1e-12 relative).
 *
 *   ps[np]        requested percentiles
 *   out_stats[3]  count, sum, avg      (as float64, like the Go map values)
 *   out_pvals[np] percentile values; NaN where percentile() returns its error
 *   out_pkeys[np] chosen bucket keys;  INT32_MIN where percentile() errors
 * Returns the exact uint64 total count.
 */
LHO_EXPORT uint64_t lho_process_histogram_p(const uint64_t *counts65536, const double *ps, int np,
                                            double *out_stats, double *out_pvals, int32_t *out_pkeys, double precision);
LHO_EXPORT uint64_t lho_process_histogram(const uint64_t *counts65536, const double *ps, int np,
                                          double *out_stats, double *out_pvals,
                                          int32_t *out_pkeys) {
    return lho_process_histogram_p(counts65536, ps, np, out_stats, out_pvals, out_pkeys, 100.0);
}
LHO_EXPORT uint64_t lho_process_histogram_p(const uint64_t *counts65536, const double *ps, int np,
                                            double *out_stats, double *out_pvals, int32_t *out_pkeys, double precision) {
    double total_sum = 0.0;
    uint64_t total_count = 0;
    for (int key = -32768; key <= 32767; key++) {
        uint64_t c = counts65536[(uint16_t)(int16_t)key];
        if (!c) continue;
        total_sum += lho_decompress_p((int16_t)key, precision) * (double)c;
        total_count += c;
    }
    out_stats[0] = (double)total_count;
    out_stats[1] = total_sum;
    out_stats[2] = total_sum / (double)total_count;
    for (int j = 0; j < np; j++) {
        out_pvals[j] = NAN;
        out_pkeys[j] = INT32_MIN;
        uint64_t sofar = 0;
        for (int key = -32768; key <= 32767; key++) {
            uint64_t c = counts65536[(uint16_t)(int16_t)key];
            if (!c) continue;
            sofar += c;
            if ((double)sofar / (double)total_count >= ps[j]) {
                out_pvals[j] = lho_decompress_p((int16_t)key, precision);
                out_pkeys[j] = key;
                break;
            }
        }
    }
    return total_count;
}

/* percentile() on explicit (value,count) pairs, for TestPercentile (metrics_test.go:111-149).
 * Returns 0 and writes *out on success, -1 on "Invalid percentile". */
typedef struct { double value; uint64_t count; } lho_proportion;
static int cmp_prop(const void *a, const void *b) {
    double x = ((const lho_proportion *)a)->value, y = ((const lho_proportion *)b)->value;
    return (x < y) ? -1 : (x > y) ? 1 : 0;
}
LHO_EXPORT int lho_percentile(uint64_t total, const double *values, const uint64_t *counts,
                              int n, double p, double *out) {
    lho_proportion *arr = (lho_proportion *)malloc(sizeof(lho_proportion) * (size_t)(n ? n : 1));
    for (int i = 0; i < n; i++) { arr[i].value = values[i]; arr[i].count = counts[i]; }
    qsort(arr, (size_t)n, sizeof(lho_proportion), cmp_prop);
    uint64_t sofar = 0;
    int rc = -1;
    for (int i = 0; i < n; i++) {
        sofar += arr[i].count;
        if ((double)sofar / (double)total >= p) { *out = arr[i].value; rc = 0; break; }
    }
    free(arr);
    return rc;
}

/* ------------------------------------------------------------------ */
/* Synthetic streams (SURVEY.md section 8d): integer-only generators so CPU and
 * GPU produce identical bits.  u_i = splitmix64(seed + i). */
static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

/* 16-entry exponent table for stream L: triangular weights over 2^17..2^24 ns. */
static const uint8_t kStreamLExp[16] = {17, 18, 18, 19, 19, 19, 20, 20, 20, 20, 21, 21, 21, 22, 22, 23};

LHO_EXPORT uint64_t lho_stream_bits(int kind, uint64_t seed, uint64_t i) {
    uint64_t u = splitmix64(seed + i);
    uint64_t mant = u & 0x000FFFFFFFFFFFFFull;
    switch (kind) {
    case 0: /* U: log-uniform over [1, 2^63) */
        return ((uint64_t)(1023 + (u >> 52) % 63) << 52) | mant;
    case 1: /* L: latency-like, clustered */
        return ((uint64_t)(1023 + kStreamLExp[(u >> 52) & 15]) << 52) | mant;
    case 2: { /* S: signed / edge mix */
        uint32_t sel = (uint32_t)(u >> 52) & 0xFFF;
        if (sel < 41) { /* ~1% negatives of U-type magnitude */
            return 0x8000000000000000ull | ((uint64_t)(1023 + (u >> 40) % 63) << 52) | mant;
        }
        if (sel < 60) { /* raw bit patterns: NaN/Inf/subnormal/huge all occur */
            return splitmix64(u);
        }
        if (sel < 80) { /* small magnitudes around the 0.005 / 0.51 region, both signs */
            return ((u >> 11) & 0x8000000000000000ull) | ((uint64_t)(1023 - 10 + (u >> 40) % 12) << 52) | mant;
        }
        if (sel < 90) { /* huge: exponents up to the top, wraps int16 */
            return ((u >> 13) & 0x8000000000000000ull) | ((uint64_t)(1023 + 63 + (u >> 40) % 961) << 52) | mant;
        }
        return ((uint64_t)(1023 + (u >> 40) % 63) << 52) | mant;
    }
    case 3: /* C: constant (degenerate heavy hitter) */
        return 0x40F86A0000000000ull; /* 100000.0 */
    case 4: { /* Z: 50% one bucket, rest L-like */
        if (u >> 63) return 0x40F86A0000000000ull;
        return ((uint64_t)(1023 + kStreamLExp[(u >> 52) & 15]) << 52) | mant;
    }
    case 6: { /* T: timer durations as int64 nanoseconds (bit pattern of an int64): the L stream truncated */
        double d = bits_to_f64(((uint64_t)(1023 + kStreamLExp[(u >> 52) & 15]) << 52) | mant);
        return (uint64_t)(int64_t)d;
    }
    case 7: /* A: counter amounts 1..16 */
        return 1 + (u >> 60);
    case 8: /* N: stream U with a random sign (50 % negative durations, readme.md:43) */
        return ((u >> 11) & 0x8000000000000000ull) | ((uint64_t)(1023 + (u >> 52) % 63) << 52) | mant;
    default:
        return u;
    }
}

LHO_EXPORT void lho_gen_stream(int kind, uint64_t seed, uint64_t start, size_t n, double *out) {
    for (size_t i = 0; i < n; i++) out[i] = bits_to_f64(lho_stream_bits(kind, seed, start + i));
}

/* ids: kind 0 uniform over H, kind 1 "Zipf-ish" = min of two draws. */
LHO_EXPORT void lho_gen_ids(int kind, uint64_t seed, uint64_t start, size_t n, uint32_t H,
                            uint32_t *out) {
    for (size_t i = 0; i < n; i++) {
        uint64_t u = splitmix64((seed ^ 0xA5A5A5A5DEADBEEFull) + start + i);
        uint32_t a = (uint32_t)((u & 0xFFFFFFFFu) % H), b = (uint32_t)((u >> 32) % H);
        out[i] = kind == 0 ? a : (a < b ? a : b);
    }
}

/* ------------------------------------------------------------------ */
/* Multi-threaded dense ingest ("best-case CPU", BASELINE.md B2): private
 * uint64[65536] per thread, merged at the end. */
typedef struct {
    const double *v; size_t n; uint64_t *counts;
} dense_job;
static void *dense_worker(void *p) {
    dense_job *j = (dense_job *)p;
    lho_ingest(j->v, j->n, j->counts);
    return NULL;
}
LHO_EXPORT void lho_ingest_mt(const double *v, size_t n, uint64_t *counts65536, int threads) {
    if (threads < 1) threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    dense_job *jobs = (dense_job *)malloc(sizeof(dense_job) * (size_t)threads);
    size_t per = n / (size_t)threads;
    for (int t = 0; t < threads; t++) {
        jobs[t].v = v + per * (size_t)t;
        jobs[t].n = (t == threads - 1) ? n - per * (size_t)t : per;
        jobs[t].counts = (uint64_t *)calloc(65536, 8);
        pthread_create(&th[t], NULL, dense_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) {
        pthread_join(th[t], NULL);
        for (int k = 0; k < 65536; k++) counts65536[k] += jobs[t].counts[k];
        free(jobs[t].counts);
    }
    free(th); free(jobs);
}

/* ------------------------------------------------------------------ */
/* Streaming full-size checkers: regenerate the synthetic stream slab by slab on every host core and bucket it on
 * the fly (no sample array is ever materialised), so that bench.py and the tests can compare a 1e9 / 1e10-sample
 * device run bucket for bucket.  Same compress(), same generators as above.
 *   single:  counts65536[(uint16)compress(stream(val_kind, val_start + i))] += 1          (metrics.go:273-295)
 *   keyed:   counts[id_i][...] += 1 with id_i = ids(id_kind, ids_start + i) % H; as_i64 != 0 treats the stream bits
 *            as int64 nanoseconds converted like TimerToken.Stop does (metrics.go:242-246)
 *   counter: counters[id_i] += amount_i (wrapping)                                         (metrics.go:251-269)
 * Keyed/counter workers add into the shared arrays with relaxed atomics (integer adds commute). */
typedef struct {
    int mode;            /* 0 single, 1 keyed, 2 counter */
    int val_kind, id_kind, as_i64;
    uint64_t seed, val_start, ids_start;
    size_t n;
    uint32_t H;
    uint64_t *out;       /* single: private [65536]; keyed: shared [H][65536]; counter: shared [H] */
} stream_job;

static inline uint32_t stream_id(int kind, uint64_t seed, uint64_t i, uint32_t H) {
    uint64_t u = splitmix64((seed ^ 0xA5A5A5A5DEADBEEFull) + i);
    uint32_t a = (uint32_t)((u & 0xFFFFFFFFu) % H), b = (uint32_t)((u >> 32) % H);
    return kind == 0 ? a : (a < b ? a : b);
}

static void *stream_worker(void *p) {
    stream_job *j = (stream_job *)p;
    for (size_t i = 0; i < j->n; i++) {
        uint64_t bits = lho_stream_bits(j->val_kind, j->seed, j->val_start + i);
        if (j->mode == 0) {
            j->out[(uint16_t)lho_compress(bits_to_f64(bits))]++;
            continue;
        }
        uint32_t id = stream_id(j->id_kind, j->seed, j->ids_start + i, j->H);
        if (j->mode == 1) {
            double v = j->as_i64 ? (double)(int64_t)bits : bits_to_f64(bits);
            __atomic_fetch_add(&j->out[(size_t)id * 65536u + (uint16_t)lho_compress(v)], 1, __ATOMIC_RELAXED);
        } else {
            __atomic_fetch_add(&j->out[id], bits, __ATOMIC_RELAXED);
        }
    }
    return NULL;
}

static void stream_run(stream_job proto, uint64_t *out, int threads) {
    if (threads < 1) threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    stream_job *jobs = (stream_job *)malloc(sizeof(stream_job) * (size_t)threads);
    size_t per = proto.n / (size_t)threads;
    for (int t = 0; t < threads; t++) {
        jobs[t] = proto;
        jobs[t].val_start = proto.val_start + per * (size_t)t;
        jobs[t].ids_start = proto.ids_start + per * (size_t)t;
        jobs[t].n = (t == threads - 1) ? proto.n - per * (size_t)t : per;
        jobs[t].out = proto.mode == 0 ? (uint64_t *)calloc(65536, 8) : out;
        pthread_create(&th[t], NULL, stream_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) {
        pthread_join(th[t], NULL);
        if (proto.mode == 0) {
            for (int k = 0; k < 65536; k++) out[k] += jobs[t].out[k];
            free(jobs[t].out);
        }
    }
    free(th); free(jobs);
}

LHO_EXPORT void lho_stream_ingest_mt(int kind, uint64_t seed, uint64_t start, size_t n, uint64_t *counts65536,
                                     int threads) {
    stream_job j = {0};
    j.mode = 0; j.val_kind = kind; j.seed = seed; j.val_start = start; j.n = n; j.H = 1;
    stream_run(j, counts65536, threads);
}

LHO_EXPORT void lho_stream_ingest_keyed_mt(int val_kind, int id_kind, int as_i64, uint64_t seed, uint64_t val_start,
                                           uint64_t ids_start, size_t n, uint32_t H, uint64_t *counts, int threads) {
    stream_job j = {0};
    j.mode = 1; j.val_kind = val_kind; j.id_kind = id_kind; j.as_i64 = as_i64; j.seed = seed;
    j.val_start = val_start; j.ids_start = ids_start; j.n = n; j.H = H;
    stream_run(j, counts, threads);
}

LHO_EXPORT void lho_stream_counter_mt(int amount_kind, int id_kind, uint64_t seed, uint64_t val_start,
                                      uint64_t ids_start, size_t n, uint32_t C, uint64_t *counters, int threads) {
    stream_job j = {0};
    j.mode = 2; j.val_kind = amount_kind; j.id_kind = id_kind; j.seed = seed;
    j.val_start = val_start; j.ids_start = ids_start; j.n = n; j.H = C;
    stream_run(j, counters, threads);
}

/* ------------------------------------------------------------------ */
/*
 * Structure-faithful port of MetricSystem (BASELINE.md B1): name-keyed maps
 * guarded by reader/writer locks, read-lock fast path + write-lock creation,
 * atomic adds on the cells -- metrics.go:251-295 -- plus the snapshot and
 * reduction semantics of metrics.go:420-506 and :590-608.
 *
 * Go maps are restated as open-addressing tables that only grow.
 */
typedef struct {
    int16_t *keys; uint64_t *vals; uint8_t *used; uint32_t cap, len;
} bucket_map; /* map[int16]*uint64 */

typedef struct {
    char *name; bucket_map buckets;
} histo_entry;

typedef struct {
    char *name; uint64_t val;
} counter_entry;

typedef struct {
    counter_entry *e; uint32_t cap, len;
} counter_map; /* map[string]*uint64 */

typedef struct {
    histo_entry *e; uint32_t cap, len;
} histo_map; /* map[string]map[int16]*uint64 */

/* sync.RWMutex restated (src/sync/rwmutex.go): the reader fast path is one
 * atomic add on readerCount for RLock and one for RUnlock -- the "2 atomic
 * RMWs on one shared cache line" that metrics.go:275/:279 pay per sample.
 * pthread_rwlock_t is NOT a fair stand-in (it collapses into futex sleeps
 * under reader contention), so the port carries Go's algorithm itself. */
#define GO_RWMUTEX_MAX_READERS (1 << 30)
typedef struct {
    pthread_mutex_t w;          /* held if there are pending writers */
    sem_t writer_sem, reader_sem;
    int32_t reader_count;       /* number of pending readers */
    int32_t reader_wait;        /* number of departing readers */
} go_rwmutex;
static void go_rw_init(go_rwmutex *rw) {
    pthread_mutex_init(&rw->w, NULL);
    sem_init(&rw->writer_sem, 0, 0); sem_init(&rw->reader_sem, 0, 0);
    rw->reader_count = 0; rw->reader_wait = 0;
}
static inline void go_rw_rlock(go_rwmutex *rw) {
    if (__atomic_add_fetch(&rw->reader_count, 1, __ATOMIC_SEQ_CST) < 0)
        while (sem_wait(&rw->reader_sem) != 0) {}          /* a writer is pending */
}
static inline void go_rw_runlock(go_rwmutex *rw) {
    if (__atomic_add_fetch(&rw->reader_count, -1, __ATOMIC_SEQ_CST) < 0)
        if (__atomic_add_fetch(&rw->reader_wait, -1, __ATOMIC_SEQ_CST) == 0)
            sem_post(&rw->writer_sem);                     /* last departing reader wakes the writer */
}
static void go_rw_lock(go_rwmutex *rw) {
    pthread_mutex_lock(&rw->w);
    int32_t r = __atomic_add_fetch(&rw->reader_count, -GO_RWMUTEX_MAX_READERS, __ATOMIC_SEQ_CST) + GO_RWMUTEX_MAX_READERS;
    if (r != 0 && __atomic_add_fetch(&rw->reader_wait, r, __ATOMIC_SEQ_CST) != 0)
        while (sem_wait(&rw->writer_sem) != 0) {}
}
static void go_rw_unlock(go_rwmutex *rw) {
    int32_t r = __atomic_add_fetch(&rw->reader_count, GO_RWMUTEX_MAX_READERS, __ATOMIC_SEQ_CST);
    for (int32_t i = 0; i < r; i++) sem_post(&rw->reader_sem);
    pthread_mutex_unlock(&rw->w);
}

typedef struct lho_ms {
    go_rwmutex histogram_mu, counter_mu, counter_store_mu, histogram_count_mu;
    histo_map histogram_cache;
    counter_map counter_cache, counter_store, histogram_count_store;
    double percentiles[32]; char plabels[32][24]; int np;
} lho_ms;

static uint64_t str_hash(const char *s) {
    uint64_t h = 1469598103934665603ull;
    for (; *s; s++) { h ^= (uint8_t)*s; h *= 1099511628211ull; }
    return h;
}

static void bucket_map_init(bucket_map *m, uint32_t cap) {
    m->cap = cap; m->len = 0;
    m->keys = (int16_t *)calloc(cap, sizeof(int16_t));
    m->vals = (uint64_t *)calloc(cap, sizeof(uint64_t));
    m->used = (uint8_t *)calloc(cap, 1);
}
static void bucket_map_free(bucket_map *m) { free(m->keys); free(m->vals); free(m->used); }
static uint64_t *bucket_map_find(bucket_map *m, int16_t key) {
    if (!m->cap) return NULL;
    uint32_t i = ((uint32_t)(uint16_t)key * 2654435761u) & (m->cap - 1);
    while (m->used[i]) {
        if (m->keys[i] == key) return &m->vals[i];
        i = (i + 1) & (m->cap - 1);
    }
    return NULL;
}
static uint64_t *bucket_map_insert(bucket_map *m, int16_t key); /* fwd */
static void bucket_map_grow(bucket_map *m) {
    bucket_map n; bucket_map_init(&n, m->cap ? m->cap * 2 : 64);
    for (uint32_t i = 0; i < m->cap; i++)
        if (m->used[i]) *bucket_map_insert(&n, m->keys[i]) = m->vals[i];
    bucket_map_free(m); *m = n;
}
static uint64_t *bucket_map_insert(bucket_map *m, int16_t key) {
    if ((m->len + 1) * 2 > m->cap) bucket_map_grow(m);
    uint32_t i = ((uint32_t)(uint16_t)key * 2654435761u) & (m->cap - 1);
    while (m->used[i]) {
        if (m->keys[i] == key) return &m->vals[i];
        i = (i + 1) & (m->cap - 1);
    }
    m->used[i] = 1; m->keys[i] = key; m->vals[i] = 0; m->len++;
    return &m->vals[i];
}

static histo_entry *histo_map_find(histo_map *m, const char *name) {
    if (!m->cap) return NULL;
    uint32_t i = (uint32_t)str_hash(name) & (m->cap - 1);
    while (m->e[i].name) {
        if (!strcmp(m->e[i].name, name)) return &m->e[i];
        i = (i + 1) & (m->cap - 1);
    }
    return NULL;
}
static histo_entry *histo_map_insert(histo_map *m, const char *name) {
    if ((m->len + 1) * 2 > m->cap) {
        histo_map n; n.cap = m->cap ? m->cap * 2 : 64; n.len = 0;
        n.e = (histo_entry *)calloc(n.cap, sizeof(histo_entry));
        for (uint32_t j = 0; j < m->cap; j++)
            if (m->e[j].name) {
                uint32_t i = (uint32_t)str_hash(m->e[j].name) & (n.cap - 1);
                while (n.e[i].name) i = (i + 1) & (n.cap - 1);
                n.e[i] = m->e[j]; n.len++;
            }
        free(m->e); *m = n;
    }
    uint32_t i = (uint32_t)str_hash(name) & (m->cap - 1);
    while (m->e[i].name) {
        if (!strcmp(m->e[i].name, name)) return &m->e[i];
        i = (i + 1) & (m->cap - 1);
    }
    m->e[i].name = strdup(name);
    memset(&m->e[i].buckets, 0, sizeof(bucket_map));
    m->len++;
    return &m->e[i];
}
static void histo_map_free(histo_map *m) {
    for (uint32_t i = 0; i < m->cap; i++)
        if (m->e[i].name) { free(m->e[i].name); bucket_map_free(&m->e[i].buckets); }
    free(m->e); memset(m, 0, sizeof(*m));
}

static counter_entry *counter_map_find(counter_map *m, const char *name) {
    if (!m->cap) return NULL;
    uint32_t i = (uint32_t)str_hash(name) & (m->cap - 1);
    while (m->e[i].name) {
        if (!strcmp(m->e[i].name, name)) return &m->e[i];
        i = (i + 1) & (m->cap - 1);
    }
    return NULL;
}
static counter_entry *counter_map_insert(counter_map *m, const char *name) {
    if ((m->len + 1) * 2 > m->cap) {
        counter_map n; n.cap = m->cap ? m->cap * 2 : 64; n.len = 0;
        n.e = (counter_entry *)calloc(n.cap, sizeof(counter_entry));
        for (uint32_t j = 0; j < m->cap; j++)
            if (m->e[j].name) {
                uint32_t i = (uint32_t)str_hash(m->e[j].name) & (n.cap - 1);
                while (n.e[i].name) i = (i + 1) & (n.cap - 1);
                n.e[i] = m->e[j]; n.len++;
            }
        free(m->e); *m = n;
    }
    uint32_t i = (uint32_t)str_hash(name) & (m->cap - 1);
    while (m->e[i].name) {
        if (!strcmp(m->e[i].name, name)) return &m->e[i];
        i = (i + 1) & (m->cap - 1);
    }
    m->e[i].name = strdup(name); m->e[i].val = 0; m->len++;
    return &m->e[i];
}
static void counter_map_free(counter_map *m) {
    for (uint32_t i = 0; i < m->cap; i++) if (m->e[i].name) free(m->e[i].name);
    free(m->e); memset(m, 0, sizeof(*m));
}

/* NewMetricSystem, metrics.go:143-195 (default percentile labels :145-155). */
LHO_EXPORT lho_ms *lho_ms_new(void) {
    lho_ms *ms = (lho_ms *)calloc(1, sizeof(lho_ms));
    go_rw_init(&ms->histogram_mu);
    go_rw_init(&ms->counter_mu);
    go_rw_init(&ms->counter_store_mu);
    go_rw_init(&ms->histogram_count_mu);
    static const char *labels[9] = {"%s_min", "%s_50", "%s_75", "%s_90", "%s_95", "%s_99", "%s_99.9", "%s_99.99", "%s_max"};
    static const double ps[9] = {0, .5, .75, .9, .95, .99, .999, .9999, 1};
    ms->np = 9;
    for (int i = 0; i < 9; i++) { strcpy(ms->plabels[i], labels[i]); ms->percentiles[i] = ps[i]; }
    return ms;
}
LHO_EXPORT void lho_ms_free(lho_ms *ms) {
    histo_map_free(&ms->histogram_cache);
    counter_map_free(&ms->counter_cache);
    counter_map_free(&ms->counter_store);
    counter_map_free(&ms->histogram_count_store);
    free(ms);
}
/* SpecifyPercentiles, metrics.go:199-201. */
LHO_EXPORT void lho_ms_specify_percentiles(lho_ms *ms, int np, const char *const *labels, const double *ps) {
    ms->np = np > 32 ? 32 : np;
    for (int i = 0; i < ms->np; i++) {
        strncpy(ms->plabels[i], labels[i], 23); ms->plabels[i][23] = 0;
        ms->percentiles[i] = ps[i];
    }
}

/* Histogram, metrics.go:273-295. */
LHO_EXPORT void lho_ms_histogram(lho_ms *ms, const char *name, double value) {
    int16_t c = lho_compress(value);
    go_rw_rlock(&ms->histogram_mu);
    histo_entry *h = histo_map_find(&ms->histogram_cache, name);
    uint64_t *cell = h ? bucket_map_find(&h->buckets, c) : NULL;
    if (cell) {
        __atomic_fetch_add(cell, 1, __ATOMIC_SEQ_CST);
        go_rw_runlock(&ms->histogram_mu);
        return;
    }
    go_rw_runlock(&ms->histogram_mu);
    go_rw_lock(&ms->histogram_mu);
    h = histo_map_insert(&ms->histogram_cache, name);
    cell = bucket_map_insert(&h->buckets, c);
    __atomic_fetch_add(cell, 1, __ATOMIC_SEQ_CST);
    go_rw_unlock(&ms->histogram_mu);
}

/* Counter, metrics.go:251-269. */
LHO_EXPORT void lho_ms_counter(lho_ms *ms, const char *name, uint64_t amount) {
    go_rw_rlock(&ms->counter_mu);
    counter_entry *e = counter_map_find(&ms->counter_cache, name);
    if (e) {
        __atomic_fetch_add(&e->val, amount, __ATOMIC_SEQ_CST);
        go_rw_runlock(&ms->counter_mu);
        return;
    }
    go_rw_runlock(&ms->counter_mu);
    go_rw_lock(&ms->counter_mu);
    e = counter_map_insert(&ms->counter_cache, name);
    __atomic_fetch_add(&e->val, amount, __ATOMIC_SEQ_CST);
    go_rw_unlock(&ms->counter_mu);
}

/*
 * collectRawMetrics + processMetrics + the reaper's _agg_* step
 * (metrics.go:420-506, 590-608), flattened into "name\0" / value records.
 *
 * emit(ctx, kind, name, key, u64, f64) is called once per datum:
 *   kind 0: raw counter (cumulative)       u64
 *   kind 1: raw rate (interval delta)      u64
 *   kind 2: raw histogram bucket           key, u64
 *   kind 3: processed metric               f64   (name already formatted)
 */
typedef void (*lho_emit_fn)(void *ctx, int kind, const char *name, int key, uint64_t u, double f);

static void fmt_label(char *dst, size_t cap, const char *label, const char *name) {
    /* labels are "%s_xxx" format strings (metrics.go:383); support exactly one %s */
    const char *p = strstr(label, "%s");
    if (!p) { strncpy(dst, label, cap - 1); dst[cap - 1] = 0; return; }
    size_t pre = (size_t)(p - label);
    size_t o = 0;
    for (size_t i = 0; i < pre && o + 1 < cap; i++) dst[o++] = label[i];
    for (const char *s = name; *s && o + 1 < cap; s++) dst[o++] = *s;
    for (const char *s = p + 2; *s && o + 1 < cap; s++) dst[o++] = *s;
    dst[o] = 0;
}

LHO_EXPORT void lho_ms_collect_and_process(lho_ms *ms, lho_emit_fn emit, void *ctx) {
    char buf[512], nm[512];
    /* swap counter cache, metrics.go:425-428 */
    go_rw_lock(&ms->counter_mu);
    counter_map fresh = ms->counter_cache;
    memset(&ms->counter_cache, 0, sizeof(counter_map));
    go_rw_unlock(&ms->counter_mu);
    /* rates :430-433; fold into store :435-453 */
    go_rw_lock(&ms->counter_store_mu);
    for (uint32_t i = 0; i < fresh.cap; i++) {
        if (!fresh.e[i].name) continue;
        emit(ctx, 1, fresh.e[i].name, 0, fresh.e[i].val, 0);
        snprintf(buf, sizeof buf, "%s_rate", fresh.e[i].name);
        emit(ctx, 3, buf, 0, 0, (double)fresh.e[i].val);
        counter_map_insert(&ms->counter_store, fresh.e[i].name)->val += fresh.e[i].val;
    }
    /* export all cumulative counters :455-457 */
    for (uint32_t i = 0; i < ms->counter_store.cap; i++) {
        if (!ms->counter_store.e[i].name) continue;
        emit(ctx, 0, ms->counter_store.e[i].name, 0, ms->counter_store.e[i].val, 0);
        emit(ctx, 3, ms->counter_store.e[i].name, 0, 0, (double)ms->counter_store.e[i].val);
    }
    go_rw_unlock(&ms->counter_store_mu);
    counter_map_free(&fresh);

    /* swap histogram cache :460-463 */
    go_rw_lock(&ms->histogram_mu);
    histo_map histos = ms->histogram_cache;
    memset(&ms->histogram_cache, 0, sizeof(histo_map));
    go_rw_unlock(&ms->histogram_mu);

    uint64_t *dense = (uint64_t *)malloc(65536 * 8);
    for (uint32_t hi = 0; hi < histos.cap; hi++) {
        histo_entry *h = &histos.e[hi];
        if (!h->name) continue;
        memset(dense, 0, 65536 * 8);
        for (uint32_t i = 0; i < h->buckets.cap; i++)
            if (h->buckets.used[i]) {
                emit(ctx, 2, h->name, h->buckets.keys[i], h->buckets.vals[i], 0);
                dense[(uint16_t)h->buckets.keys[i]] = h->buckets.vals[i];
            }
        /* processHistograms :336-387 */
        double stats[3], pv[32]; int32_t pk[32];
        uint64_t total = lho_process_histogram(dense, ms->percentiles, ms->np, stats, pv, pk);
        snprintf(buf, sizeof buf, "%s_count", h->name); emit(ctx, 3, buf, 0, 0, stats[0]);
        snprintf(buf, sizeof buf, "%s_sum", h->name);   emit(ctx, 3, buf, 0, 0, stats[1]);
        snprintf(buf, sizeof buf, "%s_avg", h->name);   emit(ctx, 3, buf, 0, 0, stats[2]);
        for (int j = 0; j < ms->np; j++) {
            if (pk[j] == INT32_MIN) continue; /* percentile() error: key omitted :380-382 */
            fmt_label(nm, sizeof nm, ms->plabels[j], h->name);
            emit(ctx, 3, nm, 0, 0, pv[j]);
        }
        /* aggregate store :359-376 and reaper :590-608 */
        go_rw_lock(&ms->histogram_count_mu);
        snprintf(buf, sizeof buf, "%s_sum", h->name);
        counter_entry *as = counter_map_insert(&ms->histogram_count_store, buf);
        as->val += lho_go_f64_to_u64(stats[1]);
        uint64_t agg_sum = as->val;
        snprintf(buf, sizeof buf, "%s_count", h->name);
        counter_entry *ac = counter_map_insert(&ms->histogram_count_store, buf);
        ac->val += total;
        uint64_t agg_count = ac->val;
        go_rw_unlock(&ms->histogram_count_mu);
        if (agg_count > 0) {
            snprintf(buf, sizeof buf, "%s_agg_avg", h->name);   emit(ctx, 3, buf, 0, 0, (double)(agg_sum / agg_count));
            snprintf(buf, sizeof buf, "%s_agg_count", h->name); emit(ctx, 3, buf, 0, 0, (double)agg_count);
            snprintf(buf, sizeof buf, "%s_agg_sum", h->name);   emit(ctx, 3, buf, 0, 0, (double)agg_sum);
        }
    }
    free(dense);
    histo_map_free(&histos);
}

/* ------------------------------------------------------------------ */
/* Baseline driver: T threads each call lho_ms_histogram(name_i, v_i) over a
 * slice of the stream, like print_benchmark.go:59-67 minus the clock reads.
 * Returns elapsed seconds. */
typedef struct {
    lho_ms *ms; const double *v; const uint32_t *ids; size_t n; const char *const *names;
} ms_job;
static void *ms_worker(void *p) {
    ms_job *j = (ms_job *)p;
    if (j->ids) for (size_t i = 0; i < j->n; i++) lho_ms_histogram(j->ms, j->names[j->ids[i]], j->v[i]);
    else        for (size_t i = 0; i < j->n; i++) lho_ms_histogram(j->ms, j->names[0], j->v[i]);
    return NULL;
}
LHO_EXPORT double lho_ms_bench_ingest(lho_ms *ms, const double *v, const uint32_t *ids, size_t n,
                                      const char *const *names, int threads) {
    if (threads < 1) threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    ms_job *jobs = (ms_job *)malloc(sizeof(ms_job) * (size_t)threads);
    size_t per = n / (size_t)threads;
    struct timespec a, b;
    clock_gettime(CLOCK_MONOTONIC, &a);
    for (int t = 0; t < threads; t++) {
        jobs[t].ms = ms; jobs[t].names = names;
        jobs[t].v = v + per * (size_t)t;
        jobs[t].ids = ids ? ids + per * (size_t)t : NULL;
        jobs[t].n = (t == threads - 1) ? n - per * (size_t)t : per;
        pthread_create(&th[t], NULL, ms_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &b);
    free(th); free(jobs);
    return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

/* Fetch one raw bucket count from the live cache (test helper). */
LHO_EXPORT uint64_t lho_ms_peek_bucket(lho_ms *ms, const char *name, int16_t key) {
    go_rw_rlock(&ms->histogram_mu);
    histo_entry *h = histo_map_find(&ms->histogram_cache, name);
    uint64_t *c = h ? bucket_map_find(&h->buckets, key) : NULL;
    uint64_t r = c ? *c : 0;
    go_rw_runlock(&ms->histogram_mu);
    return r;
}
