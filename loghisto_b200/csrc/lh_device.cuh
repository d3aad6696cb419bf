// lh_device.cuh -- device-side helpers private to the library: decompress and the synthetic stream generator.
//
// The bucket arithmetic (compress: exact_key16, fast_candidate, key16_of and Prec) and the writers' helpers live in
// the public device header include/loghisto_b200_device.cuh, which CUDA callers include to record from their own
// kernels; the library's kernels include it too, so there is one definition of the bucket function.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/loghisto_b200_device.cuh"

namespace lh {

constexpr int LH_MAX_PCT = 32;   // == LH_MAX_PERCENTILES in include/loghisto_b200.h

// math.Exp as amd64 Go evaluates it (src/math/exp_amd64.s, non-FMA path), one
// IEEE rounding per op.  Used once at context creation to fill the decompress table.
__device__ __forceinline__ double go_exp(double x) {
    const double LOG2E = 1.4426950408889634073599246810018920;
    const double LN2U = 0.69314718055966295651160180568695068359375;
    const double LN2L = 0.28235290563031577122588448175013436025525412068e-12;
    double q = __dmul_rn(LOG2E, x);
    int e = __double2int_rn(q);                  // CVTSD2SL, round-to-nearest-even
    double ef = (double)e;
    double r = __dsub_rn(x, __dmul_rn(ef, LN2U));
    r = __dsub_rn(r, __dmul_rn(ef, LN2L));
    r = __dmul_rn(r, 0.0625);
    double p = 2.4801587301587301587e-5;
    p = __dadd_rn(__dmul_rn(p, r), 1.9841269841269841270e-4);
    p = __dadd_rn(__dmul_rn(p, r), 1.3888888888888888889e-3);
    p = __dadd_rn(__dmul_rn(p, r), 8.3333333333333333333e-3);
    p = __dadd_rn(__dmul_rn(p, r), 4.1666666666666666667e-2);
    p = __dadd_rn(__dmul_rn(p, r), 1.6666666666666666667e-1);
    p = __dadd_rn(__dmul_rn(p, r), 0.5);
    p = __dadd_rn(__dmul_rn(p, r), 1.0);
    r = __dmul_rn(r, p);
    r = __dmul_rn(r, __dadd_rn(r, 2.0));
    r = __dmul_rn(r, __dadd_rn(r, 2.0));
    r = __dmul_rn(r, __dadd_rn(r, 2.0));
    r = __dmul_rn(r, __dadd_rn(r, 2.0));
    r = __dadd_rn(r, 1.0);
    int be = e + 0x3FF;
    if (be <= 0) return 0.0;
    if (be >= 0x7FF) return u64_as_f64(0x7FF0000000000000ull);
    return __dmul_rn(r, u64_as_f64((uint64_t)be << 52));
}

// decompress(), metrics.go:326-332.
__device__ __forceinline__ double go_decompress(int key, double precision) {
    double a = fabs((double)key);
    double f = __dsub_rn(go_exp(__ddiv_rn(a, precision)), 1.0);
    return key < 0 ? __dmul_rn(-1.0, f) : f;
}

// splitmix64 and the synthetic streams (SURVEY.md section 8d; integer-only so any checker can regenerate them).
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

}  // namespace lh
