/*
 * lh_stub_reduce_sparse.c -- TEST-ONLY lh_reduce_sparse_host for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_reduce_sparse_cpu.py compiles it together with lh_stub.c and oracle/loghisto_oracle.c, so that the C++
 * host mirror's processMetrics of sets it did not collect runs on the CPU.  The stub bins at the reference's
 * precision (lho_compress), so this reduces at precision 100 as well.  Stateless: no lock needed.
 *
 * Each segment is summed into a dense row (repeats wrap), reduced by the oracle, then the two answers a dense row
 * loses are restored (a key present in Go's map with a merged count of 0): p <= 0 with a total above 0 gives the
 * smallest key present, and a present +-Inf key with count 0 makes the sum and avg NaN.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "loghisto_b200.h"

/* from oracle/loghisto_oracle.c */
uint64_t lho_process_histogram_p(const uint64_t *counts65536, const double *ps, int np, double *out_stats,
                                 double *out_pvals, int32_t *out_pkeys, double precision);
double lho_decompress_p(int16_t k, double precision);

#define STUB_PRECISION 100.0

LH_API lh_status lh_reduce_sparse_host(lh_ctx *c, uint32_t n, const uint32_t *off, const int16_t *keys, const uint64_t *cnts,
                                       const double *ps, uint32_t np, uint64_t *counts, double *sums, double *avgs,
                                       int32_t *pkeys, double *pvals) {
    if (!c) return LH_ERR_INVALID;
    if (n == 0) return LH_OK;
    if (!off || np > LH_MAX_PERCENTILES || (np && !ps)) return LH_ERR_INVALID;
    for (uint32_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) return LH_ERR_INVALID;
    if (off[n] > off[0] && (!keys || !cnts)) return LH_ERR_INVALID;
    uint64_t *row = (uint64_t *)calloc(65536, 8);
    if (!row) return LH_ERR_NOMEM;
    for (uint32_t h = 0; h < n; h++) {
        int kmin = INT32_MAX, infzero = 0;
        for (uint32_t e = off[h]; e < off[h + 1]; e++) {
            row[(uint16_t)keys[e]] += cnts[e];
            if (keys[e] < kmin) kmin = keys[e];
        }
        for (uint32_t e = off[h]; e < off[h + 1]; e++)
            if (isinf(lho_decompress_p(keys[e], STUB_PRECISION)) && row[(uint16_t)keys[e]] == 0) infzero = 1;
        double stats[3], pv[LH_MAX_PERCENTILES];
        int32_t pk[LH_MAX_PERCENTILES];
        const uint64_t total = lho_process_histogram_p(row, ps, (int)np, stats, pv, pk, STUB_PRECISION);
        if (infzero) stats[1] = stats[2] = NAN;
        for (uint32_t j = 0; j < np; j++)
            if (total && ps[j] <= 0.0) { pk[j] = kmin; pv[j] = lho_decompress_p((int16_t)kmin, STUB_PRECISION); }
        if (counts) counts[h] = total;
        if (sums) sums[h] = stats[1];
        if (avgs) avgs[h] = stats[2];
        for (uint32_t j = 0; j < np; j++) {
            if (pkeys) pkeys[(size_t)h * np + j] = pk[j];
            if (pvals) pvals[(size_t)h * np + j] = pv[j];
        }
        for (uint32_t e = off[h]; e < off[h + 1]; e++) row[(uint16_t)keys[e]] = 0;
    }
    free(row);
    return LH_OK;
}
