// raw_read_client.cu -- a CUDA client of the raw device-subscription query API (include/loghisto_b200_device.cuh):
// kernels that query a raw board (lh_raw_board) through lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count,
// knowing the library only through its public headers.  Built by loghisto_b200/build.py (build_device_client) into
// tests/_build/ and used by tests/test_gpu_raw_subscription.py and tools/raw_board_probe.py.
#include <cuda_runtime.h>
#include <stdint.h>

#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

#define RRC_API extern "C" __attribute__((visibility("default")))

namespace {

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// query i: (rows[i], ps[i]) -> keys[i], vals[i], pub[i]
__global__ void k_percentiles(const lh_raw_board b, const uint32_t *rows, const double *ps, uint32_t n, int32_t *keys,
                              double *vals, unsigned long long *pub) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_percentile(b, rows[i], ps[i], &keys[i], &vals[i]);
}

// query i: (rows[i], values[i]) -> ranks[i], totals[i], pub[i]
__global__ void k_ranks(const lh_raw_board b, const uint32_t *rows, const double *values, uint32_t n, uint64_t *ranks,
                        uint64_t *totals, unsigned long long *pub) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_rank(b, rows[i], values[i], &ranks[i], &totals[i]);
}

// query i: (rows[i], keys[i]) -> counts[i], pub[i]
__global__ void k_bucket_counts(const lh_raw_board b, const uint32_t *rows, const int32_t *keys, uint32_t n,
                                uint64_t *counts, unsigned long long *pub) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_bucket_count(b, rows[i], keys[i], &counts[i]);
}

// The torn-read reader: until budget_ns of device clock have passed, every thread alternates a rank query of row 0 at
// `v` and a percentile query of row 0 at `p`, and a rank query of row 1 (never bound: always empty).  Publish j of
// row 0 holds histogram A when j is odd and B when j is even (>= 2); publish 0 is the empty row.  An answer that does
// not equal the expected one for the publish number it carries counts as bad.
// stats: [0] reads, [1] bad, [2] highest publish seen, [3] lowest non-zero publish seen, [4] publish changes
struct Expect {
    unsigned long long total[2], rank[2];   // [0] = A, [1] = B
    int32_t key[2];
};

__global__ void k_torn(const lh_raw_board b, double v, double p, Expect e, unsigned long long budget_ns,
                       unsigned long long *stats) {
    const unsigned long long deadline = now_ns() + budget_ns;
    unsigned long long reads = 0, bad = 0, hi = 0, lo = ~0ull, changes = 0, last = 0;
    while (now_ns() < deadline) {
        uint64_t rank, total;
        const uint64_t pr = lh::raw_rank(b, 0, v, &rank, &total);
        int32_t key;
        double val;
        const uint64_t pp = lh::raw_percentile(b, 0, p, &key, &val);
        uint64_t r1, t1;
        lh::raw_rank(b, 1, v, &r1, &t1);
        reads += 3;
        if (pr == 0) bad += rank != 0 || total != 0;
        else bad += rank != e.rank[(pr & 1) ? 0 : 1] || total != e.total[(pr & 1) ? 0 : 1];
        if (pp == 0) bad += key != (int32_t)0x80000000;
        else bad += key != e.key[(pp & 1) ? 0 : 1];
        bad += r1 != 0 || t1 != 0;
        const uint64_t q = pr > pp ? pr : pp;
        if (q) {
            hi = q > hi ? q : hi;
            lo = q < lo ? q : lo;
            if (last && q != last) changes++;
            last = q;
        }
    }
    atomicAdd(&stats[0], reads);
    atomicAdd(&stats[1], bad);
    atomicMax(&stats[2], hi);
    atomicMin(&stats[3], lo);
    atomicAdd(&stats[4], changes);
}

// Cost of lh::raw_percentile: one thread queries `row` `iters` times; out[0] = elapsed %globaltimer ns, out[1] = a
// checksum that keeps the queries alive.
__global__ void k_cost(const lh_raw_board b, uint32_t row, int iters, unsigned long long *out) {
    unsigned long long acc = 0;
    const unsigned long long t0 = now_ns();
    for (int it = 0; it < iters; it++) {
        int32_t key;
        double val;
        acc += lh::raw_percentile(b, row, 0.001 * (it % 1000), &key, &val) + (unsigned long long)key;
    }
    const unsigned long long t1 = now_ns();
    out[0] = t1 - t0;
    out[1] = acc;
}

uint32_t blocks(uint32_t n) { return (n + 255) / 256; }

}  // namespace

RRC_API int rrc_percentiles(const lh_raw_board *b, const void *d_rows, const void *d_ps, uint32_t n, void *d_keys,
                            void *d_vals, void *d_pub, void *stream) {
    if (!n) return 0;
    k_percentiles<<<blocks(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, (const double *)d_ps, n,
                                                                (int32_t *)d_keys, (double *)d_vals,
                                                                (unsigned long long *)d_pub);
    return (int)cudaGetLastError();
}

RRC_API int rrc_ranks(const lh_raw_board *b, const void *d_rows, const void *d_values, uint32_t n, void *d_ranks,
                      void *d_totals, void *d_pub, void *stream) {
    if (!n) return 0;
    k_ranks<<<blocks(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, (const double *)d_values, n,
                                                          (uint64_t *)d_ranks, (uint64_t *)d_totals,
                                                          (unsigned long long *)d_pub);
    return (int)cudaGetLastError();
}

RRC_API int rrc_bucket_counts(const lh_raw_board *b, const void *d_rows, const void *d_keys, uint32_t n, void *d_counts,
                              void *d_pub, void *stream) {
    if (!n) return 0;
    k_bucket_counts<<<blocks(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, (const int32_t *)d_keys,
                                                                  n, (uint64_t *)d_counts, (unsigned long long *)d_pub);
    return (int)cudaGetLastError();
}

// Starts the torn-read reader on `stream` for `budget_ns` from now (device clock), on `ctas` CTAs of 128 threads.
// d_stats: 5 uint64, [3] preset to ~0 by the caller.
RRC_API int rrc_torn_start(const lh_raw_board *b, double v, double p, const uint64_t *total, const uint64_t *rank,
                           const int32_t *key, int ctas, unsigned long long budget_ns, void *d_stats, void *stream) {
    Expect e;
    for (int i = 0; i < 2; i++) {
        e.total[i] = total[i];
        e.rank[i] = rank[i];
        e.key[i] = key[i];
    }
    k_torn<<<ctas, 128, 0, (cudaStream_t)stream>>>(*b, v, p, e, budget_ns, (unsigned long long *)d_stats);
    return (int)cudaGetLastError();
}

RRC_API int rrc_cost(const lh_raw_board *b, uint32_t row, int iters, void *d_out, void *stream) {
    k_cost<<<1, 1, 0, (cudaStream_t)stream>>>(*b, row, iters, (unsigned long long *)d_out);
    return (int)cudaGetLastError();
}
