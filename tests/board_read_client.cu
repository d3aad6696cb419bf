// board_read_client.cu -- a CUDA client of the device-subscription read API (include/loghisto_b200_device.cuh):
// kernels that read a board (lh_board) row by row through lh::read_histogram / lh::read_counter, knowing the library
// only through its public headers.  Built by loghisto_b200/build.py (build_device_client) into tests/_build/ and used
// by tests/test_gpu_device_subscription.py and tools/board_probe.py.
#include <cuda_runtime.h>
#include <stdint.h>

#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

#define BRC_API extern "C" __attribute__((visibility("default")))

namespace {

// thread i reads row i: histogram rows into out_h (the board's row layout), counter rows into out_c, and the publish
// number each read belongs to into pub[row] (histogram rows first)
__global__ void k_read_rows(const lh_board b, lh_board_hist_row *out_h, lh_board_counter_row *out_c,
                            unsigned long long *pub) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < b.k) {
        lh::HistogramStats s;
        pub[i] = lh::read_histogram(b, i, &s);
        lh_board_hist_row r{};
        r.count = s.count;
        r.sum = s.sum;
        r.avg = s.avg;
        r.present = s.present;
        for (int j = 0; j < LH_MAX_PERCENTILES; j++) { r.pvals[j] = s.pvals[j]; r.pkeys[j] = s.pkeys[j]; }
        out_h[i] = r;
    } else if (i < b.k + b.kc) {
        lh::CounterStats s;
        pub[i] = lh::read_counter(b, i - b.k, &s);
        lh_board_counter_row r{};
        r.rate = s.rate;
        r.total = s.total;
        r.present = s.present;
        out_c[i - b.k] = r;
    }
}

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Torn-read check.  Every thread reads rows until %globaltimer passes its deadline -- the only exit, which depends on
// nothing the host does.  The publisher gives, in collection j, every histogram name exactly j samples of one value
// and every counter name Counter(name, j), with percentile label 0 at p = 0.5.  So a row of publish j is consistent
// when: count == j, sum == pvals[0] * count and avg == sum / count (a single bucket); rate == j, total == j(j+1)/2.
// stats: [0] reads, [1] inconsistent rows, [2] largest publish seen, [3] smallest non-zero publish seen,
// [4] times a thread saw the publish number change.
__global__ void k_torn(const lh_board b, unsigned long long budget_ns, unsigned long long *stats) {
    const unsigned long long deadline = now_ns() + budget_ns;   // each thread runs budget_ns from its own start
    unsigned long long reads = 0, bad = 0, hi = 0, lo = ~0ull, changes = 0, last = 0;
    const uint32_t rows = b.k + b.kc, stride = gridDim.x * blockDim.x;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    while (now_ns() < deadline) {
        const uint32_t row = i % rows;
        unsigned long long p;
        bool ok;
        if (row < b.k) {
            lh::HistogramStats s;
            p = lh::read_histogram(b, row, &s);
            ok = p == 0 || (s.present && s.count == p && s.np == 1 && s.sum == __dmul_rn(s.pvals[0], (double)s.count) &&
                            s.avg == __ddiv_rn(s.sum, (double)s.count));
        } else {
            lh::CounterStats s;
            p = lh::read_counter(b, row - b.k, &s);
            ok = p == 0 || (s.present && s.rate == p && s.total == p * (p + 1) / 2);
        }
        reads++;
        if (!ok) bad++;
        if (p) {
            hi = p > hi ? p : hi;
            lo = p < lo ? p : lo;
            if (last && p != last) changes++;
            last = p;
        }
        i += stride;
    }
    atomicAdd(&stats[0], reads);
    atomicAdd(&stats[1], bad);
    atomicMax(&stats[2], hi);
    atomicMin(&stats[3], lo);
    atomicAdd(&stats[4], changes);
}

// Cost of lh::read_histogram: one thread reads `row` `iters` times; out[0] = elapsed %globaltimer ns, out[1] = a
// checksum that keeps the reads alive.
__global__ void k_read_cost(const lh_board b, uint32_t row, int iters, unsigned long long *out) {
    unsigned long long acc = 0;
    const unsigned long long t0 = now_ns();
    for (int it = 0; it < iters; it++) {
        lh::HistogramStats s;
        acc += lh::read_histogram(b, row, &s) + s.count + (unsigned long long)s.pkeys[it & 31];
    }
    const unsigned long long t1 = now_ns();
    out[0] = t1 - t0;
    out[1] = acc;
}

}  // namespace

BRC_API int brc_read_rows(const lh_board *b, void *d_out_h, void *d_out_c, void *d_pub, void *stream) {
    const uint32_t rows = b->k + b->kc;
    if (!rows) return 0;
    k_read_rows<<<(rows + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*b, (lh_board_hist_row *)d_out_h,
                                                                     (lh_board_counter_row *)d_out_c, (unsigned long long *)d_pub);
    return (int)cudaGetLastError();
}

// Starts the torn-read reader on `stream` for `budget_ns` from now (device clock), on `ctas` CTAs of 256 threads.
BRC_API int brc_torn_start(const lh_board *b, int ctas, unsigned long long budget_ns, void *d_stats, void *stream) {
    unsigned long long init[5] = {0, 0, 0, ~0ull, 0};
    cudaError_t e = cudaMemcpyAsync(d_stats, init, sizeof init, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
    k_torn<<<ctas, 256, 0, (cudaStream_t)stream>>>(*b, budget_ns, (unsigned long long *)d_stats);
    return (int)cudaGetLastError();
}

BRC_API int brc_read_cost(const lh_board *b, uint32_t row, int iters, void *d_out, void *stream) {
    k_read_cost<<<1, 1, 0, (cudaStream_t)stream>>>(*b, row, iters, (unsigned long long *)d_out);
    return (int)cudaGetLastError();
}
