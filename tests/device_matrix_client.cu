// device_matrix_client.cu -- one client of the device API (include/loghisto_b200_device.cuh), built the ways callers
// build it: loghisto_b200/build.py build_device_client() compiles it under each flag set of DEVICE_MATRIX (the library's
// own flags, --use_fast_math, -G, -maxrregcount=32, -rdc=true over two translation units, and PTX-only builds for
// compute_90 and compute_70 that the driver JITs at load) into tests/_build/device_matrix/<variant>/.  The tests call the
// extern "C" launchers below through ctypes (tests/test_gpu_device_api_builds.py) and inspect the built artefacts
// (tests/test_device_api_builds_cpu.py).  It knows the library only through its public headers.
//
// With -DLHM_PART=1 / -DLHM_PART=2 the file is one of the two translation units of the -rdc=true build: part 2 holds
// k_record_part2 and its launcher, part 1 everything else.  Both call lh::key16_of, so the out-of-line lh::exact_key16
// is reached from both and the device link must keep one copy.  Without LHM_PART the file is the whole client.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

#define LHM_API extern "C" __attribute__((visibility("default")))

#if !defined(LHM_PART) || LHM_PART == 1
#define LHM_PART1 1
#endif
#if !defined(LHM_PART) || LHM_PART == 2
#define LHM_PART2 1
#endif

namespace {

// The client's own linear thread index, so that the samples a thread takes do not depend on lh::block_thread_rank:
// a defect there shows in the BlockHistogram / BlockRecorder results, not in which samples were fed.
__device__ __forceinline__ uint32_t thread_rank() {
    return threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
}
__device__ __forceinline__ uint32_t thread_count() { return blockDim.x * blockDim.y * blockDim.z; }

int err(cudaError_t e) { return (int)e; }

// The kernels that take the caller's block shape declare the largest block, as a kernel launched with 1024 threads
// must: under -G, a kernel without it may need more registers than a 1024-thread block can have.
constexpr int kMaxThreads = 1024;

}  // namespace

#ifdef LHM_PART1
namespace {

// ---------------------------------------------------------------- the FP32 estimate, cell by cell
// Cell c of x = 1+|v| in [1, 2^64): biased exponent 1023 + (c >> 23), top 23 mantissa bits c & (2^23 - 1).  Its
// representative is the cell's smallest double X = bits 0x3FF0... + (c << 29), and v = X - 1 (exact below 2^53, and
// rounding back onto X above, where the low mantissa bits of X are even).  fast_candidate depends on v only through
// the sign and the cell of 1+|v|, so the outputs of the 2^30 representatives are the estimate's outputs for every input.
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {    // splitmix64's finaliser
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__device__ __forceinline__ double cell_value(uint32_t c) {
    return __dsub_rn(lh::u64_as_f64(0x3FF0000000000000ull + ((unsigned long long)c << 29)), 1.0);
}

// what the estimate says about one input: ~0 when it hands the sample to the exact path, (idx, bits of w) otherwise
__device__ __forceinline__ unsigned long long estimate_word(double v, const lh::Prec &pc) {
    uint32_t idx;
    bool slow;
    float w;
    lh::fast_candidate(v, pc, idx, slow, w);
    return slow ? ~0ull : ((unsigned long long)idx << 32) | __float_as_uint(w);
}

// CTA b covers cells [b * per, (b + 1) * per), per = 2^29 / gridDim.x.  hashes[b] = sum over its cells and both signs
// of mix64(cell/sign ^ mix64(output word)), mod 2^64 (order-free, so the CTA's schedule does not enter it); *left
// counts representatives whose 1 + |v| is not in their own cell.
__global__ void k_estimate(lh::Prec pc, unsigned long long *hashes, unsigned long long *left) {
    __shared__ unsigned long long s_hash, s_left;
    if (thread_rank() == 0) { s_hash = 0; s_left = 0; }
    __syncthreads();
    const uint32_t per = (1u << 29) / gridDim.x, c0 = blockIdx.x * per;
    unsigned long long h = 0, nleft = 0;
    for (uint32_t j = thread_rank(); j < per; j += thread_count()) {
        const uint32_t c = c0 + j;
        const double v = cell_value(c);
        const unsigned long long x = lh::f64_as_u64(__dadd_rn(1.0, fabs(v)));
        nleft += ((x - 0x3FF0000000000000ull) >> 29) != c;
        h += mix64(((unsigned long long)c << 1) ^ mix64(estimate_word(v, pc)));
        h += mix64(((unsigned long long)c << 1 | 1ull) ^ mix64(estimate_word(-v, pc)));
    }
    atomicAdd(&s_hash, h);
    atomicAdd(&s_left, nleft);
    __syncthreads();
    if (thread_rank() == 0) {
        hashes[blockIdx.x] = s_hash;
        if (s_left) atomicAdd(left, s_left);
    }
}

// The drill-down: the outputs of cells [c_lo, c_lo + n), both signs: entry 2j + s is cell c_lo + j with sign s
// (s = 1: -v); slow[e] = 1 when the sample goes to the exact path, and idx / w hold the estimate otherwise (0 when slow).
__global__ void k_estimate_cells(lh::Prec pc, uint32_t c_lo, uint32_t n, uint32_t *idx, uint8_t *slow, float *w) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 2 * n) return;
    const double v = cell_value(c_lo + (e >> 1));
    uint32_t i;
    bool s;
    float ww;
    lh::fast_candidate((e & 1) ? -v : v, pc, i, s, ww);
    idx[e] = s ? 0u : i;
    slow[e] = s;
    w[e] = s ? 0.0f : ww;
}

// The recorder's precision block, with c1 moved by c1_ulps float ulps (0: as the library filled it).
lh::Prec prec_of(const lh_recorder *rec, int c1_ulps) {
    lh::Prec pc = *reinterpret_cast<const lh::Prec *>(rec->prec);
    uint32_t b;
    memcpy(&b, &pc.c1, 4);
    b += (uint32_t)c1_ulps;
    memcpy(&pc.c1, &b, 4);
    return pc;
}

// ---------------------------------------------------------------- bucket keys
__global__ void k_keys(lh::Prec pc, const double *vals, size_t n, uint16_t *fast, uint16_t *exact) {
    for (size_t i = (size_t)blockIdx.x * thread_count() + thread_rank(); i < n; i += (size_t)gridDim.x * thread_count()) {
        fast[i] = (uint16_t)lh::key16_of(vals[i], pc);
        exact[i] = (uint16_t)lh::exact_key16(vals[i], pc.precision);
    }
}

// ---------------------------------------------------------------- lh::record / record_ns / count
// op 0: lh::record(ids[i], vals[i]) of float64 values; op 1: lh::record_ns of int64 nanoseconds; op 2: lh::count of
// uint64 amounts.
template <int OP>
__device__ __forceinline__ void record_one(const lh_recorder &rec, uint32_t id, const void *vals, size_t i) {
    if (OP == 0) lh::record(rec, id, static_cast<const double *>(vals)[i]);
    else if (OP == 1) lh::record_ns(rec, id, static_cast<const long long *>(vals)[i]);
    else lh::count(rec, id, static_cast<const unsigned long long *>(vals)[i]);
}

// Thread g of T = gridDim.x * thread_count() (g = blockIdx.x * thread_count() + thread_rank()) feeds samples by pattern:
//   0  every lane records: i = g, g + T, ... (the threads past n have nothing)
//   1  per-lane trip counts that differ inside a warp: thread g takes the contiguous run of base + (g % 4) samples
//      starting at g * base + 6 * (g / 4) + {0, 0, 1, 3}[g % 4], base = ceil(n / T), clipped to n
//   2  lanes return early: thread g takes the run [g * base, (g + 1) * base) clipped to n, and returns before its
//      sample k = (uint32(g) * 2654435761) % (base + 2); a lane whose k >= its run records the whole run
// Lanes may leave the kernel here because lh::record / record_ns / count never synchronise the block.
template <int OP>
__global__ void __launch_bounds__(kMaxThreads)
k_record(lh_recorder rec, int pattern, const uint32_t *ids, const void *vals, size_t n) {
    const size_t T = (size_t)gridDim.x * thread_count(), g = (size_t)blockIdx.x * thread_count() + thread_rank();
    if (pattern == 0) {
        for (size_t i = g; i < n; i += T) record_one<OP>(rec, ids[i], vals, i);
        return;
    }
    const size_t base = (n + T - 1) / T;
    if (pattern == 1) {
        const size_t r = g % 4, lo = g * base + 6 * (g / 4) + (r * (r - 1)) / 2;
        for (size_t i = lo; i < lo + base + r && i < n; i++) record_one<OP>(rec, ids[i], vals, i);
        return;
    }
    const size_t stop = (size_t)(((uint32_t)g * 2654435761u) % (uint32_t)(base + 2));
    for (size_t k = 0; k < base; k++) {
        const size_t i = g * base + k;
        if (i >= n || k == stop) return;
        record_one<OP>(rec, ids[i], vals, i);
    }
}

// ---------------------------------------------------------------- lh::BlockHistogram
// CTA b binds histogram block_ids[b], adds samples [b * chunk, min(n, (b + 1) * chunk)) in `flushes` consecutive parts
// and flushes after each.  The sub-histogram sits `off` bytes into the dynamic shared memory.
__global__ void __launch_bounds__(kMaxThreads)
k_block_histogram(lh_recorder rec, const uint32_t *block_ids, const double *vals, size_t n, size_t chunk, int flushes,
                  uint32_t off) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockHistogram bh(rec, smem + off);
    bh.init(block_ids[blockIdx.x]);
    const size_t lo = (size_t)blockIdx.x * chunk < n ? (size_t)blockIdx.x * chunk : n;
    const size_t hi = lo + chunk < n ? lo + chunk : n;
    for (int f = 0; f < flushes; f++) {
        const size_t a = lo + (hi - lo) * f / flushes, b = lo + (hi - lo) * (f + 1) / flushes;
        for (size_t i = a + thread_rank(); i < b; i += thread_count()) bh.add(vals[i]);
        bh.flush();
    }
}

// ---------------------------------------------------------------- lh::BlockRecorder
// As k_block_histogram, keyed: sample i goes to histogram ids[i] through a table asked for `entries` slots, `off`
// bytes into the dynamic shared memory.  dual != 0: two tables side by side, the second right after the first; odd
// samples go through the second.  op 0: record of float64 values, op 1: record_ns of int64 nanoseconds.
__global__ void __launch_bounds__(kMaxThreads)
k_block_recorder(lh_recorder rec, int op, const uint32_t *ids, const void *vals, size_t n, size_t chunk, int flushes,
                 uint32_t entries, uint32_t off, int dual) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br0(rec, smem + off, entries);
    lh::BlockRecorder br1(rec, smem + off + lh::BlockRecorder::smem_bytes(entries), entries);
    br0.init();
    if (dual) br1.init();
    const size_t lo = (size_t)blockIdx.x * chunk < n ? (size_t)blockIdx.x * chunk : n;
    const size_t hi = lo + chunk < n ? lo + chunk : n;
    for (int f = 0; f < flushes; f++) {
        const size_t a = lo + (hi - lo) * f / flushes, b = lo + (hi - lo) * (f + 1) / flushes;
        for (size_t i = a + thread_rank(); i < b; i += thread_count()) {
            lh::BlockRecorder &br = dual && (i & 1) ? br1 : br0;
            if (op == 0) br.record(ids[i], static_cast<const double *>(vals)[i]);
            else br.record_ns(ids[i], static_cast<const long long *>(vals)[i]);
        }
        br0.flush();
        if (dual) br1.flush();
    }
}

// ---------------------------------------------------------------- board reads
__global__ void k_raw_percentiles(const lh_raw_board b, const uint32_t *rows, const double *ps, size_t n, int32_t *keys,
                                  double *vals, unsigned long long *pub) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_percentile(b, rows[i], ps[i], &keys[i], &vals[i]);
}

__global__ void k_raw_ranks(const lh_raw_board b, const uint32_t *rows, const double *values, size_t n, uint64_t *ranks,
                            uint64_t *totals, unsigned long long *pub) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_rank(b, rows[i], values[i], &ranks[i], &totals[i]);
}

__global__ void k_raw_bucket_counts(const lh_raw_board b, const uint32_t *rows, const int32_t *keys, size_t n,
                                    uint64_t *counts, unsigned long long *pub) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pub[i] = lh::raw_bucket_count(b, rows[i], keys[i], &counts[i]);
}

// query i reads histogram row rows[i] into out[i] (the board's row layout)
__global__ void k_read_histograms(const lh_board b, const uint32_t *rows, size_t n, lh_board_hist_row *out,
                                  unsigned long long *pub) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    lh::HistogramStats s;
    pub[i] = lh::read_histogram(b, rows[i], &s);
    lh_board_hist_row r{};
    r.count = s.count;
    r.sum = s.sum;
    r.avg = s.avg;
    r.present = s.present;
    for (int j = 0; j < LH_MAX_PERCENTILES; j++) { r.pvals[j] = s.pvals[j]; r.pkeys[j] = s.pkeys[j]; }
    out[i] = r;
}

unsigned blocks_of(size_t n) { return (unsigned)((n + 255) / 256); }

// raises the kernel's dynamic shared-memory limit to `bytes` and launches it
template <typename Kernel, typename... Args>
int launch_smem(Kernel k, unsigned grid, dim3 block, uint32_t bytes, void *stream, Args... args) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return err(e);
    k<<<grid, block, bytes, (cudaStream_t)stream>>>(args...);
    return err(cudaGetLastError());
}

}  // namespace

// Every launcher enqueues its kernels on `stream` and returns the cudaError_t of the launch.  They run on this library's
// current device, which must be the device of the context the recorder or board came from.
LHM_API int lhm_set_device(int device) { return err(cudaSetDevice(device)); }

// k_estimate at the recorder's precision (c1 moved by c1_ulps float ulps) on `grid` CTAs (a power of two <= 2^20) of
// `threads`: d_hashes gets `grid` uint64, and the cells that left their cell are added to *d_left.
LHM_API int lhm_estimate(const lh_recorder *rec, int c1_ulps, unsigned grid, unsigned threads, void *d_hashes,
                         void *d_left, void *stream) {
    if (!grid || (grid & (grid - 1)) || grid > (1u << 20) || !threads) return err(cudaErrorInvalidValue);
    k_estimate<<<grid, threads, 0, (cudaStream_t)stream>>>(prec_of(rec, c1_ulps), (unsigned long long *)d_hashes,
                                                            (unsigned long long *)d_left);
    return err(cudaGetLastError());
}

LHM_API int lhm_estimate_cells(const lh_recorder *rec, int c1_ulps, uint32_t c_lo, uint32_t n, void *d_idx, void *d_slow,
                               void *d_w, void *stream) {
    if (!n) return 0;
    k_estimate_cells<<<blocks_of(2 * (size_t)n), 256, 0, (cudaStream_t)stream>>>(prec_of(rec, c1_ulps), c_lo, n,
                                                                                 (uint32_t *)d_idx, (uint8_t *)d_slow,
                                                                                 (float *)d_w);
    return err(cudaGetLastError());
}

// (uint16) lh::key16_of and lh::exact_key16 of n values at the recorder's precision
LHM_API int lhm_keys(const lh_recorder *rec, const void *d_vals, size_t n, void *d_fast, void *d_exact, void *stream) {
    if (!n) return 0;
    k_keys<<<264, 256, 0, (cudaStream_t)stream>>>(prec_of(rec, 0), (const double *)d_vals, n, (uint16_t *)d_fast,
                                                  (uint16_t *)d_exact);
    return err(cudaGetLastError());
}

// k_record<op> (op 0 record, 1 record_ns, 2 count) with `pattern` on `grid` CTAs of (bx, by, bz) threads
LHM_API int lhm_record(const lh_recorder *rec, int op, int pattern, const void *d_ids, const void *d_vals, size_t n,
                       unsigned grid, unsigned bx, unsigned by, unsigned bz, void *stream) {
    if (op < 0 || op > 2 || pattern < 0 || pattern > 2) return err(cudaErrorInvalidValue);
    if (!n) return 0;
    const dim3 block(bx, by, bz);
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t *ids = (const uint32_t *)d_ids;
    if (op == 0) k_record<0><<<grid, block, 0, s>>>(*rec, pattern, ids, d_vals, n);
    else if (op == 1) k_record<1><<<grid, block, 0, s>>>(*rec, pattern, ids, d_vals, n);
    else k_record<2><<<grid, block, 0, s>>>(*rec, pattern, ids, d_vals, n);
    return err(cudaGetLastError());
}

// k_block_histogram on `grid` CTAs (d_block_ids holds `grid` ids) with rec->block_smem_bytes + off bytes
LHM_API int lhm_block_histogram(const lh_recorder *rec, const void *d_block_ids, const void *d_vals, size_t n,
                                size_t chunk, int flushes, uint32_t off, unsigned grid, unsigned bx, unsigned by,
                                unsigned bz, void *stream) {
    if (!chunk || flushes < 1) return err(cudaErrorInvalidValue);
    return launch_smem(k_block_histogram, grid, dim3(bx, by, bz), rec->block_smem_bytes + off, stream, *rec,
                       (const uint32_t *)d_block_ids, (const double *)d_vals, n, chunk, flushes, off);
}

// k_block_recorder on `grid` CTAs with off + (dual ? 2 : 1) * BlockRecorder::smem_bytes(entries) bytes
LHM_API int lhm_block_recorder(const lh_recorder *rec, int op, const void *d_ids, const void *d_vals, size_t n,
                               size_t chunk, int flushes, uint32_t entries, uint32_t off, int dual, unsigned grid,
                               unsigned bx, unsigned by, unsigned bz, void *stream) {
    if (!chunk || flushes < 1 || op < 0 || op > 1) return err(cudaErrorInvalidValue);
    const uint32_t bytes = off + (dual ? 2u : 1u) * lh::BlockRecorder::smem_bytes(entries);
    return launch_smem(k_block_recorder, grid, dim3(bx, by, bz), bytes, stream, *rec, op, (const uint32_t *)d_ids,
                       d_vals, n, chunk, flushes, entries, off, dual);
}

// query i: (rows[i], ps[i]) -> keys[i], vals[i], pub[i]
LHM_API int lhm_raw_percentiles(const lh_raw_board *b, const void *d_rows, const void *d_ps, size_t n, void *d_keys,
                                void *d_vals, void *d_pub, void *stream) {
    if (!n) return 0;
    k_raw_percentiles<<<blocks_of(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, (const double *)d_ps,
                                                                      n, (int32_t *)d_keys, (double *)d_vals,
                                                                      (unsigned long long *)d_pub);
    return err(cudaGetLastError());
}

// query i: (rows[i], values[i]) -> ranks[i], totals[i], pub[i]
LHM_API int lhm_raw_ranks(const lh_raw_board *b, const void *d_rows, const void *d_values, size_t n, void *d_ranks,
                          void *d_totals, void *d_pub, void *stream) {
    if (!n) return 0;
    k_raw_ranks<<<blocks_of(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, (const double *)d_values,
                                                                n, (uint64_t *)d_ranks, (uint64_t *)d_totals,
                                                                (unsigned long long *)d_pub);
    return err(cudaGetLastError());
}

// query i: (rows[i], keys[i]) -> counts[i], pub[i]
LHM_API int lhm_raw_bucket_counts(const lh_raw_board *b, const void *d_rows, const void *d_keys, size_t n,
                                  void *d_counts, void *d_pub, void *stream) {
    if (!n) return 0;
    k_raw_bucket_counts<<<blocks_of(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows,
                                                                        (const int32_t *)d_keys, n, (uint64_t *)d_counts,
                                                                        (unsigned long long *)d_pub);
    return err(cudaGetLastError());
}

// query i: histogram row rows[i] -> out[i] (lh_board_hist_row), pub[i]
LHM_API int lhm_read_histograms(const lh_board *b, const void *d_rows, size_t n, void *d_out, void *d_pub,
                                void *stream) {
    if (!n) return 0;
    k_read_histograms<<<blocks_of(n), 256, 0, (cudaStream_t)stream>>>(*b, (const uint32_t *)d_rows, n,
                                                                      (lh_board_hist_row *)d_out,
                                                                      (unsigned long long *)d_pub);
    return err(cudaGetLastError());
}
#endif  // LHM_PART1

#ifdef LHM_PART2
namespace {

// lh::record of float64 values, every lane, from the second translation unit of the -rdc=true build
__global__ void __launch_bounds__(kMaxThreads)
k_record_part2(lh_recorder rec, const uint32_t *ids, const double *vals, size_t n) {
    for (size_t i = (size_t)blockIdx.x * thread_count() + thread_rank(); i < n; i += (size_t)gridDim.x * thread_count())
        lh::record(rec, ids[i], vals[i]);
}

}  // namespace

LHM_API int lhm_record_part2(const lh_recorder *rec, const void *d_ids, const void *d_vals, size_t n, unsigned grid,
                             unsigned threads, void *stream) {
    if (!n) return 0;
    k_record_part2<<<grid, threads, 0, (cudaStream_t)stream>>>(*rec, (const uint32_t *)d_ids, (const double *)d_vals, n);
    return err(cudaGetLastError());
}
#endif  // LHM_PART2
