// block_recorder_client.cu -- a CUDA translation unit that records into a loghisto context through lh::BlockRecorder,
// the per-CTA shared-memory combining table of the device API, knowing the library only through its two public headers.
// Built by loghisto_b200/build.py build_device_client() into tests/_build/; tests/test_gpu_block_recorder.py and
// tools/device_record_probe.py call the extern "C" launchers below through ctypes, with a recorder from a record scope
// and a stream of the same scope.
//
// Every launcher takes `chunk` and `entries`: CTA b handles samples [b*chunk, min(n, (b+1)*chunk)) through a table
// asked for `entries` slots (BlockRecorder::smem_bytes(entries) of dynamic shared memory).
#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

namespace {

constexpr int kThreads = 256;

struct Range {
    size_t lo, mid, hi;
};

// this CTA's samples; mid splits them where the kernel flushes once before the end (mid = hi: no mid-chunk flush)
__device__ Range cta_range(size_t n, size_t chunk, int mid_flush) {
    Range r;
    r.lo = (size_t)blockIdx.x * chunk;
    r.hi = r.lo + chunk < n ? r.lo + chunk : n;
    r.mid = mid_flush ? r.lo + (r.hi - r.lo) / 2 : r.hi;
    return r;
}

// keyed records; ids == nullptr: every sample goes to histogram 0
__global__ void __launch_bounds__(kThreads) k_br_record(lh_recorder rec, const uint32_t *ids, const double *vals, size_t n,
                                                        size_t chunk, uint32_t entries, int mid_flush) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, entries);
    br.init();
    const Range r = cta_range(n, chunk, mid_flush);
    for (size_t i = r.lo + threadIdx.x; i < r.mid; i += kThreads) br.record(ids ? ids[i] : 0u, vals[i]);
    if (mid_flush) br.flush();
    for (size_t i = r.mid + threadIdx.x; i < r.hi; i += kThreads) br.record(ids ? ids[i] : 0u, vals[i]);
    br.flush();
}

// only the samples whose lowest bit of the float64 pattern is set are recorded: a data-dependent subset of the lanes
__global__ void __launch_bounds__(kThreads) k_br_record_subset(lh_recorder rec, const uint32_t *ids, const double *vals,
                                                               size_t n, size_t chunk, uint32_t entries) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, entries);
    br.init();
    const Range r = cta_range(n, chunk, 0);
    for (size_t i = r.lo + threadIdx.x; i < r.hi; i += kThreads) {
        const double v = vals[i];
        if (__double_as_longlong(v) & 1) br.record(ids[i], v);
    }
    br.flush();
}

__global__ void __launch_bounds__(kThreads) k_br_record_ns(lh_recorder rec, const uint32_t *ids, const long long *ns,
                                                           size_t n, size_t chunk, uint32_t entries) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, entries);
    br.init();
    const Range r = cta_range(n, chunk, 1);
    for (size_t i = r.lo + threadIdx.x; i < r.mid; i += kThreads) br.record_ns(ids[i], ns[i]);
    br.flush();
    for (size_t i = r.mid + threadIdx.x; i < r.hi; i += kThreads) br.record_ns(ids[i], ns[i]);
    br.flush();
}

// spin until %globaltimer has advanced by at least `ns`
__device__ void spin_ns(uint64_t ns) {
    const uint64_t t0 = lh::globaltimer_ns();
    while (lh::globaltimer_ns() - t0 < ns) {}
}

// StartTimer(ids[i]) / Stop() through the table around a spin of (i % 17) * 100 ns; the durations go to out
__global__ void __launch_bounds__(kThreads) k_br_stop(lh_recorder rec, const uint32_t *ids, long long *out, size_t n,
                                                      size_t chunk, uint32_t entries) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, entries);
    br.init();
    const Range r = cta_range(n, chunk, 0);
    for (size_t i = r.lo + threadIdx.x; i < r.hi; i += kThreads) {
        const lh::TimerToken t = lh::start_timer(ids[i]);
        spin_ns((i % 17) * 100);
        out[i] = br.stop(t);
    }
    br.flush();
}

// ceil(n / chunk) CTAs with the table's shared memory, after raising the kernel's dynamic shared-memory limit to it
template <typename Kernel, typename... Args>
int launch(Kernel k, size_t n, size_t chunk, uint32_t entries, void *stream, Args... args) {
    if (!n || !chunk) return 0;
    const uint32_t bytes = lh::BlockRecorder::smem_bytes(entries);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return (int)e;
    const size_t grid = (n + chunk - 1) / chunk;
    k<<<(unsigned)grid, kThreads, bytes, (cudaStream_t)stream>>>(args...);
    return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

// The launchers run on this TU's current device: it must be the device of the context the recorder came from.
int brc_set_device(int device) { return (int)cudaSetDevice(device); }

// Each launcher enqueues one kernel on `stream` and returns the cudaError_t of the launch.
// mid_flush != 0: every CTA flushes after the first half of its chunk as well as at the end.
int brc_record(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, size_t chunk,
               uint32_t entries, int mid_flush, void *stream) {
    return launch(k_br_record, n, chunk, entries, stream, *rec, d_ids, d_vals, n, chunk, entries, mid_flush);
}

int brc_record_subset(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, size_t chunk,
                      uint32_t entries, void *stream) {
    return launch(k_br_record_subset, n, chunk, entries, stream, *rec, d_ids, d_vals, n, chunk, entries);
}

int brc_record_ns(const lh_recorder *rec, const uint32_t *d_ids, const int64_t *d_ns, size_t n, size_t chunk,
                  uint32_t entries, void *stream) {
    return launch(k_br_record_ns, n, chunk, entries, stream, *rec, d_ids, reinterpret_cast<const long long *>(d_ns), n,
                  chunk, entries);
}

int brc_stop(const lh_recorder *rec, const uint32_t *d_ids, int64_t *d_out, size_t n, size_t chunk, uint32_t entries,
             void *stream) {
    return launch(k_br_stop, n, chunk, entries, stream, *rec, d_ids, reinterpret_cast<long long *>(d_out), n, chunk,
                  entries);
}

}  // extern "C"
