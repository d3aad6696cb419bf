// device_record_client.cu -- a CUDA translation unit that records into a loghisto context from its own kernels, knowing
// the library only through its two public headers (no link against libloghisto_b200.so: the recorder carries every
// device pointer).  Built by loghisto_b200/build.py build_device_client() into tests/_build/; the tests and
// tools/device_record_probe.py call the extern "C" launchers below through ctypes, with a recorder from
// Engine.record_begin and a stream of the same scope.
#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

namespace {

constexpr int kThreads = 256;

int grid_for(size_t n, int per_sm) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t need = (n + kThreads - 1) / kThreads;
    const size_t cap = (size_t)sms * per_sm;
    return (int)(need < 1 ? 1 : (need < cap ? need : cap));
}

// ids == nullptr: every sample goes to histogram 0
__global__ void __launch_bounds__(kThreads) k_record(lh_recorder rec, const uint32_t *ids, const double *vals, size_t n) {
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        lh::record(rec, ids ? ids[i] : 0u, vals[i]);
}

// only the samples whose lowest bit of the float64 pattern is set are recorded: a data-dependent subset of the lanes
__global__ void __launch_bounds__(kThreads) k_record_subset(lh_recorder rec, const uint32_t *ids, const double *vals, size_t n) {
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
        const double v = vals[i];
        if (__double_as_longlong(v) & 1) lh::record(rec, ids[i], v);
    }
}

__global__ void __launch_bounds__(kThreads) k_record_ns(lh_recorder rec, const uint32_t *ids, const long long *ns, size_t n) {
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        lh::record_ns(rec, ids[i], ns[i]);
}

__global__ void __launch_bounds__(kThreads) k_count(lh_recorder rec, const uint32_t *ids, const unsigned long long *amounts, size_t n) {
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        lh::count(rec, ids[i], amounts[i]);
}

// CTA b records samples [b*chunk, min(n, (b+1)*chunk)) into histogram block_ids[b], flushing once after the first
// half of its chunk and once at the end (so a sub-histogram is reused after a flush)
__global__ void __launch_bounds__(kThreads) k_block(lh_recorder rec, const uint32_t *block_ids, const double *vals, size_t n, size_t chunk) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockHistogram bh(rec, smem);
    bh.init(block_ids[blockIdx.x]);
    const size_t lo = (size_t)blockIdx.x * chunk;
    const size_t hi = lo + chunk < n ? lo + chunk : n;
    const size_t mid = lo + (hi - lo) / 2;
    for (size_t i = lo + threadIdx.x; i < mid; i += kThreads) bh.add(vals[i]);
    bh.flush();
    for (size_t i = mid + threadIdx.x; i < hi; i += kThreads) bh.add(vals[i]);
    bh.flush();
}

}  // namespace

extern "C" {

// The launchers run on this TU's current device: it must be the device of the context the recorder came from.
int lhc_set_device(int device) { return (int)cudaSetDevice(device); }

// Each launcher enqueues one kernel on `stream` and returns the cudaError_t of the launch.
int lhc_record(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, void *stream) {
    if (n) k_record<<<grid_for(n, 8), kThreads, 0, (cudaStream_t)stream>>>(*rec, d_ids, d_vals, n);
    return (int)cudaGetLastError();
}

int lhc_record_subset(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, void *stream) {
    if (n) k_record_subset<<<grid_for(n, 8), kThreads, 0, (cudaStream_t)stream>>>(*rec, d_ids, d_vals, n);
    return (int)cudaGetLastError();
}

int lhc_record_ns(const lh_recorder *rec, const uint32_t *d_ids, const int64_t *d_ns, size_t n, void *stream) {
    if (n) k_record_ns<<<grid_for(n, 8), kThreads, 0, (cudaStream_t)stream>>>(*rec, d_ids, reinterpret_cast<const long long *>(d_ns), n);
    return (int)cudaGetLastError();
}

int lhc_count(const lh_recorder *rec, const uint32_t *d_ids, const uint64_t *d_amounts, size_t n, void *stream) {
    if (n) k_count<<<grid_for(n, 8), kThreads, 0, (cudaStream_t)stream>>>(*rec, d_ids, reinterpret_cast<const unsigned long long *>(d_amounts), n);
    return (int)cudaGetLastError();
}

// ceil(n / chunk) CTAs; d_block_ids holds one histogram id per CTA
int lhc_block(const lh_recorder *rec, const uint32_t *d_block_ids, const double *d_vals, size_t n, size_t chunk, void *stream) {
    if (!n || !chunk) return 0;
    cudaError_t e = cudaFuncSetAttribute(k_block, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rec->block_smem_bytes);
    if (e != cudaSuccess) return (int)e;
    const size_t grid = (n + chunk - 1) / chunk;
    k_block<<<(unsigned)grid, kThreads, rec->block_smem_bytes, (cudaStream_t)stream>>>(*rec, d_block_ids, d_vals, n, chunk);
    return (int)cudaGetLastError();
}

}  // extern "C"
