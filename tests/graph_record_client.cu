// graph_record_client.cu -- a CUDA translation unit that records through the device API from kernels meant to be
// captured into CUDA graphs, with the recorder of a graph recorder (lh_graph_recorder_create), knowing the library only
// through its two public headers.  Built by loghisto_b200/build.py build_device_client() into tests/_build/;
// tests/test_gpu_graph_recorder.py and tools/graph_record_probe.py call the extern "C" functions below through ctypes.
#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

namespace {

constexpr int kThreads = 256;

// lh::record of (ids[i], vals[i]), lh::record_ns of (ns_ids[i], ns[i]), lh::count of (cids[i], amounts[i])
__global__ void __launch_bounds__(kThreads) k_gr_scalar(lh_recorder rec, const uint32_t *ids, const double *vals, size_t n,
                                                        const uint32_t *ns_ids, const long long *ns, size_t n_ns,
                                                        const uint32_t *cids, const unsigned long long *amounts, size_t n_c) {
    const size_t stride = (size_t)gridDim.x * kThreads;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) lh::record(rec, ids[i], vals[i]);
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n_ns; i += stride) lh::record_ns(rec, ns_ids[i], ns[i]);
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n_c; i += stride) lh::count(rec, cids[i], amounts[i]);
}

// CTA b feeds samples [b*chunk, (b+1)*chunk) of vals into histogram `id` through lh::BlockHistogram
__global__ void __launch_bounds__(kThreads) k_gr_block_hist(lh_recorder rec, uint32_t id, const double *vals, size_t n,
                                                            size_t chunk) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockHistogram bh(rec, smem);
    bh.init(id);
    const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
    for (size_t i = lo + threadIdx.x; i < hi; i += kThreads) bh.add(vals[i]);
    bh.flush();
}

// the same through lh::BlockRecorder with a table asked for `entries` slots, under ids[i]
__global__ void __launch_bounds__(kThreads) k_gr_block_rec(lh_recorder rec, const uint32_t *ids, const double *vals,
                                                           size_t n, size_t chunk, uint32_t entries) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, entries);
    br.init();
    const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
    for (size_t i = lo + threadIdx.x; i < hi; i += kThreads) br.record(ids[i], vals[i]);
    br.flush();
}

unsigned grid_of(size_t n, size_t chunk) { return (unsigned)((n + chunk - 1) / chunk); }

}  // namespace

extern "C" {

int grc_set_device(int device) { return (int)cudaSetDevice(device); }

// Raises the dynamic shared-memory limits the launchers need; call it before a capture (and once per process).
int grc_prepare(uint32_t block_smem_bytes, uint32_t entries) {
    cudaError_t e = cudaFuncSetAttribute(k_gr_block_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)block_smem_bytes);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(k_gr_block_rec, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)lh::BlockRecorder::smem_bytes(entries));
    return (int)e;
}

// One step of a client: enqueues on `stream` (capturable: launches only) the lh::record / record_ns / count kernel,
// BlockHistogram of vals into histogram bh_id and BlockRecorder of (ids, vals) with `entries` slots.  Returns the
// cudaError_t of the launches.
int grc_step(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, const uint32_t *d_ns_ids,
             const int64_t *d_ns, size_t n_ns, const uint32_t *d_cids, const uint64_t *d_amounts, size_t n_c,
             uint32_t bh_id, uint32_t entries, size_t chunk, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const size_t most = n > n_ns ? (n > n_c ? n : n_c) : (n_ns > n_c ? n_ns : n_c);
    if (most) {
        k_gr_scalar<<<grid_of(most, 4 * kThreads) < 1024 ? grid_of(most, 4 * kThreads) : 1024, kThreads, 0, s>>>(
            *rec, d_ids, d_vals, n, d_ns_ids, reinterpret_cast<const long long *>(d_ns), n_ns, d_cids,
            reinterpret_cast<const unsigned long long *>(d_amounts), n_c);
    }
    if (n) {
        k_gr_block_hist<<<grid_of(n, chunk), kThreads, rec->block_smem_bytes, s>>>(*rec, bh_id, d_vals, n, chunk);
        k_gr_block_rec<<<grid_of(n, chunk), kThreads, lh::BlockRecorder::smem_bytes(entries), s>>>(*rec, d_ids, d_vals, n,
                                                                                                    chunk, entries);
    }
    return (int)cudaGetLastError();
}

// Only lh::record of (ids, vals) through a BlockRecorder (entries slots, 0 = every sample on the direct path): the
// replay-cost workload of tools/graph_record_probe.py.
int grc_block_record(const lh_recorder *rec, const uint32_t *d_ids, const double *d_vals, size_t n, uint32_t entries,
                     size_t chunk, void *stream) {
    if (!n) return 0;
    k_gr_block_rec<<<grid_of(n, chunk), kThreads, lh::BlockRecorder::smem_bytes(entries), (cudaStream_t)stream>>>(
        *rec, d_ids, d_vals, n, chunk, entries);
    return (int)cudaGetLastError();
}

}  // extern "C"
