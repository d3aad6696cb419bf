// named_record_client.cu -- a CUDA translation unit that records under MetricSystem names from its own kernels: the ids
// come from a name-bound record scope (MetricSystem::BeginRecording / lhms_record_begin, MetricSystem.recording in
// Python), the recorder is passed by value.  It knows the library only through its two public headers.  Built by
// loghisto_b200/build.py build_device_client() into tests/_build/; tests/test_gpu_named_recording.py and
// tools/globaltimer_probe.py call the extern "C" launchers below through ctypes.
#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

namespace {

constexpr int kThreads = 256;

unsigned grid_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// n samples of one histogram id
__global__ void __launch_bounds__(kThreads) k_record_one(lh_recorder rec, uint32_t id, const double *vals, size_t n) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) lh::record(rec, id, vals[i]);
}

// n counter ops of `amount` on one counter id
__global__ void __launch_bounds__(kThreads) k_count_one(lh_recorder rec, uint32_t id, unsigned long long amount, size_t n) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) lh::count(rec, id, amount);
}

// spin until %globaltimer has advanced by at least `ns` (a duration to measure)
__device__ void spin_ns(uint64_t ns) {
    const uint64_t t0 = lh::globaltimer_ns();
    while (lh::globaltimer_ns() - t0 < ns) {}
}

// StartTimer / Stop in one thread around a spin of (i % 17) * 250 ns; the durations are written to out
__global__ void __launch_bounds__(kThreads) k_timer_pair(lh_recorder rec, uint32_t id, long long *out, size_t n) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const lh::TimerToken t = lh::start_timer(id);
    spin_ns((i % 17) * 250);
    out[i] = lh::stop(rec, t);
}

// the producer half: tokens written to memory, stopped by a later kernel
__global__ void __launch_bounds__(kThreads) k_timer_start(lh::TimerToken *tok, uint32_t id, size_t n) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) tok[i] = lh::start_timer(id);
}
__global__ void __launch_bounds__(kThreads) k_timer_stop(lh_recorder rec, const lh::TimerToken *tok, long long *out, size_t n) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) out[i] = lh::stop(rec, tok[i]);
}

// One thread reads %globaltimer back to back and keeps the first n values that differ from the previous one.
__global__ void k_globaltimer_probe(unsigned long long *out, int n, unsigned long long max_reads) {
    uint64_t prev = lh::globaltimer_ns();
    int k = 0;
    for (unsigned long long r = 0; r < max_reads && k < n; r++) {
        const uint64_t t = lh::globaltimer_ns();
        if (t != prev) { out[k++] = t; prev = t; }
    }
    for (; k < n; k++) out[k] = 0;
}

}  // namespace

extern "C" {

int nrc_set_device(int device) { return (int)cudaSetDevice(device); }

// Each launcher enqueues one kernel on `stream` and returns the cudaError_t of the launch.
int nrc_record_one(const lh_recorder *rec, uint32_t id, const double *d_vals, size_t n, void *stream) {
    if (n) k_record_one<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(*rec, id, d_vals, n);
    return (int)cudaGetLastError();
}

int nrc_count_one(const lh_recorder *rec, uint32_t id, uint64_t amount, size_t n, void *stream) {
    if (n) k_count_one<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(*rec, id, (unsigned long long)amount, n);
    return (int)cudaGetLastError();
}

int nrc_timer_pair(const lh_recorder *rec, uint32_t id, int64_t *d_out, size_t n, void *stream) {
    if (n) k_timer_pair<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(*rec, id, reinterpret_cast<long long *>(d_out), n);
    return (int)cudaGetLastError();
}

// d_tokens: n * 16 bytes
int nrc_timer_start(void *d_tokens, uint32_t id, size_t n, void *stream) {
    if (n) k_timer_start<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(static_cast<lh::TimerToken *>(d_tokens), id, n);
    return (int)cudaGetLastError();
}

int nrc_timer_stop(const lh_recorder *rec, const void *d_tokens, int64_t *d_out, size_t n, void *stream) {
    if (n)
        k_timer_stop<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(*rec, static_cast<const lh::TimerToken *>(d_tokens),
                                                                         reinterpret_cast<long long *>(d_out), n);
    return (int)cudaGetLastError();
}

int nrc_globaltimer_probe(uint64_t *d_out, int n, uint64_t max_reads, void *stream) {
    k_globaltimer_probe<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<unsigned long long *>(d_out), n,
                                                           (unsigned long long)max_reads);
    return (int)cudaGetLastError();
}

}  // extern "C"
