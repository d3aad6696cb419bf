// gpu_timer_client.cu -- stream work of a known length for the GPU timer tests (tests/test_gpu_stream_timer.py) and
// tools/gpu_timer_probe.py: one thread spins until %globaltimer, the clock the timers read, has advanced by at least
// the requested number of nanoseconds.  Built by loghisto_b200/build.py build_device_client() into tests/_build/.
#include "loghisto_b200_device.cuh"

namespace {

__global__ void k_spin_ns(unsigned long long ns) {
    const uint64_t t0 = lh::globaltimer_ns();
    while (lh::globaltimer_ns() - t0 < ns) {}
}

}  // namespace

extern "C" {

int gtc_set_device(int device) { return (int)cudaSetDevice(device); }

// Enqueues one spin of at least `ns` on `stream` (0 = the legacy default stream) and returns the launch's cudaError_t.
int gtc_spin(uint64_t ns, void *stream) {
    k_spin_ns<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned long long)ns);
    return (int)cudaGetLastError();
}

}  // extern "C"
