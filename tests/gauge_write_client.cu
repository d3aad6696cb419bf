// gauge_write_client.cu -- a CUDA client of the device-gauge write API (include/loghisto_b200_device.cuh): kernels that
// write gauge cells with lh::set_gauge or with plain stores, knowing the library only through its public headers.
// Built by loghisto_b200/build.py (build_device_client) into tests/_build/ and used by tests/test_gpu_device_gauges.py.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

#define GWC_API extern "C" __attribute__((visibility("default")))

namespace {

template <typename T>
__device__ void set_bits(void *p, unsigned long long bits) {
    T v;
    __builtin_memcpy(&v, &bits, sizeof v);
    lh::set_gauge(static_cast<T *>(p), v);
}

// one thread: lh::set_gauge of the LH_GAUGE_* type `dtype` whose bit pattern is the low bytes of `bits`
__global__ void k_set(void *p, uint32_t dtype, unsigned long long bits) {
    switch (dtype) {
    case LH_GAUGE_F64: set_bits<double>(p, bits); break;
    case LH_GAUGE_F32: set_bits<float>(p, bits); break;
    case LH_GAUGE_F16: set_bits<__half>(p, bits); break;
    case LH_GAUGE_BF16: set_bits<__nv_bfloat16>(p, bits); break;
    case LH_GAUGE_I64: set_bits<int64_t>(p, bits); break;
    case LH_GAUGE_I32: set_bits<int32_t>(p, bits); break;
    default: set_bits<uint64_t>(p, bits); break;
    }
}

struct Flip {
    unsigned long long a[3], b[3];   // the two patterns of cells 0 (float64), 1 (int64), 2 (uint64)
};

// threads 0..2 alternate cell t between a[t] and b[t], `iters` times, with a short sleep between stores: strong stores
// through lh::set_gauge, or plain 8-byte stores (a compiler barrier keeps every one of them)
__global__ void k_flip(unsigned long long *cells, Flip f, int strong, unsigned long long iters) {
    const int t = threadIdx.x;
    if (t >= 3) return;
    for (unsigned long long i = 0; i < iters; i++) {
        const unsigned long long v = (i & 1) ? f.b[t] : f.a[t];
        if (strong) {
            if (t == 0) lh::set_gauge(reinterpret_cast<double *>(cells), __longlong_as_double((long long)v));
            else if (t == 1) lh::set_gauge(reinterpret_cast<int64_t *>(cells + 1), (int64_t)v);
            else lh::set_gauge(reinterpret_cast<uint64_t *>(cells + 2), (uint64_t)v);
        } else {
            cells[t] = v;
            asm volatile("" ::: "memory");
        }
        __nanosleep(100);
    }
}

}  // namespace

GWC_API int gwc_set(void *p, uint32_t dtype, uint64_t bits, void *stream) {
    k_set<<<1, 1, 0, (cudaStream_t)stream>>>(p, dtype, (unsigned long long)bits);
    return (int)cudaGetLastError();
}

GWC_API int gwc_flip(void *cells, const uint64_t *a, const uint64_t *b, int strong, uint64_t iters, void *stream) {
    Flip f;
    for (int i = 0; i < 3; i++) { f.a[i] = a[i]; f.b[i] = b[i]; }
    k_flip<<<1, 32, 0, (cudaStream_t)stream>>>((unsigned long long *)cells, f, strong, (unsigned long long)iters);
    return (int)cudaGetLastError();
}
