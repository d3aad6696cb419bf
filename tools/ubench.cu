// ubench.cu -- shared-memory primitive costs that decide the keyed-path design:
// returning vs non-returning ATOMS on ~132 spread addresses (one per SM-owner), MATCH.ANY, ballot-built peer masks, plain LDS/STS.
// Prints cycles per warp-level operation per SM at a given number of resident warps.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu && tools/ubench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int ITERS = 2048;
constexpr int UNROLL = 4;

__device__ __forceinline__ uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}

template <int MODE>
__global__ void __launch_bounds__(1024, 1) k_bench(uint32_t nbins, unsigned long long *out_cycles, uint32_t *sink) {
    extern __shared__ uint32_t sm[];
    for (uint32_t i = threadIdx.x; i < 8192; i += blockDim.x) sm[i] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *wsm = sm + 4096;                 // scratch beyond the bins
    uint32_t acc = 0;
    uint32_t state = mix(threadIdx.x * 2654435761u + blockIdx.x);
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
            state = state * 1664525u + 1013904223u;
            const uint32_t bin = __umulhi(state, nbins);       // uniform in [0, nbins)
            if (MODE == 0) { acc += bin; }                                             // baseline: index generation only
            if (MODE == 1) { acc += atomicAdd(&sm[bin], 1u); }                        // returning ATOMS.ADD
            if (MODE == 2) { atomicAdd(&sm[bin], 1u); }                               // non-returning (POPC.INC)
            if (MODE == 3) { atomicAdd(&sm[bin], (state >> 28) | 1u); }                // non-returning, arbitrary addend
            if (MODE == 4) { atomicOr(&sm[bin], 1u << lane); }                        // non-returning OR
            if (MODE == 5) { acc += __match_any_sync(0xFFFFFFFFu, bin); }             // MATCH.ANY
            if (MODE == 6) {                                                          // peers from 8 ballots
                uint32_t peers = 0xFFFFFFFFu;
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    const uint32_t m = __ballot_sync(0xFFFFFFFFu, (bin >> b) & 1u);
                    peers &= ((bin >> b) & 1u) ? m : ~m;
                }
                acc += peers;
            }
            if (MODE == 7) { acc += sm[bin]; }                                        // LDS, random bank
            if (MODE == 8) { sm[bin] = state; }                                       // STS, random bank
            if (MODE == 9) {                                                          // match + leader-only returning ATOMS + shfl
                const uint32_t peers = __match_any_sync(0xFFFFFFFFu, bin);
                const uint32_t leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd(&sm[bin], __popc(peers));
                base = __shfl_sync(0xFFFFFFFFu, base, leader);
                acc += base + __popc(peers & ((1u << lane) - 1u));
            }
            if (MODE == 10) {                                                         // warp-private counters: ballot peers + LDS + leader STS
                uint32_t peers = 0xFFFFFFFFu;
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    const uint32_t m = __ballot_sync(0xFFFFFFFFu, (bin >> b) & 1u);
                    peers &= ((bin >> b) & 1u) ? m : ~m;
                }
                uint32_t *cnt = wsm + warp * 160;     // needs warps*160 <= 4096 words
                const uint32_t base = cnt[bin];
                const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
                __syncwarp();
                if (rank == 0) cnt[bin] = base + __popc(peers);
                __syncwarp();
                acc += base + rank;
            }
            if (MODE == 11) {                                                         // same with MATCH.ANY
                const uint32_t peers = __match_any_sync(0xFFFFFFFFu, bin);
                uint32_t *cnt = wsm + warp * 160;
                const uint32_t base = cnt[bin];
                const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
                __syncwarp();
                if (rank == 0) cnt[bin] = base + __popc(peers);
                __syncwarp();
                acc += base + rank;
            }
            if (MODE == 12) { acc += atomicAdd(&sm[bin], 1u); acc += atomicAdd(&sm[2048 + bin], 1u); }   // two returning
            if (MODE == 13) { acc += atomicExch(&sm[bin], state); }                   // returning EXCH
            if (MODE == 14) {                                                         // 16-bit store to a random (bin, pos) slot
                reinterpret_cast<unsigned short *>(sm)[bin * 16 + (state >> 28)] = (unsigned short)state;
            }
        }
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) out_cycles[blockIdx.x] = (unsigned long long)(t1 - t0);
    if (acc == 0x12345678u) sink[0] = acc;
}

template <int MODE>
double run(const char *name, int warps, uint32_t nbins, double base, unsigned long long *d_cyc, uint32_t *d_sink) {
    const int grid = 148;
    cudaFuncSetAttribute(k_bench<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 4);
    k_bench<MODE><<<grid, warps * 32, 8192 * 4>>>(nbins, d_cyc, d_sink);
    k_bench<MODE><<<grid, warps * 32, 8192 * 4>>>(nbins, d_cyc, d_sink);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); return 0; }
    unsigned long long h[148];
    cudaMemcpy(h, d_cyc, sizeof h, cudaMemcpyDeviceToHost);
    double avg = 0; for (int i = 0; i < grid; i++) avg += (double)h[i]; avg /= grid;
    const double per_warp_op = avg / ((double)ITERS * UNROLL * warps);     // SM cycles per warp-level op
    printf("%-44s warps=%2d bins=%5u  cycles/warp-op/SM = %7.2f  (minus baseline %7.2f)  -> %6.2f samples/clk/SM\n",
           name, warps, nbins, per_warp_op, per_warp_op - base, 32.0 / per_warp_op);
    return per_warp_op;
}

int main() {
    unsigned long long *d_cyc; uint32_t *d_sink;
    cudaMalloc(&d_cyc, 148 * 8); cudaMalloc(&d_sink, 4);
    for (int warps : {8, 16, 32}) {
        for (uint32_t nbins : {148u, 4368u}) {
            if (nbins > 2048) {   // modes using two arrays / warp scratch assume bins <= 2048
                double b = run<0>("baseline (index generation)", warps, nbins, 0, d_cyc, d_sink);
                run<1>("ATOMS.ADD returning", warps, nbins, b, d_cyc, d_sink);
                run<2>("ATOMS.POPC.INC non-returning", warps, nbins, b, d_cyc, d_sink);
                run<3>("ATOMS.ADD non-returning, any addend", warps, nbins, b, d_cyc, d_sink);
                run<7>("LDS random", warps, nbins, b, d_cyc, d_sink);
                run<8>("STS random", warps, nbins, b, d_cyc, d_sink);
                continue;
            }
            double b = run<0>("baseline (index generation)", warps, nbins, 0, d_cyc, d_sink);
            run<1>("ATOMS.ADD returning", warps, nbins, b, d_cyc, d_sink);
            run<12>("2x ATOMS.ADD returning", warps, nbins, b, d_cyc, d_sink);
            run<13>("ATOMS.EXCH returning", warps, nbins, b, d_cyc, d_sink);
            run<2>("ATOMS.POPC.INC non-returning", warps, nbins, b, d_cyc, d_sink);
            run<3>("ATOMS.ADD non-returning, any addend", warps, nbins, b, d_cyc, d_sink);
            run<4>("ATOMS.OR non-returning", warps, nbins, b, d_cyc, d_sink);
            run<5>("MATCH.ANY", warps, nbins, b, d_cyc, d_sink);
            run<6>("peers from 8 ballots", warps, nbins, b, d_cyc, d_sink);
            run<7>("LDS random", warps, nbins, b, d_cyc, d_sink);
            run<8>("STS random", warps, nbins, b, d_cyc, d_sink);
            run<14>("STS.U16 random slot", warps, nbins, b, d_cyc, d_sink);
            run<9>("match + leader ATOMS + shfl", warps, nbins, b, d_cyc, d_sink);
            if (warps * 160 <= 4096) {
                run<10>("warp-private counters (ballot peers)", warps, nbins, b, d_cyc, d_sink);
                run<11>("warp-private counters (MATCH.ANY)", warps, nbins, b, d_cyc, d_sink);
            }
        }
    }
    return 0;
}
