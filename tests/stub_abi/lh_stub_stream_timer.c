/*
 * lh_stub_stream_timer.c -- TEST-ONLY GPU timers for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_stream_timer_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c and
 * oracle/loghisto_oracle.c, so that MetricSystem::StartGpuTimer / GpuTimerToken::Stop
 * (loghisto_b200/host/metric_system.cc) run on the CPU.  The host's CLOCK_MONOTONIC stands in for %globaltimer, and a
 * stop records its one sample through the stub's lh_ingest_f64 (lh_stub_record.c).  It adds:
 *   lh_stub_gpu_timer_pool     forgets every pool and sets the slots of the pools made after it (default 65536);
 *   lh_stub_gpu_timer_stream   the stream the latest start or stop was given (the Python stream mapping shows here);
 *   lh_stub_gpu_timer_stops    how many stops were recorded.
 * There is no device, so a released slot is free at once.  "Device" pointers are host pointers.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <time.h>

#include "loghisto_b200.h"

#define MAX_CTX 64

static pthread_mutex_t g_tmu = PTHREAD_MUTEX_INITIALIZER;
static uint32_t g_pool_size = 65536;
static void *g_last_stream = 0;
static uint64_t g_stops = 0;
static struct { lh_ctx *ctx; uint32_t n; uint64_t *start; uint32_t *gen; uint8_t *held; } g_pools[MAX_CTX];

/* forgets every pool (a context created after a destroyed one may reuse its address) and sizes the next ones */
LH_API void lh_stub_gpu_timer_pool(uint32_t n) {
    pthread_mutex_lock(&g_tmu);
    for (int i = 0; i < MAX_CTX; i++) {
        free(g_pools[i].start); free(g_pools[i].gen); free(g_pools[i].held);
        g_pools[i].ctx = 0; g_pools[i].start = 0; g_pools[i].gen = 0; g_pools[i].held = 0; g_pools[i].n = 0;
    }
    g_pool_size = n;
    g_stops = 0;
    g_last_stream = 0;
    pthread_mutex_unlock(&g_tmu);
}
LH_API void *lh_stub_gpu_timer_stream(void) {
    pthread_mutex_lock(&g_tmu);
    void *s = g_last_stream;
    pthread_mutex_unlock(&g_tmu);
    return s;
}
LH_API uint64_t lh_stub_gpu_timer_stops(void) {
    pthread_mutex_lock(&g_tmu);
    uint64_t n = g_stops;
    pthread_mutex_unlock(&g_tmu);
    return n;
}

static uint64_t now_ns(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}

/* the pool of ctx, created on first use (called locked) */
static int pool_of(lh_ctx *ctx) {
    for (int i = 0; i < MAX_CTX; i++)
        if (g_pools[i].ctx == ctx) return i;
    for (int i = 0; i < MAX_CTX; i++)
        if (!g_pools[i].ctx) {
            g_pools[i].ctx = ctx;
            g_pools[i].n = g_pool_size;
            g_pools[i].start = (uint64_t *)calloc(g_pool_size, 8);
            g_pools[i].gen = (uint32_t *)calloc(g_pool_size, 4);
            g_pools[i].held = (uint8_t *)calloc(g_pool_size, 1);
            return i;
        }
    return -1;
}

/* handle = pool index (8 bits) | generation (32 bits) | slot (24 bits); the held slot it names, or -1 (called locked) */
static uint64_t handle_of(int p, uint32_t k) { return (uint64_t)(p + 1) << 56 | (uint64_t)g_pools[p].gen[k] << 24 | k; }
static int slot_of(lh_ctx *ctx, const lh_gpu_timer *t, int *pool) {
    const int p = t ? pool_of(ctx) : -1;
    if (p < 0) return -1;
    const uint32_t k = (uint32_t)(t->handle & 0xFFFFFFu);
    if (k >= g_pools[p].n || !g_pools[p].held[k] || t->handle != handle_of(p, k)) return -1;
    *pool = p;
    return (int)k;
}

LH_API lh_status lh_gpu_timer_start(lh_ctx *ctx, void *stream, lh_gpu_timer *out) {
    if (!ctx || !out) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_tmu);
    g_last_stream = stream;
    const int p = pool_of(ctx);
    lh_status st = p < 0 ? LH_ERR_NOMEM : LH_ERR_RANGE;
    for (uint32_t k = 0; p >= 0 && k < g_pools[p].n; k++)
        if (!g_pools[p].held[k]) {
            g_pools[p].held[k] = 1;
            g_pools[p].start[k] = now_ns();
            out->handle = handle_of(p, k);
            st = LH_OK;
            break;
        }
    pthread_mutex_unlock(&g_tmu);
    return st;
}

LH_API lh_status lh_gpu_timer_stop(lh_ctx *ctx, const lh_gpu_timer *t, uint32_t histogram_id, void *stream,
                                   int64_t *d_duration_ns) {
    if (!ctx) return LH_ERR_INVALID;
    if (histogram_id >= ((const lh_config *)ctx)->max_histograms) return LH_ERR_RANGE;
    pthread_mutex_lock(&g_tmu);
    g_last_stream = stream;
    int p = -1;
    const int k = slot_of(ctx, t, &p);
    const int64_t ns = k < 0 ? 0 : (int64_t)(now_ns() - g_pools[p].start[k]);
    if (k >= 0) g_stops++;
    pthread_mutex_unlock(&g_tmu);
    if (k < 0) return LH_ERR_INVALID;
    const double v = (double)ns;
    if (d_duration_ns) *d_duration_ns = ns;
    return lh_ingest_f64(ctx, histogram_id, &v, 1, stream);
}

LH_API lh_status lh_gpu_timer_release(lh_ctx *ctx, const lh_gpu_timer *t) {
    if (!ctx) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_tmu);
    int p = -1;
    const int k = slot_of(ctx, t, &p);
    if (k >= 0) {
        g_pools[p].held[k] = 0;
        g_pools[p].gen[k]++;
    }
    pthread_mutex_unlock(&g_tmu);
    return k < 0 ? LH_ERR_INVALID : LH_OK;
}
