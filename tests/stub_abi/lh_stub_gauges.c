/*
 * lh_stub_gauges.c -- TEST-ONLY device gauges for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_device_gauges_cpu.py compiles it with lh_stub.c and oracle/loghisto_oracle.c, so that
 * MetricSystem::RegisterDeviceGauge and the gauge step of collectRawMetrics (loghisto_b200/host/metric_system.cc) run
 * on the CPU.  "Device" memory here is host memory handed out by lh_stub_gauge_alloc: lh_gauges_read refuses, as the
 * real library does, any address that is not inside such an allocation, so freeing one (lh_stub_gauge_free) makes
 * every later read that includes it fail.  Values are converted as Go's float64(x) is.  lh_stub_gauge_reads counts the
 * reads that got past validation (the real library launches its kernel only then).
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_ALLOCS 64

static pthread_mutex_t g_gmu = PTHREAD_MUTEX_INITIALIZER;
static struct { char *p; size_t bytes; } g_allocs[MAX_ALLOCS];
static uint64_t g_reads;

static const uint32_t kBytes[] = {8, 4, 2, 2, 8, 4, 8};

static int inside(const void *p, size_t n) {
    for (int i = 0; i < MAX_ALLOCS; i++)
        if (g_allocs[i].p && (const char *)p >= g_allocs[i].p && (const char *)p + n <= g_allocs[i].p + g_allocs[i].bytes)
            return 1;
    return 0;
}

static double half_to_double(uint16_t h) {
    const int e = (h >> 10) & 31, m = h & 1023;
    const double s = (h & 0x8000) ? -1.0 : 1.0;
    if (e == 31) return m ? NAN : s * INFINITY;
    if (e == 0) return s * ldexp((double)m, -24);
    return s * ldexp((double)(m | 1024), e - 25);
}

LH_API lh_status lh_gauges_read(lh_ctx *ctx, const lh_gauge_src *h_srcs, uint32_t n, double *h_out) {
    if (!ctx || (n && (!h_srcs || !h_out))) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_gmu);
    for (uint32_t i = 0; i < n; i++) {
        const lh_gauge_src *s = &h_srcs[i];
        if (s->dtype > LH_GAUGE_U64 || s->reserved || !s->d_value || ((uintptr_t)s->d_value & (kBytes[s->dtype] - 1)) ||
            !inside(s->d_value, kBytes[s->dtype])) {
            pthread_mutex_unlock(&g_gmu);
            return LH_ERR_INVALID;
        }
    }
    if (n) g_reads++;
    for (uint32_t i = 0; i < n; i++) {
        const void *p = h_srcs[i].d_value;
        switch (h_srcs[i].dtype) {
        case LH_GAUGE_F64: h_out[i] = *(const double *)p; break;
        case LH_GAUGE_F32: h_out[i] = (double)*(const float *)p; break;
        case LH_GAUGE_F16: h_out[i] = half_to_double(*(const uint16_t *)p); break;
        case LH_GAUGE_BF16: {
            const uint32_t u = (uint32_t)*(const uint16_t *)p << 16;
            float f;
            memcpy(&f, &u, 4);
            h_out[i] = (double)f;
            break;
        }
        case LH_GAUGE_I64: h_out[i] = (double)*(const int64_t *)p; break;
        case LH_GAUGE_I32: h_out[i] = (double)*(const int32_t *)p; break;
        default: h_out[i] = (double)*(const uint64_t *)p; break;
        }
    }
    pthread_mutex_unlock(&g_gmu);
    return LH_OK;
}

/* zeroed "device" memory that lh_gauges_read accepts, 8-byte aligned */
LH_API void *lh_stub_gauge_alloc(size_t bytes) {
    pthread_mutex_lock(&g_gmu);
    for (int i = 0; i < MAX_ALLOCS; i++) {
        if (g_allocs[i].p) continue;
        g_allocs[i].p = (char *)calloc(1, bytes ? bytes : 1);
        g_allocs[i].bytes = bytes;
        pthread_mutex_unlock(&g_gmu);
        return g_allocs[i].p;
    }
    pthread_mutex_unlock(&g_gmu);
    return 0;
}

LH_API void lh_stub_gauge_free(void *p) {
    pthread_mutex_lock(&g_gmu);
    for (int i = 0; i < MAX_ALLOCS; i++)
        if (g_allocs[i].p == p) { free(p); g_allocs[i].p = 0; g_allocs[i].bytes = 0; }
    pthread_mutex_unlock(&g_gmu);
}

/* lh_gauges_read calls with n > 0 that passed validation */
LH_API uint64_t lh_stub_gauge_reads(void) {
    pthread_mutex_lock(&g_gmu);
    const uint64_t n = g_reads;
    pthread_mutex_unlock(&g_gmu);
    return n;
}
