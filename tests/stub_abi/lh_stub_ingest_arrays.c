/*
 * lh_stub_ingest_arrays.c -- TEST-ONLY lh_ingest_arrays for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_array_ingest_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c and
 * oracle/loghisto_oracle.c, so that RecordScope::Arrays (loghisto_b200/host/metric_system.cc), lhms_arrays_scope and
 * the Python marshalling run on the CPU; built with lh_stub_batch.c and lh_stub_graph.c as well, its
 * lh_graph_recorder_ingest_arrays runs GraphRecorder::Arrays and lhms_arrays_graph_recorder, through lh_stub_graph.c's
 * lh_graph_recorder_ingest.  It validates the call as the library does (nothing is recorded when an item
 * is refused), then converts every element to float64 as C converts it (floats and int32 exactly, int64 / uint64 to
 * nearest) and records it through the stub's lh_ingest_f64.  It adds:
 *   lh_stub_arrays_calls   how many calls were accepted with at least one sample;
 *   lh_stub_arrays_last    the items and the stream of the latest call (accepted or not).
 * "Device" pointers are host pointers here.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_KEPT 4096

static pthread_mutex_t g_amu = PTHREAD_MUTEX_INITIALIZER;
static uint64_t g_calls = 0;
static lh_array_src g_last[MAX_KEPT];
static uint32_t g_last_n = 0;
static void *g_last_stream = 0;
static const uint32_t k_bytes[] = {8, 4, 2, 2, 8, 4, 8};

LH_API uint64_t lh_stub_arrays_calls(void) {
    pthread_mutex_lock(&g_amu);
    uint64_t n = g_calls;
    pthread_mutex_unlock(&g_amu);
    return n;
}
/* copies up to `cap` items of the latest call to out; returns its n_srcs and sets *stream */
LH_API uint32_t lh_stub_arrays_last(lh_array_src *out, uint32_t cap, void **stream) {
    pthread_mutex_lock(&g_amu);
    const uint32_t n = g_last_n;
    memcpy(out, g_last, sizeof(lh_array_src) * (n < cap ? n : cap));
    if (stream) *stream = g_last_stream;
    pthread_mutex_unlock(&g_amu);
    return n;
}

static double f16_to_double(uint16_t h) {
    const uint32_t e = (h >> 10) & 31u, m = h & 1023u;
    double v;
    if (e == 0) v = (double)m * (1.0 / 16777216.0);                  /* m * 2^-24 */
    else if (e == 31) v = m ? __builtin_nan("") : __builtin_inf();
    else v = (double)(m | 1024u) * (double)(1ull << e) / 33554432.0;  /* (1024 + m) * 2^(e - 25) */
    return (h & 0x8000u) ? -v : v;
}

static double element(const void *p, uint32_t dtype, uint64_t j) {
    switch (dtype) {
    case LH_GAUGE_F64: return ((const double *)p)[j];
    case LH_GAUGE_F32: return (double)((const float *)p)[j];
    case LH_GAUGE_F16: return f16_to_double(((const uint16_t *)p)[j]);
    case LH_GAUGE_BF16: {
        const uint32_t b = (uint32_t)((const uint16_t *)p)[j] << 16;
        float f;
        memcpy(&f, &b, 4);
        return (double)f;
    }
    case LH_GAUGE_I64: return (double)((const int64_t *)p)[j];
    case LH_GAUGE_I32: return (double)((const int32_t *)p)[j];
    default: return (double)((const uint64_t *)p)[j];
    }
}

LH_API lh_status lh_ingest_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs, void *stream) {
    if (!ctx) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_amu);
    g_last_n = h_srcs ? n_srcs : 0;
    if (h_srcs) memcpy(g_last, h_srcs, sizeof(lh_array_src) * (n_srcs < MAX_KEPT ? n_srcs : MAX_KEPT));
    g_last_stream = stream;
    pthread_mutex_unlock(&g_amu);
    if (n_srcs && !h_srcs) return LH_ERR_INVALID;
    const uint32_t H = ((const lh_config *)ctx)->max_histograms;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n_srcs; i++) {
        const lh_array_src *a = &h_srcs[i];
        if (a->dtype > LH_GAUGE_U64) return LH_ERR_INVALID;
        if (!a->n) continue;
        if (!a->d_values || ((uintptr_t)a->d_values & (k_bytes[a->dtype] - 1u))) return LH_ERR_INVALID;
        if (a->histogram_id >= H) return LH_ERR_RANGE;
        total += a->n;
    }
    if (!total) return LH_OK;
    for (uint32_t i = 0; i < n_srcs; i++) {
        const lh_array_src *a = &h_srcs[i];
        if (!a->n) continue;
        double *v = (double *)malloc(sizeof(double) * (size_t)a->n);
        if (!v) return LH_ERR_NOMEM;
        for (uint64_t j = 0; j < a->n; j++) v[j] = element(a->d_values, a->dtype, j);
        lh_status st = lh_ingest_f64(ctx, a->histogram_id, v, (size_t)a->n, stream);
        free(v);
        if (st != LH_OK) return st;
    }
    pthread_mutex_lock(&g_amu);
    g_calls++;
    pthread_mutex_unlock(&g_amu);
    return LH_OK;
}

/* The graph recorder form (needs lh_stub_graph.c): the items checked as lh_ingest_arrays checks them, converted, then
 * handed to the stub's lh_graph_recorder_ingest as float64 items in one call, which checks the ids against the
 * recorder's k before it records anything. */
LH_API lh_status lh_graph_recorder_ingest_arrays(lh_ctx *ctx, const lh_graph_recorder *g, const lh_array_src *h_srcs,
                                                 uint32_t n_srcs, void *stream) {
    if (!ctx || !g || (n_srcs && !h_srcs)) return LH_ERR_INVALID;
    for (uint32_t i = 0; i < n_srcs; i++) {
        const lh_array_src *a = &h_srcs[i];
        if (a->dtype > LH_GAUGE_U64) return LH_ERR_INVALID;
        if (a->n && (!a->d_values || ((uintptr_t)a->d_values & (k_bytes[a->dtype] - 1u)))) return LH_ERR_INVALID;
    }
    lh_batch_item *items = (lh_batch_item *)calloc(n_srcs ? n_srcs : 1, sizeof(lh_batch_item));
    double **vals = (double **)calloc(n_srcs ? n_srcs : 1, sizeof(double *));
    lh_status st = items && vals ? LH_OK : LH_ERR_NOMEM;
    for (uint32_t i = 0; st == LH_OK && i < n_srcs; i++) {
        const lh_array_src *a = &h_srcs[i];
        vals[i] = (double *)malloc(sizeof(double) * (size_t)(a->n ? a->n : 1));
        if (!vals[i]) { st = LH_ERR_NOMEM; break; }
        for (uint64_t j = 0; j < a->n; j++) vals[i][j] = element(a->d_values, a->dtype, j);
        items[i] = (lh_batch_item){vals[i], a->n, a->histogram_id, LH_VALUES_F64};
    }
    if (st == LH_OK) st = lh_graph_recorder_ingest(ctx, g, items, n_srcs, stream);
    for (uint32_t i = 0; vals && i < n_srcs; i++) free(vals[i]);
    free(vals);
    free(items);
    return st;
}
