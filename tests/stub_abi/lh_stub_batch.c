/*
 * lh_stub_batch.c -- TEST-ONLY lh_ingest_batch for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_batch_ingest_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c and
 * oracle/loghisto_oracle.c, so that RecordScope::Histograms (loghisto_b200/host/metric_system.cc) and
 * Engine.ingest_batch's marshalling run on the CPU.  It validates a batch as the library does (nothing is recorded when
 * an item is refused), then records every item through the stub's lh_ingest_f64 (lh_stub_record.c); int64 nanoseconds
 * become float64(ns), round-to-nearest.  It adds:
 *   lh_stub_batch_calls   how many calls were accepted with at least one sample;
 *   lh_stub_batch_last    the items and the stream of the latest call (accepted or not).
 * "Device" pointers are host pointers here.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_KEPT 4096

static pthread_mutex_t g_bmu = PTHREAD_MUTEX_INITIALIZER;
static uint64_t g_calls = 0;
static lh_batch_item g_last[MAX_KEPT];
static uint32_t g_last_n = 0;
static void *g_last_stream = 0;

LH_API uint64_t lh_stub_batch_calls(void) {
    pthread_mutex_lock(&g_bmu);
    uint64_t n = g_calls;
    pthread_mutex_unlock(&g_bmu);
    return n;
}
/* copies up to `cap` items of the latest call to out; returns its n_items and sets *stream */
LH_API uint32_t lh_stub_batch_last(lh_batch_item *out, uint32_t cap, void **stream) {
    pthread_mutex_lock(&g_bmu);
    const uint32_t n = g_last_n;
    memcpy(out, g_last, sizeof(lh_batch_item) * (n < cap ? n : cap));
    if (stream) *stream = g_last_stream;
    pthread_mutex_unlock(&g_bmu);
    return n;
}

LH_API lh_status lh_ingest_batch(lh_ctx *ctx, const lh_batch_item *h_items, uint32_t n_items, void *stream) {
    if (!ctx) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_bmu);
    g_last_n = h_items ? n_items : 0;
    if (h_items) memcpy(g_last, h_items, sizeof(lh_batch_item) * (n_items < MAX_KEPT ? n_items : MAX_KEPT));
    g_last_stream = stream;
    pthread_mutex_unlock(&g_bmu);
    if (n_items && !h_items) return LH_ERR_INVALID;
    const uint32_t H = ((const lh_config *)ctx)->max_histograms;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n_items; i++) {
        const lh_batch_item *it = &h_items[i];
        if (it->kind != LH_VALUES_F64 && it->kind != LH_VALUES_I64NS) return LH_ERR_INVALID;
        if (!it->n) continue;
        if (!it->d_values || ((uintptr_t)it->d_values & 7u)) return LH_ERR_INVALID;
        if (it->histogram_id >= H) return LH_ERR_RANGE;
        total += it->n;
    }
    if (!total) return LH_OK;
    for (uint32_t i = 0; i < n_items; i++) {
        const lh_batch_item *it = &h_items[i];
        if (!it->n) continue;
        lh_status st;
        if (it->kind == LH_VALUES_F64) {
            st = lh_ingest_f64(ctx, it->histogram_id, (const double *)it->d_values, (size_t)it->n, stream);
        } else {
            double *v = (double *)malloc(sizeof(double) * (size_t)it->n);
            if (!v) return LH_ERR_NOMEM;
            for (uint64_t j = 0; j < it->n; j++) v[j] = (double)((const int64_t *)it->d_values)[j];
            st = lh_ingest_f64(ctx, it->histogram_id, v, (size_t)it->n, stream);
            free(v);
        }
        if (st != LH_OK) return st;
    }
    pthread_mutex_lock(&g_bmu);
    g_calls++;
    pthread_mutex_unlock(&g_bmu);
    return LH_OK;
}
