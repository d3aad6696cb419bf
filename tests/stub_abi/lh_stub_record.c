/*
 * lh_stub_record.c -- TEST-ONLY record scopes for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_named_recording_cpu.py compiles it together with lh_stub.c, lh_stub_reduce_sparse.c and
 * oracle/loghisto_oracle.c, so that MetricSystem::BeginRecording (loghisto_b200/host/metric_system.cc) runs on the CPU.
 * It implements lh_record_begin / lh_record_end and lh_ingest_f64 over the stub's public entry points, and adds:
 *   lh_stub_record / lh_stub_count   what lh::record / lh::count do in a kernel, for one sample of an open scope
 *                                    (through a one-sample staging batch, so ids >= max_* are dropped and counted);
 *   lh_stub_record_hook              a callback run at the start of every lh_record_begin, before the scope opens --
 *                                    the tests run collections from it, between the binding's lookup and its check;
 *   lh_stub_record_begins            how many times lh_record_begin ran (retries of the binding show here).
 * The stub's lh_snapshot_begin does not wait for scopes; the tests that need that run on the real library.
 * "Device" pointers are host pointers here.  lh_stub.c's lh_ctx begins with its lh_config, which is where the
 * recorder's max_histograms / max_counters come from.
 */
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_SCOPES 256

static pthread_mutex_t g_rmu = PTHREAD_MUTEX_INITIALIZER;
static struct { uint64_t ticket; lh_ctx *ctx; } g_open[MAX_SCOPES];
static uint64_t g_next_ticket = 1, g_begins = 0;
static void (*g_hook)(void *, uint64_t) = 0;
static void *g_hook_arg = 0;

LH_API void lh_stub_record_hook(void (*fn)(void *, uint64_t), void *arg) {
    pthread_mutex_lock(&g_rmu);
    g_hook = fn; g_hook_arg = arg;
    pthread_mutex_unlock(&g_rmu);
}
LH_API uint64_t lh_stub_record_begins(void) {
    pthread_mutex_lock(&g_rmu);
    uint64_t n = g_begins;
    pthread_mutex_unlock(&g_rmu);
    return n;
}

LH_API lh_status lh_record_begin(lh_ctx *ctx, void *stream, lh_recorder *out) {
    (void)stream;
    if (!ctx || !out) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_rmu);
    const uint64_t call = g_begins++;
    void (*fn)(void *, uint64_t) = g_hook;
    void *arg = g_hook_arg;
    pthread_mutex_unlock(&g_rmu);
    if (fn) fn(arg, call);                                   /* no lock held: the hook collects */
    const lh_config *cfg = (const lh_config *)ctx;
    memset(out, 0, sizeof *out);
    out->max_histograms = cfg->max_histograms;
    out->max_counters = cfg->max_counters;
    pthread_mutex_lock(&g_rmu);
    for (int i = 0; i < MAX_SCOPES; i++)
        if (!g_open[i].ticket) {
            g_open[i].ticket = out->scope = g_next_ticket++;
            g_open[i].ctx = ctx;
            pthread_mutex_unlock(&g_rmu);
            return LH_OK;
        }
    pthread_mutex_unlock(&g_rmu);
    return LH_ERR_NOMEM;
}

/* the context of an open scope, or NULL (and, with `close`, the scope is closed) */
static lh_ctx *scope_ctx(const lh_recorder *rec, int close) {
    lh_ctx *c = 0;
    pthread_mutex_lock(&g_rmu);
    for (int i = 0; i < MAX_SCOPES; i++)
        if (rec && g_open[i].ticket && g_open[i].ticket == rec->scope) {
            c = g_open[i].ctx;
            if (close) g_open[i].ticket = 0;
            break;
        }
    pthread_mutex_unlock(&g_rmu);
    return c;
}

LH_API lh_status lh_record_end(lh_ctx *ctx, const lh_recorder *rec) {
    lh_ctx *c = scope_ctx(rec, 1);
    return c && c == ctx ? LH_OK : LH_ERR_INVALID;
}

static uint16_t id16(uint32_t id) { return id > 0xFFFFu ? 0xFFFFu : (uint16_t)id; }

/* n (value, id) pairs into the active interval, as one or more staging batches */
static lh_status commit_pairs(lh_ctx *c, const void *vals, uint32_t id, size_t n, int counter) {
    while (n) {
        lh_staging s;
        lh_status st = lh_staging_acquire(c, &s);
        if (st != LH_OK) return st;
        const uint64_t cap = (s.bytes / 10) & ~(uint64_t)15;
        const size_t k = n < cap ? n : (size_t)cap;
        uint16_t *ids = (uint16_t *)((char *)s.host + cap * 8);
        memcpy(s.host, vals, k * 8);
        for (size_t i = 0; i < k; i++) ids[i] = id16(id);
        st = counter ? lh_staging_commit_counter_u16(c, &s, k, cap * 8) : lh_staging_commit_keyed_f64_u16(c, &s, k, cap * 8);
        if (st != LH_OK) return st;
        vals = (const char *)vals + k * 8;
        n -= k;
    }
    return LH_OK;
}

LH_API lh_status lh_stub_record(const lh_recorder *rec, uint32_t id, double v) {
    lh_ctx *c = scope_ctx(rec, 0);
    return c ? commit_pairs(c, &v, id, 1, 0) : LH_ERR_STATE;
}
LH_API lh_status lh_stub_count(const lh_recorder *rec, uint32_t id, uint64_t amount) {
    lh_ctx *c = scope_ctx(rec, 0);
    return c ? commit_pairs(c, &amount, id, 1, 1) : LH_ERR_STATE;
}

LH_API lh_status lh_ingest_f64(lh_ctx *ctx, uint32_t histogram_id, const double *d_values, size_t n, void *stream) {
    (void)stream;
    if (!ctx || (n && !d_values)) return LH_ERR_INVALID;
    if (histogram_id >= ((const lh_config *)ctx)->max_histograms) return LH_ERR_RANGE;
    return commit_pairs(ctx, d_values, histogram_id, n, 0);
}
