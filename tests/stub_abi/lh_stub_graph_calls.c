/*
 * lh_stub_graph_calls.c -- TEST-ONLY captured keyed samples, counter adds and GPU-timed spans of graph recorders
 * (lh_graph_recorder_ingest_keyed_* / counter_add_* / timer_*) for the oracle-backed stub of the C ABI.
 *
 * It includes lh_stub_graph.c, whose recorders it extends, so tests/test_graph_recorder_calls_cpu.py compiles this file
 * in its place (with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c, lh_stub_batch.c and
 * oracle/loghisto_oracle.c); compiled with lh_stub_graph.c instead, the stub is a library that predates these calls.
 * The calls validate as the library does and then record on the host into the recorder's pending values, which every
 * drain moves into the active interval: a sample or amount under a local id >= k (>= kc) is dropped and counted at
 * once.  A timer's duration is the stub's clock at the stop minus its clock at the start.  It adds:
 *   lh_stub_graph_set_clock   the stub's device clock, which the graph timers read;
 *   lh_stub_graph_calls       how many calls of the six entry points below ran (any status).
 */
#include "lh_stub_graph.c"

/* timer start marks per recorder slot, valid for the recorder whose handle is mark_owner (a new recorder in the slot
 * starts with every mark never started) */
static uint64_t *g_marks[MAX_GRAPHS];
static uint64_t g_mark_owner[MAX_GRAPHS];
static uint64_t g_clock_ns;
static uint64_t g_calls;

LH_API void lh_stub_graph_set_clock(uint64_t ns) {
    pthread_mutex_lock(&g_gmu);
    g_clock_ns = ns;
    pthread_mutex_unlock(&g_gmu);
}

LH_API uint64_t lh_stub_graph_calls(void) {
    pthread_mutex_lock(&g_gmu);
    uint64_t n = g_calls;
    pthread_mutex_unlock(&g_gmu);
    return n;
}

/* the start marks of live recorder g (with g_gmu held) */
static uint64_t *marks_of(Graph *g) {
    const int i = (int)(g - g_graphs);
    if (g_mark_owner[i] != g->handle) {
        free(g_marks[i]);
        g_marks[i] = (uint64_t *)malloc(8 * (size_t)(g->k + 1));
        for (uint32_t j = 0; j < g->k; j++) g_marks[i][j] = UINT64_MAX;
        g_mark_owner[i] = g->handle;
    }
    return g_marks[i];
}

/* one sample or amount under local id `id` of a table of `limit`: kept, or dropped and counted at once */
static lh_status keep(Graph *g, Vals *rows, uint32_t limit, uint32_t id, const void *v, int counter) {
    if (id < limit) { push(&rows[id], v, 1); return LH_OK; }
    return commit(g->ctx, v, LH_GRAPH_UNBOUND, 1, counter);
}

static lh_status keyed(lh_ctx *ctx, const lh_graph_recorder *gr, const void *ids, size_t id_bytes, const void *vals,
                       uint32_t kind, size_t n) {
    pthread_mutex_lock(&g_gmu);
    g_calls++;
    Graph *g = find(ctx, gr);
    lh_status st = LH_OK;
    if (!g || (kind != LH_VALUES_F64 && kind != LH_VALUES_I64NS) || (n && (!ids || !vals)) || ((uintptr_t)vals & 7u) ||
        ((uintptr_t)ids & (id_bytes - 1)))
        st = LH_ERR_INVALID;
    for (size_t i = 0; st == LH_OK && i < n; i++) {
        const uint32_t id = id_bytes == 2 ? ((const uint16_t *)ids)[i] : ((const uint32_t *)ids)[i];
        const double v = kind == LH_VALUES_F64 ? ((const double *)vals)[i] : (double)((const int64_t *)vals)[i];
        st = keep(g, g->rows, g->k, id, &v, 0);
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

static lh_status counters(lh_ctx *ctx, const lh_graph_recorder *gr, const void *ids, size_t id_bytes, const uint64_t *amounts,
                          size_t n) {
    pthread_mutex_lock(&g_gmu);
    g_calls++;
    Graph *g = find(ctx, gr);
    lh_status st = LH_OK;
    if (!g || (n && (!ids || !amounts)) || ((uintptr_t)amounts & 7u) || ((uintptr_t)ids & (id_bytes - 1))) st = LH_ERR_INVALID;
    for (size_t i = 0; st == LH_OK && i < n; i++) {
        const uint32_t id = id_bytes == 2 ? ((const uint16_t *)ids)[i] : ((const uint32_t *)ids)[i];
        st = keep(g, g->ctrs, g->kc, id, &amounts[i], 1);
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_graph_recorder_ingest_keyed_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                    const void *d_values, uint32_t kind, size_t n, void *stream) {
    (void)stream;
    return keyed(ctx, g, d_ids, 2, d_values, kind, n);
}
LH_API lh_status lh_graph_recorder_ingest_keyed_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                    const void *d_values, uint32_t kind, size_t n, void *stream) {
    (void)stream;
    return keyed(ctx, g, d_ids, 4, d_values, kind, n);
}
LH_API lh_status lh_graph_recorder_counter_add_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                   const uint64_t *d_amounts, size_t n, void *stream) {
    (void)stream;
    return counters(ctx, g, d_ids, 2, d_amounts, n);
}
LH_API lh_status lh_graph_recorder_counter_add_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                   const uint64_t *d_amounts, size_t n, void *stream) {
    (void)stream;
    return counters(ctx, g, d_ids, 4, d_amounts, n);
}

LH_API lh_status lh_graph_recorder_timer_start(lh_ctx *ctx, const lh_graph_recorder *gr, uint32_t histogram, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_gmu);
    g_calls++;
    Graph *g = find(ctx, gr);
    lh_status st = !g ? LH_ERR_INVALID : histogram >= g->k ? LH_ERR_RANGE : LH_OK;
    if (st == LH_OK) marks_of(g)[histogram] = g_clock_ns;
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_graph_recorder_timer_stop(lh_ctx *ctx, const lh_graph_recorder *gr, uint32_t histogram, void *stream,
                                              int64_t *d_duration_ns) {
    (void)stream;
    pthread_mutex_lock(&g_gmu);
    g_calls++;
    Graph *g = find(ctx, gr);
    lh_status st = !g ? LH_ERR_INVALID : histogram >= g->k ? LH_ERR_RANGE : ((uintptr_t)d_duration_ns & 7u) ? LH_ERR_INVALID : LH_OK;
    if (st == LH_OK) {
        const uint64_t mark = marks_of(g)[histogram];
        if (mark == UINT64_MAX) {
            const double v = 0.0;
            st = commit(g->ctx, &v, LH_GRAPH_UNBOUND, 1, 0);     /* never started: dropped and counted */
        } else {
            const int64_t ns = (int64_t)(g_clock_ns - mark);
            const double v = (double)ns;
            push(&g->rows[histogram], &v, 1);
            if (d_duration_ns) *d_duration_ns = ns;
        }
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}
