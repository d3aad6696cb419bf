/*
 * lh_stub_graph.c -- TEST-ONLY graph recorders for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_graph_recorder_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c,
 * lh_stub_batch.c and oracle/loghisto_oracle.c, so that MetricSystem::NewGraphRecorder and the binding step of
 * collectRawMetrics (loghisto_b200/host/metric_system.cc) run on the CPU.  A recorder here keeps the samples recorded
 * into it as plain values per local row (and amounts per local counter) instead of bucket rows, and drains them into the
 * active interval through the stub's staging calls, under the target ids, at every lh_graph_recorder_bind and at
 * lh_graph_recorder_destroy.  The mirror binds every open recorder just before lh_snapshot_begin, so a drain at bind
 * lands in the interval that collection freezes, as the library's drain inside lh_snapshot_begin does.  Unbound rows
 * and counters are committed under an id >= max_*, which the stub drops and counts per sample (per counter op).
 * It adds:
 *   lh_stub_graph_record / lh_stub_graph_count   what lh::record / lh::count do in a replayed kernel (a local id >= k
 *                                                 or >= kc is dropped and counted at once);
 *   lh_stub_graph_alive                           how many recorders are live;
 *   lh_stub_graph_target                          the target id local row (counter) i of a recorder is bound to.
 * The recorder of a stub lh_recorder is found through its d_buckets, which here points at the stub's record of it.
 * "Device" pointers are host pointers here.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_GRAPHS 64

typedef struct {
    double *v;
    size_t n, cap;
} Vals;

typedef struct {
    uint64_t handle;                 /* 0 = free */
    lh_ctx *ctx;
    uint32_t k, kc;
    uint32_t *hid, *cid;
    Vals *rows, *ctrs;               /* pending values / amounts (as float64 bit patterns for counters) */
} Graph;

static pthread_mutex_t g_gmu = PTHREAD_MUTEX_INITIALIZER;
static Graph g_graphs[MAX_GRAPHS];
static uint64_t g_next = 1;

static const lh_config *cfg_of(lh_ctx *c) { return (const lh_config *)c; }

static Graph *of_rec(const lh_recorder *rec) {
    for (int i = 0; rec && i < MAX_GRAPHS; i++)
        if (g_graphs[i].handle && (void *)rec->d_buckets == (void *)&g_graphs[i]) return &g_graphs[i];
    return 0;
}

static Graph *find(lh_ctx *ctx, const lh_graph_recorder *g) {
    if (!ctx || !g) return 0;
    for (int i = 0; i < MAX_GRAPHS; i++)
        if (g_graphs[i].handle && g_graphs[i].handle == g->handle && g_graphs[i].ctx == ctx) return &g_graphs[i];
    return 0;
}

static int ids_ok(const uint32_t *ids, uint32_t n, uint32_t limit) {
    for (uint32_t i = 0; ids && i < n; i++)
        if (ids[i] >= limit && ids[i] != LH_GRAPH_UNBOUND) return 0;
    return 1;
}

static void push(Vals *a, const void *p, size_t n) {
    if (a->n + n > a->cap) {
        a->cap = (a->n + n) * 2 + 16;
        a->v = (double *)realloc(a->v, a->cap * 8);
    }
    memcpy(a->v + a->n, p, n * 8);
    a->n += n;
}

/* n 8-byte items under one uint16 id (0xFFFF when id does not fit: dropped by the stub) into the active interval */
static lh_status commit(lh_ctx *c, const void *vals, uint32_t id, size_t n, int counter) {
    const uint16_t id16 = id > 0xFFFEu ? 0xFFFFu : (uint16_t)id;
    while (n) {
        lh_staging s;
        lh_status st = lh_staging_acquire(c, &s);
        if (st != LH_OK) return st;
        const uint64_t cap = (s.bytes / 10) & ~(uint64_t)15;
        const size_t m = n < cap ? n : (size_t)cap;
        uint16_t *ids = (uint16_t *)((char *)s.host + cap * 8);
        memcpy(s.host, vals, m * 8);
        for (size_t i = 0; i < m; i++) ids[i] = id16;
        st = counter ? lh_staging_commit_counter_u16(c, &s, m, cap * 8) : lh_staging_commit_keyed_f64_u16(c, &s, m, cap * 8);
        if (st != LH_OK) return st;
        vals = (const char *)vals + m * 8;
        n -= m;
    }
    return LH_OK;
}

static lh_status drain(Graph *g) {
    for (uint32_t i = 0; i < g->k; i++) {
        lh_status st = commit(g->ctx, g->rows[i].v, g->hid[i], g->rows[i].n, 0);
        if (st != LH_OK) return st;
        g->rows[i].n = 0;
    }
    for (uint32_t i = 0; i < g->kc; i++) {
        lh_status st = commit(g->ctx, g->ctrs[i].v, g->cid[i], g->ctrs[i].n, 1);
        if (st != LH_OK) return st;
        g->ctrs[i].n = 0;
    }
    return LH_OK;
}

LH_API lh_status lh_graph_recorder_create(lh_ctx *ctx, uint32_t k, uint32_t kc, const uint32_t *hist_ids,
                                          const uint32_t *counter_ids, lh_graph_recorder *out) {
    if (!ctx || !out || (k == 0 && kc == 0)) return LH_ERR_INVALID;
    const lh_config *cfg = cfg_of(ctx);
    if (k > cfg->max_histograms || kc > cfg->max_counters) return LH_ERR_RANGE;
    if (!ids_ok(hist_ids, k, cfg->max_histograms) || !ids_ok(counter_ids, kc, cfg->max_counters)) return LH_ERR_RANGE;
    pthread_mutex_lock(&g_gmu);
    for (int i = 0; i < MAX_GRAPHS; i++) {
        Graph *g = &g_graphs[i];
        if (g->handle) continue;
        memset(g, 0, sizeof *g);
        g->handle = g_next++;
        g->ctx = ctx;
        g->k = k;
        g->kc = kc;
        g->hid = (uint32_t *)malloc(4 * (size_t)(k + 1));
        g->cid = (uint32_t *)malloc(4 * (size_t)(kc + 1));
        for (uint32_t j = 0; j < k; j++) g->hid[j] = hist_ids ? hist_ids[j] : LH_GRAPH_UNBOUND;
        for (uint32_t j = 0; j < kc; j++) g->cid[j] = counter_ids ? counter_ids[j] : LH_GRAPH_UNBOUND;
        g->rows = (Vals *)calloc(k + 1, sizeof(Vals));
        g->ctrs = (Vals *)calloc(kc + 1, sizeof(Vals));
        memset(out, 0, sizeof *out);
        out->handle = g->handle;
        out->rec.d_buckets = (uint64_t *)(void *)g;   /* identifies the recorder to lh_stub_graph_* */
        out->rec.max_histograms = k;
        out->rec.max_counters = kc;
        pthread_mutex_unlock(&g_gmu);
        return LH_OK;
    }
    pthread_mutex_unlock(&g_gmu);
    return LH_ERR_NOMEM;
}

LH_API lh_status lh_graph_recorder_bind(lh_ctx *ctx, const lh_graph_recorder *gr, const uint32_t *hist_ids,
                                        const uint32_t *counter_ids) {
    pthread_mutex_lock(&g_gmu);
    Graph *g = find(ctx, gr);
    lh_status st = LH_ERR_INVALID;
    if (g) {
        st = LH_ERR_RANGE;
        if (ids_ok(hist_ids, g->k, cfg_of(ctx)->max_histograms) && ids_ok(counter_ids, g->kc, cfg_of(ctx)->max_counters)) {
            if (hist_ids) memcpy(g->hid, hist_ids, 4 * (size_t)g->k);
            if (counter_ids) memcpy(g->cid, counter_ids, 4 * (size_t)g->kc);
            st = drain(g);
        }
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_graph_recorder_ingest(lh_ctx *ctx, const lh_graph_recorder *gr, const lh_batch_item *items,
                                          uint32_t n_items, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_gmu);
    Graph *g = find(ctx, gr);
    lh_status st = g ? LH_OK : LH_ERR_INVALID;
    if (g && n_items && !items) st = LH_ERR_INVALID;
    for (uint32_t i = 0; st == LH_OK && i < n_items; i++) {
        const lh_batch_item *it = &items[i];
        if (it->kind != LH_VALUES_F64 && it->kind != LH_VALUES_I64NS) st = LH_ERR_INVALID;
        else if (it->n && (!it->d_values || ((uintptr_t)it->d_values & 7u))) st = LH_ERR_INVALID;
        else if (it->n && it->histogram_id >= g->k) st = LH_ERR_RANGE;
    }
    for (uint32_t i = 0; st == LH_OK && i < n_items; i++) {
        const lh_batch_item *it = &items[i];
        for (uint64_t j = 0; j < it->n; j++) {
            double v = it->kind == LH_VALUES_F64 ? ((const double *)it->d_values)[j]
                                                 : (double)((const int64_t *)it->d_values)[j];
            push(&g->rows[it->histogram_id], &v, 1);
        }
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_graph_recorder_destroy(lh_ctx *ctx, const lh_graph_recorder *gr, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_gmu);
    Graph *g = find(ctx, gr);
    lh_status st = LH_ERR_INVALID;
    if (g) {
        st = drain(g);
        for (uint32_t i = 0; i < g->k; i++) free(g->rows[i].v);
        for (uint32_t i = 0; i < g->kc; i++) free(g->ctrs[i].v);
        free(g->rows); free(g->ctrs); free(g->hid); free(g->cid);
        memset(g, 0, sizeof *g);
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_stub_graph_record(const lh_recorder *rec, uint32_t id, double v) {
    pthread_mutex_lock(&g_gmu);
    Graph *g = of_rec(rec);
    lh_status st = g ? LH_OK : LH_ERR_INVALID;
    if (g && id < g->k) push(&g->rows[id], &v, 1);
    else if (g) st = commit(g->ctx, &v, LH_GRAPH_UNBOUND, 1, 0);
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_stub_graph_count(const lh_recorder *rec, uint32_t id, uint64_t amount) {
    pthread_mutex_lock(&g_gmu);
    Graph *g = of_rec(rec);
    lh_status st = g ? LH_OK : LH_ERR_INVALID;
    if (g && id < g->kc) push(&g->ctrs[id], &amount, 1);
    else if (g) st = commit(g->ctx, &amount, LH_GRAPH_UNBOUND, 1, 1);
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API uint32_t lh_stub_graph_alive(void) {
    uint32_t n = 0;
    pthread_mutex_lock(&g_gmu);
    for (int i = 0; i < MAX_GRAPHS; i++) n += g_graphs[i].handle != 0;
    pthread_mutex_unlock(&g_gmu);
    return n;
}

/* target of local row i (counter: counter != 0) of the recorder of `rec`, or 0xFFFFFFFE if there is none */
LH_API uint32_t lh_stub_graph_target(const lh_recorder *rec, uint32_t i, int counter) {
    uint32_t t = 0xFFFFFFFEu;
    pthread_mutex_lock(&g_gmu);
    const Graph *g = of_rec(rec);
    if (g && (counter ? i < g->kc : i < g->k)) t = counter ? g->cid[i] : g->hid[i];
    pthread_mutex_unlock(&g_gmu);
    return t;
}
