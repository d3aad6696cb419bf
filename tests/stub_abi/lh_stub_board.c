/*
 * lh_stub_board.c -- TEST-ONLY device subscription boards for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_device_subscription_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c,
 * lh_stub_batch.c, lh_stub_graph.c and oracle/loghisto_oracle.c, so that MetricSystem::NewDeviceSubscription and the
 * publish step of collectRawMetrics (loghisto_b200/host/metric_system.cc) run on the CPU.  A board here is host memory
 * in the layout of include/loghisto_b200.h.  lh_snapshot_publish fills it from the open snapshot's export (the stub
 * keeps no reduction results to read): a bound histogram row gets count = the sum of its exported counts and
 * present = (count != 0), with sum, avg and the percentile slots left as an untouched row; a bound counter row gets its
 * exported delta; unbound rows are untouched rows; totals are the caller's.  It also records the id every row was
 * bound to (lh_stub_board_bound).  "Device" pointers are host pointers; lh_board_read is a memcpy.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

#define MAX_BOARDS 64

typedef struct {
    uint64_t handle;                 /* 0 = free */
    lh_ctx *ctx;
    lh_board b;
    uint32_t *bound;                 /* [k + kc] id of each row at the latest publish */
} Board;

static pthread_mutex_t g_bmu = PTHREAD_MUTEX_INITIALIZER;
static Board g_boards[MAX_BOARDS];
static uint64_t g_bnext = 1;

static const lh_config *cfg_of(lh_ctx *c) { return (const lh_config *)c; }

static Board *find(lh_ctx *ctx, const lh_board *b) {
    if (!ctx || !b) return 0;
    for (int i = 0; i < MAX_BOARDS; i++)
        if (g_boards[i].handle && g_boards[i].handle == b->handle && g_boards[i].ctx == ctx &&
            g_boards[i].b.d_board == b->d_board) return &g_boards[i];
    return 0;
}

static void untouched_row(lh_board_hist_row *r) {
    memset(r, 0, sizeof *r);
    r->avg = NAN;
    for (int j = 0; j < LH_MAX_PERCENTILES; j++) { r->pvals[j] = NAN; r->pkeys[j] = INT32_MIN; }
}

LH_API lh_status lh_board_create(lh_ctx *ctx, uint32_t k, uint32_t kc, lh_board *out) {
    if (!ctx || !out || (k == 0 && kc == 0)) return LH_ERR_INVALID;
    if (k > cfg_of(ctx)->max_histograms || kc > cfg_of(ctx)->max_counters) return LH_ERR_RANGE;
    pthread_mutex_lock(&g_bmu);
    for (int i = 0; i < MAX_BOARDS; i++) {
        Board *s = &g_boards[i];
        if (s->handle) continue;
        s->handle = g_bnext++;
        s->ctx = ctx;
        s->b.handle = s->handle;
        s->b.k = k;
        s->b.kc = kc;
        s->b.bytes = sizeof(lh_board_header) + (uint64_t)k * sizeof(lh_board_hist_row) + (uint64_t)kc * sizeof(lh_board_counter_row);
        s->b.d_board = calloc(1, s->b.bytes);
        s->bound = (uint32_t *)malloc(((size_t)k + kc) * 4);
        for (uint32_t r = 0; r < k + kc; r++) s->bound[r] = LH_GRAPH_UNBOUND;
        *out = s->b;
        pthread_mutex_unlock(&g_bmu);
        return LH_OK;
    }
    pthread_mutex_unlock(&g_bmu);
    return LH_ERR_NOMEM;
}

LH_API lh_status lh_snapshot_publish(lh_ctx *ctx, const lh_board *b, const uint32_t *hist_ids,
                                     const uint32_t *counter_ids, const uint64_t *counter_totals) {
    pthread_mutex_lock(&g_bmu);
    Board *s = find(ctx, b);
    lh_status st = s ? LH_OK : LH_ERR_INVALID;
    lh_sparse sp;
    if (st == LH_OK) st = lh_snapshot_export(ctx, &sp);   /* LH_ERR_STATE outside a snapshot */
    for (uint32_t i = 0; st == LH_OK && i < s->b.k; i++)
        if (hist_ids && hist_ids[i] != LH_GRAPH_UNBOUND && hist_ids[i] >= cfg_of(ctx)->max_histograms) st = LH_ERR_RANGE;
    for (uint32_t i = 0; st == LH_OK && i < s->b.kc; i++)
        if (counter_ids && counter_ids[i] != LH_GRAPH_UNBOUND && counter_ids[i] >= cfg_of(ctx)->max_counters) st = LH_ERR_RANGE;
    if (st != LH_OK) { pthread_mutex_unlock(&g_bmu); return st; }
    char *base = (char *)s->b.d_board;
    lh_board_header *h = (lh_board_header *)base;
    lh_board_hist_row *rows = (lh_board_hist_row *)(base + sizeof *h);
    lh_board_counter_row *crows = (lh_board_counter_row *)(rows + s->b.k);
    h->seq++;
    h->np = 0;
    for (int j = 0; j < LH_MAX_PERCENTILES; j++) h->percentiles[j] = NAN;
    for (uint32_t i = 0; i < s->b.k; i++) {
        const uint32_t id = hist_ids ? hist_ids[i] : LH_GRAPH_UNBOUND;
        untouched_row(&rows[i]);
        s->bound[i] = id;
        if (id == LH_GRAPH_UNBOUND) continue;
        uint64_t c = 0;
        for (uint32_t e = sp.offsets[id]; e < sp.offsets[id + 1]; e++) c += sp.counts[e];
        rows[i].count = c;
        rows[i].present = c != 0;
    }
    for (uint32_t i = 0; i < s->b.kc; i++) {
        const uint32_t id = counter_ids ? counter_ids[i] : LH_GRAPH_UNBOUND;
        s->bound[s->b.k + i] = id;
        crows[i].rate = id == LH_GRAPH_UNBOUND ? 0 : sp.counter_deltas[id];
        crows[i].present = id != LH_GRAPH_UNBOUND;
        crows[i].total = counter_totals ? counter_totals[i] : 0;
    }
    h->seq++;
    h->publishes = h->seq / 2;
    pthread_mutex_unlock(&g_bmu);
    return LH_OK;
}

LH_API lh_status lh_board_read(lh_ctx *ctx, const lh_board *b, void *d_out, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_bmu);
    Board *s = find(ctx, b);
    if (s && d_out) memcpy(d_out, s->b.d_board, s->b.bytes);
    pthread_mutex_unlock(&g_bmu);
    return s && d_out ? LH_OK : LH_ERR_INVALID;
}

LH_API lh_status lh_board_destroy(lh_ctx *ctx, const lh_board *b) {
    pthread_mutex_lock(&g_bmu);
    Board *s = find(ctx, b);
    if (s) {
        free(s->b.d_board);
        free(s->bound);
        memset(s, 0, sizeof *s);
    }
    pthread_mutex_unlock(&g_bmu);
    return s ? LH_OK : LH_ERR_INVALID;
}

/* boards alive (created and not destroyed) */
LH_API uint32_t lh_stub_board_alive(void) {
    uint32_t n = 0;
    pthread_mutex_lock(&g_bmu);
    for (int i = 0; i < MAX_BOARDS; i++) n += g_boards[i].handle != 0;
    pthread_mutex_unlock(&g_bmu);
    return n;
}

/* the id row `row` (histogram rows first, then counter rows) was bound to at the latest publish */
LH_API uint32_t lh_stub_board_bound(const lh_board *b, uint32_t row) {
    uint32_t id = LH_GRAPH_UNBOUND;
    pthread_mutex_lock(&g_bmu);
    for (int i = 0; i < MAX_BOARDS; i++)
        if (g_boards[i].handle && g_boards[i].handle == b->handle && row < g_boards[i].b.k + g_boards[i].b.kc)
            id = g_boards[i].bound[row];
    pthread_mutex_unlock(&g_bmu);
    return id;
}
