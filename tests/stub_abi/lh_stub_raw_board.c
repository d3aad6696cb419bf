/*
 * lh_stub_raw_board.c -- TEST-ONLY raw device subscription boards for the oracle-backed stub of the C ABI (lh_stub.c).
 *
 * tests/test_raw_subscription_cpu.py compiles it with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c,
 * lh_stub_batch.c, lh_stub_graph.c, lh_stub_board.c and oracle/loghisto_oracle.c, so that
 * MetricSystem::NewRawDeviceSubscription and the raw publish step of collectRawMetrics
 * (loghisto_b200/host/metric_system.cc) run on the CPU.  A raw board here is host memory in the layout of
 * include/loghisto_b200.h.  lh_snapshot_publish_raw fills it from the open snapshot's export: a bound row with samples
 * gets running counts over all 65 536 keys, anything else is an empty row.  The query calls answer on the CPU from
 * those arrays with the reference's rules (percentile: the first non-empty key, ascending, whose running count c has
 * float64(c)/float64(total) >= p; rank: the running count at the oracle's compress(v)).  It also records the id every
 * row was bound to (lh_stub_raw_bound).  "Device" pointers are host pointers.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "loghisto_b200.h"

int16_t lho_compress_p(double value, double precision);
double lho_decompress_p(int16_t k, double precision);

#define MAX_RAW_BOARDS 64

typedef struct {
    uint64_t handle;                 /* 0 = free */
    lh_ctx *ctx;
    lh_raw_board b;
    double precision;
    double *decomp;                  /* [65536] by (uint16)key */
    uint32_t *bound;                 /* [k] id of each row at the latest publish */
} RawBoard;

static pthread_mutex_t g_rmu = PTHREAD_MUTEX_INITIALIZER;
static RawBoard g_raw[MAX_RAW_BOARDS];
static uint64_t g_rnext = 1;

static const lh_config *raw_cfg_of(lh_ctx *c) { return (const lh_config *)c; }

static RawBoard *raw_find(lh_ctx *ctx, const lh_raw_board *b) {
    if (!ctx || !b) return 0;
    for (int i = 0; i < MAX_RAW_BOARDS; i++)
        if (g_raw[i].handle && g_raw[i].handle == b->handle && g_raw[i].ctx == ctx && g_raw[i].b.d_rows == b->d_rows)
            return &g_raw[i];
    return 0;
}

static lh_raw_row_header *hdr(RawBoard *s, uint32_t row) { return (lh_raw_row_header *)s->b.d_rows + row; }
static uint64_t *cells(RawBoard *s, uint32_t row) {
    return (uint64_t *)((char *)s->b.d_rows + LH_RAW_CELLS_OFFSET(s->b.k)) + (size_t)row * 65536u;
}
static uint64_t running(RawBoard *s, uint32_t row, int key) {
    const lh_raw_row_header *h = hdr(s, row);
    if (key < h->key_lo) return 0;
    if (key > h->key_hi) return h->total;
    return cells(s, row)[key + 32768];
}

LH_API lh_status lh_raw_board_create(lh_ctx *ctx, uint32_t k, lh_raw_board *out) {
    if (!ctx || !out || k == 0) return LH_ERR_INVALID;
    if (k > raw_cfg_of(ctx)->max_histograms) return LH_ERR_RANGE;
    pthread_mutex_lock(&g_rmu);
    for (int i = 0; i < MAX_RAW_BOARDS; i++) {
        RawBoard *s = &g_raw[i];
        if (s->handle) continue;
        s->handle = g_rnext++;
        s->ctx = ctx;
        memset(&s->b, 0, sizeof s->b);
        s->b.handle = s->handle;
        s->b.k = k;
        s->b.d_rows = calloc(1, LH_RAW_CELLS_OFFSET(k) + (size_t)k * 65536u * 8u);
        s->precision = raw_cfg_of(ctx)->precision ? (double)raw_cfg_of(ctx)->precision : 100.0;
        s->decomp = (double *)malloc(65536 * sizeof(double));
        for (int key = -32768; key < 32768; key++) s->decomp[(uint16_t)key] = lho_decompress_p((int16_t)key, s->precision);
        s->b.d_decomp = s->decomp;
        for (uint32_t r = 0; r < k; r++) hdr(s, r)->key_hi = -1;   /* empty rows of publish 0, as the library's */
        s->bound = (uint32_t *)malloc((size_t)k * 4);
        for (uint32_t r = 0; r < k; r++) s->bound[r] = LH_GRAPH_UNBOUND;
        *out = s->b;
        pthread_mutex_unlock(&g_rmu);
        return LH_OK;
    }
    pthread_mutex_unlock(&g_rmu);
    return LH_ERR_NOMEM;
}

LH_API lh_status lh_snapshot_publish_raw(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *hist_ids) {
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    lh_status st = s ? LH_OK : LH_ERR_INVALID;
    lh_sparse sp;
    if (st == LH_OK) st = lh_snapshot_export(ctx, &sp);   /* LH_ERR_STATE outside a snapshot */
    for (uint32_t i = 0; st == LH_OK && i < s->b.k; i++)
        if (hist_ids && hist_ids[i] != LH_GRAPH_UNBOUND && hist_ids[i] >= raw_cfg_of(ctx)->max_histograms) st = LH_ERR_RANGE;
    if (st != LH_OK) { pthread_mutex_unlock(&g_rmu); return st; }
    for (uint32_t i = 0; i < s->b.k; i++) {
        const uint32_t id = hist_ids ? hist_ids[i] : LH_GRAPH_UNBOUND;
        lh_raw_row_header *h = hdr(s, i);
        s->bound[i] = id;
        h->seq++;
        h->total = 0;
        h->key_lo = 0;
        h->key_hi = -1;
        if (id != LH_GRAPH_UNBOUND && sp.offsets[id] != sp.offsets[id + 1]) {
            uint64_t *c = cells(s, i);
            memset(c, 0, 65536u * 8u);
            for (uint32_t e = sp.offsets[id]; e < sp.offsets[id + 1]; e++) c[sp.keys[e] + 32768] += sp.counts[e];
            for (uint32_t x = 1; x < 65536u; x++) c[x] += c[x - 1];
            h->total = c[65535];
            h->key_lo = -32768;
            h->key_hi = 32767;
        }
        h->seq++;
        h->publishes = h->seq / 2;
    }
    pthread_mutex_unlock(&g_rmu);
    return LH_OK;
}

static void answer_pct(RawBoard *s, uint32_t row, double p, int32_t *key, double *val, uint64_t *pub) {
    *key = INT32_MIN;
    *val = NAN;
    *pub = row < s->b.k ? hdr(s, row)->seq / 2 : 0;
    if (row >= s->b.k || !hdr(s, row)->total) return;
    const uint64_t total = hdr(s, row)->total;
    for (int k = -32768; k < 32768; k++) {
        const uint64_t c = running(s, row, k);
        if (c != running(s, row, k - 1) && (double)c / (double)total >= p) {
            *key = k;
            *val = s->decomp[(uint16_t)k];
            return;
        }
    }
}

static void answer_rank(RawBoard *s, uint32_t row, double v, uint64_t *rank, uint64_t *total, uint64_t *pub) {
    *rank = *total = *pub = 0;
    if (row >= s->b.k) return;
    *rank = running(s, row, lho_compress_p(v, s->precision));
    *total = hdr(s, row)->total;
    *pub = hdr(s, row)->seq / 2;
}

static int ptr_ok(const void *p, uintptr_t a) { return p && ((uintptr_t)p & (a - 1u)) == 0; }

LH_API lh_status lh_raw_percentiles(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_ps,
                                    uint32_t n, int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    lh_status st = !s ? LH_ERR_INVALID : n && !(ptr_ok(d_rows, 4) && ptr_ok(d_ps, 8) && ptr_ok(d_keys, 4) &&
                                              ptr_ok(d_vals, 8) && ptr_ok(d_publish, 8)) ? LH_ERR_INVALID : LH_OK;
    for (uint32_t i = 0; st == LH_OK && i < n; i++) answer_pct(s, d_rows[i], d_ps[i], &d_keys[i], &d_vals[i], &d_publish[i]);
    pthread_mutex_unlock(&g_rmu);
    return st;
}

LH_API lh_status lh_raw_ranks(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_values,
                              uint32_t n, uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    lh_status st = !s ? LH_ERR_INVALID : n && !(ptr_ok(d_rows, 4) && ptr_ok(d_values, 8) && ptr_ok(d_ranks, 8) &&
                                              ptr_ok(d_totals, 8) && ptr_ok(d_publish, 8)) ? LH_ERR_INVALID : LH_OK;
    for (uint32_t i = 0; st == LH_OK && i < n; i++)
        answer_rank(s, d_rows[i], d_values[i], &d_ranks[i], &d_totals[i], &d_publish[i]);
    pthread_mutex_unlock(&g_rmu);
    return st;
}

LH_API lh_status lh_raw_percentiles_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_ps, uint32_t m,
                                         int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    lh_status st = !s ? LH_ERR_INVALID : m && !(ptr_ok(d_ps, 8) && ptr_ok(d_keys, 4) && ptr_ok(d_vals, 8) &&
                                              ptr_ok(d_publish, 8)) ? LH_ERR_INVALID : LH_OK;
    for (uint32_t r = 0; st == LH_OK && r < s->b.k; r++)
        for (uint32_t j = 0; j < m; j++) {
            const size_t i = (size_t)r * m + j;
            answer_pct(s, r, d_ps[j], &d_keys[i], &d_vals[i], &d_publish[i]);
        }
    pthread_mutex_unlock(&g_rmu);
    return st;
}

LH_API lh_status lh_raw_ranks_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_values, uint32_t m,
                                   uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream) {
    (void)stream;
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    lh_status st = !s ? LH_ERR_INVALID : m && !(ptr_ok(d_values, 8) && ptr_ok(d_ranks, 8) && ptr_ok(d_totals, 8) &&
                                              ptr_ok(d_publish, 8)) ? LH_ERR_INVALID : LH_OK;
    for (uint32_t r = 0; st == LH_OK && r < s->b.k; r++)
        for (uint32_t j = 0; j < m; j++) {
            const size_t i = (size_t)r * m + j;
            uint64_t total;
            answer_rank(s, r, d_values[j], &d_ranks[i], &total, &d_publish[i]);
            if (j == 0) d_totals[r] = total;
        }
    pthread_mutex_unlock(&g_rmu);
    return st;
}

LH_API lh_status lh_raw_board_destroy(lh_ctx *ctx, const lh_raw_board *b) {
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    if (s) {
        free(s->b.d_rows);
        free(s->decomp);
        free(s->bound);
        memset(s, 0, sizeof *s);
    }
    pthread_mutex_unlock(&g_rmu);
    return s ? LH_OK : LH_ERR_INVALID;
}

/* raw boards alive (created and not destroyed) */
LH_API uint32_t lh_stub_raw_alive(void) {
    uint32_t n = 0;
    pthread_mutex_lock(&g_rmu);
    for (int i = 0; i < MAX_RAW_BOARDS; i++) n += g_raw[i].handle != 0;
    pthread_mutex_unlock(&g_rmu);
    return n;
}

/* the id row `row` was bound to at the latest publish */
LH_API uint32_t lh_stub_raw_bound(const lh_raw_board *b, uint32_t row) {
    uint32_t id = LH_GRAPH_UNBOUND;
    pthread_mutex_lock(&g_rmu);
    for (int i = 0; i < MAX_RAW_BOARDS; i++)
        if (g_raw[i].handle && g_raw[i].handle == b->handle && row < g_raw[i].b.k) id = g_raw[i].bound[row];
    pthread_mutex_unlock(&g_rmu);
    return id;
}
