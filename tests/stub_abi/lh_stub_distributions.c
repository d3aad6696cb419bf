/*
 * lh_stub_distributions.c -- TEST-ONLY distribution gauges (lh_snapshot_ingest_arrays) for the oracle-backed stub of
 * the C ABI.
 *
 * It includes lh_stub.c, which it extends, so tests/test_device_distributions_cpu.py compiles this file in its place
 * (with lh_stub_gauges.c, lh_stub_record.c and oracle/loghisto_oracle.c).  MetricSystem::RegisterDeviceDistribution and the distribution
 * step of collectRawMetrics (loghisto_b200/host/metric_system.cc) then run on the CPU.  "Device" memory is host memory
 * handed out by lh_stub_gauge_alloc.  lh_snapshot_ingest_arrays validates as the library does before its state check:
 * every element must be readable by lh_gauges_read (which refuses any address outside such an allocation, so freeing
 * one makes every later call that includes it fail), and histogram_id must be below max_histograms.  The values are
 * lh_gauges_read's float64(x), counted into the frozen buffer with the oracle's bucket key.  The state check refuses
 * the call unless a snapshot of that context is open and neither reduce nor export has read it yet.  The call log is
 * one for the process.  It adds:
 *   lh_stub_dist_log    the successful calls of begin (B), ingest_arrays (A), reduce (R), export (E) and end (N), in
 *                       order, as a string (reading it empties it);
 *   lh_stub_dist_last   the entries of the latest successful ingest_arrays call.
 */
#define lh_snapshot_begin lh_snapshot_begin_base
#define lh_snapshot_reduce lh_snapshot_reduce_base
#define lh_snapshot_export lh_snapshot_export_base
#define lh_snapshot_end lh_snapshot_end_base
#include "lh_stub.c"
#undef lh_snapshot_begin
#undef lh_snapshot_reduce
#undef lh_snapshot_export
#undef lh_snapshot_end

#define LOG_CAP 4096
#define MAX_KEPT 256

static char g_log[LOG_CAP];
static size_t g_log_n;
/* contexts whose open snapshot was reduced or exported (lh_stub_ranks.c keeps its per-context state alike) */
#define MAX_CTX 64
static lh_ctx *g_read[MAX_CTX];

static void set_read(lh_ctx *c, int read) {   /* with g_mu held */
    for (int i = 0; i < MAX_CTX; i++)
        if (g_read[i] == c) { if (!read) g_read[i] = 0; return; }
    if (read)
        for (int i = 0; i < MAX_CTX; i++)
            if (!g_read[i]) { g_read[i] = c; return; }
}
static int was_read(lh_ctx *c) {   /* with g_mu held */
    for (int i = 0; i < MAX_CTX; i++)
        if (g_read[i] == c) return 1;
    return 0;
}
static lh_array_src g_last[MAX_KEPT];
static uint32_t g_last_n;

/* logs `call` and marks ctx's open snapshot read or not */
static void log_call(lh_ctx *ctx, char call, int read) {
    pthread_mutex_lock(&g_mu);
    if (g_log_n + 1 < LOG_CAP) g_log[g_log_n++] = call;
    set_read(ctx, read);
    pthread_mutex_unlock(&g_mu);
}

LH_API size_t lh_stub_dist_log(char *out, size_t cap) {
    pthread_mutex_lock(&g_mu);
    const size_t n = g_log_n < cap ? g_log_n : cap;
    memcpy(out, g_log, n);
    g_log_n = 0;
    pthread_mutex_unlock(&g_mu);
    return n;
}

LH_API uint32_t lh_stub_dist_last(lh_array_src *out, uint32_t cap) {
    pthread_mutex_lock(&g_mu);
    const uint32_t n = g_last_n;
    memcpy(out, g_last, sizeof(lh_array_src) * (n < cap ? n : cap));
    pthread_mutex_unlock(&g_mu);
    return n;
}

LH_API lh_status lh_snapshot_begin(lh_ctx *c) {
    const lh_status st = lh_snapshot_begin_base(c);
    if (st == LH_OK) log_call(c, 'B', 0);
    return st;
}
LH_API lh_status lh_snapshot_reduce(lh_ctx *c, const double *ps, uint32_t np, uint64_t *counts, double *sums, double *avgs,
                                    int32_t *pkeys, double *pvals) {
    const lh_status st = lh_snapshot_reduce_base(c, ps, np, counts, sums, avgs, pkeys, pvals);
    if (st == LH_OK) log_call(c, 'R', 1);
    return st;
}
LH_API lh_status lh_snapshot_export(lh_ctx *c, lh_sparse *out) {
    const lh_status st = lh_snapshot_export_base(c, out);
    if (st == LH_OK) log_call(c, 'E', 1);
    return st;
}
LH_API lh_status lh_snapshot_end(lh_ctx *c) {
    const lh_status st = lh_snapshot_end_base(c);
    if (st == LH_OK) log_call(c, 'N', 0);
    return st;
}

/* every element of a as float64 through lh_gauges_read (lh_stub_gauges.c), or its refusal */
static lh_status convert(lh_ctx *c, const lh_array_src *a, double *out) {
    static const uint32_t bytes[] = {8, 4, 2, 2, 8, 4, 8};
    lh_gauge_src s[256];
    for (uint64_t i = 0; i < a->n;) {
        uint32_t m = 0;
        for (; m < 256 && i + m < a->n; m++) {
            s[m].d_value = (const char *)a->d_values + (i + m) * bytes[a->dtype];
            s[m].dtype = a->dtype;
            s[m].reserved = 0;
        }
        const lh_status st = lh_gauges_read(c, s, m, out + i);
        if (st != LH_OK) return st;
        i += m;
    }
    return LH_OK;
}

LH_API lh_status lh_snapshot_ingest_arrays(lh_ctx *c, const lh_array_src *h_srcs, uint32_t n_srcs) {
    if (!c || (n_srcs && !h_srcs)) return LH_ERR_INVALID;
    double **vals = (double **)calloc(n_srcs ? n_srcs : 1, sizeof(double *));
    lh_status st = LH_OK;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n_srcs && st == LH_OK; i++) {
        const lh_array_src *a = &h_srcs[i];
        if (a->dtype > LH_GAUGE_U64) { st = LH_ERR_INVALID; break; }
        if (!a->n) continue;
        if (a->histogram_id >= c->cfg.max_histograms) { st = LH_ERR_RANGE; break; }
        vals[i] = (double *)malloc(sizeof(double) * (size_t)a->n);
        st = convert(c, a, vals[i]);
        total += a->n;
    }
    pthread_mutex_lock(&g_mu);
    if (st == LH_OK && (!c->frozen || was_read(c))) {
        snprintf(c->err, sizeof c->err, "lh_snapshot_ingest_arrays needs an open snapshot whose rows nothing has read yet");
        st = LH_ERR_STATE;
    }
    if (st == LH_OK) {
        uint64_t *fb = c->buckets[c->active ^ 1];
        for (uint32_t i = 0; i < n_srcs; i++)
            for (uint64_t j = 0; j < h_srcs[i].n; j++)
                fb[(size_t)h_srcs[i].histogram_id * 65536u + (uint16_t)lho_compress(vals[i][j])]++;
        c->samples += total;
        g_last_n = n_srcs < MAX_KEPT ? n_srcs : MAX_KEPT;
        memcpy(g_last, h_srcs, sizeof(lh_array_src) * g_last_n);
        if (g_log_n + 1 < LOG_CAP) g_log[g_log_n++] = 'A';
    }
    pthread_mutex_unlock(&g_mu);
    for (uint32_t i = 0; i < n_srcs; i++) free(vals[i]);
    free(vals);
    return st;
}
