/*
 * lh_stub_ranks.c -- TEST-ONLY joined ranks (lh_comm_export / lh_comm_import / lh_comm_info / lh_snapshot_rows /
 * lh_snapshot_allreduce_rows / lh_snapshot_copy_histogram) for the oracle-backed stub of the C ABI.
 *
 * It includes lh_stub.c, which it extends, so tests/test_ranks_cpu.py compiles this file in its place (with
 * lh_stub_reduce_sparse.c, lh_stub_record.c, lh_stub_batch.c and oracle/loghisto_oracle.c).  The ranks are stub
 * contexts in one process, one thread each.  A handle carries the context's address.  The all-reduce validates as the
 * library does and then, unlike the library's kernel, blocks its caller: it waits until every rank of the group has
 * called it for the same sequence number, sums each job-wide row g from every rank's frozen row map[r][g] (nothing for
 * LH_ROW_ABSENT), waits until every rank has summed, and writes the sums over its own frozen arrays, row g at index g
 * and nothing at or above n_rows.  The snapshot's reduce, export and copy then read the job-wide rows.  It adds:
 *   lh_stub_rows_calls   how many lh_snapshot_allreduce_rows calls got past validation (would have launched).
 */
#define lh_destroy lh_destroy_base   /* wrapped below: a destroyed context leaves its group */
#include "lh_stub.c"
#undef lh_destroy

#include <errno.h>
#include <time.h>

static pthread_cond_t g_rcv = PTHREAD_COND_INITIALIZER;
static uint64_t g_rows_calls;

struct stub_comm {
    lh_ctx *ctx;
    uint32_t rank, world;
    lh_ctx *peers[LH_MAX_RANKS];
    uint64_t seq;           /* last all-reduce */
    uint64_t arrived, summed;
    uint32_t status;
    uint64_t reduced_at;    /* snapshot number (lh_stats.snapshots) of the last all-reduce */
};
static struct stub_comm g_comm[64];

static struct stub_comm *comm_of(lh_ctx *c) {
    for (int i = 0; i < 64; i++)
        if (g_comm[i].ctx == c) return &g_comm[i];
    for (int i = 0; i < 64; i++)
        if (!g_comm[i].ctx) { memset(&g_comm[i], 0, sizeof g_comm[i]); g_comm[i].ctx = c; return &g_comm[i]; }
    return NULL;
}

LH_API lh_status lh_destroy(lh_ctx *c) {
    pthread_mutex_lock(&g_mu);
    for (int i = 0; i < 64; i++)
        if (g_comm[i].ctx == c) memset(&g_comm[i], 0, sizeof g_comm[i]);
    pthread_mutex_unlock(&g_mu);
    return lh_destroy_base(c);
}

LH_API uint64_t lh_stub_rows_calls(void) {
    pthread_mutex_lock(&g_mu);
    uint64_t n = g_rows_calls;
    pthread_mutex_unlock(&g_mu);
    return n;
}

LH_API lh_status lh_comm_export(lh_ctx *c, lh_peer_handle *out) {
    if (!c || !out) return LH_ERR_INVALID;
    memset(out, 0, sizeof *out);
    memcpy(out->bytes, &c, sizeof c);
    return LH_OK;
}

LH_API lh_status lh_comm_import(lh_ctx *c, uint32_t rank, uint32_t world, const lh_peer_handle *all) {
    if (!c || !all || world < 1 || world > LH_MAX_RANKS || rank >= world) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    struct stub_comm *m = comm_of(c);
    lh_status st = LH_OK;
    if (c->frozen) st = LH_ERR_STATE;
    for (uint32_t r = 0; st == LH_OK && r < world; r++) {
        lh_ctx *p;
        memcpy(&p, all[r].bytes, sizeof p);
        if ((r == rank && p != c) || p->cfg.max_histograms != c->cfg.max_histograms ||
            p->cfg.max_counters != c->cfg.max_counters || p->cfg.precision != c->cfg.precision)
            st = LH_ERR_INVALID;
        else
            m->peers[r] = p;
    }
    if (st == LH_OK) { m->rank = rank; m->world = world; }
    pthread_mutex_unlock(&g_mu);
    return st;
}

LH_API lh_status lh_comm_info(lh_ctx *c, lh_comm_stats *out) {
    if (!c || !out) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    struct stub_comm *m = comm_of(c);
    memset(out, 0, sizeof *out);
    out->rank = m->rank; out->world = m->world; out->status = m->status; out->allreduces = m->seq;
    pthread_mutex_unlock(&g_mu);
    return LH_OK;
}

LH_API lh_status lh_snapshot_copy_histogram(lh_ctx *c, uint32_t hid, uint64_t *out) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    lh_status st = !c->frozen ? LH_ERR_STATE : hid >= c->cfg.max_histograms ? LH_ERR_RANGE : !out ? LH_ERR_INVALID : LH_OK;
    if (st == LH_OK) memcpy(out, c->buckets[c->active ^ 1] + (size_t)hid * 65536u, 65536u * 8u);
    pthread_mutex_unlock(&g_mu);
    return st;
}

/* the open snapshot was all-reduced (lh_snapshot_rows and a second all-reduce refuse); with g_mu held */
static int reduced(lh_ctx *c) { return c->frozen && comm_of(c)->reduced_at == c->snapshots; }

LH_API lh_status lh_snapshot_rows(lh_ctx *c, uint8_t *touched, uint64_t *deltas, uint32_t *frozen) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    lh_status st = !c->frozen || reduced(c) ? LH_ERR_STATE : LH_OK;
    if (st == LH_OK) {
        const uint64_t *fb = c->buckets[c->active ^ 1];
        for (uint32_t h = 0; touched && h < c->cfg.max_histograms; h++) {
            touched[h] = 0;
            for (uint32_t k = 0; k < 65536u; k++)
                if (fb[(size_t)h * 65536u + k]) { touched[h] = 1; break; }
        }
        if (deltas) memcpy(deltas, c->counters[c->active ^ 1], (size_t)c->cfg.max_counters * 8);
        if (frozen) *frozen = (uint32_t)(c->active ^ 1);
    }
    pthread_mutex_unlock(&g_mu);
    return st;
}

/* wait, with g_mu held, until every peer's field reached seq; 0 on timeout */
static int wait_peers(struct stub_comm *m, uint64_t seq, int summed) {
    struct timespec dl;
    clock_gettime(CLOCK_REALTIME, &dl);
    dl.tv_sec += 10;
    for (;;) {
        int all = 1;
        for (uint32_t r = 0; r < m->world; r++) {
            struct stub_comm *p = comm_of(m->peers[r]);
            if ((summed ? p->summed : p->arrived) < seq) all = 0;
        }
        if (all) return 1;
        if (pthread_cond_timedwait(&g_rcv, &g_mu, &dl) == ETIMEDOUT) return 0;
    }
}

LH_API lh_status lh_snapshot_allreduce_rows(lh_ctx *c, uint64_t seq, const uint32_t *frozen, uint32_t n_rows,
                                            const uint32_t *hist_map, uint32_t n_counter_rows,
                                            const uint32_t *counter_map, uint64_t *seq_out) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    struct stub_comm *m = comm_of(c);
    const uint32_t H = c->cfg.max_histograms, C = c->cfg.max_counters, W = m->world;
    lh_status st = LH_OK;
    if (!c->frozen || W < 2 || reduced(c)) st = LH_ERR_STATE;
    else if (!frozen || n_rows > H || n_counter_rows > C || (n_rows && !hist_map) || (n_counter_rows && !counter_map) ||
             seq <= m->seq)
        st = LH_ERR_INVALID;
    for (uint32_t r = 0; st == LH_OK && r < W; r++)
        if (frozen[r] > 1) st = LH_ERR_INVALID;
    if (st == LH_OK && frozen[m->rank] != (uint32_t)(c->active ^ 1)) st = LH_ERR_INVALID;
    for (size_t i = 0; st == LH_OK && i < (size_t)W * n_rows; i++)
        if (hist_map[i] != LH_ROW_ABSENT && hist_map[i] >= H) st = LH_ERR_RANGE;
    for (size_t i = 0; st == LH_OK && i < (size_t)W * n_counter_rows; i++)
        if (counter_map[i] != LH_ROW_ABSENT && counter_map[i] >= C) st = LH_ERR_RANGE;
    if (st != LH_OK) { pthread_mutex_unlock(&g_mu); return st; }
    g_rows_calls++;
    m->seq = seq;
    m->arrived = seq;
    pthread_cond_broadcast(&g_rcv);
    const int ok = wait_peers(m, seq, 0);
    uint64_t *hs = (uint64_t *)calloc((size_t)(n_rows ? n_rows : 1) * 65536u, 8);
    uint64_t *cs = (uint64_t *)calloc(C, 8);
    const uint32_t r0 = ok ? 0 : m->rank, r1 = ok ? W : m->rank + 1;
    for (uint32_t r = r0; r < r1; r++) {
        const lh_ctx *p = m->peers[r];
        const uint64_t *pb = p->buckets[frozen[r]], *pc = p->counters[frozen[r]];
        for (uint32_t g = 0; g < n_rows; g++) {
            const uint32_t h = hist_map[(size_t)r * n_rows + g];
            if (h == LH_ROW_ABSENT) continue;
            for (uint32_t k = 0; k < 65536u; k++) hs[(size_t)g * 65536u + k] += pb[(size_t)h * 65536u + k];
        }
        for (uint32_t g = 0; g < n_counter_rows; g++) {
            const uint32_t i = counter_map[(size_t)r * n_counter_rows + g];
            if (i != LH_ROW_ABSENT) cs[g] += pc[i];
        }
    }
    m->summed = seq;
    pthread_cond_broadcast(&g_rcv);
    if (ok && !wait_peers(m, seq, 1)) m->status = 1;
    else m->status = ok ? 0 : 1;
    uint64_t *fb = c->buckets[c->active ^ 1];
    memset(fb, 0, (size_t)H * 65536u * 8);
    memcpy(fb, hs, (size_t)n_rows * 65536u * 8);
    memcpy(c->counters[c->active ^ 1], cs, (size_t)C * 8);
    free(hs);
    free(cs);
    m->reduced_at = c->snapshots;
    if (seq_out) *seq_out = seq;
    pthread_mutex_unlock(&g_mu);
    return LH_OK;
}
