/*
 * lh_stub_rows_pack.c -- TEST-ONLY joined ranks through the caller's all-reduce (lh_snapshot_row_levels /
 * lh_snapshot_pack_rows / lh_snapshot_unpack_rows) for the oracle-backed stub of the C ABI.
 *
 * It includes lh_stub_ranks.c (and through it lh_stub.c), which it extends, so tests/test_ranks_allreduce_cpu.py
 * compiles this file in their place, with the same companions.  The calls validate as the library does.  "Device"
 * buffers are host memory: the pack writes this rank's frozen rows into a send payload laid out as the header states,
 * the caller sums the payloads of every rank into recv, and the unpack writes recv (or send) over the frozen arrays,
 * row g at index g, counters below n_counter_rows, nothing else, so the snapshot's reduce, export and copy read the
 * job-wide rows (as lh_stub_ranks.c's all-reduce leaves them).  lh_snapshot_begin is wrapped to forget the previous
 * snapshot's pack.  It adds:
 *   lh_stub_pack_calls     how many lh_snapshot_pack_rows calls got past validation (would have launched);
 *   lh_stub_unpack_calls   the same for lh_snapshot_unpack_rows.
 */
#define lh_snapshot_begin lh_snapshot_begin_base
#include "lh_stub_ranks.c"
#undef lh_snapshot_begin

#include <math.h>

struct stub_pack {
    lh_ctx *ctx;
    int packed;
    uint32_t n_rows, n_counter_rows;
    uint8_t *levels;              /* [max_histograms] */
    uint64_t words, cap;
    uint64_t *send, *recv;
};
static struct stub_pack g_pack[64];
static uint64_t g_pack_calls, g_unpack_calls;

/* with g_mu held */
static struct stub_pack *pack_of(lh_ctx *c) {
    for (int i = 0; i < 64; i++)
        if (g_pack[i].ctx == c) return &g_pack[i];
    for (int i = 0; i < 64; i++)
        if (!g_pack[i].ctx) { g_pack[i].ctx = c; return &g_pack[i]; }
    return NULL;
}

LH_API uint64_t lh_stub_pack_calls(void) {
    pthread_mutex_lock(&g_mu);
    uint64_t n = g_pack_calls;
    pthread_mutex_unlock(&g_mu);
    return n;
}

LH_API uint64_t lh_stub_unpack_calls(void) {
    pthread_mutex_lock(&g_mu);
    uint64_t n = g_unpack_calls;
    pthread_mutex_unlock(&g_mu);
    return n;
}

LH_API lh_status lh_snapshot_begin(lh_ctx *c) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    pack_of(c)->packed = 0;
    pthread_mutex_unlock(&g_mu);
    return lh_snapshot_begin_base(c);
}

static uint32_t stub_win(const lh_ctx *c) {
    const double P = c->cfg.precision ? (double)c->cfg.precision : 100.0;
    return (uint32_t)floor(P * 63.0 * 0.6931471805599453094172321 + 0.5) + 1u;
}

/* payload word j of a row at `level` -> its cell */
static uint32_t row_cell(uint32_t level, uint32_t j, uint32_t win) {
    return level == 3 || j < win ? j : j + 65537u - 2u * win;
}
static uint32_t row_words(uint32_t level, uint32_t win) { return level == 0 ? 0 : level == 1 ? 2u * win - 1u : 65536u; }

LH_API lh_status lh_snapshot_row_levels(lh_ctx *c, uint8_t *levels) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    lh_status st = !c->frozen || reduced(c) ? LH_ERR_STATE : !levels ? LH_ERR_INVALID : LH_OK;
    if (st == LH_OK) {
        const uint32_t win = stub_win(c);
        const uint64_t *fb = c->buckets[c->active ^ 1];
        for (uint32_t h = 0; h < c->cfg.max_histograms; h++) {
            uint8_t lv = 0;
            for (uint32_t k = 0; k < 65536u; k++) {
                if (!fb[(size_t)h * 65536u + k]) continue;
                if (k < win || k >= 65536u - (win - 1u)) lv = lv ? lv : 1;
                else { lv = 3; break; }
            }
            levels[h] = lv;
        }
    }
    pthread_mutex_unlock(&g_mu);
    return st;
}

LH_API lh_status lh_snapshot_pack_rows(lh_ctx *c, uint32_t n_rows, const uint32_t *hist_rows, const uint8_t *levels,
                                       uint32_t n_counter_rows, const uint32_t *counter_rows, uint64_t **d_send,
                                       uint64_t **d_recv, uint64_t *n_words, void **stream) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    struct stub_pack *p = pack_of(c);
    const uint32_t H = c->cfg.max_histograms, C = c->cfg.max_counters;
    lh_status st = LH_OK;
    if (!c->frozen || reduced(c) || p->packed) st = LH_ERR_STATE;
    else if (n_rows > H || n_counter_rows > C || (n_rows && (!hist_rows || !levels)) || (n_counter_rows && !counter_rows) ||
             !d_send || !d_recv || !n_words || !stream)
        st = LH_ERR_INVALID;
    for (uint32_t g = 0; st == LH_OK && g < n_rows; g++)
        if (levels[g] != 0 && levels[g] != 1 && levels[g] != 3) st = LH_ERR_INVALID;
    for (uint32_t g = 0; st == LH_OK && g < n_rows; g++)
        if (hist_rows[g] != LH_ROW_ABSENT && hist_rows[g] >= H) st = LH_ERR_RANGE;
    for (uint32_t g = 0; st == LH_OK && g < n_counter_rows; g++)
        if (counter_rows[g] != LH_ROW_ABSENT && counter_rows[g] >= C) st = LH_ERR_RANGE;
    if (st != LH_OK) { pthread_mutex_unlock(&g_mu); return st; }
    const uint32_t win = stub_win(c);
    uint64_t words = n_counter_rows;
    for (uint32_t g = 0; g < n_rows; g++) words += row_words(levels[g], win);
    if (words > p->cap) {
        free(p->send); free(p->recv);
        p->send = (uint64_t *)calloc(words, 8);
        p->recv = (uint64_t *)calloc(words, 8);
        p->cap = words;
    }
    if (!p->levels) p->levels = (uint8_t *)calloc(H, 1);
    const uint64_t *fb = c->buckets[c->active ^ 1], *fc = c->counters[c->active ^ 1];
    uint64_t at = 0;
    for (uint32_t g = 0; g < n_rows; g++) {
        const uint32_t n = row_words(levels[g], win);
        for (uint32_t j = 0; j < n; j++)
            p->send[at + j] = hist_rows[g] == LH_ROW_ABSENT ? 0 : fb[(size_t)hist_rows[g] * 65536u + row_cell(levels[g], j, win)];
        at += n;
        p->levels[g] = levels[g];
    }
    for (uint32_t g = 0; g < n_counter_rows; g++) p->send[at + g] = counter_rows[g] == LH_ROW_ABSENT ? 0 : fc[counter_rows[g]];
    p->packed = 1;
    p->n_rows = n_rows;
    p->n_counter_rows = n_counter_rows;
    p->words = words;
    g_pack_calls++;
    *d_send = p->send;
    *d_recv = p->recv;
    *n_words = words;
    *stream = NULL;
    pthread_mutex_unlock(&g_mu);
    return LH_OK;
}

LH_API lh_status lh_snapshot_unpack_rows(lh_ctx *c, uint32_t summed) {
    if (!c) return LH_ERR_INVALID;
    pthread_mutex_lock(&g_mu);
    struct stub_pack *p = pack_of(c);
    if (!c->frozen || reduced(c) || !p->packed) { pthread_mutex_unlock(&g_mu); return LH_ERR_STATE; }
    const uint32_t H = c->cfg.max_histograms, C = c->cfg.max_counters, win = stub_win(c);
    const uint64_t *src = summed ? p->recv : p->send;
    uint64_t *fb = c->buckets[c->active ^ 1], *fc = c->counters[c->active ^ 1];
    memset(fb, 0, (size_t)H * 65536u * 8);
    memset(fc, 0, (size_t)C * 8);
    uint64_t at = 0;
    for (uint32_t g = 0; g < p->n_rows; g++) {
        const uint32_t n = row_words(p->levels[g], win);
        for (uint32_t j = 0; j < n; j++) fb[(size_t)g * 65536u + row_cell(p->levels[g], j, win)] = src[at + j];
        at += n;
    }
    for (uint32_t g = 0; g < p->n_counter_rows; g++) fc[g] = src[at + g];
    comm_of(c)->reduced_at = c->snapshots;
    g_unpack_calls++;
    pthread_mutex_unlock(&g_mu);
    return LH_OK;
}
