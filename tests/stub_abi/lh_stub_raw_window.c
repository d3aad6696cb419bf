/*
 * lh_stub_raw_window.c -- TEST-ONLY window boards (lh_raw_board_create_window) for the oracle-backed stub of the C ABI.
 *
 * tests/test_raw_window_cpu.py compiles it INSTEAD of lh_stub_raw_board.c (with lh_stub.c, lh_stub_reduce_sparse.c,
 * lh_stub_record.c, lh_stub_batch.c, lh_stub_graph.c, lh_stub_board.c and oracle/loghisto_oracle.c).  It includes
 * lh_stub_raw_board.c with that file's create / publish / destroy renamed, so the plain boards, the queries,
 * lh_stub_raw_alive and lh_stub_raw_bound are that file's, and wraps them: a window board keeps, per row, the dense
 * counts of its last `window` entering intervals in host memory, and after the plain stub has written a publish's
 * running counts it rewrites each row from the sum of those intervals (all 65 536 keys, or an empty row when every
 * interval in the window is empty; key_hi + LH_RAW_KEY_WRAPPED when the running count passed 2^64).  A second publish
 * to a window board in one snapshot is refused with LH_ERR_STATE, as the library refuses it.
 */
#define lh_raw_board_create lh_stub_plain_raw_board_create
#define lh_snapshot_publish_raw lh_stub_plain_publish_raw
#define lh_raw_board_destroy lh_stub_plain_raw_board_destroy
#include "lh_stub_raw_board.c"
#undef lh_raw_board_create
#undef lh_snapshot_publish_raw
#undef lh_raw_board_destroy

typedef struct {
    uint64_t handle;                 /* the board's handle; 0 = free */
    uint32_t window;
    uint64_t published;              /* publishes so far: the next replaces slot published % window */
    uint64_t snapshot;               /* lh_stats.snapshots at the latest publish */
    uint64_t *slots;                 /* [k][window][65536] dense counts by key + 32768 */
} WinBoard;

static WinBoard g_win[MAX_RAW_BOARDS];

static WinBoard *win_find(uint64_t handle) {
    for (int i = 0; i < MAX_RAW_BOARDS; i++)
        if (g_win[i].handle && g_win[i].handle == handle) return &g_win[i];
    return 0;
}

LH_API lh_status lh_raw_board_create(lh_ctx *ctx, uint32_t k, lh_raw_board *out) {
    return lh_stub_plain_raw_board_create(ctx, k, out);
}

LH_API lh_status lh_raw_board_create_window(lh_ctx *ctx, uint32_t k, uint32_t window, lh_raw_board *out) {
    if (window == 0) return LH_ERR_INVALID;
    if (window == 1) return lh_stub_plain_raw_board_create(ctx, k, out);
    if (window > LH_RAW_MAX_WINDOW) return LH_ERR_RANGE;
    lh_status st = lh_stub_plain_raw_board_create(ctx, k, out);
    if (st != LH_OK) return st;
    pthread_mutex_lock(&g_rmu);
    WinBoard *w = win_find(0);
    for (int i = 0; !w && i < MAX_RAW_BOARDS; i++)
        if (!g_win[i].handle) w = &g_win[i];
    w->handle = out->handle;
    w->window = window;
    w->published = 0;
    w->snapshot = 0;
    w->slots = (uint64_t *)calloc((size_t)k * window * 65536u, 8);
    pthread_mutex_unlock(&g_rmu);
    return LH_OK;
}

LH_API lh_status lh_snapshot_publish_raw(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *hist_ids) {
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    WinBoard *w = s ? win_find(s->handle) : 0;
    lh_stats stats;
    memset(&stats, 0, sizeof stats);
    if (w) {
        lh_get_stats(ctx, &stats);
        if (w->published && w->snapshot == stats.snapshots) { pthread_mutex_unlock(&g_rmu); return LH_ERR_STATE; }
    }
    pthread_mutex_unlock(&g_rmu);
    lh_status st = lh_stub_plain_publish_raw(ctx, b, hist_ids);
    if (st != LH_OK || !w) return st;
    pthread_mutex_lock(&g_rmu);
    const uint32_t slot = (uint32_t)(w->published % w->window);
    for (uint32_t r = 0; r < s->b.k; r++) {
        lh_raw_row_header *h = hdr(s, r);
        uint64_t *c = cells(s, r);
        uint64_t *in = w->slots + ((size_t)r * w->window + slot) * 65536u;
        for (uint32_t x = 0; x < 65536u; x++)   /* the plain publish wrote all keys or none */
            in[x] = h->key_lo > h->key_hi ? 0 : c[x] - (x ? c[x - 1] : 0);
        int any = 0, wrap = 0;
        uint64_t run = 0;
        for (uint32_t x = 0; x < 65536u; x++) {
            uint64_t sum = 0;
            for (uint32_t j = 0; j < w->window; j++) sum += w->slots[((size_t)r * w->window + j) * 65536u + x];
            for (uint32_t j = 0; j < w->window && !any; j++) any = w->slots[((size_t)r * w->window + j) * 65536u + x] != 0;
            run += sum;
            wrap |= run < sum;
            c[x] = run;
        }
        h->total = any ? run : 0;             /* seq / publishes: the plain publish already advanced them */
        h->key_lo = any ? -32768 : 0;
        h->key_hi = any ? 32767 + (wrap ? LH_RAW_KEY_WRAPPED : 0) : -1;
    }
    w->published++;
    w->snapshot = stats.snapshots;
    pthread_mutex_unlock(&g_rmu);
    return LH_OK;
}

LH_API lh_status lh_raw_board_destroy(lh_ctx *ctx, const lh_raw_board *b) {
    pthread_mutex_lock(&g_rmu);
    RawBoard *s = raw_find(ctx, b);
    WinBoard *w = s ? win_find(s->handle) : 0;
    if (w) {
        free(w->slots);
        memset(w, 0, sizeof *w);
    }
    pthread_mutex_unlock(&g_rmu);
    return lh_stub_plain_raw_board_destroy(ctx, b);
}
