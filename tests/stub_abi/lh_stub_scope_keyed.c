/*
 * lh_stub_scope_keyed.c -- TEST-ONLY mapped keyed samples and counter adds (lh_ingest_keyed_mapped_* /
 * lh_counter_add_mapped_*) for the oracle-backed stub of the C ABI.
 *
 * It includes lh_stub_graph_calls.c, which it extends, so tests/test_scope_keyed_cpu.py compiles this file in its place
 * (with lh_stub.c, lh_stub_reduce_sparse.c, lh_stub_record.c, lh_stub_batch.c and oracle/loghisto_oracle.c); compiled
 * with lh_stub_graph_calls.c instead, the stub is a library that predates these calls.  The calls validate as the
 * library does, then apply the map on the host and commit each sample or amount under its row into the active
 * interval: a local id >= k, or a row of LH_GRAPH_UNBOUND, is dropped and counted.  It adds:
 *   lh_stub_mapped_calls   how many of the four entry points below got past validation (i.e. would have enqueued work).
 */
#include "lh_stub_graph_calls.c"

static uint64_t g_mapped_calls;

LH_API uint64_t lh_stub_mapped_calls(void) {
    pthread_mutex_lock(&g_gmu);
    uint64_t n = g_mapped_calls;
    pthread_mutex_unlock(&g_gmu);
    return n;
}

static lh_status check_map(const lh_ctx *ctx, const uint32_t *h_map, uint32_t k, uint32_t limit) {
    if (k > LH_MAP_MAX_IDS || (k && !h_map)) return LH_ERR_INVALID;
    for (uint32_t i = 0; i < k; i++)
        if (h_map[i] != LH_GRAPH_UNBOUND && h_map[i] >= limit) return LH_ERR_RANGE;
    (void)ctx;
    return LH_OK;
}

static uint32_t row_of(const uint32_t *h_map, uint32_t k, uint32_t id) { return id < k ? h_map[id] : LH_GRAPH_UNBOUND; }

static lh_status mapped_keyed(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const void *ids, size_t id_bytes,
                              const void *vals, uint32_t kind, size_t n) {
    if (!ctx) return LH_ERR_INVALID;
    if ((kind != LH_VALUES_F64 && kind != LH_VALUES_I64NS) || (n && (!ids || !vals)) || ((uintptr_t)vals & 7u) ||
        ((uintptr_t)ids & (id_bytes - 1)))
        return LH_ERR_INVALID;
    lh_status st = check_map(ctx, h_map, k, ((const lh_config *)ctx)->max_histograms);
    if (st != LH_OK || n == 0) return st;
    pthread_mutex_lock(&g_gmu);
    g_mapped_calls++;
    for (size_t i = 0; st == LH_OK && i < n; i++) {
        const uint32_t id = id_bytes == 2 ? ((const uint16_t *)ids)[i] : ((const uint32_t *)ids)[i];
        const double v = kind == LH_VALUES_F64 ? ((const double *)vals)[i] : (double)((const int64_t *)vals)[i];
        st = commit(ctx, &v, row_of(h_map, k, id), 1, 0);
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

static lh_status mapped_counters(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const void *ids, size_t id_bytes,
                                 const uint64_t *amounts, size_t n) {
    if (!ctx) return LH_ERR_INVALID;
    if ((n && (!ids || !amounts)) || ((uintptr_t)amounts & 7u) || ((uintptr_t)ids & (id_bytes - 1))) return LH_ERR_INVALID;
    lh_status st = check_map(ctx, h_map, kc, ((const lh_config *)ctx)->max_counters);
    if (st != LH_OK || n == 0) return st;
    pthread_mutex_lock(&g_gmu);
    g_mapped_calls++;
    for (size_t i = 0; st == LH_OK && i < n; i++) {
        const uint32_t id = id_bytes == 2 ? ((const uint16_t *)ids)[i] : ((const uint32_t *)ids)[i];
        st = commit(ctx, &amounts[i], row_of(h_map, kc, id), 1, 1);
    }
    pthread_mutex_unlock(&g_gmu);
    return st;
}

LH_API lh_status lh_ingest_keyed_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint16_t *d_ids,
                                            const void *d_values, uint32_t kind, size_t n, void *stream) {
    (void)stream;
    return mapped_keyed(ctx, h_map, k, d_ids, 2, d_values, kind, n);
}
LH_API lh_status lh_ingest_keyed_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint32_t *d_ids,
                                            const void *d_values, uint32_t kind, size_t n, void *stream) {
    (void)stream;
    return mapped_keyed(ctx, h_map, k, d_ids, 4, d_values, kind, n);
}
LH_API lh_status lh_counter_add_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint16_t *d_ids,
                                           const uint64_t *d_amounts, size_t n, void *stream) {
    (void)stream;
    return mapped_counters(ctx, h_map, kc, d_ids, 2, d_amounts, n);
}
LH_API lh_status lh_counter_add_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint32_t *d_ids,
                                           const uint64_t *d_amounts, size_t n, void *stream) {
    (void)stream;
    return mapped_counters(ctx, h_map, kc, d_ids, 4, d_amounts, n);
}
