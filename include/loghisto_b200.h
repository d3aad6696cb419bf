/*
 * loghisto_b200.h -- C ABI of the H100-native loghisto ingest/reduction engine.
 *
 * This is the drop-in boundary for ONE path of spacejam/loghisto: the bodies of
 *   MetricSystem.Histogram      (metrics.go:273-295)  + compress (metrics.go:316-322)
 *   MetricSystem.Counter        (metrics.go:251-269)
 *   TimerToken.Stop             (metrics.go:242-246)   (its Histogram() call)
 *   collectRawMetrics           (metrics.go:420-479)   (cache swap = snapshot)
 *   processHistograms/percentile(metrics.go:336-418)   + decompress (metrics.go:326-332)
 * The reference has no FFI of its own (it is pure Go); these entry points are
 * what a cgo shim that keeps loghisto's exported Go API binds (INTEGRATION.md).
 *
 * Conventions (mirroring the reference's: ingest never fails loudly, never
 * blocks on consumers, metrics.go:570-573/632-636):
 *   - every function returns an lh_status (0 = LH_OK, negative = error); nothing
 *     throws, nothing calls back into the caller;
 *   - all functions are thread-safe; ingest may run concurrently with a
 *     snapshot (double-buffered bucket arrays), and may be issued from any
 *     number of streams and of contexts on one device (launches of the
 *     write-combining keyed kernel on a device are serialised);
 *   - `stream` arguments are a cudaStream_t passed as void* (NULL = the
 *     context's own ingest stream); device pointers are plain pointers;
 *   - names never cross the boundary: the caller interns name -> dense id.
 *
 * Bucket layout: one dense uint64[65536] per histogram, indexed by
 * (uint16_t)key where key is the reference's int16 bucket.  Samples whose id is
 * >= max_histograms are dropped and counted (lh_stats.dropped).
 *
 * There is NO CPU fallback: without a CUDA device lh_create fails with
 * LH_ERR_NO_DEVICE.
 */
#ifndef LOGHISTO_B200_H_
#define LOGHISTO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LH_API __attribute__((visibility("default")))
#else
#define LH_API
#endif

#define LH_ABI_VERSION 2
#define LH_KEYS_PER_HISTOGRAM 65536
#define LH_MAX_PERCENTILES 32
#define LH_MAX_PRECISION 250     /* buckets per unit of ln(1+|v|); the reference's constant is 100 (metrics.go:40-43) */
#define LH_MAX_RANKS 16          /* GPUs one lh_comm group may span (one node) */
#define LH_PEER_HANDLE_BYTES 1024

typedef int32_t lh_status;
enum {
    LH_OK = 0,
    LH_ERR_INVALID = -1,    /* bad argument */
    LH_ERR_CUDA = -2,       /* a CUDA runtime call failed; see lh_last_error */
    LH_ERR_NOMEM = -3,      /* host or device allocation failed */
    LH_ERR_NO_DEVICE = -4,  /* no usable CUDA device: there is no CPU fallback */
    LH_ERR_STATE = -5,      /* call out of order (e.g. reduce without a snapshot) */
    LH_ERR_RANGE = -6       /* id / size out of the configured range */
};

typedef struct lh_ctx lh_ctx;

typedef struct lh_config {
    uint32_t struct_size;     /* = sizeof(lh_config) */
    int32_t device;           /* CUDA ordinal */
    uint32_t max_histograms;  /* H >= 1: ids 0..H-1 */
    uint32_t max_counters;    /* C >= 1: ids 0..C-1 */
    uint64_t staging_bytes;   /* bytes per pinned staging slot (0 = 32 MiB) */
    uint32_t staging_slots;   /* slots in the ring (0 = 3) */
    uint32_t flags;           /* reserved, 0 */
    uint32_t precision;       /* `precision` of compress/decompress (metrics.go:40-43, 316-332): key =
                               * int16(precision*ln(1+|v|)+0.5).  0 = the reference's 100; 1..LH_MAX_PRECISION */
    uint32_t reserved[3];     /* 0 */
} lh_config;

/* ---- lifecycle ------------------------------------------------------- */
LH_API lh_status lh_create(const lh_config *cfg, lh_ctx **out);
LH_API lh_status lh_destroy(lh_ctx *ctx);
LH_API const char *lh_strerror(lh_status st);
/* Last error detail recorded on this context (thread-unsafe snapshot, for logs). */
LH_API const char *lh_last_error(const lh_ctx *ctx);
LH_API uint32_t lh_abi_version(void);

/* ---- ingest, device-resident inputs ------------------------------------
 * Replaces compress + the map lookup + atomic.AddUint64 of metrics.go:273-295.
 * All launches are asynchronous on `stream`. */

/* n samples of ONE histogram (the single-name loop of print_benchmark.go:59-67). */
LH_API lh_status lh_ingest_f64(lh_ctx *ctx, uint32_t histogram_id, const double *d_values, size_t n,
                        void *stream);
/* (id,value) pairs, the name->histogram dispatch path.  ids are dense ids. */
LH_API lh_status lh_ingest_keyed_f64_u16(lh_ctx *ctx, const uint16_t *d_ids, const double *d_values,
                                  size_t n, void *stream);
LH_API lh_status lh_ingest_keyed_f64_u32(lh_ctx *ctx, const uint32_t *d_ids, const double *d_values,
                                  size_t n, void *stream);
/* Timer samples: value = float64(duration.Nanoseconds()), metrics.go:242-246. */
LH_API lh_status lh_ingest_keyed_i64ns_u16(lh_ctx *ctx, const uint16_t *d_ids, const int64_t *d_nanos,
                                    size_t n, void *stream);

/* A batch of Histogram samples AND a batch of Timer samples (metrics.go:242-246 then :273-295) in one call: above a few
 * million pairs both are binned by ONE launch of the write-combining kernel, so its fixed costs are paid once per batch
 * (configs[4]: 50 % Histogram / 25 % Timer ops).  Same semantics as lh_ingest_keyed_f64_u16 followed by
 * lh_ingest_keyed_i64ns_u16; either count may be 0. */
LH_API lh_status lh_ingest_keyed_pair_u16(lh_ctx *ctx, const uint16_t *d_ids_f64, const double *d_values, size_t n_f64,
                                          const uint16_t *d_ids_ns, const int64_t *d_nanos, size_t n_ns, void *stream);
/* Many device arrays, each under its own histogram id, in one call (per-layer tensors, per-endpoint latency batches):
 * the bucket counts are exactly those of issuing, for every item,
 *   LH_VALUES_F64    lh_ingest_f64(ctx, histogram_id, d_values, n, stream)           Histogram(name, v), metrics.go:273-295
 *   LH_VALUES_I64NS  the int64 nanoseconds of lh_ingest_keyed_i64ns_u16, float64(ns) round-to-nearest
 *                                                                                     TimerToken.Stop, metrics.go:242-246
 * but the call is ONE write bracket: one sequence number (lh_kernel_ms covers all its launches), lh_stats.samples += the
 * sum of n, and every item lands in the same interval (a concurrent lh_snapshot_begin comes before all of it or after
 * all of it).  Items may repeat ids, alias or overlap each other's memory and come in any order.
 *
 * Routing: an F64 item of at least 2^20 samples is ingested by the single-histogram kernel, as lh_ingest_f64 would;
 * every other item goes to one kernel that deals the concatenation of the items to CTAs in pieces and counts them
 * through a shared-memory combining table, up to 1024 items per launch.  A batch of a few hundred samples runs on one
 * CTA, not the whole machine.
 * Measured on an H100 80GB HBM3 at 700 W (DESIGN.md section 5): 64 arrays of 64 samples take 0.050 ms to a
 * synchronise, against 0.73 ms as 64 lh_ingest_f64 calls; 4096 arrays of 1024 samples 0.36 ms against 48 ms.  A single
 * short array is slower than one lh_ingest_f64 (17 vs 9 us of kernel time).
 *
 * Every item is validated before anything is enqueued; on error nothing is launched, counted or sequenced:
 * LH_ERR_INVALID for h_items NULL with n_items > 0 or an unknown kind, and, for an item with n > 0, d_values NULL or
 * not 8-byte aligned; LH_ERR_RANGE for an item with n > 0 and histogram_id >= max_histograms (as lh_ingest_f64, not
 * the keyed calls' drop-and-count).  Items with n == 0 are skipped; a call without samples returns LH_OK with no
 * bracket and no launch.  h_items may be reused when the call returns; the device arrays must stay valid until the
 * stream's work completes.  The call never waits for the device and allocates nothing. */
#define LH_VALUES_F64 0     /* float64 values */
#define LH_VALUES_I64NS 1   /* int64 nanoseconds */
typedef struct lh_batch_item {
    const void *d_values;   /* device memory, 8-byte aligned */
    uint64_t n;
    uint32_t histogram_id;
    uint32_t kind;          /* LH_VALUES_* */
} lh_batch_item;
LH_API lh_status lh_ingest_batch(lh_ctx *ctx, const lh_batch_item *h_items, uint32_t n_items, void *stream);

/* Counter(name, amount), metrics.go:251-269: wrapping uint64 adds.  NULL inputs with n > 0, amounts not 8-byte aligned
 * or ids not naturally aligned give LH_ERR_INVALID, before anything is enqueued. */
LH_API lh_status lh_counter_add_u16(lh_ctx *ctx, const uint16_t *d_ids, const uint64_t *d_amounts,
                             size_t n, void *stream);
LH_API lh_status lh_counter_add_u32(lh_ctx *ctx, const uint32_t *d_ids, const uint64_t *d_amounts,
                             size_t n, void *stream);

/* Keyed samples and counter adds under local ids, for callers whose global ids are not stable (MetricSystem record
 * scopes: interned names whose ids are recycled).  h_map (host memory, k entries, reusable when the call returns) maps
 * local id l < k to histogram / counter h_map[l]; a local id >= k, or an entry of LH_GRAPH_UNBOUND, drops the sample or
 * op and counts 1 in lh_stats.dropped (k = 0 drops everything).  Entries may repeat.  Otherwise the semantics are those
 * of lh_ingest_keyed_* (values of `kind` LH_VALUES_F64, or LH_VALUES_I64NS recorded as float64(ns)) and
 * lh_counter_add_* (wrapping uint64): one write bracket and sequence number, lh_stats.samples / counter_ops, and
 * lh_keyed_kernel_name reports the route.  The keyed kernels are those of lh_ingest_keyed_*, planned on k ids instead of
 * max_histograms, so a call over a few names takes the shared-memory privatised kernel.
 * Errors, before anything is enqueued: LH_ERR_INVALID for k > 4096, h_map NULL with k > 0, an unknown kind, NULL
 * inputs with n > 0, values / amounts not 8-byte aligned or ids not naturally aligned; LH_ERR_RANGE for an entry
 * >= max_histograms (max_counters) other than LH_GRAPH_UNBOUND.  n = 0 returns LH_OK with no bracket. */
#define LH_MAP_MAX_IDS 4096
LH_API lh_status lh_ingest_keyed_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint16_t *d_ids,
                                            const void *d_values, uint32_t kind, size_t n, void *stream);
LH_API lh_status lh_ingest_keyed_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint32_t *d_ids,
                                            const void *d_values, uint32_t kind, size_t n, void *stream);
LH_API lh_status lh_counter_add_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint16_t *d_ids,
                                           const uint64_t *d_amounts, size_t n, void *stream);
LH_API lh_status lh_counter_add_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint32_t *d_ids,
                                           const uint64_t *d_amounts, size_t n, void *stream);

/* ---- ingest, host-resident inputs ----------------------------------------
 * Same semantics, inputs in host memory.  Copies are chunked and overlapped
 * with the kernels.  On return the host buffers may be reused; the work may
 * still be in flight on the context's ingest stream. */
LH_API lh_status lh_ingest_f64_host(lh_ctx *ctx, uint32_t histogram_id, const double *h_values, size_t n);
LH_API lh_status lh_ingest_keyed_f64_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const double *h_values,
                                       size_t n);
LH_API lh_status lh_ingest_keyed_i64ns_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const int64_t *h_nanos,
                                         size_t n);
LH_API lh_status lh_counter_add_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const uint64_t *h_amounts,
                                  size_t n);

/* ---- merging snapshots --------------------------------------------------
 * Adds n sparse (histogram id, int16 key, uint64 count) triples -- the format lh_snapshot_export returns -- into
 * the ACTIVE bucket arrays.  Bucket counts are a commutative monoid, so snapshots taken on other hosts or GPUs
 * merge exactly (SURVEY.md section 8f rank 3); it also lets a caller re-reduce a RawMetricSet it holds. */
LH_API lh_status lh_merge_counts_host(lh_ctx *ctx, const uint32_t *h_ids, const int16_t *h_keys,
                                      const uint64_t *h_counts, size_t n);

/* ---- pinned staging ring (the cgo-friendly feed) ------------------------
 * cgo forbids C code from keeping Go pointers after a call returns, so the
 * shim fills C-owned pinned memory instead.  A slot of `staging_bytes` is laid
 * out by the caller as it likes and committed with one of the calls below,
 * which enqueue H2D + kernel and recycle the slot when the copy has landed.
 * lh_staging_acquire blocks only when every slot is still in flight. */
typedef struct lh_staging {
    void *host;        /* pinned host memory, `bytes` long, 256-byte aligned */
    uint64_t bytes;
    uint32_t slot;
    uint32_t reserved;
} lh_staging;
LH_API lh_status lh_staging_acquire(lh_ctx *ctx, lh_staging *out);
/* slot holds n float64 values of one histogram */
LH_API lh_status lh_staging_commit_f64(lh_ctx *ctx, const lh_staging *s, uint32_t histogram_id, size_t n);
/* slot holds n float64 values at offset 0 followed, at byte offset
 * ids_offset (multiple of 16), by n uint16 ids */
LH_API lh_status lh_staging_commit_keyed_f64_u16(lh_ctx *ctx, const lh_staging *s, size_t n,
                                          uint64_t ids_offset);
/* slot holds n uint64 amounts at offset 0 and n uint16 ids at ids_offset */
LH_API lh_status lh_staging_commit_counter_u16(lh_ctx *ctx, const lh_staging *s, size_t n,
                                        uint64_t ids_offset);
/* give a slot back unused */
LH_API lh_status lh_staging_abandon(lh_ctx *ctx, const lh_staging *s);

/* ---- recording from CUDA code (include/loghisto_b200_device.cuh) ----------
 * A record scope lets the caller's own kernels add samples with lh::record / lh::record_ns / lh::count /
 * lh::BlockHistogram, without materialising (id, value) pairs in memory first.
 *
 *   lh_record_begin  orders `stream` (NULL = the context's ingest stream) after the zeroing of the active interval's
 *                    arrays, fills *out with them and opens a scope.  Never blocks.
 *   lh_record_end    marks the end of the scope on its stream (the snapshot of the interval is ordered after it) and
 *                    closes it.  LH_ERR_INVALID for an unknown ticket or one already closed.
 *
 * Contract: kernels that use a recorder are enqueued on the scope's stream between the two calls, and the recorder
 * (passed to them by value) is not used after lh_record_end.  While scopes of the active interval are open,
 * lh_snapshot_begin makes the spare arrays active (scopes opened from then on record into the next interval) and
 * waits until every scope of the interval being frozen has been ended; it returns LH_ERR_STATE instead when the
 * calling thread itself holds such a scope.  Ingest calls never wait for scopes.  lh_destroy returns LH_ERR_STATE
 * while a scope is open.  Records do not count in lh_stats.samples / counter_ops; dropped ids count in
 * lh_stats.dropped. */
typedef struct lh_recorder {          /* passed by value to kernels; valid only inside its scope */
    uint64_t *d_buckets;              /* [max_histograms][65536] of the interval */
    uint32_t *d_flags;                /* [max_histograms] */
    uint64_t *d_counters;             /* [max_counters] interval deltas */
    uint64_t *d_dropped;              /* the context's dropped tally */
    uint32_t max_histograms, max_counters;
    uint32_t block_smem_bytes;        /* shared memory one lh::BlockHistogram needs at this precision */
    uint32_t reserved;
    uint64_t scope;                   /* ticket for lh_record_end */
    uint8_t prec[48];                 /* lh::Prec, opaque to C */
} lh_recorder;
LH_API lh_status lh_record_begin(lh_ctx *ctx, void *stream, lh_recorder *out);
LH_API lh_status lh_record_end(lh_ctx *ctx, const lh_recorder *rec);

/* ---- recording from CUDA graphs ---------------------------------------------------------------------------------
 * A record scope hands out the active interval's rows, which a captured kernel would keep writing at every replay,
 * after the snapshot froze them.  A graph recorder owns its rows instead: `rec` is an ordinary lh_recorder whose
 * d_buckets / d_flags / d_counters are k histogram rows (local ids 0 .. k-1) and kc counters that no snapshot swaps or
 * clears, so lh::record / record_ns / count / stop / BlockHistogram / BlockRecorder work unchanged in kernels captured
 * into a CUDA graph and replayed any number of times.  Each lh_snapshot_begin drains every live recorder into the
 * interval it freezes: one kernel on the snapshot stream takes every non-zero cell with an atomic exchange to 0 and
 * adds it to the row of the histogram (counter) id the local row is bound to at that moment.  Replays running
 * meanwhile keep adding, so each count is taken by exactly one drain; the host never waits for a replay.  A count
 * lands in the interval of the first collection whose drain finds it, so a caller that wants a replay in a given
 * interval synchronises the replay's stream before collecting.
 *
 *   lh_graph_recorder_create   allocates and zeroes k rows of uint64[65536] (512 KiB each), k flags and kc counters
 *                              (and k timer start marks, set to never started, in the same allocation),
 *                              k <= max_histograms, kc <= max_counters, k + kc >= 1, and binds them: hist_ids[i] /
 *                              counter_ids[i] (NULL = all unbound) is the context id local row i drains into.  The
 *                              recorder has max_histograms = k and max_counters = kc (a local id >= k is dropped and
 *                              counted, as in a scope), the context's d_dropped and precision, and a `scope` that
 *                              lh_record_end refuses with LH_ERR_INVALID.  Call it outside any stream capture; it
 *                              waits for the zeroing.
 *   lh_graph_recorder_bind     sets the target ids of the rows (either array may be NULL: unchanged).  Takes effect at
 *                              the next drain.  LH_GRAPH_UNBOUND: that row's drained counts are dropped and counted in
 *                              lh_stats.dropped (for a counter, its drained amount).
 *   lh_graph_recorder_ingest   lh_ingest_batch into the recorder's rows: the same items, kinds, validation (ids are
 *                              local: LH_ERR_RANGE for histogram_id >= k) and kernels, but no write bracket, event,
 *                              sequence number, lh_stats.samples or allocation -- it only enqueues kernels, so it may be
 *                              captured into a CUDA graph (or called on an ordinary stream).  On error nothing is
 *                              enqueued.
 *   lh_graph_recorder_ingest_keyed_u16 / _u32
 *                              n (local id, value) pairs into the recorder's rows: values of `kind` LH_VALUES_F64 or
 *                              LH_VALUES_I64NS as in lh_ingest_batch, ids local (an id >= k is dropped and counted in
 *                              lh_stats.dropped, also when k = 0).  Validation as lh_ingest_keyed_*: NULL inputs with
 *                              n > 0, values not 8-byte aligned, ids not naturally aligned or any other kind give
 *                              LH_ERR_INVALID.  One sm_90a kernel (k_ingest_keyed_graph) per up to 2^31 samples per CTA.
 *   lh_graph_recorder_counter_add_u16 / _u32
 *                              n (local id, amount) pairs: wrapping uint64 adds into the recorder's kc counters; an op
 *                              with id >= kc counts 1 in lh_stats.dropped.  NULL inputs with n > 0, or amounts / ids not
 *                              naturally aligned, give LH_ERR_INVALID.
 *   lh_graph_recorder_timer_start / _stop
 *                              a GPU-timed span of local histogram `histogram` (LH_ERR_RANGE when >= k): the start
 *                              writes the device clock into the histogram's start mark, the stop records
 *                              float64(now - mark) into its row and, when d_duration_ns is not NULL (8-byte aligned
 *                              device memory, else LH_ERR_INVALID), writes the int64 duration there.  A stop whose mark
 *                              was never started records nothing, writes nothing and counts 1 in lh_stats.dropped.  The
 *                              mark stays after a stop, so a span may be stopped again.  The caller orders a start
 *                              before its stop: the same stream, or its own fork / join inside the capture.  A histogram
 *                              has one mark per recorder, so one open span at a time; sequential spans (one per layer)
 *                              are fine, concurrent spans of one histogram on parallel branches need two recorders or
 *                              lh::start_timer in a kernel.
 *                              These six calls, like lh_graph_recorder_ingest, only enqueue kernels on `stream` (NULL =
 *                              the ingest stream): no event, host wait, allocation, write bracket, sequence number or
 *                              lh_stats.samples / counter_ops, so they may be captured in any capture mode or called on
 *                              an ordinary stream.  Every check runs first; on error, and for n = 0, nothing is enqueued.
 *   lh_graph_recorder_destroy  enqueues a final drain on `stream` (NULL = the ingest stream) into the active interval
 *                              as one write bracket, as an ingest call, and frees the rows, stream-ordered, after it and
 *                              after every collection drain already issued.  The caller guarantees that no replay that
 *                              uses the recorder is pending or will be launched.  lh_destroy frees every recorder left.
 *
 * A handle carries its context: a destroyed or foreign handle gets LH_ERR_INVALID and touches nothing.  Every call
 * that takes the context's lock (the snapshot calls, lh_sync, lh_destroy and the host-fed ingest calls among them)
 * switches the calling thread to cudaStreamCaptureModeRelaxed for its duration, so a collection from another thread
 * neither fails nor invalidates a capture that some thread runs in the global mode (torch.cuda.graph's default). */
#define LH_GRAPH_UNBOUND 0xFFFFFFFFu
typedef struct lh_graph_recorder {
    uint64_t handle;          /* opaque */
    lh_recorder rec;          /* pass by value to captured kernels */
} lh_graph_recorder;
LH_API lh_status lh_graph_recorder_create(lh_ctx *ctx, uint32_t n_histograms, uint32_t n_counters,
                                          const uint32_t *hist_ids, const uint32_t *counter_ids,
                                          lh_graph_recorder *out);
LH_API lh_status lh_graph_recorder_bind(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *hist_ids,
                                        const uint32_t *counter_ids);
LH_API lh_status lh_graph_recorder_ingest(lh_ctx *ctx, const lh_graph_recorder *g, const lh_batch_item *h_items,
                                          uint32_t n_items, void *stream);
LH_API lh_status lh_graph_recorder_ingest_keyed_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                    const void *d_values, uint32_t kind, size_t n, void *stream);
LH_API lh_status lh_graph_recorder_ingest_keyed_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                    const void *d_values, uint32_t kind, size_t n, void *stream);
LH_API lh_status lh_graph_recorder_counter_add_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                   const uint64_t *d_amounts, size_t n, void *stream);
LH_API lh_status lh_graph_recorder_counter_add_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                   const uint64_t *d_amounts, size_t n, void *stream);
LH_API lh_status lh_graph_recorder_timer_start(lh_ctx *ctx, const lh_graph_recorder *g, uint32_t histogram, void *stream);
LH_API lh_status lh_graph_recorder_timer_stop(lh_ctx *ctx, const lh_graph_recorder *g, uint32_t histogram, void *stream,
                                              int64_t *d_duration_ns);
LH_API lh_status lh_graph_recorder_destroy(lh_ctx *ctx, const lh_graph_recorder *g, void *stream);

/* ---- device subscriptions: each collection's processed metrics in device memory --------------------------------
 * SubscribeToProcessedMetrics (metrics.go:218, 508-525) for consumers on the GPU.  A board is device memory the library
 * owns; lh_snapshot_publish writes the named rows of the open snapshot's reduction into it, on the snapshot stream,
 * and kernels (include/loghisto_b200_device.cuh: lh::read_histogram / lh::read_counter) or lh_board_read read the
 * latest publish from there with no host call, also from CUDA-graph replays.  A board is guarded by a seqlock:
 * `seq` is odd while a publish writes it and advances by 2 per publish, so every read is of one publish.
 *
 * Layout (bytes): lh_board_header at 0, k lh_board_hist_row, then kc lh_board_counter_row.
 *
 *   lh_board_create      allocates a board of k histogram rows and kc counter rows (k <= max_histograms,
 *                        kc <= max_counters, k + kc >= 1) and zeroes it: every row unbound, np = 0, publishes = 0.
 *                        Call it outside any stream capture; it waits for the zeroing.
 *   lh_snapshot_publish  fills every row from the most recent lh_snapshot_reduce / lh_snapshot_reduce_async of the
 *                        open snapshot (LH_ERR_STATE without one, or outside a snapshot):
 *                          histogram row i, hist_ids[i] = h: count, sum, avg, pkeys[0..np), pvals[0..np) bit for bit
 *                            as that reduction reports h (the all-reduced values after lh_snapshot_allreduce), and
 *                            present = whether h holds a non-empty bucket (count != 0, or a count that wrapped);
 *                          hist_ids[i] = LH_GRAPH_UNBOUND (or hist_ids NULL): an untouched histogram as the reduction
 *                            reports one (count 0, sum 0, avg NaN, keys INT32_MIN, values NaN), present = 0;
 *                          counter row i, counter_ids[i] = c: rate = the interval delta lh_snapshot_export reports in
 *                            counter_deltas[c], present = 1; LH_GRAPH_UNBOUND (or counter_ids NULL): rate 0, present 0;
 *                            total = counter_totals[i] either way (0 when counter_totals is NULL).
 *                        Percentile slots j >= np hold INT32_MIN / NaN.  LH_ERR_RANGE for an id >= max_histograms /
 *                        max_counters other than LH_GRAPH_UNBOUND.  The publish is enqueued on the snapshot stream after
 *                        that reduction (so it may follow lh_snapshot_reduce_async before lh_snapshot_result); it never
 *                        waits and never allocates.
 *   lh_board_read        enqueues ONE kernel on `stream` (NULL = the ingest stream) that copies a consistent image of the
 *                        whole board (b->bytes, the board's layout, even seq) to device memory d_out (8-byte aligned).
 *                        It only enqueues a kernel, so it may be captured into a CUDA graph: a replay copies whatever
 *                        publish is the latest when it runs.
 *   lh_board_destroy     frees the board, stream-ordered after every publish already issued.  The caller guarantees
 *                        that no read of the board (lh_board_read or a kernel) is pending.  lh_destroy frees every
 *                        board left.
 * A destroyed or foreign handle gets LH_ERR_INVALID. */
typedef struct lh_board_header {
    uint64_t seq;                             /* seqlock word: odd while a publish writes, +2 per publish */
    uint64_t publishes;                       /* publishes so far (= seq / 2 when even) */
    uint32_t np;                              /* percentiles of the latest publish */
    uint32_t reserved[3];
    double percentiles[LH_MAX_PERCENTILES];   /* [0, np) of the latest publish, NaN beyond */
} lh_board_header;
typedef struct lh_board_hist_row {
    uint64_t count;
    double sum, avg;
    uint32_t present;                         /* a non-empty bucket (count != 0 unless the uint64 count wrapped) */
    uint32_t reserved;
    double pvals[LH_MAX_PERCENTILES];         /* NaN where pkeys is INT32_MIN, and beyond np */
    int32_t pkeys[LH_MAX_PERCENTILES];
} lh_board_hist_row;
typedef struct lh_board_counter_row {
    uint64_t rate;                            /* interval delta */
    uint64_t total;                           /* the caller's running total */
    uint32_t present;
    uint32_t reserved;
} lh_board_counter_row;
typedef struct lh_board {                     /* pass by value to kernels */
    uint64_t handle;                          /* opaque */
    void *d_board;                            /* device memory: header, k histogram rows, kc counter rows */
    uint32_t k, kc;
    uint64_t bytes;                           /* size of an image (lh_board_read) */
} lh_board;
#ifdef __cplusplus
#define LH_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define LH_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif
LH_STATIC_ASSERT(sizeof(lh_board_header) == 288 && offsetof(lh_board_header, percentiles) == 32,
                 "lh_board_header is 288 bytes: seq, publishes, np, reserved, percentiles");
LH_STATIC_ASSERT(sizeof(lh_board_hist_row) == 416 && offsetof(lh_board_hist_row, pvals) == 32 &&
                 offsetof(lh_board_hist_row, pkeys) == 288, "lh_board_hist_row is 416 bytes");
LH_STATIC_ASSERT(sizeof(lh_board_counter_row) == 24, "lh_board_counter_row is 24 bytes");
LH_STATIC_ASSERT(sizeof(lh_board) == 32, "lh_board is 32 bytes");
LH_API lh_status lh_board_create(lh_ctx *ctx, uint32_t k, uint32_t kc, lh_board *out);
LH_API lh_status lh_snapshot_publish(lh_ctx *ctx, const lh_board *b, const uint32_t *hist_ids,
                                     const uint32_t *counter_ids, const uint64_t *counter_totals);
LH_API lh_status lh_board_read(lh_ctx *ctx, const lh_board *b, void *d_out, void *stream);
LH_API lh_status lh_board_destroy(lh_ctx *ctx, const lh_board *b);

/* ---- raw device subscriptions: each collection's bucket counts in device memory ---------------------------------
 * SubscribeToRawMetrics (metrics.go:203-215, 508-525) for consumers on the GPU.  A raw board holds k histogram rows;
 * lh_snapshot_publish_raw writes the running bucket counts of the open snapshot's histograms into them, and kernels
 * (include/loghisto_b200_device.cuh: lh::raw_percentile / raw_rank / raw_bucket_count) or the capturable query calls
 * below answer exact percentile, rank and bucket queries from the latest publish with no host call.
 *
 * Layout (bytes, from d_rows): k lh_raw_row_header, then from LH_RAW_CELLS_OFFSET(k) k rows of uint64[65536]: cell
 * key + 32768 of row i holds the number of samples of that publish whose int16 bucket key is <= key (ascending int16
 * key order, the order K3 and lh_snapshot_reduce rank in), mod 2^64 as Go's uint64 running count.  Only keys
 * [key_lo, key_hi] of the header are written by a publish: a key below key_lo reads as 0 and a key above key_hi as
 * total.  A row whose running count passed 2^64 (counts summing to 2^64 or more: the cells are not monotone and total
 * may be 0) stores key_hi + LH_RAW_KEY_WRAPPED, so a stored key_hi above 32767 marks it; the device queries then apply
 * the percentile rule to every written key.  An empty row has key_lo > key_hi (and total 0).
 * Each row has its own seqlock: `seq` is odd while a publish writes the row and advances by 2 per publish, so
 * seq / 2 is the publish number (0 before the first) and every query answer is of one publish.
 *
 *   lh_raw_board_create      allocates a board of 1 <= k <= max_histograms rows and writes every header as an empty
 *                            row of publish 0 (total 0, key_lo 0, key_hi -1), so that queries before the first publish
 *                            answer as for an empty row and read no cell.  512 KiB per row.  Call it outside any stream
 *                            capture; it waits for the headers to be written.
 *   lh_snapshot_publish_raw  writes row i from histogram hist_ids[i] of the open snapshot (its frozen counts, or the
 *                            all-reduced ones after lh_snapshot_allreduce: publish after the all-reduce, before
 *                            lh_snapshot_end).  hist_ids[i] = LH_GRAPH_UNBOUND (or hist_ids NULL), or a histogram the
 *                            interval never touched: an empty row.  No reduction is needed.  LH_ERR_STATE outside a
 *                            snapshot, LH_ERR_RANGE for an id >= max_histograms other than LH_GRAPH_UNBOUND.  Enqueued on
 *                            the snapshot stream; it never waits and never allocates.
 *   lh_raw_percentiles       query i: (d_keys[i], d_vals[i]) = what lh_snapshot_reduce reports for row d_rows[i]'s
 *                            histogram with percentile d_ps[i], bit for bit (INT32_MIN / NaN where no bucket satisfies
 *                            the rule: p > 1 unless the row's running counts wrapped, NaN, an empty row; the smallest
 *                            non-empty key for p <= 0).
 *   lh_raw_ranks             query i: d_ranks[i] = samples of row d_rows[i] whose key is <= compress(d_values[i]) (the
 *                            bucket lh::record gives the value; NaN and +-Inf have key 0), d_totals[i] = its total.
 *   lh_raw_percentiles_grid / lh_raw_ranks_grid
 *                            the same for every row r < k and input j < m: answers at [r * m + j]; d_totals[r] is the
 *                            total of the publish query (r, 0) read.  LH_ERR_RANGE when k * m >= 2^32.
 *                            Every query call writes d_publish[i] = the publish number its answer comes from, enqueues ONE
 *                            kernel on `stream` (NULL = the ingest stream) and nothing else, so it may be captured into a
 *                            CUDA graph: a replay answers from the publish latest when it runs.  Different queries may
 *                            come from different publishes.  A row >= k answers as an empty row of publish 0.  Arrays are
 *                            device memory, naturally aligned (LH_ERR_INVALID otherwise, or NULL, with n > 0: nothing is
 *                            enqueued); n == 0 enqueues nothing.
 *   lh_raw_board_destroy     frees the board, stream-ordered after every publish already issued.  The caller guarantees
 *                            that no query of the board is pending.  lh_destroy frees every raw board left.
 * A destroyed or foreign handle gets LH_ERR_INVALID.
 *
 * Window boards: lh_raw_board_create_window(ctx, k, window, out) creates a board whose row i answers for the
 * histogram whose per-key counts are the sums, mod 2^64, of row i's last `window` publishes (fewer before the board
 * has seen `window`), i.e. what a board of lh_raw_board_create would answer had those intervals been merged into one
 * snapshot: the same layout, header, seqlock and LH_RAW_KEY_WRAPPED rule (applied to the window's own running counts,
 * so a window may wrap when none of its intervals does, and stops being wrapped when the interval that wrapped it
 * leaves), so every query call, the device functions and the bindings work on it unchanged.
 *   window == 1 is lh_raw_board_create; window == 0 gives LH_ERR_INVALID, window > LH_RAW_MAX_WINDOW LH_ERR_RANGE, a
 *   failed allocation LH_ERR_NOMEM with nothing left allocated; the other checks are lh_raw_board_create's.  Device
 *   memory: (window + 1) x 512 KiB per row beyond the board's 512 KiB (a dense sum row and one slot per publish of the
 *   window), plus window + 8 bytes of bookkeeping per row.
 *   lh_snapshot_publish_raw on a window board takes row i's entering interval as on any board (hist_ids[i]'s frozen or
 *   all-reduced counts; unbound or untouched: empty), drops the row's oldest one from the window and writes the row
 *   from the new window, all inside the row's seqlock, in one kernel (plus the same staging launches for k > 4096),
 *   without waiting or allocating.  Its traffic follows the key ranges of the intervals in the window (the fast window's
 *   keys unless one of them has a count outside it), not `window`.  A second publish to a window board in the same
 *   snapshot gives LH_ERR_STATE and enqueues nothing, since it would count one interval twice. */
typedef struct lh_raw_row_header {
    uint64_t seq;                             /* seqlock word: odd while a publish writes the row, +2 per publish */
    uint64_t publishes;                       /* publishes so far (= seq / 2 when even) */
    uint64_t total;                           /* samples of the row in the latest publish */
    int32_t key_lo, key_hi;                   /* the key range that publish wrote (key_lo > key_hi: empty row); key_hi
                                               * + LH_RAW_KEY_WRAPPED when the running counts wrapped */
} lh_raw_row_header;
#define LH_RAW_KEY_WRAPPED 65536
typedef struct lh_raw_board {                 /* pass by value to kernels */
    uint64_t handle;                          /* opaque */
    void *d_rows;                             /* device memory: k headers, then k rows of running counts */
    const double *d_decomp;                   /* the context's decompress table, indexed by (uint16)key */
    uint32_t k;
    uint32_t reserved;
    uint8_t prec[48];                         /* lh::Prec of the context (raw_rank's bucket function), opaque to C */
} lh_raw_board;
LH_STATIC_ASSERT(sizeof(lh_raw_row_header) == 32 && offsetof(lh_raw_row_header, key_lo) == 24,
                 "lh_raw_row_header is 32 bytes: seq, publishes, total, key_lo, key_hi");
LH_STATIC_ASSERT(sizeof(lh_raw_board) == 80 && offsetof(lh_raw_board, prec) == 32, "lh_raw_board is 80 bytes");
/* byte offset of row 0's cells from d_rows: the headers rounded up to 256 bytes */
#define LH_RAW_CELLS_OFFSET(k) ((((uint64_t)(k) * 32u) + 255u) & ~(uint64_t)255u)
#define LH_RAW_MAX_WINDOW 4096
LH_API lh_status lh_raw_board_create(lh_ctx *ctx, uint32_t k, lh_raw_board *out);
LH_API lh_status lh_raw_board_create_window(lh_ctx *ctx, uint32_t k, uint32_t window, lh_raw_board *out);
LH_API lh_status lh_snapshot_publish_raw(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *hist_ids);
LH_API lh_status lh_raw_percentiles(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_ps,
                                    uint32_t n, int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream);
LH_API lh_status lh_raw_ranks(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_values,
                              uint32_t n, uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream);
LH_API lh_status lh_raw_percentiles_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_ps, uint32_t m,
                                         int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream);
LH_API lh_status lh_raw_ranks_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_values, uint32_t m,
                                   uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream);
LH_API lh_status lh_raw_board_destroy(lh_ctx *ctx, const lh_raw_board *b);

/* ---- device gauges: RegisterGaugeFunc (metrics.go:299-310) for values that live in device memory -----------------
 * lh_gauges_read reads n scalars from device memory, one per lh_gauge_src, and returns them to the host as float64.  It
 * is stateless: the registry of names lives in the caller (MetricSystem::RegisterDeviceGauge).
 *
 *   Values    h_out[i] is Go's float64(x) of the value x at d_value: exact for F64, F32, F16, BF16 and I32;
 *             round-to-nearest-even for I64 and U64 (what amd64 Go does: CVTSQ2SD, and the halve-and-double
 *             sequence for uint64 >= 2^63).  A NaN stays a NaN; its payload is unspecified.
 *   Loads     each value is read with one naturally aligned strong load (ld.relaxed.gpu), so a value written by a
 *             single aligned store is never torn (see lh::set_gauge in include/loghisto_b200_device.cuh).
 *   Ordering  the read is enqueued on the context's snapshot stream only.  It never waits for ingest streams, record
 *             scopes, graph replays or any caller stream: it reads whatever is in memory when the kernel runs, as a Go
 *             gauge function reads the current state.
 *   Waiting   the call returns once the values are in h_out.  It does not hold the context's lock while it waits for
 *             the device, so ingest calls from other threads are not held up.
 *   Checks    everything is validated before anything is launched; on a failed check nothing is launched:
 *             h_srcs / h_out NULL with n > 0, an unknown dtype, a non-zero `reserved`, a NULL d_value or one not
 *             naturally aligned for its dtype, and a d_value that is not device or managed memory of the context's
 *             device (cudaPointerGetAttributes: host memory, pinned or not, and another GPU's memory are refused) all
 *             return LH_ERR_INVALID.  The last check is what keeps the kernel from ever faulting on a bad address.
 *   Sizes     n == 0 returns LH_OK with no launch.  Any n is accepted: tables larger than one launch's parameter block
 *             (1 024 entries) are split across launches on the same stream, with one wait at the end.
 * The call returns host values, so it cannot be captured into a CUDA graph.  It does not change lh_stats.samples,
 * lh_stats.counter_ops or the ingest sequence. */
#define LH_GAUGE_F64 0
#define LH_GAUGE_F32 1
#define LH_GAUGE_F16 2
#define LH_GAUGE_BF16 3
#define LH_GAUGE_I64 4
#define LH_GAUGE_I32 5
#define LH_GAUGE_U64 6
typedef struct lh_gauge_src {
    const void *d_value;                      /* device or managed memory of the context's device */
    uint32_t dtype;                           /* LH_GAUGE_* */
    uint32_t reserved;                        /* 0 */
} lh_gauge_src;
LH_STATIC_ASSERT(sizeof(lh_gauge_src) == 16 && offsetof(lh_gauge_src, dtype) == 8 &&
                 offsetof(lh_gauge_src, reserved) == 12, "lh_gauge_src is 16 bytes: d_value, dtype, reserved");
LH_API lh_status lh_gauges_read(lh_ctx *ctx, const lh_gauge_src *h_srcs, uint32_t n, double *h_out);

/* ---- distribution gauges: a device array's current values as one histogram, once per collection -----------------
 * lh_snapshot_ingest_arrays records every element x of n_srcs device arrays, one per lh_array_src, as a sample
 * float64(x) of its histogram_id, into the interval the open snapshot froze.  It is stateless: the registry of names
 * lives in the caller (MetricSystem::RegisterDeviceDistribution), which calls it once per collection.
 *
 *   Values    each element is converted as lh_gauges_read converts a gauge (Go's float64(x)) and counted as one
 *             Histogram(name, float64(x)) would count it.  The samples join every other sample of that id in the
 *             frozen interval, and every reader of the snapshot sees them.
 *   Loads     each element is read with one naturally aligned strong load (ld.relaxed.gpu) of its width, so an
 *             element written by a single aligned store is never torn.
 *   Ordering  the kernels are enqueued on the context's snapshot stream only, into the frozen rows.  They never wait for
 *             ingest streams, record scopes, graph replays or any caller stream: they read whatever is in memory when
 *             they run, as a Go gauge function reads the current state.  The call does not wait for them.
 *   Checks    everything is validated before the state check and before anything is launched; on a failed check
 *             nothing is launched: h_srcs NULL with n_srcs > 0, an unknown dtype, and, for an array with n > 0, a NULL
 *             or not naturally aligned d_values, a d_values that is not device or managed memory of the context's
 *             device, or a range [d_values, d_values + n * size) that does not lie inside one allocation
 *             (cuMemGetAddressRange) return LH_ERR_INVALID; a histogram_id >= max_histograms returns LH_ERR_RANGE.  The
 *             range check is what keeps the kernel from ever reading past an allocation.
 *   State     then LH_ERR_STATE unless a snapshot is open (lh_snapshot_begin) and nothing has read its rows yet:
 *             reduce (sync or async), export, copy_histogram, rows, row_levels, pack_rows, the all-reduces, publish,
 *             publish_raw and lh_snapshot_device all read them.  Call it right after lh_snapshot_begin.
 *   Sizes     n_srcs == 0, or every n == 0, returns LH_OK with no launch.  One launch takes up to 1 024 arrays and as
 *             many samples as its CTAs' uint32 tables allow; longer tables and arrays are split across launches.
 *   Counting  lh_stats.samples grows by the sum of n.  The call is not an ingest: it takes no ingest sequence number
 *             and no kernel timing.
 * A collection is never captured, so neither is this call. */
typedef struct lh_array_src {
    const void *d_values;                     /* n elements of dtype, in one allocation of the context's device */
    uint64_t n;
    uint32_t dtype;                           /* LH_GAUGE_* */
    uint32_t histogram_id;
} lh_array_src;
LH_STATIC_ASSERT(sizeof(lh_array_src) == 24 && offsetof(lh_array_src, n) == 8 && offsetof(lh_array_src, dtype) == 16 &&
                 offsetof(lh_array_src, histogram_id) == 20, "lh_array_src is 24 bytes: d_values, n, dtype, histogram_id");
LH_API lh_status lh_snapshot_ingest_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs);

/* ---- stream-ordered ingest of device arrays of any gauge dtype -------------------------------------------------
 * lh_ingest_arrays records every element x of n_srcs device arrays (lh_array_src above, dtype LH_GAUGE_*) as one
 * Histogram(histogram_id, float64(x)), without widening the arrays to float64 first: a float32 or int32 sample is read
 * as 4 bytes and a float16 or bfloat16 one as 2.  The conversion is lh_gauges_read's (Go's float64(x)): floats and int32
 * exactly, subnormals kept; int64 and uint64 round to nearest even, so an LH_GAUGE_I64 array of nanoseconds counts
 * exactly as LH_VALUES_I64NS does and an LH_GAUGE_F64 array as LH_VALUES_F64.
 *
 * In every other respect it is lh_ingest_batch: one write bracket and one ingest sequence number on `stream` (NULL =
 * the context's ingest stream), every sample in one interval, lh_stats.samples += the sum of n; items may repeat ids,
 * alias or overlap and come in any order; the call never waits for the device and allocates nothing.  The arrays are
 * read in stream order with streaming loads and must stay valid until the stream's work completes.
 *
 * Routing: an F64 item of at least 2^20 samples goes to the single-histogram kernel (as in lh_ingest_batch), an F32 or
 * I32 item of at least 2^20 to its 4-byte form, an F16 or BF16 item of at least 2^20 to its 16-bit form (a per-context
 * key table from each 16-bit magnitude to its bucket, built at lh_create); every other item, and every I64 / U64 one,
 * to the kernel of lh_snapshot_ingest_arrays with streaming loads.
 *
 * Every item is validated before anything is enqueued; on error nothing is launched, counted or sequenced:
 * LH_ERR_INVALID for h_srcs NULL with n_srcs > 0 or an unknown dtype, and, for an item with n > 0, d_values NULL or not
 * naturally aligned for its dtype; LH_ERR_RANGE for an item with n > 0 and histogram_id >= max_histograms.  The memory
 * kind and the allocation range are not checked (the arrays are read in stream order, as lh_ingest_batch's are).
 *
 * lh_graph_recorder_ingest_arrays is lh_ingest_arrays into a graph recorder's rows (as lh_graph_recorder_ingest is
 * lh_ingest_batch): kernels only, capturable, ids local (histogram_id >= the recorder's k returns LH_ERR_RANGE), no
 * bracket, sequence number or sample tally. */
LH_API lh_status lh_ingest_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs, void *stream);
LH_API lh_status lh_graph_recorder_ingest_arrays(lh_ctx *ctx, const lh_graph_recorder *g, const lh_array_src *h_srcs,
                                                 uint32_t n_srcs, void *stream);

/* ---- GPU timers: StartTimer / Stop (metrics.go:232-246) from host code, timed on the device ------------------
 * Host StartTimer / Stop around CUDA work time the enqueue.  These calls put the two ends of the span on the GPU
 * instead: each end is a one-thread kernel on `stream` that reads %globaltimer (the clock of lh::start_timer), and
 * the duration is recorded on the device; it never crosses to the host.  A span includes the launch latency of its
 * two marks.  `stream` NULL = the context's ingest stream, as everywhere.
 *
 *   lh_gpu_timer_start    takes a free slot of the context's pool of 64-bit start marks (allocated on first use;
 *                         65536 slots, or lh_tune(ctx, "gpu_timer_slots", n) before the first start), enqueues the
 *                         mark on `stream` and records the slot's start event.  Never blocks.  LH_ERR_RANGE when
 *                         every slot is held or still in use by kernels that have not completed.
 *   lh_gpu_timer_stop     an ingest call of one sample: float64(now - start) into histogram `histogram_id` of the
 *                         active interval, inside one write bracket (one sequence number, one lh_stats.samples), so a
 *                         stop issued after lh_snapshot_begin lands in the next interval.  If d_duration_ns is not
 *                         NULL (device memory) the kernel also writes the duration there.  When `stream` is not the
 *                         start's stream, `stream` first waits for the start's mark, so the stop never reads an
 *                         unwritten slot; ordering after the WORK on the start's stream stays the caller's job.  A
 *                         token may be stopped any number of times (one sample each, from the same start).
 *                         LH_ERR_RANGE for histogram_id >= max_histograms.
 *   lh_gpu_timer_release  gives the slot back.  It is handed out again only after every kernel that read or wrote it
 *                         has completed (events on each stream that touched it), so releasing before the GPU has run
 *                         a stop never changes that stop's duration.
 *
 * A handle carries its slot, a generation and its context: a released, stale or foreign handle gets LH_ERR_INVALID
 * and touches no slot.  Start and stop on a stream in CUDA-graph capture return LH_ERR_STATE and enqueue nothing
 * (graph replay is not supported).  lh_destroy frees the pool whatever tokens are outstanding. */
typedef struct lh_gpu_timer { uint64_t handle; } lh_gpu_timer;   /* opaque */
LH_API lh_status lh_gpu_timer_start(lh_ctx *ctx, void *stream, lh_gpu_timer *out);
LH_API lh_status lh_gpu_timer_stop(lh_ctx *ctx, const lh_gpu_timer *t, uint32_t histogram_id, void *stream,
                                   int64_t *d_duration_ns);
LH_API lh_status lh_gpu_timer_release(lh_ctx *ctx, const lh_gpu_timer *t);

/* ---- snapshot = collectRawMetrics' cache swap (metrics.go:425-428, 460-463)
 *
 * lh_snapshot_begin   freezes the active bucket/counter arrays and makes the
 *                     spare (zeroed) pair active; ingest continues unblocked.
 * lh_snapshot_device  exposes the frozen device arrays so a multi-GPU caller
 *                     can all-reduce them in place (sum of uint64) before
 *                     reducing; work must be ordered on the returned stream.
 * lh_snapshot_reduce  processHistograms for every histogram (count, sum, avg,
 *                     percentiles), results copied to caller arrays.
 * lh_snapshot_export  sparse (key,count) lists + counter deltas, enough to
 *                     rebuild RawMetricSet.Histograms / Rates exactly.
 * lh_snapshot_end     zeroes the frozen arrays and returns them to the pool.
 */
typedef struct lh_device_view {
    uint64_t *d_buckets;   /* [max_histograms][65536] */
    uint64_t *d_counters;  /* [max_counters] interval deltas */
    uint64_t n_bucket_words;
    uint64_t n_counter_words;
    void *stream;          /* cudaStream_t the snapshot work is ordered on */
    uint32_t *d_flags;     /* [max_histograms] 0 = untouched this interval, 1 = counts inside the fast window only,
                            * 3 = also outside it.  A caller that reduces d_buckets in place across GPUs must reduce
                            * these with MAX (= bitwise OR) too: the reduction / export kernels scan only what the
                            * flags cover */
    uint64_t n_flag_words;
} lh_device_view;

LH_API lh_status lh_snapshot_begin(lh_ctx *ctx);
LH_API lh_status lh_snapshot_device(lh_ctx *ctx, lh_device_view *out);

/* Output arrays are caller-allocated host memory:
 *   counts[H]           uint64 totals, mod 2^64 as Go's (0 when the histogram is absent this interval, and also when
 *                       counts merged into it sum to a multiple of 2^64: presence is a non-empty bucket, which the
 *                       export's offsets show)
 *   sums[H], avgs[H]    as the reference's float64 map values (avg = sum / float64(count): NaN when absent, +-Inf or
 *                       NaN for a wrapped count of 0)
 *   pkeys[H*np]         chosen bucket key per percentile, INT32_MIN where the
 *                       reference's percentile() returns its error (no bucket satisfies the rule: p>1 unless the
 *                       running count wrapped, NaN, absent)
 *   pvals[H*np]         decompress(key); NaN where pkeys is INT32_MIN
 * Any output pointer may be NULL to skip it. */
LH_API lh_status lh_snapshot_reduce(lh_ctx *ctx, const double *percentiles, uint32_t np,
                             uint64_t *counts, double *sums, double *avgs, int32_t *pkeys,
                             double *pvals);

/* Asynchronous form for pipelined callers (the reaper overlaps the next interval's ingest with this
 * interval's reduction): enqueue the reduction of the open snapshot and get a ticket.  The frozen
 * arrays may be released with lh_snapshot_end right away; lh_snapshot_result waits for the ticket and
 * copies its results out.  Two tickets may be in flight; a ticket expires when the second-next is issued. */
LH_API lh_status lh_snapshot_reduce_async(lh_ctx *ctx, const double *percentiles, uint32_t np, uint64_t *ticket);
LH_API lh_status lh_snapshot_result(lh_ctx *ctx, uint64_t ticket, uint64_t *counts, double *sums, double *avgs,
                                    int32_t *pkeys, double *pvals);

typedef struct lh_sparse {
    const uint32_t *offsets;   /* [H+1] prefix offsets into keys/counts */
    const int16_t *keys;       /* ascending per histogram */
    const uint64_t *counts;
    const uint64_t *counter_deltas; /* [max_counters] */
    uint64_t total_entries;
} lh_sparse;
/* Pointers stay valid until the next lh_snapshot_export / lh_destroy. */
LH_API lh_status lh_snapshot_export(lh_ctx *ctx, lh_sparse *out);
/* Dense copy of one frozen histogram into host memory (uint64[65536]). */
LH_API lh_status lh_snapshot_copy_histogram(lh_ctx *ctx, uint32_t histogram_id, uint64_t *h_out65536);
LH_API lh_status lh_snapshot_end(lh_ctx *ctx);

/* ---- reducing sparse histograms the caller holds ----------------------------
 * processHistograms + percentile (metrics.go:336-418) over caller-supplied sparse histograms, independent of the
 * context's bucket arrays and snapshot state.  Histogram i is entries [offsets[i], offsets[i+1]) of keys/counts
 * (the lh_sparse layout, so an export can be passed back verbatim); keys may come in any order and may repeat
 * (repeats are summed, wrapping uint64, as a merge would).  Outputs as lh_snapshot_reduce, n_histograms long.
 *
 * The answer for histogram i is processHistograms' for the Go map map[int16]*uint64 its entries form, including
 * keys whose merged count is 0: with a total above 0, p <= 0 returns the smallest key present; a present key whose
 * decompress is +-Inf (precision <= 46) with a merged count of 0 makes the sum and avg NaN (Inf * 0).
 * n_histograms is not bounded by max_histograms.  Inputs are host memory (pageable or pinned); the call is
 * synchronous.  LH_ERR_INVALID, before anything is launched, when offsets decrease, np > LH_MAX_PERCENTILES, or an
 * input is NULL while there are entries; n_histograms == 0 is a no-op.  Thread-safe beside ingest, snapshots,
 * the all-reduce and other calls of this function; the context's bucket arrays, snapshot results and stats
 * counters of samples / snapshots are left as they were. */
LH_API lh_status lh_reduce_sparse_host(lh_ctx *ctx, uint32_t n_histograms, const uint32_t *h_offsets,
                                       const int16_t *h_keys, const uint64_t *h_counts,
                                       const double *percentiles, uint32_t np,
                                       uint64_t *counts, double *sums, double *avgs, int32_t *pkeys, double *pvals);

/* ---- multi-GPU: sharded sample stream, bucket arrays summed at snapshot time (SURVEY.md section 8e) -------------
 * One context per GPU (one process per GPU, or one thread per GPU in one process).  Each rank ingests its shard
 * into its own arrays; between lh_snapshot_begin and the reduction, lh_snapshot_allreduce sums the live window of
 * every rank's frozen arrays into this rank's view of the snapshot with ONE small kernel that reads the peers'
 * memory directly over NVLink (peer mappings: CUDA IPC between processes, peer access inside one process) -- no
 * library collective, nothing to link.  uint64 sums are associative, so every rank ends with exactly the bucket
 * counts a single GPU would have produced (metrics.go:273-295 over the whole stream).
 *
 *   lh_comm_export   opaque handle describing this context's arrays; the host exchanges the handles of all ranks
 *                    by any means it has (a file, a pipe, MPI, torch.distributed, Go channels in one process)
 *   lh_comm_import   maps every peer; handles[rank] must be this context's own.  Collective: every rank calls it
 *                    before any rank calls lh_snapshot_allreduce
 *   lh_snapshot_allreduce  collective, between lh_snapshot_begin and lh_snapshot_reduce/_export: ranks must take
 *                    their snapshots in lock-step (same number, same order).  Enqueued on the snapshot stream; the
 *                    kernel waits on the device for the peers' frozen arrays (no host synchronisation) and returns
 *                    LH_OK immediately.  A peer that never arrives makes the kernel give up after 10 s (status 1);
 *                    ranks that froze different halves of their double buffers, because one took a snapshot
 *                    without the collective, are found at once (status 2, on every rank).  Either way the snapshot's
 *                    reduction, export and counter deltas are then this rank's own frozen counts only, and nothing
 *                    was written into a peer's arrays by this rank.  lh_comm_info.status and last_bytes_from_peers
 *                    describe the most recent all-reduce (0 bytes when it failed): a failure does not outlive it,
 *                    so the all-reduce after the ranks are back in lock-step sums again.  Limit: a timeout can be
 *                    one-sided -- a peer that did arrive may still read this rank's frozen arrays, or (two-shot
 *                    form) push its sums into this rank's reduced arrays, after this rank gave up; only status 2 is
 *                    known to be seen by every rank alike
 *   lh_comm_allreduce_ms   device time of all-reduce `seq` (CUDA events around the kernel on the snapshot stream)
 */
typedef struct lh_peer_handle { uint8_t bytes[LH_PEER_HANDLE_BYTES]; } lh_peer_handle;
typedef struct lh_comm_stats {
    uint32_t rank, world;
    uint32_t status;                 /* most recent all-reduce: 0 ok, 1 a peer did not arrive in time, 2 peers froze
                                        different buffers (1 and 2: the snapshot holds this rank's counts only) */
    uint32_t reserved;
    uint64_t allreduces;
    uint64_t last_bytes_from_peers;  /* bytes read over NVLink by the most recent all-reduce */
} lh_comm_stats;
LH_API lh_status lh_comm_export(lh_ctx *ctx, lh_peer_handle *out);
LH_API lh_status lh_comm_import(lh_ctx *ctx, uint32_t rank, uint32_t world, const lh_peer_handle *handles);
LH_API lh_status lh_snapshot_allreduce(lh_ctx *ctx, uint32_t include_counters, uint64_t *seq);
LH_API lh_status lh_comm_allreduce_ms(lh_ctx *ctx, uint64_t seq, float *ms);
LH_API lh_status lh_comm_info(lh_ctx *ctx, lh_comm_stats *out);

/* ---- multi-GPU by rows: the all-reduce over job-wide rows whose ids differ per rank ---------------------------------
 * lh_snapshot_allreduce sums row h of every rank into row h.  When each rank keeps a name under its own id (MetricSystem
 * interns and recycles per rank), the ranks first agree on job-wide rows g and then sum through maps:
 *
 *   lh_snapshot_rows  between lh_snapshot_begin and any all-reduce: hist_touched[h] = 1 when histogram row h of the
 *                     frozen interval holds data (flag != 0), counter_deltas[c] = the frozen counter delta of c, and
 *                     *frozen = the half of the double buffer this snapshot froze (0 or 1), which the ranks exchange
 *                     for lh_snapshot_allreduce_rows (any pointer may be NULL).  One D2H on the snapshot stream, behind
 *                     what lh_snapshot_begin ordered there.  LH_ERR_STATE without a snapshot or after an all-reduce.
 *   lh_snapshot_allreduce_rows  collective, as lh_snapshot_allreduce, over job-wide rows: rank r contributes its frozen
 *                     row hist_map[r * n_rows + g] to row g (nothing for LH_ROW_ABSENT), and counter_map[r *
 *                     n_counter_rows + g] to counter g.  Afterwards the snapshot's reduce, export, publish and
 *                     lh_snapshot_copy_histogram see job-wide row g at index g, and nothing at or above n_rows
 *                     (n_counter_rows).  seq and frozen[world] (the buffer each rank froze: 0 or 1) come from the
 *                     host's own exchange, so every rank uses one agreed sequence number and reads each peer's own
 *                     frozen half; seq must exceed this context's last all-reduce.  The form (one-shot / two-shot) is
 *                     chosen from n_rows * (2*win - 1) * 8 bytes.  On failure (lh_comm_info.status != 0) the
 *                     snapshot holds this rank's own counts through hist_map[rank] / counter_map[rank].  Errors
 *                     before anything is launched: LH_ERR_STATE without a snapshot or lh_comm_import, LH_ERR_INVALID
 *                     for n_rows > max_histograms, n_counter_rows > max_counters, a NULL map with rows, a NULL frozen,
 *                     a frozen[r] > 1, frozen[rank] other than this snapshot's buffer, or seq not above the last,
 *                     LH_ERR_RANGE for a map entry neither LH_ROW_ABSENT nor below max_histograms (max_counters).
 */
#define LH_ROW_ABSENT 0xFFFFFFFFu
LH_API lh_status lh_snapshot_rows(lh_ctx *ctx, uint8_t *hist_touched, uint64_t *counter_deltas, uint32_t *frozen);
LH_API lh_status lh_snapshot_allreduce_rows(lh_ctx *ctx, uint64_t seq, const uint32_t *frozen, uint32_t n_rows,
                                            const uint32_t *hist_map, uint32_t n_counter_rows,
                                            const uint32_t *counter_map, uint64_t *seq_out);

/* ---- multi-GPU by rows through the caller's all-reduce ---------------------------------------------------------------
 * The peer all-reduce needs CUDA IPC mappings, which exist only between processes of one host.  Ranks on different
 * hosts agree on job-wide rows as above and then sum a payload through a transport the caller owns (gloo, NCCL, MPI):
 *
 *   lh_snapshot_row_levels  between lh_snapshot_begin and any all-reduce: levels[h] (uint8[max_histograms]) = the level
 *                     of frozen row h: 0 no data, 1 every count inside the fast window, 3 some count beyond it.
 *   lh_snapshot_pack_rows  between lh_snapshot_begin and any all-reduce, once per snapshot: gathers job-wide row g from
 *                     this rank's frozen row hist_rows[g] (zeros for LH_ROW_ABSENT) at the agreed levels[g], then
 *                     counter g from frozen counter counter_rows[g], into a payload of *n_words uint64: rows g = 0 ..
 *                     n_rows-1 in order (level 0: nothing; 1: the 2*win-1 cells [0, win) then [65536-(win-1), 65536);
 *                     3: all 65536 cells), then the n_counter_rows counters.  Every rank that passes the same n_rows,
 *                     levels and n_counter_rows gets the same layout.  *d_send holds the payload and *d_recv is as
 *                     large; both are owned by the context, grow on demand and stay valid until the next pack or
 *                     lh_destroy.  The pack is enqueued on the snapshot stream, returned in *stream: the caller's
 *                     all-reduce (d_recv = the element-wise wrapping uint64 sum of every rank's d_send) goes on it, or
 *                     completes before lh_snapshot_unpack_rows.  Needs no lh_comm_import.
 *   lh_snapshot_unpack_rows  after a pack in the same snapshot: summed = 1 writes d_recv (the job-wide sums), 0 writes
 *                     d_send (this rank's own counts, e.g. after a failed transport) into the reduced arrays: row g
 *                     at index g with flag levels[g], counters 0 .. n_counter_rows-1, nothing above.  Afterwards the
 *                     snapshot's reduce, export, publish and lh_snapshot_copy_histogram read them, as after
 *                     lh_snapshot_allreduce_rows.  A snapshot that ends after a pack without an unpack read its own
 *                     frozen arrays throughout.
 * Errors, before anything is launched: LH_ERR_STATE without a snapshot, after an all-reduce or unpack, for a second
 * pack, or for an unpack without a pack; LH_ERR_INVALID for n_rows > max_histograms, n_counter_rows > max_counters, a
 * NULL map or NULL levels with rows, a level other than 0 / 1 / 3, or a NULL output pointer; LH_ERR_RANGE for a map
 * entry neither LH_ROW_ABSENT nor below max_histograms (max_counters).
 */
LH_API lh_status lh_snapshot_row_levels(lh_ctx *ctx, uint8_t *levels);
LH_API lh_status lh_snapshot_pack_rows(lh_ctx *ctx, uint32_t n_rows, const uint32_t *hist_rows, const uint8_t *levels,
                                       uint32_t n_counter_rows, const uint32_t *counter_rows, uint64_t **d_send,
                                       uint64_t **d_recv, uint64_t *n_words, void **stream);
LH_API lh_status lh_snapshot_unpack_rows(lh_ctx *ctx, uint32_t summed);

/* ---- scalar helpers, evaluated ON THE DEVICE (parity probes for tests) --- */
/* out[i] = compress(values[i]) exactly as the ingest kernels compute it
 * (mode 0: production fast path + exact fallback; mode 1: exact path only) */
LH_API lh_status lh_compress_f64(lh_ctx *ctx, const double *d_values, size_t n, int16_t *d_out, int mode,
                          void *stream);
/* copy of the device decompress table: out[(uint16)key] = decompress(key) */
LH_API lh_status lh_decompress_table(lh_ctx *ctx, double *h_out65536);
/* max |fast-path estimate - exact 100*ln(1+|v|)| over the inputs, in bucket
 * units, restricted to samples the fast path accepts; margin evidence for EPS */
LH_API lh_status lh_fastpath_margin(lh_ctx *ctx, const double *d_values, size_t n, double *h_max_err,
                             uint64_t *h_n_slow, void *stream);
/* the same per estimator (1: fast_candidate, 2: the packed-FP32 form of the single-histogram kernels), for the
 * inputs of the last lh_fastpath_margin call */
LH_API lh_status lh_fastpath_margin_detail(lh_ctx *ctx, double *h_err_estimator1, double *h_err_estimator2);
/* Exhaustive check of the FP32 estimate behind every fast path, on the device, at every precision of
 * [p_lo, p_hi] (1 <= p_lo <= p_hi <= LH_MAX_PRECISION; independent of the context's own precision).  Every cell of
 * x = 1+|v| in [1, 2^64) (biased exponent, top 23 mantissa bits: the estimate depends on nothing else) is fed with
 * both signs through each shipped form of the estimate and compared with FP64 P*ln at both ends of the cell.
 * h_out[(p - p_lo) * 4 + form], form 0: fast_candidate (keyed vec / scalar kernels, fix-ups, device API),
 * 1: the packed form of the single-histogram kernels with the sign folded into the slot, 2: the same with negatives
 * flagged (also the few-histogram keyed kernel), 3: the slot-index form of the write-combining keyed kernel.
 * A correct form has wrong == out_of_range == unflagged_outside == over_flagged == input_mismatch == 0. */
typedef struct lh_certify_form {
    uint64_t samples;            /* samples inside the window (x < 2^63; v >= 0 for forms 2 and 3) */
    uint64_t flagged;            /* ... of them sent to the exact path */
    uint64_t wrong;              /* unflagged, and some double of the cell is not in the returned bucket, or lies
                                  * within 2^-30 bucket units of its boundary */
    uint64_t out_of_range;       /* unflagged, with a slot outside the window's sub-histogram */
    uint64_t unflagged_outside;  /* unflagged although outside the window (x >= 2^63; v < 0 for forms 2 and 3) */
    uint64_t over_flagged;       /* flagged, though farther from every bucket boundary than eps plus its error */
    uint64_t input_mismatch;     /* inputs v for which 1+|v| did not land on the intended cell */
    double max_err;              /* max |estimate - P*ln x| over samples with x < 2^63, bucket units */
    double min_margin;           /* smallest distance of an unflagged cell from a bucket boundary, bucket units */
} lh_certify_form;
LH_API lh_status lh_fastpath_certify(lh_ctx *ctx, uint32_t p_lo, uint32_t p_hi, lh_certify_form *h_out);

/* ---- synthetic streams (bench / tests; SURVEY.md section 8d) ------------- */
/* kind: 0=U log-uniform, 1=L latency-like, 2=S signed/edge mix, 3=C constant, 4=Z heavy hitter,
 *       6=timer durations (int64 ns bit patterns), 7=counter amounts 1..16, 8=N (stream U with a random sign) */
LH_API lh_status lh_gen_stream_f64(lh_ctx *ctx, int kind, uint64_t seed, uint64_t start, size_t n,
                            double *d_out, void *stream);
LH_API lh_status lh_gen_ids_u16(lh_ctx *ctx, int kind, uint64_t seed, uint64_t start, size_t n,
                         uint32_t n_ids, uint16_t *d_out, void *stream);

/* ---- misc ---------------------------------------------------------------- */
typedef struct lh_stats {
    uint64_t samples;        /* samples accepted by host-issued ingest calls (host-side tally; device records
                              * through lh_recorder are not counted) */
    uint64_t counter_ops;    /* likewise */
    uint64_t dropped;        /* samples with id out of range (device-side tally, device records included) */
    uint64_t kernel_launches;
    uint64_t h2d_bytes;
    uint64_t d2h_bytes;
    uint64_t snapshots;
} lh_stats;
LH_API lh_status lh_get_stats(lh_ctx *ctx, lh_stats *out);
/* wait for all work issued through this context */
LH_API lh_status lh_sync(lh_ctx *ctx);
/* cudaStream_t of the context's own ingest stream, as void* */
LH_API void *lh_ingest_stream(lh_ctx *ctx);
/* device allocation helpers so non-CUDA hosts (ctypes, cgo) can own device buffers */
LH_API lh_status lh_device_alloc(lh_ctx *ctx, size_t bytes, void **d_out);
LH_API lh_status lh_device_free(lh_ctx *ctx, void *d_ptr);
LH_API lh_status lh_host_alloc_pinned(lh_ctx *ctx, size_t bytes, void **h_out);
LH_API lh_status lh_host_free_pinned(lh_ctx *ctx, void *h_ptr);
/* lh_memcpy_h2d returns once the bytes are in device memory, so that work on any stream may read them */
LH_API lh_status lh_memcpy_h2d(lh_ctx *ctx, void *d_dst, const void *h_src, size_t bytes);
LH_API lh_status lh_memcpy_d2h(lh_ctx *ctx, void *h_dst, const void *d_src, size_t bytes);
/* kernel-variant selection for profiling: key "k1" -> variant number,
 * "k1_grid_mult", "k1_reserve_sms" (SMs the ingest kernels leave free so that a concurrent
 * snapshot / all-reduce kernel can run beside them), "keyed_blocks_per_sm", "keyed_mode" (0 auto, 1 L2-atomic
 * kernel, 2 owner-partitioned write-combining kernel whatever the batch size), and that kernel's knobs: "kp_chunk"
 * (samples per chunk, default 256 M), "wc_spt" (tile shape code: 6 = 896 threads x 4 samples (default), 4 = 1024 x 4,
 * 3 = 768 x 4, 8 = 512 x 8), "wc_flush" (samples a CTA bins between two flushes of its owner buffers, default 24576),
 * "wc_pf" (L2 prefetch distance of its input in tiles, default 1, 0 = off), "gpu_timer_slots" (size of the GPU
 * timer pool, 1 ... 2^20, default 65536; LH_ERR_STATE once the pool exists) */
LH_API lh_status lh_tune(lh_ctx *ctx, const char *key, int64_t value);
LH_API int32_t lh_k1_variant_count(void);
LH_API int32_t lh_k1_variant_current(lh_ctx *ctx);
LH_API const char *lh_k1_variant_name(lh_ctx *ctx, int32_t i);
/* name of the kernel the most recent keyed ingest dispatched to */
LH_API const char *lh_keyed_kernel_name(lh_ctx *ctx);
/* Ingest timing: two CUDA events on the launch stream bracket the kernels of one sequence number, which is
 *   - one device-pointer ingest call, lh_ingest_keyed_pair_u16 and lh_ingest_batch included whichever kernels they take;
 *   - one staging chunk of a host-fed call (lh_*_host); its H2D copy is outside the bracket;
 *   - one lh_staging_commit_* call;
 *   - one lh_gpu_timer_stop.
 * A call with no samples may take none.
 * lh_last_kernel_ms = device time of the latest sequence number in ms;
 * lh_ingest_seq = sequence numbers issued so far (the latest one, 1-based);
 * lh_kernel_ms = device time of sequence number `seq` (its events stay available for the next 15) */
LH_API lh_status lh_last_kernel_ms(lh_ctx *ctx, float *ms);
LH_API uint64_t lh_ingest_seq(lh_ctx *ctx);
LH_API lh_status lh_kernel_ms(lh_ctx *ctx, uint64_t seq, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* LOGHISTO_B200_H_ */
