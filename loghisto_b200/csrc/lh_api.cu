// lh_api.cu -- C ABI (include/loghisto_b200.h) over the sm_90a kernels.
//
// Host-side bookkeeping only: double-buffered bucket/counter arrays, stream
// and event ordering between ingest and snapshot, the pinned staging ring,
// kernel-variant dispatch.  No bucket arithmetic happens on the CPU.
#include "../../include/loghisto_b200.h"
#include "lh_kernels.cuh"

#include <cuda.h>   // driver types of cuMemGetAddressRange only: the library does not link libcuda

#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>
#include <unistd.h>

using namespace lh;

namespace {

// Owners of one CUDA handle each (move-only): the handle is released when its owner is reset or destroyed.  out()
// releases what is held and hands the slot to an allocating call.
template <typename H, cudaError_t (*Release)(H)>
class Owned {
    H h_ = nullptr;
public:
    Owned() = default;
    Owned(Owned &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Owned &operator=(Owned &&o) noexcept { if (this != &o) { reset(); h_ = o.h_; o.h_ = nullptr; } return *this; }
    ~Owned() { reset(); }
    H get() const { return h_; }
    H *out() { reset(); return &h_; }
    void reset() { if (h_) Release(h_); h_ = nullptr; }
};
template <typename T> cudaError_t free_device(T *p) { return cudaFree(p); }
template <typename T> cudaError_t free_pinned(T *p) { return cudaFreeHost(p); }
template <typename T> using DevPtr = Owned<T *, free_device<T>>;      // cudaMalloc
template <typename T> using PinnedPtr = Owned<T *, free_pinned<T>>;   // cudaMallocHost, cudaHostAlloc
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;

// stream-ordered device memory (cudaMallocAsync), freed on the stream it was given, or on the one passed to reset
class AsyncPtr {
    char *p_ = nullptr;
    cudaStream_t s_ = nullptr;
public:
    explicit AsyncPtr(cudaStream_t s = nullptr) : s_(s) {}
    AsyncPtr(AsyncPtr &&o) noexcept : p_(o.p_), s_(o.s_) { o.p_ = nullptr; }
    AsyncPtr &operator=(AsyncPtr &&o) noexcept { if (this != &o) { reset(); p_ = o.p_; s_ = o.s_; o.p_ = nullptr; } return *this; }
    ~AsyncPtr() { reset(); }
    char *get() const { return p_; }
    char **out() { reset(); return &p_; }
    cudaError_t reset() { return reset(s_); }
    cudaError_t reset(cudaStream_t s) { const cudaError_t e = p_ ? cudaFreeAsync(p_, s) : cudaSuccess; p_ = nullptr; return e; }
};

struct WriterEvent { cudaStream_t stream; Event ev; };

// an open record scope (lh_record_begin .. lh_record_end): device code is writing buffer `buf` from `stream`
struct Scope { uint64_t ticket; int buf; cudaStream_t stream; std::thread::id thread; };
static_assert(sizeof(Prec) == sizeof(((lh_recorder *)0)->prec) && offsetof(lh_recorder, prec) % alignof(Prec) == 0,
              "lh_recorder.prec must hold an lh::Prec");

// one slot of the GPU timer pool (lh_gpu_timer_*)
enum TimerState : uint8_t { TIMER_FRESH = 0 /* never handed out */, TIMER_HELD = 1, TIMER_RELEASED = 2 };
struct TimerSlot {
    uint32_t gen = 0;                  // bumped at every release: handles of earlier tokens stop matching
    uint8_t state = TIMER_FRESH;
    cudaStream_t start_stream = nullptr;
    Event started;                     // after the mark (created on the slot's first use, kept)
    std::vector<WriterEvent> stops;    // after the latest stop on each stream that stopped the token
};

// a graph recorder (lh_graph_recorder_*): rows it owns, drained into the frozen interval at every lh_snapshot_begin
struct GraphRec {
    uint64_t handle;
    AsyncPtr mem;                    // the one allocation behind rec and d_marks
    lh_recorder rec;                 // what the caller was given (rows, flags, counters in one allocation)
    unsigned long long *d_marks;     // [k] start marks of lh_graph_recorder_timer_* (kTimerNeverStarted until a start)
    std::vector<uint32_t> hid, cid;  // target id of each local row / counter (LH_GRAPH_UNBOUND = drop and count)
};

struct Buffer {
    DevPtr<unsigned long long> d_buckets;      // [H][65536]
    DevPtr<unsigned long long> d_counters;     // [C]
    DevPtr<uint32_t> d_flags;                  // [H] 0 untouched / 1 window only / 3 also outside the window
    DevPtr<unsigned int> d_hot;                // [hot_replicas][H][2*win] uint32 window of the keyed path
    unsigned long long hot_pending = 0;        // samples added to d_hot since it was last drained
    Event cleared;                             // zeroing finished
    std::vector<WriterEvent> writers;          // last ingest per stream
};

enum SlotState { SLOT_FREE = 0, SLOT_ACQUIRED = 1 /* handed to the caller (lh_staging_acquire) */, SLOT_INFLIGHT = 2,
                 SLOT_WAITED = 3 /* a thread is waiting for its kernel, mutex released */,
                 SLOT_FILLING = 4 /* lh_*_host is copying pageable memory into it, mutex released */ };
struct Slot {
    PinnedPtr<void> h; DevPtr<void> d;
    Event done;                      // kernel that consumed the slot has finished
    Event copied;                    // H2D copy into the slot has landed
    int state = SLOT_FREE;
    uint64_t seq = 0;
};

struct K1Variant {
    const char *name;
    void (*launch)(int grid, size_t smem, cudaStream_t s, const double *v32, size_t nvec,
                   const double *head, int nhead, const double *tail, int ntail, unsigned long long *counts,
                   uint32_t *flag, const Prec &pc);
    const void *func;
    int threads;
    size_t smem_fixed;   // bytes besides the sub-histogram (ring + barriers)
    int blocks_per_sm;   // filled at create
    size_t smem;         // filled at create: smem_fixed + sub-histogram for the context's precision
};

template <int THREADS, int UNROLL, int MINB>
void launch_ldg(int grid, size_t smem, cudaStream_t s, const double *v32, size_t nvec, const double *head, int nhead,
                const double *tail, int ntail, unsigned long long *counts, uint32_t *flag, const Prec &pc) {
    k_ingest_single_ldg<THREADS, UNROLL, MINB><<<grid, THREADS, smem, s>>>(v32, nvec, head, nhead, tail, ntail, counts, flag, pc);
}
template <int CW, int STAGES, int STAGE_BYTES, int MINB, bool FOLD>
void launch_bulk(int grid, size_t smem, cudaStream_t s, const double *v32, size_t nvec, const double *head, int nhead,
                 const double *tail, int ntail, unsigned long long *counts, uint32_t *flag, const Prec &pc) {
    k_ingest_single_bulk<CW, STAGES, STAGE_BYTES, MINB, FOLD><<<grid, (CW + 1) * 32, smem, s>>>(v32, nvec, head, nhead, tail, ntail, counts, flag, pc);
}
void launch_probe(int grid, size_t, cudaStream_t s, const double *v32, size_t nvec, const double *head, int nhead,
                  const double *tail, int ntail, unsigned long long *counts, uint32_t *flag, const Prec &pc) {
    k_stream_probe<512, 4><<<grid, 512, 0, s>>>(v32, nvec, head, nhead, tail, ntail, counts, flag, pc);
}

#define LDG_VARIANT(T, U, M) \
    { "ldg_t" #T "_u" #U "_b" #M, launch_ldg<T, U, M>, (const void *)k_ingest_single_ldg<T, U, M>, T, 0, 0, 0 }
#define BULK_VARIANT(W, S, B, M, F) \
    { "bulk2_w" #W "_s" #S "_" #B "_b" #M "_sign" #F, launch_bulk<W, S, B, M, F != 0>, (const void *)k_ingest_single_bulk<W, S, B, M, F != 0>, (W + 1) * 32, \
      (size_t)S * B + (size_t)S * 16, 0, 0 }

// The shipped kernel plus what the parity tests compare it with (the winners of a sweep of 27 shapes and the
// independent first version).
K1Variant g_k1_variants[] = {
    BULK_VARIANT(16, 4, 32768, 1, 1),   // 0: default (sign folded into the slot)
    BULK_VARIANT(16, 3, 65536, 1, 1),   // 1
    BULK_VARIANT(8, 4, 16384, 2, 1),    // 2
    LDG_VARIANT(512, 2, 2),             // 3: first version (scalar fast_candidate, register double-buffering)
    // 4: read-only diagnostic, produces no counts (never selected by default)
    { "probe_read_only_t512_u4", launch_probe, (const void *)k_stream_probe<512, 4>, 512, 0, 0, 0 },
    BULK_VARIANT(16, 4, 32768, 1, 0),   // 5: negatives flagged to the fix-up instead of folded (2 instructions less per sample)
    BULK_VARIANT(16, 3, 65536, 1, 0),   // 6
};
constexpr int kNumK1Variants = (int)(sizeof(g_k1_variants) / sizeof(g_k1_variants[0]));

// The narrow forms of K1 that lh_ingest_arrays routes long float32 / int32 (4-byte form) and float16 / bfloat16
// (16-bit form, key table) items to.  One shape each, chosen to fit kSmemBudget beside the sub-histogram at every
// precision 1..250 (87 KB at 250): 4 x 32 KiB stages for the 4-byte form, 2 x 32 KiB plus the 64 KiB key table for
// the 16-bit form; 16 consumer warps, negatives folded into the slot.
constexpr int kK1nCW = 16, kK1nStage = 32768;
constexpr int kK1nStages4 = 4, kK1nStages2 = 2;
struct K1Narrow {
    void (*launch)(int grid, size_t smem, cudaStream_t s, const void *v32, size_t nvec, const void *head, int nhead,
                   const void *tail, int ntail, unsigned long long *counts, uint32_t *flag, const Prec &pc,
                   const uint16_t *keys);
    const void *func;
    uint32_t bytes;      // element size
    size_t smem_fixed;   // ring + barriers (+ key table)
    int blocks_per_sm;   // filled at create
    size_t smem;         // filled at create
};
template <typename Cv, int STAGES>
void launch_narrow(int grid, size_t smem, cudaStream_t s, const void *v32, size_t nvec, const void *head, int nhead,
                   const void *tail, int ntail, unsigned long long *counts, uint32_t *flag, const Prec &pc,
                   const uint16_t *keys) {
    using T = typename Cv::T;
    k_ingest_single_bulk<kK1nCW, STAGES, kK1nStage, 1, true, Cv><<<grid, (kK1nCW + 1) * 32, smem, s>>>(
        (const T *)v32, nvec, (const T *)head, nhead, (const T *)tail, ntail, counts, flag, pc, keys);
}
#define NARROW_FORM(CV, S, TABLE) \
    { launch_narrow<CV, S>, (const void *)k_ingest_single_bulk<kK1nCW, S, kK1nStage, 1, true, CV>, \
      (uint32_t)sizeof(CV::T), (size_t)S * (kK1nStage + 16) + (TABLE), 0, 0 }
const K1Narrow g_k1_narrow[4] = {   // by k1n_index
    NARROW_FORM(K1F32, kK1nStages4, 0),
    NARROW_FORM(K1I32, kK1nStages4, 0),
    NARROW_FORM(K1F16, kK1nStages2, 65536),
    NARROW_FORM(K1BF16, kK1nStages2, 65536),
};
#undef NARROW_FORM
// index into g_k1_narrow of dtype LH_GAUGE_*, -1: no narrow form (F64 takes K1 itself, I64 / U64 k_ingest_arrays)
int k1n_index(uint32_t dtype) {
    switch (dtype) {
    case LH_GAUGE_F32: return 0;
    case LH_GAUGE_I32: return 1;
    case LH_GAUGE_F16: return 2;
    case LH_GAUGE_BF16: return 3;
    default: return -1;
    }
}
constexpr int kDefaultK1Variant = 6;   // 3 x 64 KB stages, negatives through the fix-up: best sustained time of the bulk variants (within 2 % of each other on H100)

// Everything the kernels derive from `precision` (metrics.go:40-43), see lh_device.cuh.
Prec make_prec(uint32_t precision) {
    Prec pc{};
    const double P = (double)precision;
    const double c1 = P * 0.6931471805599453094172321;
    pc.precision = P;
    pc.a_int = (uint32_t)std::floor(c1);
    pc.c1 = (float)c1;
    pc.c2 = (float)(c1 - (double)pc.a_int);
    pc.kb = (float)(-1023.0 * (double)pc.c2);
    const float eps = 0.000244140625f * (precision > 100 ? (float)P / 100.0f : 1.0f);
    pc.thresh = 0.5f - eps;
    pc.win = (uint32_t)std::floor(P * 63.0 * 0.6931471805599453094172321 + 0.5) + 1u;
    pc.a4 = pc.a_int * 4u;
    pc.coff = 0u - 1023u * pc.a4 - (0x4B400000u << 2);
    pc.coff0 = 0u - 1023u * pc.a_int - 0x4B400000u;
    return pc;
}

constexpr int kMaxRanks = LH_MAX_RANKS;
constexpr int kCommWords = 2 * LH_MAX_RANKS;       // arrive[16], depart[16]
constexpr uint32_t kPeerMagic = 0x4C485052u;       // "LHPR"

// what lh_comm_export hands to the peers (fits lh_peer_handle)
struct PeerWire {
    uint32_t magic, abi, H, C;
    uint32_t precision, device;
    int64_t pid;
    uint64_t ctx_id;                               // distinguishes contexts of one process
    uint64_t ptr_buckets[2], ptr_flags[2], ptr_counters[2], ptr_comm, ptr_red;
    cudaIpcMemHandle_t ipc_buckets[2], ipc_flags[2], ipc_counters[2], ipc_comm, ipc_red;
};
static_assert(sizeof(PeerWire) <= LH_PEER_HANDLE_BYTES, "lh_peer_handle too small");

struct PeerMap {                                   // one remote rank as mapped into this process
    unsigned long long *buckets[2] = {nullptr, nullptr};
    uint32_t *flags[2] = {nullptr, nullptr};
    unsigned long long *counters[2] = {nullptr, nullptr};
    unsigned long long *comm = nullptr;
    unsigned long long *red = nullptr;             // the rank's REDUCED bucket array: owners of a slice push their sums into it
    bool ipc = false;                              // pointers came from cudaIpcOpenMemHandle (must be closed)
};

// a live raw board (lh_raw_board_create / _window) and the host's bookkeeping of its window
struct RawBoard {
    lh_raw_board b{};
    AsyncPtr mem;                 // the one allocation behind b.d_rows
    uint32_t window = 1;          // publishes summed per row (1: a plain board, published by k_raw_publish)
    uint64_t published = 0;       // publishes issued; a window board's next one replaces slot published % window
    uint64_t snapshot = 0;        // stats.snapshots at its latest publish: a window board takes one per snapshot
};

// a live board (lh_board_create): what the caller was given, and the allocation behind b.d_board
struct Board {
    lh_board b{};
    AsyncPtr mem;
};

}  // namespace

struct lh_ctx {
    // The streams come first: members are destroyed in reverse order, and stream-ordered allocations (graph recorders,
    // boards) are freed on snap_stream, so the streams must outlive every other member.  This order must hold.
    Stream ingest_stream, snap_stream, copy_stream;
    Stream rs_stream;                    // lh_reduce_sparse_host's own (created on first use)
    lh_config cfg{};
    int device = 0;
    int sm_count = 0;
    uint32_t H = 0, C = 0;
    Prec pc{};
    Buffer buf[2];
    int active = 0;
    bool frozen = false;
    bool rows_read = false;              // a reader has read the frozen rows (rows_read()): too late to add to them
    bool freezing = false;               // lh_snapshot_begin flipped the buffers and waits for record scopes to end
    bool nnz_valid = false;
    DevPtr<double> d_decomp;
    DevPtr<unsigned long long> d_dropped;
    // reduce / export scratch
    // two result slots (ticket & 1): packed [count H][sum H][avg H][pvals H*np][pkeys H*np]; slot 2 is scratch for
    // lh_snapshot_export when no reduction has produced the non-empty-bucket counts yet (never holds a ticket)
    DevPtr<double> d_ps[3];
    DevPtr<char> d_res[3];
    PinnedPtr<char> h_res[3];
    Event res_done[3];
    uint32_t res_np[3] = {0, 0, 0};
    uint64_t res_ticket[2] = {0, 0};
    uint64_t next_ticket = 1;
    DevPtr<uint32_t> d_nnz, d_offsets;                   // d_nnz: [3][H], the non-empty buckets K3 counted per result slot
    int nnz_slot = 0;                                    // the slot whose counts k_scan_nnz reads (the latest K3)
    DevPtr<short> d_x_keys; DevPtr<unsigned long long> d_x_counts; size_t x_cap = 0;
    // pinned host mirrors
    PinnedPtr<uint32_t> h_offsets;
    PinnedPtr<short> h_x_keys; PinnedPtr<unsigned long long> h_x_counts; size_t hx_cap = 0;
    PinnedPtr<unsigned long long> h_counter_deltas;
    // staging ring
    std::vector<Slot> slots;
    uint64_t slot_seq = 0;
    size_t staging_bytes = 0;
    // tuning
    unsigned long long last_margin[2] = {0, 0};
    int k1_variant = kDefaultK1Variant;
    int k1_grid_mult = 1;
    int k1_reserve_sms = 0;   // SMs left free for concurrent snapshot / collective kernels
    int keyed_blocks_per_sm = 8;
    uint32_t hot_replicas = 1;          // copies of the hot window (all L2-resident); only the vector RED kernel spreads over them
    int keyed_mode = 0;                 // 0 auto, 1 force L2-atomic kernel, 2 force the write-combining owner kernel
    int64_t kp_chunk = 256 << 20;       // samples per chunk of the owner-partitioned kernel (16 / 32 / 64 / 128 / 256 M: 319 / 339 / 354 / 363 / 368 G samples/s, keyed_pf_probe_r02q/r.txt)
    uint32_t wc_pf_tiles = 1;           // L2 prefetch distance of that kernel's input, in tiles past the one being loaded (0 = off; 1: +12 %)
    uint32_t wc_flush_samples = 24576;  // samples a CTA bins between two flushes of its owner buffers
    int wc_spt = 6;                     // tile shape of that kernel (6: 896 threads x 4 samples; 4: 1024 x 4; 3: 768 x 4; 8: 512 x 8)
    // owner-partitioned keyed kernel scratch (allocated on first use)
    DevPtr<unsigned short> d_kp_queues;
    DevPtr<unsigned int> d_kp_cnt;        // per-(owner, writer) record counts, then the grid-barrier word
    DevPtr<uint4> d_kp_rare;              // per-CTA lists of samples set aside for the exact path
    size_t kp_cap = 0;
    int kp_parts = 0;
    const char *keyed_kernel = "";       // kernel the last keyed launch used
    // lh_ingest_batch: CTAs of k_ingest_batch per SM (filled at create) and the parameter block being filled (locked)
    int batch_blocks_per_sm = 1;
    BatchParams batch_prm{};
    // multi-GPU (lh_comm_*): peer mappings of every rank's arrays + this rank's reduced output arrays
    uint32_t comm_rank = 0, comm_world = 0;
    DevPtr<unsigned long long> d_comm;            // this rank's comm block (uint64[kCommWords])
    DevPtr<unsigned int> d_comm_aux;              // [0] block counter, [1] status, [2..3] cells (both of the last all-reduce)
    PeerMap peers[kMaxRanks];
    DevPtr<unsigned long long> d_red_buckets;     // [H][65536] sums over ranks (valid for the open snapshot after lh_snapshot_allreduce)
    DevPtr<uint32_t> d_red_flags;
    DevPtr<unsigned long long> d_red_counters;
    bool view_reduced = false;                    // the open snapshot's reduce/export read the reduced arrays
    bool view_counters_reduced = false;
    uint64_t comm_seq = 0;
    bool comm_two_shot = false;                    // form of the last all-reduce (lh_comm_info's byte count)
    static constexpr int kCommRing = 8;
    Event comm_t0[kCommRing], comm_t1[kCommRing];
    // lh_snapshot_allreduce_rows: the row maps ([world][H] then [world][C] uint32, allocated at lh_comm_import), their
    // pinned staging, and an event behind the last upload (staging is rewritten only after it)
    DevPtr<uint32_t> d_row_maps;
    PinnedPtr<uint32_t> h_row_maps;
    Event row_maps_copied;
    // lh_snapshot_rows: pinned staging of the frozen flags and counters (allocated on first use)
    PinnedPtr<uint32_t> h_rows_flags;
    PinnedPtr<unsigned long long> h_rows_counters;
    // lh_snapshot_pack_rows / lh_snapshot_unpack_rows: the row table ([H] RowsEntry, then [C] counter rows) with its
    // pinned staging and an event behind the last upload (allocated on first use); the send and recv payloads (grown
    // on demand, rows_cap words each); the open snapshot's pack
    DevPtr<unsigned char> d_rows_table;
    PinnedPtr<unsigned char> h_rows_table;
    Event rows_table_copied;
    DevPtr<unsigned long long> d_rows_send, d_rows_recv;
    size_t rows_cap = 0;
    bool rows_packed = false;
    uint32_t rows_n = 0, rows_nc = 0;
    uint64_t rows_words = 0;
    uint64_t ctx_id = 0;
    // lh_reduce_sparse_host: its own stream (rs_stream) and K6_BATCH scratch rows (allocated on first use), serialised
    // by rs_mu; none of the arrays above is touched by it
    std::mutex rs_mu;
    DevPtr<unsigned long long> d_rs_rows;         // [K6_BATCH][65536], all zero between calls
    DevPtr<uint32_t> d_rs_flags, d_rs_nnz;
    bool rs_dirty = false;                        // a call failed part-way: zero the rows before the next one
    K1Variant k1[kNumK1Variants];
    // lh_ingest_arrays: the narrow forms of K1 (by K1Narrow index, occupancy filled at create) and the key tables of
    // the 16-bit form ([2][32768] uint16, k_fill_key16: float16, then bfloat16)
    K1Narrow k1n[4];
    DevPtr<uint16_t> d_key16;
    // timing of ingest: CUDA events bracket the kernels of every write_bracket (one sequence number); a ring keeps the
    // last kTimingRing pairs
    static constexpr int kTimingRing = 16;
    Event ev_t0s[kTimingRing], ev_t1s[kTimingRing];
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;   // the pair of the bracket being issued
    uint64_t ingest_seq = 0;                         // brackets opened so far
    bool timing_valid = false;
    // GPU timers: a pool of 64-bit start marks on the device (allocated by the first lh_gpu_timer_start)
    uint32_t timer_slots_n = 65536;
    DevPtr<unsigned long long> d_timer_marks;
    std::vector<TimerSlot> timer_slots;
    std::vector<uint32_t> timer_released;            // released slots, oldest first, reused once their kernels are done
    uint32_t timer_fresh = 0;                         // slots [timer_fresh, n) have never been handed out
    std::vector<Event> timer_spare_events;            // stop events of recycled slots
    // graph recorders, and the parameter block of their drain kernel (filled under the lock)
    std::vector<GraphRec> graphs;
    uint64_t next_graph = 1;
    Event graph_drained;                               // after the latest collection drain (created with the first recorder)
    DrainParams drain_prm{};
    // device subscriptions (lh_board_*): live boards, and the parameter block of their publish kernel (filled under the
    // lock); pub_slot is the result slot of the open snapshot's latest lh_snapshot_reduce(_async), -1 when there is none
    std::vector<Board> boards;
    uint64_t next_board = 1;
    int pub_slot = -1;
    BoardParams board_prm{};
    // raw device subscriptions (lh_raw_board_*): live boards, and the parameter block of their publish kernels (filled
    // under the lock)
    std::vector<RawBoard> raw_boards;
    uint64_t next_raw_board = 1;
    RawPublishParams raw_prm{};
    // device gauges (lh_gauges_read): calls are serialised by gauge_mu (taken before mu), since they share the output
    // buffer, mapped pinned memory that k_gauge_read writes into (grown on demand); gauge_done follows the last launch
    std::mutex gauge_mu;
    PinnedPtr<double> h_gauges;
    double *d_gauges = nullptr;                        // h_gauges as the device sees it
    uint32_t gauge_cap = 0;
    Event gauge_done;
    GaugeParams gauge_prm{};
    // distribution gauges (lh_snapshot_ingest_arrays): the parameter block of k_ingest_arrays (filled under the lock)
    ArrayParams array_prm{};
    // stats
    lh_stats stats{};
    std::mutex mu;
    std::condition_variable slot_cv;     // a staging slot came back (see slot_wait_free)
    std::vector<Scope> scopes;           // open record scopes
    uint64_t next_scope = 1;
    std::condition_variable scope_cv;    // a record scope ended (see lh_snapshot_begin)
    std::string last_error;
};

namespace {

lh_status fail(lh_ctx *ctx, lh_status st, const char *what, cudaError_t e = cudaSuccess) {
    if (ctx) {
        char buf[512];
        if (e != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
        else snprintf(buf, sizeof buf, "%s", what);
        ctx->last_error = buf;
    }
    return st;
}

// The calling thread in cudaStreamCaptureModeRelaxed for the scope of one entry point.  In the global mode (what
// torch.cuda.graph uses by default) a capture on ANY thread makes calls such as cudaEventSynchronize or cudaMalloc fail
// on every other thread and invalidates the capture; the library's own calls never touch a capturing stream, so a
// collection from a reaper thread may run beside a capture.
struct RelaxedCapture {
    cudaStreamCaptureMode prev = cudaStreamCaptureModeRelaxed;
    RelaxedCapture() { cudaThreadExchangeStreamCaptureMode(&prev); }
    ~RelaxedCapture() { cudaThreadExchangeStreamCaptureMode(&prev); }
};

#define LH_CUDA(ctx, call)                                                      \
    do {                                                                        \
        cudaError_t _e = (call);                                                \
        if (_e != cudaSuccess) return fail((ctx), LH_ERR_CUDA, #call, _e);      \
    } while (0)

// Every reader of the open snapshot's rows calls this before it reads them: lh_snapshot_ingest_arrays may add to the
// rows only until then, so that every reader of one snapshot sees the same interval.
void mark_rows_read(lh_ctx *ctx) { ctx->rows_read = true; }

// order `s` after the zeroing of buffer b, and remember `s` as a writer of b
lh_status before_write(lh_ctx *ctx, int b, cudaStream_t s) {
    LH_CUDA(ctx, cudaStreamWaitEvent(s, ctx->buf[b].cleared.get(), 0));
    return LH_OK;
}
lh_status after_write(lh_ctx *ctx, int b, cudaStream_t s) {
    for (auto &w : ctx->buf[b].writers)
        if (w.stream == s) { LH_CUDA(ctx, cudaEventRecord(w.ev.get(), s)); return LH_OK; }
    WriterEvent w{s, {}};
    LH_CUDA(ctx, cudaEventCreateWithFlags(w.ev.out(), cudaEventDisableTiming));
    LH_CUDA(ctx, cudaEventRecord(w.ev.get(), s));
    ctx->buf[b].writers.push_back(std::move(w));
    return LH_OK;
}

void next_timing_slot(lh_ctx *ctx) {
    const int i = (int)(ctx->ingest_seq % lh_ctx::kTimingRing);
    ctx->ev_t0 = ctx->ev_t0s[i].get();
    ctx->ev_t1 = ctx->ev_t1s[i].get();
    ctx->ingest_seq++;
}

cudaStream_t pick_stream(lh_ctx *ctx, void *stream) { return stream ? (cudaStream_t)stream : ctx->ingest_stream.get(); }

int grid_1d(lh_ctx *ctx, size_t n, int threads, int per_thread, int blocks_per_sm) {
    size_t need = (n + (size_t)threads * per_thread - 1) / ((size_t)threads * per_thread);
    size_t cap = (size_t)ctx->sm_count * blocks_per_sm;
    return (int)std::max<size_t>(1, std::min(need, cap));
}

// The SMs the ingest kernels may spread over: all but the k1_reserve_sms left to concurrent snapshot / collective work.
int ingest_sms(const lh_ctx *ctx) { return std::max(1, ctx->sm_count - ctx->k1_reserve_sms); }
// Samples one launch of `grid` CTAs may take when each CTA counts into uint32 cells of its own (K1's sub-histograms, the
// tables of k_ingest_batch / k_ingest_keyed_graph): work is dealt round-robin, so 2^31 per CTA keeps every cell < 2^32.
size_t launch_cap(int grid) { return std::min((size_t)1 << 36, (size_t)grid << 31); }
// The vector body of n samples of val_bytes each (8 unless given; naturally aligned) at `vals`: `head` scalar samples
// (at most 32 / val_bytes - 1) up to the first 32-byte aligned value, then n4 32-byte groups (of 4 samples when they are
// 8-byte); ids_ok: the ids (id_bytes each; 0: none) are aligned to 4 ids there.  Each caller decides what a misaligned
// or short piece takes instead.
struct VecSplit { size_t head, n4; bool ids_ok; };
VecSplit vec_split(const void *vals, size_t n, const void *ids = nullptr, size_t id_bytes = 0, size_t val_bytes = 8) {
    const size_t head = std::min<size_t>(n, ((32u - ((uintptr_t)vals & 31u)) & 31u) / val_bytes);
    return {head, (n - head) / (32 / val_bytes), !id_bytes || (((uintptr_t)ids + head * id_bytes) & (4 * id_bytes - 1)) == 0};
}

// The write protocol of every timed ingest (locked): order `s` after the zeroing of the active buffer, bracket
// body(b) with the CUDA events of one sequence number, then register `s` as a writer of b, which is what
// lh_snapshot_begin orders the snapshot after.  The body only issues kernels into buffer b and counts them in stats;
// when it fails, its status is returned without the end event or the writer registration.
template <typename Body>
lh_status write_bracket(lh_ctx *ctx, cudaStream_t s, Body body) {
    const int b = ctx->active;
    lh_status st = before_write(ctx, b, s);
    if (st != LH_OK) return st;
    next_timing_slot(ctx);
    LH_CUDA(ctx, cudaEventRecord(ctx->ev_t0, s));
    st = body(b);
    if (st != LH_OK) return st;
    LH_CUDA(ctx, cudaEventRecord(ctx->ev_t1, s));
    ctx->timing_valid = true;
    return after_write(ctx, b, s);
}

// ---- ingest bodies (run on validated input: inside write_bracket, or into a graph recorder's rows) ----
// The rows of buffer b as a recorder: the target the bodies below write, like a graph recorder's.
lh_recorder buffer_target(lh_ctx *ctx, int b) {
    lh_recorder rec;
    memset(&rec, 0, sizeof rec);
    rec.d_buckets = reinterpret_cast<uint64_t *>(ctx->buf[b].d_buckets.get());
    rec.d_flags = ctx->buf[b].d_flags.get();
    rec.d_counters = reinterpret_cast<uint64_t *>(ctx->buf[b].d_counters.get());
    rec.d_dropped = reinterpret_cast<uint64_t *>(ctx->d_dropped.get());
    rec.max_histograms = ctx->H;
    rec.max_counters = ctx->C;
    memcpy(rec.prec, &ctx->pc, sizeof ctx->pc);
    return rec;
}

// K1 into one row (counts, flag); the caller counts the samples in stats
lh_status launch_single(lh_ctx *ctx, unsigned long long *counts, uint32_t *flag, const double *d_values, size_t n, cudaStream_t s) {
    const K1Variant &kv = ctx->k1[ctx->k1_variant];
    const int grid = ingest_sms(ctx) * kv.blocks_per_sm * ctx->k1_grid_mult;
    const size_t cap = launch_cap(grid);
    size_t done = 0;
    while (done < n) {
        size_t m = std::min(n - done, cap);
        const double *p = d_values + done;
        const VecSplit v = vec_split(p, m);
        const double *body = p + v.head;
        const double *tail = body + v.n4 * 4;
        kv.launch(grid, kv.smem, s, body, v.n4, p, (int)v.head, tail, (int)(m - v.head - v.n4 * 4), counts, flag, ctx->pc);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        done += m;
    }
    return LH_OK;
}
// launch_single for a long array of 4-byte or 16-bit elements: the narrow form k1n of K1 (g_k1_narrow), with the grid
// and per-launch bound of launch_single.  The caller counts the samples in stats.
lh_status launch_narrow_single(lh_ctx *ctx, int k1n, unsigned long long *counts, uint32_t *flag, const void *d_values,
                               size_t n, cudaStream_t s) {
    const K1Narrow &f = ctx->k1n[k1n];
    const int grid = ingest_sms(ctx) * f.blocks_per_sm * ctx->k1_grid_mult;
    const size_t cap = launch_cap(grid);
    const uint16_t *keys = ctx->d_key16.get() + (k1n == 3 ? 32768 : 0);   // the 16-bit forms' table (bfloat16 second)
    for (size_t done = 0; done < n;) {
        const size_t m = std::min(n - done, cap);
        const char *p = (const char *)d_values + done * f.bytes;
        const VecSplit v = vec_split(p, m, nullptr, 0, f.bytes);
        const char *body = p + v.head * f.bytes;
        const char *tail = body + v.n4 * 32;
        f.launch(grid, f.smem, s, body, v.n4, p, (int)v.head, tail, (int)(m - v.head - v.n4 * (32 / f.bytes)), counts, flag,
                 ctx->pc, keys);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        done += m;
    }
    return LH_OK;
}
// n samples of histogram hid into buffer b, counted in stats
lh_status ingest_single(lh_ctx *ctx, int b, uint32_t hid, const double *d_values, size_t n, cudaStream_t s) {
    lh_status st = launch_single(ctx, ctx->buf[b].d_buckets.get() + (size_t)hid * 65536u, ctx->buf[b].d_flags.get() + hid, d_values, n, s);
    if (st == LH_OK) ctx->stats.samples += n;
    return st;
}

lh_status fold_hot(lh_ctx *ctx, int b, cudaStream_t s) {
    const size_t cells = (size_t)ctx->H * 2u * ctx->pc.win;
    int grid = (int)std::min<size_t>((cells + 255) / 256, (size_t)ctx->sm_count * 16);
    k_fold_hot<<<grid, 256, 0, s>>>(ctx->buf[b].d_hot.get(), ctx->buf[b].d_buckets.get(), ctx->buf[b].d_flags.get(), cells, ctx->hot_replicas, ctx->pc.win);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    ctx->buf[b].hot_pending = 0;
    return LH_OK;
}

KeyedOut keyed_out(lh_ctx *ctx, int b) {
    KeyedOut o{};
    o.hot = ctx->buf[b].d_hot.get(); o.buckets = ctx->buf[b].d_buckets.get(); o.flags = ctx->buf[b].d_flags.get();
    o.dropped = ctx->d_dropped.get(); o.H = ctx->H;
    return o;
}

// The scalar keyed kernel over a ragged piece (a head before the aligned body, a tail after it); nothing when n == 0.
// With an IdMap (record-scope ids), its mapped form, which copies the map into shared memory.
template <typename IdT, typename ValT, typename Map>
void launch_keyed_scalar(lh_ctx *ctx, const KeyedOut &ko, const IdT *ids, const ValT *vals, size_t n, cudaStream_t s,
                         const Map &map) {
    if (!n) return;
    constexpr int T = 256;
    const int grid = grid_1d(ctx, n, T, 1, ctx->keyed_blocks_per_sm);
    k_ingest_keyed<IdT, ValT, T, Map><<<grid, T, map_smem_bytes(map), s>>>(ids, vals, n, ko, ctx->pc, map);
    ctx->stats.kernel_launches++;
}

// Few histograms: their windows fit in shared memory (K1-style privatisation).  Up to KS_MAX_PASSES passes over id
// sub-ranges match or beat the L2-atomic kernel (each pass is HBM-bound at 10 B/sample) and, unlike it, do not depend
// on how clustered the values are.
constexpr uint32_t KS_MAX_PASSES = 4;

// Owner-partitioned write-combining kernel: used when the histograms cannot be privatised per CTA in a few
// passes but P owner CTAs (one per SM) can hold them all, and the batch is big enough to amortise the
// cooperative launch.
constexpr size_t kSmemBudget = 227 * 1024;
// the narrow forms of K1 fit beside the largest sub-histogram (precision 250: win 10 918)
static_assert(kK1nStages4 * (kK1nStage + 16) + (2 * 10918 + 8) * 4 <= kSmemBudget, "4-byte form of K1");
static_assert(kK1nStages2 * (kK1nStage + 16) + 65536 + (2 * 10918 + 8) * 4 <= kSmemBudget, "16-bit form of K1");

// Samples one launch of k_ingest_keyed_wc may take, both arrays of a fused pair together: its owner windows are uint32
// cells flushed once, at the end of the launch, so no cell may receive 2^32 samples in one launch.
constexpr size_t kWcMaxLaunch = 0xFFFFFFFFu;

// The write-combining tile shape of a wc_spt value (6, 4 or 3; any other value is 8): f(std::integral_constant<int, SPT>),
// so that f can name WcShape<SPT> and the kernels of that shape.
template <typename F>
auto with_wc_shape(int spt, F f) {
    switch (spt) {
    case 6: return f(std::integral_constant<int, 6>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 3: return f(std::integral_constant<int, 3>{});
    default: return f(std::integral_constant<int, 8>{});
    }
}

// What launch_keyed issues for one piece of a batch, or launch_keyed_pair for a pair (plan_keyed).
struct KeyedPlan {
    // the kernel of the vector body (the ragged ends always go through k_ingest_keyed); APART: a pair the
    // write-combining kernel does not take, ingested one array after the other
    enum Route { SCALAR /* no vector body */, SMALL, WC, VEC, APART } route = SCALAR;
    const char *name = "k_ingest_keyed";  // what lh_keyed_kernel_name reports after the launch
    size_t head = 0, n4 = 0;              // scalar samples before the vector body (32-byte aligned values), groups of 4 in it
    size_t taken = 0, taken2 = 0;         // samples the body kernel bins, of each array; the rest is the scalar tail
    int grid = 0;                         // CTAs: small, or P, the owners of the write-combining kernel
    size_t smem = 0;                      // dynamic shared memory (small, write-combining)
    uint32_t per = 0;                     // small: ids per pass
    int spt = 0, threads = 0;             // write-combining: tile shape (wc_spt resolved to 3, 4, 6 or 8)
    WcParams wc{};                        // write-combining: the parameter block but for the arrays and the scratch
};

// The route of keyed samples (ids, vals, n) over `nids` ids in play (ctx->H; a mapped call's k) and everything its
// launches need; no CUDA call and no change to ctx.  No ids in play: the scalar kernel, which drops every sample.
// A pair (float64 samples ids/vals/n, int64 samples ids2/vals2/n2) is one write-combining launch for both arrays when
// both are vector-aligned, together at most kWcMaxLaunch samples, and that kernel takes them, else APART.
KeyedPlan plan_keyed(const lh_ctx *ctx, uint32_t nids, size_t id_bytes, const void *ids, const void *vals, size_t n, bool pair = false,
                     const void *ids2 = nullptr, const void *vals2 = nullptr, size_t n2 = 0) {
    KeyedPlan p;
    if (!nids) return p;
    const uint32_t ks_per_max = std::max<uint32_t>(1, (uint32_t)(KS_SMEM_BYTES / ((size_t)ctx->pc.win * 4)));
    const uint32_t ks_passes = (nids + ks_per_max - 1) / ks_per_max;
    const bool small = ks_passes <= KS_MAX_PASSES && ctx->keyed_mode == 0;
    if (pair) {
        // few histograms: the shared-memory privatised kernel of launch_keyed is the better one, per array
        auto aligned = [&](const void *v, const void *i) { return ((uintptr_t)v & 31u) == 0 && ((uintptr_t)i & (4 * id_bytes - 1)) == 0; };
        p.route = KeyedPlan::APART;
        if (!n || !n2 || ctx->keyed_mode == 1 || small || !aligned(vals, ids) || !aligned(vals2, ids2)) return p;
        if (n + n2 > kWcMaxLaunch) return p;   // apart, each array split by launch_keyed
    } else {
        const VecSplit v = vec_split(vals, n, ids, id_bytes);
        if (!v.ids_ok) return p;                                                          // misaligned: the scalar kernel only
        p.head = v.head; p.n4 = v.n4;
        if (!p.n4) return p;                                                              // short: the scalar kernel only
        n = p.taken = p.n4 * 4;                                  // the vector body, all the write-combining kernel is offered
        if (small && p.n4 >= 4096) {
            p.route = KeyedPlan::SMALL; p.name = "k_ingest_keyed_small";
            p.per = (nids + ks_passes - 1) / ks_passes;
            p.smem = ((size_t)p.per * ctx->pc.win + 4) * 4;
            // one CTA per SM; fewer when the batch is small, so that the per-CTA flush stays negligible
            p.grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)ingest_sms(ctx), p.n4 / (KS_THREADS * 16)));
            return p;
        }
        p.route = KeyedPlan::VEC; p.name = "k_ingest_keyed_vec";
        if (ctx->keyed_mode == 1) return p;
    }
    // the write-combining kernel, or keep the route above when it declines
    const int P = std::min(ingest_sms(ctx), (int)WC_MAX_PARTS);
    if (P < 8) return p;
    const uint32_t ids_per = (nids + P - 1) / P;
    const size_t hist_bytes = (((size_t)ids_per * ctx->pc.win + 3) & ~(size_t)3) * 4;
    // the owners' windows first, then the largest per-owner buffers that still fit (fewer SMs for ingest = more ids per
    // owner = less room; on H100, 256 records at P = 131 for H = 1024)
    uint32_t row_cap = 0;
    size_t smem = 0;
    for (uint32_t cap_try : {256u, 192u, 128u}) {
        smem = hist_bytes + 2 * WC_MAX_PARTS * 4 + (size_t)(P + 1) * (cap_try + WC_ROW_EXTRA) * 2;
        if (smem <= kSmemBudget) { row_cap = cap_try; break; }
    }
    if (!row_cap || (size_t)ids_per * ctx->pc.win > 65535) return p;           // records are 16-bit (lid*win + slot)
    if (ctx->keyed_mode != 2 && n + n2 < ((size_t)1 << 22)) return p;          // small batches: the L2-atomic kernel
    int spt = 0, tile = 0, threads = 0;
    with_wc_shape(ctx->wc_spt, [&](auto c) { spt = c; tile = WcShape<c>::TILE; threads = WcShape<c>::THREADS; });
    const size_t taken = n / tile * tile, taken2 = n2 / tile * tile;   // whole tiles only
    if (taken + taken2 == 0) return p;
    p.route = KeyedPlan::WC; p.name = "k_ingest_keyed_wc";
    p.taken = taken; p.taken2 = taken2; p.grid = P; p.smem = smem; p.spt = spt; p.threads = threads;
    WcParams &w = p.wc;
    w.n = taken; w.n2 = taken2; w.ids_per = ids_per; w.row_cap = row_cap; w.row_stride = row_cap + WC_ROW_EXTRA;
    w.inv_p = (uint32_t)(((uint64_t)1 << 32) / (uint64_t)P) + 1u;
    w.pf_tiles = ctx->wc_pf_tiles;
    // chunks of about kp_chunk samples, EQUAL in size: with the nominal slice a short last chunk would be binned by a
    // few CTAs at full slice length while the others idle, a whole chunk time per launch)
    const size_t slice_max = std::max<size_t>(1, ((size_t)ctx->kp_chunk + (size_t)P * tile - 1) / ((size_t)P * tile));
    const size_t tiles_all = taken / tile + taken2 / tile;
    const size_t nchunks = (tiles_all + slice_max * P - 1) / (slice_max * P);
    w.slice_tiles = (uint32_t)std::max<size_t>(1, (tiles_all + nchunks * P - 1) / (nchunks * P));
    // every (owner, writer) pair has its own sub-queue: 1.25x the expected records per pair per chunk, plus slack
    // (records that do not fit take the exact L2 route, so this only trades speed on heavily skewed ids)
    const size_t expect = slice_max * tile / P;       // sized for the nominal slice: the allocation does not follow the batch size
    w.cap = (uint32_t)(((expect * 5 / 4 + 3 * WC_LINE + WC_LINE - 1) / WC_LINE) * WC_LINE);
    // samples between two flushes of the shared-memory owner buffers: the flush costs about the same whatever it moves,
    // so as many as the buffers hold at 4 sigma (wc_flush_samples; default 24576)
    // ... and an owner's expected share m of one interval must leave room for the carried-over remainder (< 64) and the
    // binomial spread: m + 3.5 sqrt(m) + 63 <= row_cap
    const double room = (double)row_cap - 63.0;
    const double m_max = std::pow((-3.5 + std::sqrt(3.5 * 3.5 + 4.0 * room)) / 2.0, 2.0);
    const uint32_t flush_samples = std::min<uint32_t>(ctx->wc_flush_samples, (uint32_t)(m_max * P));
    w.flush_tiles = std::max<uint32_t>(1u, flush_samples / tile);
    return p;
}

// Every write-combining launch on a device is ordered after the previous one, whatever its stream or context.  A
// context's scratch (record sub-queues, grid-barrier word) is shared by all the streams it ingests from, and a launch
// zeroes the barrier word on its own stream: two launches in flight together could clear it under a running grid and
// mix their records.  Ordering across contexts as well means no two cooperative grids are ever outstanding at once.
// A grid holds one CTA on every SM it uses, so two of them never ran side by side anyway.
std::mutex g_wc_mu;                      // guards g_wc_done; held from the wait through the record of each launch
std::vector<cudaEvent_t> g_wc_done;      // [device]: after the device's last write-combining launch

// the device's completion event (created on first use; lives as long as the process); call with g_wc_mu held
cudaError_t wc_done_event(int device, cudaEvent_t *out) {
    if ((size_t)device >= g_wc_done.size()) g_wc_done.resize((size_t)device + 1, nullptr);
    if (!g_wc_done[device]) {
        cudaError_t e = cudaEventCreateWithFlags(&g_wc_done[device], cudaEventDisableTiming);
        if (e != cudaSuccess) { g_wc_done[device] = nullptr; return e; }
    }
    *out = g_wc_done[device];
    return cudaSuccess;
}

// The write-combining launch of plan p: its first p.taken samples of (ids, vals) and, in a fused pair, the first
// p.taken2 int64 samples of (ids2, vals2).  A fused pair is never mapped.
template <typename IdT, typename ValT, typename Map>
lh_status launch_keyed_wc(lh_ctx *ctx, int b, const KeyedPlan &p, const IdT *ids, const ValT *vals, cudaStream_t s,
                          const Map &map, const IdT *ids2 = nullptr, const long long *vals2 = nullptr) {
    const int P = p.grid;
    if (!ctx->d_kp_queues.get() || ctx->kp_cap != p.wc.cap || ctx->kp_parts != P) {
        if (ctx->d_kp_queues.get()) {
            // a launch on another stream may still be using the old scratch
            cudaEvent_t done;
            {
                std::lock_guard<std::mutex> lk(g_wc_mu);
                LH_CUDA(ctx, wc_done_event(ctx->device, &done));
            }
            LH_CUDA(ctx, cudaEventSynchronize(done));
        }
        ctx->d_kp_queues.reset(); ctx->d_kp_cnt.reset(); ctx->d_kp_rare.reset();
        DevPtr<unsigned short> queues; DevPtr<unsigned int> cnt; DevPtr<uint4> rare;
        LH_CUDA(ctx, cudaMalloc(rare.out(), (size_t)P * WC_RARE_CAP * sizeof(uint4)));
        LH_CUDA(ctx, cudaMalloc(queues.out(), (size_t)2 * P * P * p.wc.cap * sizeof(unsigned short)));
        LH_CUDA(ctx, cudaMalloc(cnt.out(), ((size_t)2 * P * P + 1) * sizeof(unsigned int)));
        ctx->d_kp_queues = std::move(queues); ctx->d_kp_cnt = std::move(cnt); ctx->d_kp_rare = std::move(rare);
        ctx->kp_cap = p.wc.cap; ctx->kp_parts = P;
    }
    // the kernel of the planned tile shape; with an int64 second segment, its PAIR form (on the float64 instantiation)
    const void *fn = with_wc_shape(p.spt, [&](auto c) {
        if constexpr (kMapped<Map>) return (const void *)k_ingest_keyed_wc<IdT, ValT, c, false, Map>;
        else return !p.taken2 ? (const void *)k_ingest_keyed_wc<IdT, ValT, c, false> : (const void *)k_ingest_keyed_wc<IdT, double, c, true>;
    });
    // the attribute belongs to the function on the device, not to this context: one value for every context
    LH_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    WcParams prm = p.wc;
    prm.ids = ids; prm.vals = vals; prm.ids2 = ids2; prm.vals2 = vals2;
    prm.queues = ctx->d_kp_queues.get(); prm.q_cnt = ctx->d_kp_cnt.get(); prm.barrier = ctx->d_kp_cnt.get() + (size_t)2 * P * P;
    prm.rare = ctx->d_kp_rare.get(); prm.o = keyed_out(ctx, b);
    Prec pc = ctx->pc;
    void *args[] = {&prm, &pc, (void *)&map};
    {
        std::lock_guard<std::mutex> lk(g_wc_mu);
        cudaEvent_t done;
        LH_CUDA(ctx, wc_done_event(ctx->device, &done));
        LH_CUDA(ctx, cudaStreamWaitEvent(s, done, 0));
        LH_CUDA(ctx, cudaMemsetAsync(prm.barrier, 0, sizeof(unsigned int), s));
        LH_CUDA(ctx, cudaLaunchCooperativeKernel(fn, dim3(P), dim3(p.threads), args, p.smem, s));
        LH_CUDA(ctx, cudaEventRecord(done, s));
    }
    ctx->stats.kernel_launches++;
    return LH_OK;
}

// With an IdMap, ids are local to it (record-scope calls): the plan counts map.k ids and the kernels are the mapped forms.
template <typename IdT, typename ValT, typename Map>
lh_status launch_keyed(lh_ctx *ctx, int b, const IdT *d_ids, const ValT *d_vals, size_t n, cudaStream_t s, const Map &map) {
    constexpr int T = 256;
    uint32_t nids = ctx->H;
    if constexpr (kMapped<Map>) nids = map.k;
    const KeyedOut ko = keyed_out(ctx, b);
    size_t done = 0;
    while (done < n) {
        // no uint32 cell may wrap: the write-combining kernel's owner windows hold a whole launch (kWcMaxLaunch), and
        // the hot window of the small and vector kernels everything since its last drain, which comes before 2^32
        const unsigned long long kCap = kWcMaxLaunch;
        if (ctx->buf[b].hot_pending >= kCap - (1ull << 30)) {
            // the tally is host-side and counts what every stream has issued: the fold must come after all of it, not
            // only after this stream's kernels (each writer event follows the last bracket issued on its stream)
            for (const WriterEvent &w : ctx->buf[b].writers)
                if (w.stream != s) LH_CUDA(ctx, cudaStreamWaitEvent(s, w.ev.get(), 0));
            lh_status st = fold_hot(ctx, b, s);
            if (st != LH_OK) return st;
        }
        size_t m = (size_t)std::min<unsigned long long>(n - done, kCap - ctx->buf[b].hot_pending);
        const IdT *ids = d_ids + done;
        const ValT *vals = d_vals + done;
        const KeyedPlan p = plan_keyed(ctx, nids, sizeof(IdT), ids, vals, m);
        launch_keyed_scalar(ctx, ko, ids, vals, p.head, s, map);
        if (p.route == KeyedPlan::SMALL) {
            // per device, not per context: a value of this context's H could be overwritten by another context's
            // between here and the launch
            const void *fn = (const void *)k_ingest_keyed_small<IdT, ValT, Map>;
            LH_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
            for (uint32_t lo = 0; lo < nids; lo += p.per) {
                const uint32_t cnt = std::min(p.per, nids - lo);
                k_ingest_keyed_small<IdT, ValT, Map><<<p.grid, KS_THREADS, p.smem, s>>>(ids + p.head, vals + p.head, p.n4, lo, cnt, ko, ctx->pc, map);
                ctx->stats.kernel_launches++;
            }
        } else if (p.route == KeyedPlan::WC) {
            lh_status st = launch_keyed_wc<IdT, ValT>(ctx, b, p, ids + p.head, vals + p.head, s, map);
            if (st != LH_OK) return st;
        } else if (p.route == KeyedPlan::VEC) {
            const int grid = grid_1d(ctx, p.n4, T, 1, ctx->keyed_blocks_per_sm);
            k_ingest_keyed_vec<IdT, ValT, T, Map><<<grid, T, map_smem_bytes(map), s>>>(ids + p.head, vals + p.head, p.n4, ctx->hot_replicas, ko, ctx->pc, map);
            ctx->stats.kernel_launches++;
        }
        ctx->keyed_kernel = p.name;
        const size_t tail_off = p.head + p.taken;   // after whole tiles of the write-combining kernel: a ragged remainder
        launch_keyed_scalar(ctx, ko, ids + tail_off, vals + tail_off, m - tail_off, s, map);
        LH_CUDA(ctx, cudaGetLastError());
        // only k_ingest_keyed_small / _vec count into the uint32 hot window
        if (p.route == KeyedPlan::SMALL || p.route == KeyedPlan::VEC) ctx->buf[b].hot_pending += p.taken;
        done += m;
    }
    ctx->stats.samples += n;
    return LH_OK;
}

// Histogram samples (float64) and Timer samples (int64 ns, metrics.go:242-246) of one batch in ONE launch of the
// write-combining kernel: its fixed costs (zeroing and flushing the owners' windows, the last partly filled chunk) are
// paid once.  Unless plan_keyed fuses them, launch_keyed for each array in turn; either way one body, one sequence number.
template <typename IdT>
lh_status launch_keyed_pair(lh_ctx *ctx, int b, const IdT *ids_f, const double *vals_f, size_t n_f, const IdT *ids_ns,
                            const long long *vals_ns, size_t n_ns, cudaStream_t s) {
    const KeyedPlan p = plan_keyed(ctx, ctx->H, sizeof(IdT), ids_f, vals_f, n_f, true, ids_ns, vals_ns, n_ns);
    if (p.route == KeyedPlan::APART) {
        lh_status st = launch_keyed<IdT, double>(ctx, b, ids_f, vals_f, n_f, s, IdIdentity{});
        if (st != LH_OK) return st;
        return launch_keyed<IdT, long long>(ctx, b, ids_ns, vals_ns, n_ns, s, IdIdentity{});
    }
    lh_status st = launch_keyed_wc<IdT, double>(ctx, b, p, ids_f, vals_f, s, IdIdentity{}, ids_ns, vals_ns);
    if (st != LH_OK) return st;
    ctx->keyed_kernel = p.name;
    const KeyedOut ko = keyed_out(ctx, b);
    launch_keyed_scalar(ctx, ko, ids_f + p.taken, vals_f + p.taken, n_f - p.taken, s, IdIdentity{});   // the ragged ends
    launch_keyed_scalar(ctx, ko, ids_ns + p.taken2, vals_ns + p.taken2, n_ns - p.taken2, s, IdIdentity{});
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.samples += n_f + n_ns;
    return LH_OK;
}

// (id, amount) pairs into `counters` (C of them, ids >= C dropped and counted); the caller counts the ops in stats.
// With an IdMap, ids are local: C is map.k (<= LH_MAP_MAX, so always the shared-memory kernels, whose mapped forms take
// the map after the 2C halves: 12 B per id, 48 KiB at most) and an op under an unbound row is dropped and counted.
static_assert(LH_MAP_MAX <= (uint32_t)K2_SMEM_COUNTERS, "k_counter_add has no mapped form");
template <typename IdT, typename Map>
lh_status launch_counter(lh_ctx *ctx, unsigned long long *counters, uint32_t C, const IdT *d_ids, const uint64_t *d_amounts,
                         size_t n, cudaStream_t s, const Map &map) {
    if (n) {
        constexpr int T = 512;
        const unsigned long long *amts = reinterpret_cast<const unsigned long long *>(d_amounts);
        if (kMapped<Map> || C <= (uint32_t)K2_SMEM_COUNTERS) {
            // privatised per CTA (lo/hi halves in shared memory).  Vector body where the alignment allows: 4 ops per
            // thread and iteration; ragged head / tail through the scalar form of the same kernel.
            const VecSplit v = vec_split(amts, n, d_ids, sizeof(IdT));
            size_t head = v.head, n4 = v.n4;
            if (!v.ids_ok || ((uintptr_t)amts & 7u) != 0 || n4 < 4096) { head = 0; n4 = 0; }
            const size_t tail_off = head + n4 * 4;
            const size_t smem = (size_t)C * 8 + map_smem_bytes(map);
            auto scalar = [&](int grid, size_t off, size_t cnt) {
                k_counter_add_smem<IdT, T, Map><<<grid, T, smem, s>>>(d_ids + off, amts + off, cnt, counters, C, ctx->d_dropped.get(), map);
                ctx->stats.kernel_launches++;
            };
            if (head) scalar(1, 0, head);
            if (n4) {
                // one CTA per SM (the per-CTA flush is C global atomics), fewer for small batches
                const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)ingest_sms(ctx) * 2, n4 / (T * 4)));
                k_counter_add_smem_vec<IdT, T, Map><<<grid, T, smem, s>>>(d_ids + head, amts + head, n4, counters, C, ctx->d_dropped.get(), map);
                ctx->stats.kernel_launches++;
            }
            if (tail_off < n) scalar(grid_1d(ctx, n - tail_off, T, 8, 2), tail_off, n - tail_off);
        } else if constexpr (!kMapped<Map>) {
            int grid = grid_1d(ctx, n, T, 4, 4);
            k_counter_add<IdT, T><<<grid, T, 0, s>>>(d_ids, amts, n, counters, C, ctx->d_dropped.get());
            ctx->stats.kernel_launches++;
        }
        LH_CUDA(ctx, cudaGetLastError());
    }
    return LH_OK;
}
// n counter ops into buffer b's counters (C of them; a mapped call's kc), counted in stats
template <typename IdT, typename Map>
lh_status add_counters(lh_ctx *ctx, int b, uint32_t C, const IdT *d_ids, const uint64_t *d_amounts, size_t n, cudaStream_t s,
                       const Map &map) {
    lh_status st = launch_counter<IdT>(ctx, ctx->buf[b].d_counters.get(), C, d_ids, d_amounts, n, s, map);
    if (st == LH_OK) ctx->stats.counter_ops += n;
    return st;
}

// lh_ingest_batch routing.  An F64 item this long pays back K1's full-grid launch (launch_single); shorter ones and every
// I64NS item go to k_ingest_batch.
constexpr size_t kBatchK1Min = 1024 * 1024;

// Items of a validated batch (lh_ingest_batch, lh_graph_recorder_ingest) into the rows of `target`: the long float64
// ones through launch_single, the rest through as few launches of k_ingest_batch as the parameter block and the uint32
// table counts allow.  An item that does not fit the launch being filled is split across launches.  Kernels only (the
// graph recorder's form is captured); the caller counts the samples in stats.
// The grid of k_ingest_batch (and of k_ingest_keyed_graph, which has its launch bounds and table).
int batch_grid_max(const lh_ctx *ctx) { return ingest_sms(ctx) * ctx->batch_blocks_per_sm; }

lh_status launch_batch(lh_ctx *ctx, const lh_recorder &target, const lh_batch_item *items, uint32_t n_items, cudaStream_t s) {
    BatchParams &prm = ctx->batch_prm;
    prm.rec = target;
    const int grid_max = batch_grid_max(ctx);
    const unsigned long long cap = launch_cap(grid_max);
    uint32_t k = 0;
    unsigned long long total = 0;
    auto launch = [&]() -> lh_status {
        if (!k) return LH_OK;
        prm.n_items = k;
        const unsigned long long pieces = (total + BI_PIECE - 1) / BI_PIECE;
        const int grid = (int)std::min<unsigned long long>((unsigned long long)grid_max, pieces);
        k_ingest_batch<<<grid, BI_THREADS, BlockRecorder::smem_bytes(BI_TABLE_ENTRIES), s>>>(prm);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        k = 0;
        total = 0;
        return LH_OK;
    };
    for (uint32_t i = 0; i < n_items; i++) {
        const lh_batch_item &it = items[i];
        if (it.n == 0) continue;
        if (it.kind == LH_VALUES_F64 && it.n >= kBatchK1Min) {
            unsigned long long *row = reinterpret_cast<unsigned long long *>(target.d_buckets) + (size_t)it.histogram_id * 65536u;
            lh_status st = launch_single(ctx, row, target.d_flags + it.histogram_id, (const double *)it.d_values, (size_t)it.n, s);
            if (st != LH_OK) return st;
            continue;
        }
        const unsigned long long *p = (const unsigned long long *)it.d_values;
        unsigned long long left = it.n;
        while (left) {
            if (k == (uint32_t)BI_MAX_ITEMS || total == cap) {
                lh_status st = launch();
                if (st != LH_OK) return st;
            }
            const unsigned long long m = std::min(left, cap - total);
            prm.seg[k] = BatchSeg{p, it.histogram_id, it.kind};
            prm.start[k] = total;
            total += m;
            prm.start[k + 1] = total;
            k++;
            p += m;
            left -= m;
        }
    }
    return launch();
}

// Validated (id, value) pairs into the rows of `target` (lh_graph_recorder_ingest_keyed_*): k_ingest_keyed_graph, over
// as many launches as launch_batch's bound on the samples of one launch requires, with launch_batch's grid.  The
// vector body starts at the first 32-byte aligned value; when the ids are not 4*sizeof(IdT)-aligned there, every sample
// goes one per thread.  Kernels only, so it may be captured; the caller counts nothing in stats but the launches.
template <typename IdT>
lh_status launch_keyed_graph(lh_ctx *ctx, const lh_recorder &target, const IdT *ids, const unsigned long long *vals, size_t n,
                             bool ns, cudaStream_t s) {
    const int grid_max = batch_grid_max(ctx);
    const size_t cap = launch_cap(grid_max);
    for (size_t done = 0; done < n;) {
        const size_t m = std::min(n - done, cap);
        const IdT *ip = ids + done;
        const unsigned long long *vp = vals + done;
        const VecSplit v = vec_split(vp, m, ip, sizeof(IdT));
        const size_t head = v.ids_ok ? v.head : m, n4 = v.ids_ok ? v.n4 : 0;   // misaligned ids: one sample per thread
        const int grid = (int)std::min<size_t>((size_t)grid_max, (m + BI_PIECE - 1) / BI_PIECE);
        k_ingest_keyed_graph<IdT><<<grid, BI_THREADS, BlockRecorder::smem_bytes(BI_TABLE_ENTRIES), s>>>(target, ip, vp, head, n4, m, ns);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        done += m;
    }
    return LH_OK;
}

// Validation of lh_ingest_batch / lh_graph_recorder_ingest against `limit` histogram ids; the samples of the batch
lh_status check_batch(lh_ctx *ctx, const lh_batch_item *h_items, uint32_t n_items, uint32_t limit, unsigned long long *n_out) {
    if (n_items && !h_items) return fail(ctx, LH_ERR_INVALID, "h_items is NULL");
    unsigned long long n = 0;
    for (uint32_t i = 0; i < n_items; i++) {
        const lh_batch_item &it = h_items[i];
        if (it.kind != LH_VALUES_F64 && it.kind != LH_VALUES_I64NS) return fail(ctx, LH_ERR_INVALID, "unknown item kind");
        if (it.n == 0) continue;
        if (!it.d_values) return fail(ctx, LH_ERR_INVALID, "item d_values is NULL");
        if (((uintptr_t)it.d_values & 7u) != 0) return fail(ctx, LH_ERR_INVALID, "item d_values must be 8-byte aligned");
        if (it.histogram_id >= limit) return fail(ctx, LH_ERR_RANGE, "item histogram_id >= max_histograms");
        n += it.n;
    }
    *n_out = n;
    return LH_OK;
}

// One launch of k_graph_drain per DR_MAX_ENTRIES rows and counters of `graphs` (all live recorders, or one), into the
// rows of buffer b, on s.
lh_status drain_graphs(lh_ctx *ctx, const GraphRec *graphs, size_t n_graphs, int b, cudaStream_t s) {
    DrainParams &p = ctx->drain_prm;
    p.buckets = ctx->buf[b].d_buckets.get();
    p.flags = ctx->buf[b].d_flags.get();
    p.counters = ctx->buf[b].d_counters.get();
    p.dropped = ctx->d_dropped.get();
    p.win = ctx->pc.win;
    p.n = 0;
    auto launch = [&]() -> lh_status {
        if (!p.n) return LH_OK;
        k_graph_drain<<<p.n, DR_THREADS, 0, s>>>(p);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        p.n = 0;
        return LH_OK;
    };
    auto add = [&](unsigned long long *src, uint32_t *flag, uint32_t target) -> lh_status {
        if (p.n == (uint32_t)DR_MAX_ENTRIES) {
            lh_status st = launch();
            if (st != LH_OK) return st;
        }
        p.e[p.n++] = DrainEntry{src, flag, target, 0};
        return LH_OK;
    };
    for (size_t g = 0; g < n_graphs; g++) {
        const GraphRec &gr = graphs[g];
        unsigned long long *rows = reinterpret_cast<unsigned long long *>(gr.rec.d_buckets);
        unsigned long long *ctrs = reinterpret_cast<unsigned long long *>(gr.rec.d_counters);
        for (uint32_t i = 0; i < gr.rec.max_histograms; i++) {
            lh_status st = add(rows + (size_t)i * 65536u, gr.rec.d_flags + i, gr.hid[i]);
            if (st != LH_OK) return st;
        }
        for (uint32_t i = 0; i < gr.rec.max_counters; i++) {
            lh_status st = add(ctrs + i, nullptr, gr.cid[i]);
            if (st != LH_OK) return st;
        }
    }
    return launch();
}

// ---- staging ring (locked) ----
// Called with ctx->mu held through `lk`.  The host-side wait for an in-flight slot happens with the mutex RELEASED
// (the slot is parked as SLOT_WAITED meanwhile so nobody else takes it): other ingest threads are never held up by
// it, and a thread that finds every slot either acquired or being waited for sleeps on slot_cv until one comes back.
lh_status slot_wait_free(lh_ctx *ctx, std::unique_lock<std::mutex> &lk, int *out) {
    for (;;) {
        // prefer a free slot that already has memory, then an in-flight one that has already finished, then a fresh
        // slot (allocating its pinned + device memory), and only then wait for the oldest in-flight one
        int best = -1, fresh = -1, waited = 0;
        for (size_t i = 0; i < ctx->slots.size(); i++) {
            if (ctx->slots[i].state == SLOT_WAITED || ctx->slots[i].state == SLOT_FILLING) waited++;   // will come back by itself
            if (ctx->slots[i].state != SLOT_FREE) continue;
            if (ctx->slots[i].h.get()) { *out = (int)i; return LH_OK; }
            if (fresh < 0) fresh = (int)i;
        }
        for (size_t i = 0; i < ctx->slots.size(); i++)
            if (ctx->slots[i].state == SLOT_INFLIGHT && cudaEventQuery(ctx->slots[i].done.get()) == cudaSuccess) {
                ctx->slots[i].state = SLOT_FREE;
                *out = (int)i;
                return LH_OK;
            }
        cudaGetLastError();   // cudaErrorNotReady from the queries above is not an error
        if (fresh >= 0) {
            PinnedPtr<void> h; DevPtr<void> d;
            cudaError_t e = cudaMallocHost(h.out(), ctx->staging_bytes);
            if (e == cudaSuccess) e = cudaMalloc(d.out(), ctx->staging_bytes);
            if (e != cudaSuccess)
                return fail(ctx, e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA, "allocating a staging slot", e);
            ctx->slots[fresh].h = std::move(h);
            ctx->slots[fresh].d = std::move(d);
            *out = fresh;
            return LH_OK;
        }
        for (size_t i = 0; i < ctx->slots.size(); i++)
            if (ctx->slots[i].state == SLOT_INFLIGHT && (best < 0 || ctx->slots[i].seq < ctx->slots[best].seq)) best = (int)i;
        if (best >= 0) {
            ctx->slots[best].state = SLOT_WAITED;
            cudaEvent_t ev = ctx->slots[best].done.get();
            lk.unlock();
            cudaError_t e = cudaEventSynchronize(ev);
            lk.lock();
            ctx->slots[best].state = SLOT_FREE;
            ctx->slot_cv.notify_all();
            if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "cudaEventSynchronize(slot)", e);
            *out = best;
            return LH_OK;
        }
        if (!waited) return fail(ctx, LH_ERR_STATE, "every staging slot is acquired and none is in flight");
        ctx->slot_cv.wait(lk);   // other threads are waiting for kernels: one of them will free a slot (or take it; then retry)
    }
}

// close the IPC mappings of the peers (lh_comm_import), if any
void comm_unmap(lh_ctx *ctx) {
    for (int r = 0; r < kMaxRanks; r++) {
        PeerMap &pm = ctx->peers[r];
        if (pm.ipc) {
            for (int b = 0; b < 2; b++) {
                if (pm.buckets[b]) cudaIpcCloseMemHandle(pm.buckets[b]);
                if (pm.flags[b]) cudaIpcCloseMemHandle(pm.flags[b]);
                if (pm.counters[b]) cudaIpcCloseMemHandle(pm.counters[b]);
            }
            if (pm.comm) cudaIpcCloseMemHandle(pm.comm);
            if (pm.red) cudaIpcCloseMemHandle(pm.red);
        }
        pm = PeerMap{};
    }
    ctx->comm_world = 0;
}

// the arrays the all-reduce writes (this rank's own kernel and, for its slices, every peer's)
lh_status comm_alloc_reduced(lh_ctx *ctx) {
    if (ctx->d_red_buckets.get()) return LH_OK;
    const size_t bucket_bytes = (size_t)ctx->H * 65536u * 8u;
    cudaStream_t s = ctx->snap_stream.get();
    DevPtr<unsigned long long> buckets, counters; DevPtr<uint32_t> flags;
    LH_CUDA(ctx, cudaMalloc(buckets.out(), bucket_bytes));
    LH_CUDA(ctx, cudaMalloc(flags.out(), (size_t)ctx->H * 4));
    LH_CUDA(ctx, cudaMalloc(counters.out(), (size_t)ctx->C * 8));
    LH_CUDA(ctx, cudaMemsetAsync(buckets.get(), 0, bucket_bytes, s));
    LH_CUDA(ctx, cudaMemsetAsync(flags.get(), 0, (size_t)ctx->H * 4, s));
    LH_CUDA(ctx, cudaMemsetAsync(counters.get(), 0, (size_t)ctx->C * 8, s));
    LH_CUDA(ctx, cudaStreamSynchronize(s));
    ctx->d_red_buckets = std::move(buckets); ctx->d_red_flags = std::move(flags); ctx->d_red_counters = std::move(counters);
    return LH_OK;
}

// the row maps of lh_snapshot_allreduce_rows, sized for the largest world
lh_status comm_alloc_row_maps(lh_ctx *ctx) {
    if (ctx->d_row_maps.get()) return LH_OK;
    const size_t bytes = (size_t)kMaxRanks * ((size_t)ctx->H + ctx->C) * 4u;
    DevPtr<uint32_t> d; PinnedPtr<uint32_t> h; Event copied;
    LH_CUDA(ctx, cudaMalloc(d.out(), bytes));
    LH_CUDA(ctx, cudaMallocHost(h.out(), bytes));
    LH_CUDA(ctx, cudaEventCreateWithFlags(copied.out(), cudaEventDisableTiming));
    ctx->d_row_maps = std::move(d); ctx->h_row_maps = std::move(h); ctx->row_maps_copied = std::move(copied);
    return LH_OK;
}

// pinned staging of lh_snapshot_rows and lh_snapshot_row_levels
lh_status alloc_rows_staging(lh_ctx *ctx) {
    if (ctx->h_rows_flags.get()) return LH_OK;
    PinnedPtr<uint32_t> flags; PinnedPtr<unsigned long long> counters;
    LH_CUDA(ctx, cudaMallocHost(flags.out(), (size_t)ctx->H * 4));
    LH_CUDA(ctx, cudaMallocHost(counters.out(), (size_t)ctx->C * 8));
    ctx->h_rows_flags = std::move(flags); ctx->h_rows_counters = std::move(counters);
    return LH_OK;
}

bool is_pinned_or_managed(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

}  // namespace

// =========================================================== lifecycle
extern "C" uint32_t lh_abi_version(void) { return LH_ABI_VERSION; }

extern "C" const char *lh_strerror(lh_status st) {
    switch (st) {
    case LH_OK: return "ok";
    case LH_ERR_INVALID: return "invalid argument";
    case LH_ERR_CUDA: return "CUDA runtime error";
    case LH_ERR_NOMEM: return "out of memory";
    case LH_ERR_NO_DEVICE: return "no usable CUDA device (there is no CPU fallback)";
    case LH_ERR_STATE: return "call out of order";
    case LH_ERR_RANGE: return "id or size out of range";
    default: return "unknown status";
    }
}

extern "C" const char *lh_last_error(const lh_ctx *ctx) { return ctx ? ctx->last_error.c_str() : ""; }

extern "C" lh_status lh_create(const lh_config *cfg, lh_ctx **out) {
    if (!cfg || !out || cfg->struct_size != sizeof(lh_config) || cfg->max_histograms == 0 || cfg->max_counters == 0)
        return LH_ERR_INVALID;
    if (cfg->precision > LH_MAX_PRECISION) return LH_ERR_RANGE;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return LH_ERR_NO_DEVICE; }
    if (cfg->device < 0 || cfg->device >= ndev) return LH_ERR_NO_DEVICE;
    // released through lh_destroy on every failure below, handed out at the end
    std::unique_ptr<lh_ctx, lh_status (*)(lh_ctx *)> ctx(new (std::nothrow) lh_ctx(), lh_destroy);
    if (!ctx) return LH_ERR_NOMEM;
    ctx->cfg = *cfg;
    ctx->device = cfg->device;
    ctx->H = cfg->max_histograms;
    ctx->C = cfg->max_counters;
    ctx->pc = make_prec(cfg->precision ? cfg->precision : 100);
    {
        static std::mutex id_mu;
        static uint64_t next_id = 1;
        std::lock_guard<std::mutex> lk(id_mu);
        ctx->ctx_id = next_id++;
    }
    {   // replicas of the keyed hot window: as many as keep all copies within ~20 MB (L2-resident in H100's 50 MB
        // L2 next to the streamed input), at most 32
        const size_t one = (size_t)ctx->H * 2u * ctx->pc.win * 4u;
        ctx->hot_replicas = (uint32_t)std::max<size_t>(1, std::min<size_t>(32, ((size_t)20 << 20) / one));
    }
    ctx->staging_bytes = cfg->staging_bytes ? (size_t)cfg->staging_bytes : ((size_t)32 << 20);
    ctx->staging_bytes = (ctx->staging_bytes + 255) & ~(size_t)255;
    const uint32_t nslots = cfg->staging_slots ? cfg->staging_slots : 3;

#define LH_CREATE_CUDA(call)                                                            \
    do {                                                                                \
        cudaError_t _e = (call);                                                        \
        if (_e != cudaSuccess) {                                                        \
            fprintf(stderr, "loghisto_b200: lh_create: %s failed: %s\n", #call, cudaGetErrorString(_e)); \
            return _e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA;        \
        }                                                                               \
    } while (0)

    LH_CREATE_CUDA(cudaSetDevice(ctx->device));
    cudaDeviceProp prop;
    LH_CREATE_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code runs on compute capability 9.0 only
        fprintf(stderr, "loghisto_b200: device %d is sm_%d%d; this library is built for sm_90a only\n", ctx->device, prop.major, prop.minor);
        return LH_ERR_NO_DEVICE;
    }
    ctx->sm_count = prop.multiProcessorCount;
    LH_CREATE_CUDA(cudaStreamCreateWithFlags(ctx->ingest_stream.out(), cudaStreamNonBlocking));
    LH_CREATE_CUDA(cudaStreamCreateWithFlags(ctx->copy_stream.out(), cudaStreamNonBlocking));
    {   // the snapshot stream outranks ingest: its small kernels slot in as soon as any ingest CTA retires
        int least = 0, greatest = 0;
        LH_CREATE_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        LH_CREATE_CUDA(cudaStreamCreateWithPriority(ctx->snap_stream.out(), cudaStreamNonBlocking, greatest));
    }
    for (int i = 0; i < lh_ctx::kTimingRing; i++) {
        LH_CREATE_CUDA(cudaEventCreate(ctx->ev_t0s[i].out()));
        LH_CREATE_CUDA(cudaEventCreate(ctx->ev_t1s[i].out()));
    }
    for (int i = 0; i < lh_ctx::kCommRing; i++) {
        LH_CREATE_CUDA(cudaEventCreate(ctx->comm_t0[i].out()));
        LH_CREATE_CUDA(cudaEventCreate(ctx->comm_t1[i].out()));
    }

    const size_t bucket_bytes = (size_t)ctx->H * 65536u * 8u, counter_bytes = (size_t)ctx->C * 8u;
    const size_t hot_bytes = (size_t)ctx->hot_replicas * ctx->H * 2u * ctx->pc.win * 4u;
    for (int b = 0; b < 2; b++) {
        LH_CREATE_CUDA(cudaMalloc(ctx->buf[b].d_buckets.out(), bucket_bytes));
        LH_CREATE_CUDA(cudaMalloc(ctx->buf[b].d_counters.out(), counter_bytes));
        LH_CREATE_CUDA(cudaMalloc(ctx->buf[b].d_flags.out(), (size_t)ctx->H * 4u));
        LH_CREATE_CUDA(cudaMemsetAsync(ctx->buf[b].d_buckets.get(), 0, bucket_bytes, ctx->snap_stream.get()));
        LH_CREATE_CUDA(cudaMemsetAsync(ctx->buf[b].d_counters.get(), 0, counter_bytes, ctx->snap_stream.get()));
        LH_CREATE_CUDA(cudaMemsetAsync(ctx->buf[b].d_flags.get(), 0, (size_t)ctx->H * 4u, ctx->snap_stream.get()));
        LH_CREATE_CUDA(cudaMalloc(ctx->buf[b].d_hot.out(), hot_bytes));
        LH_CREATE_CUDA(cudaMemsetAsync(ctx->buf[b].d_hot.get(), 0, hot_bytes, ctx->snap_stream.get()));
        LH_CREATE_CUDA(cudaEventCreateWithFlags(ctx->buf[b].cleared.out(), cudaEventDisableTiming));
        LH_CREATE_CUDA(cudaEventRecord(ctx->buf[b].cleared.get(), ctx->snap_stream.get()));
    }
    LH_CREATE_CUDA(cudaMalloc(ctx->d_decomp.out(), 65536 * sizeof(double)));
    k_fill_decompress<<<65536 / 256, 256, 0, ctx->snap_stream.get()>>>(ctx->d_decomp.get(), ctx->pc.precision);
    LH_CREATE_CUDA(cudaGetLastError());
    LH_CREATE_CUDA(cudaMalloc(ctx->d_comm.out(), kCommWords * 8));
    LH_CREATE_CUDA(cudaMemsetAsync(ctx->d_comm.get(), 0, kCommWords * 8, ctx->snap_stream.get()));
    LH_CREATE_CUDA(cudaMalloc(ctx->d_comm_aux.out(), 16));
    LH_CREATE_CUDA(cudaMemsetAsync(ctx->d_comm_aux.get(), 0, 16, ctx->snap_stream.get()));
    LH_CREATE_CUDA(cudaMalloc(ctx->d_dropped.out(), 8));
    LH_CREATE_CUDA(cudaMemsetAsync(ctx->d_dropped.get(), 0, 8, ctx->snap_stream.get()));
    for (int i = 0; i < 3; i++) {
        const size_t res_bytes = (size_t)ctx->H * (24 + LH_MAX_PERCENTILES * 12);
        LH_CREATE_CUDA(cudaMalloc(ctx->d_ps[i].out(), LH_MAX_PERCENTILES * sizeof(double)));
        LH_CREATE_CUDA(cudaMalloc(ctx->d_res[i].out(), res_bytes));
        LH_CREATE_CUDA(cudaMallocHost(ctx->h_res[i].out(), res_bytes));
        LH_CREATE_CUDA(cudaEventCreateWithFlags(ctx->res_done[i].out(), cudaEventDisableTiming));
    }
    LH_CREATE_CUDA(cudaMalloc(ctx->d_nnz.out(), (size_t)3 * ctx->H * 4));
    LH_CREATE_CUDA(cudaMalloc(ctx->d_offsets.out(), ((size_t)ctx->H + 1) * 4));
    LH_CREATE_CUDA(cudaMallocHost(ctx->h_offsets.out(), ((size_t)ctx->H + 1) * 4));
    LH_CREATE_CUDA(cudaMallocHost(ctx->h_counter_deltas.out(), counter_bytes));

    ctx->slots.resize(nslots);   // pinned + device memory of a slot is allocated the first time it is handed out
    for (auto &sl : ctx->slots) {
        LH_CREATE_CUDA(cudaEventCreateWithFlags(sl.done.out(), cudaEventDisableTiming));
        LH_CREATE_CUDA(cudaEventCreateWithFlags(sl.copied.out(), cudaEventDisableTiming));
    }

    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_peer_allreduce, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_peer_allreduce_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_counter_add_smem<unsigned short, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, K2_SMEM_COUNTERS * 8));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_counter_add_smem<unsigned int, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, K2_SMEM_COUNTERS * 8));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_counter_add_smem_vec<unsigned short, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, K2_SMEM_COUNTERS * 8));
    LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_counter_add_smem_vec<unsigned int, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, K2_SMEM_COUNTERS * 8));
    for (int i = 0; i < kNumK1Variants; i++) {
        ctx->k1[i] = g_k1_variants[i];
        const bool probe = ctx->k1[i].launch == launch_probe;
        const size_t hist = ((size_t)2 * ctx->pc.win + 8) * 4;
        ctx->k1[i].smem = probe ? 0 : ctx->k1[i].smem_fixed + hist;
        if (ctx->k1[i].smem > kSmemBudget) {
            // this ring does not fit beside the sub-histogram at this precision: take the next smaller ring with the same
            // arithmetic, and the register-pipelined kernel when none fits
            static const int smaller[] = {5, 0, 2, 3};
            for (int j : smaller) {
                if (g_k1_variants[j].smem_fixed + hist <= kSmemBudget) {
                    const char *name = ctx->k1[i].name;
                    ctx->k1[i] = g_k1_variants[j];
                    ctx->k1[i].name = name;
                    ctx->k1[i].smem = g_k1_variants[j].smem_fixed + hist;
                    break;
                }
            }
        }
        // the limit is an attribute of the function on the device, shared by every context: a value of this precision
        // would make an older context of a higher precision fail its launches.  Every launch asks for at most the budget.
        LH_CREATE_CUDA(cudaFuncSetAttribute(ctx->k1[i].func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
        int nb = 0;
        LH_CREATE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, ctx->k1[i].func, ctx->k1[i].threads, ctx->k1[i].smem));
        ctx->k1[i].blocks_per_sm = std::max(nb, 1);
    }
    {   // the attribute is per function on the device, so the same budget as every other kernel with a large table
        const void *fn = (const void *)k_ingest_batch;
        LH_CREATE_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
        int nb = 0;
        LH_CREATE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fn, BI_THREADS, BlockRecorder::smem_bytes(BI_TABLE_ENTRIES)));
        ctx->batch_blocks_per_sm = std::max(nb, 1);
        // k_ingest_keyed_graph: the same launch bounds and table, so the same occupancy and grid (batch_grid_max)
        LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_ingest_keyed_graph<unsigned short>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
        LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_ingest_keyed_graph<unsigned int>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
        // k_ingest_arrays (lh_snapshot_ingest_arrays, and lh_ingest_arrays' short items): likewise
        LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_ingest_arrays<gauge::Relaxed>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
        LH_CREATE_CUDA(cudaFuncSetAttribute((const void *)k_ingest_arrays<gauge::Streaming>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    }
    {   // lh_ingest_arrays' narrow forms of K1 and the key tables of the 16-bit one (before any capture can need them)
        LH_CREATE_CUDA(cudaMalloc(ctx->d_key16.out(), 65536 * sizeof(uint16_t)));
        k_fill_key16<<<65536 / 256, 256, 0, ctx->snap_stream.get()>>>(ctx->d_key16.get(), ctx->pc.precision, ctx->pc.win);
        LH_CREATE_CUDA(cudaGetLastError());
        const size_t hist = (size_t)subhist_words(ctx->pc.win) * 4;
        for (int i = 0; i < 4; i++) {
            K1Narrow &f = ctx->k1n[i];
            f = g_k1_narrow[i];
            f.smem = f.smem_fixed + hist;   // <= kSmemBudget at every precision (static_assert beside kSmemBudget)
            LH_CREATE_CUDA(cudaFuncSetAttribute(f.func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
            int nb = 0;
            LH_CREATE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, f.func, (kK1nCW + 1) * 32, f.smem));
            f.blocks_per_sm = std::max(nb, 1);
        }
    }
    LH_CREATE_CUDA(cudaStreamSynchronize(ctx->snap_stream.get()));
#undef LH_CREATE_CUDA
    *out = ctx.release();
    return LH_OK;
}

extern "C" lh_status lh_destroy(lh_ctx *ctx) {
    if (!ctx) return LH_OK;
    RelaxedCapture relaxed;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (!ctx->scopes.empty()) return fail(ctx, LH_ERR_STATE, "lh_destroy with record scopes open");
    }
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    comm_unmap(ctx);
    delete ctx;           // every other resource is released by its owner, the streams last (see lh_ctx)
    cudaGetLastError();   // a release that failed leaves no error behind for the caller's next CUDA call
    return LH_OK;
}

// =========================================================== ingest (device)
#define LH_ENTER(ctx)                                   \
    if (!(ctx)) return LH_ERR_INVALID;                  \
    RelaxedCapture _relaxed;                            \
    std::unique_lock<std::mutex> _lk((ctx)->mu);        \
    LH_CUDA((ctx), cudaSetDevice((ctx)->device))

namespace {
// A device (ids, values | amounts) pair of n entries: not NULL when n > 0, the 8-byte values or amounts 8-byte aligned
// and the ids naturally aligned, so that no kernel makes a misaligned load.
template <typename IdT>
lh_status check_pairs(lh_ctx *ctx, const IdT *ids, const void *vals, size_t n) {
    if (n && (!ids || !vals)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    if (((uintptr_t)vals & 7u) || ((uintptr_t)ids & (sizeof(IdT) - 1)))
        return fail(ctx, LH_ERR_INVALID, "values / amounts not 8-byte aligned or ids not naturally aligned");
    return LH_OK;
}
lh_status check_kind(lh_ctx *ctx, uint32_t kind) {
    if (kind != LH_VALUES_F64 && kind != LH_VALUES_I64NS) return fail(ctx, LH_ERR_INVALID, "unknown values kind");
    return LH_OK;
}

template <typename IdT, typename ValT>
lh_status ingest_keyed(lh_ctx *ctx, const IdT *d_ids, const ValT *d_vals, size_t n, void *stream) {
    if (lh_status st = check_pairs(ctx, d_ids, d_vals, n); st != LH_OK) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) { return launch_keyed<IdT, ValT>(ctx, b, d_ids, d_vals, n, s, IdIdentity{}); });
}
}  // namespace

extern "C" lh_status lh_ingest_f64(lh_ctx *ctx, uint32_t hid, const double *d_values, size_t n, void *stream) {
    LH_ENTER(ctx);
    if (n && !d_values) return fail(ctx, LH_ERR_INVALID, "d_values is NULL");
    if (n == 0) return LH_OK;
    if (hid >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram_id >= max_histograms");
    if (((uintptr_t)d_values & 7u) != 0) return fail(ctx, LH_ERR_INVALID, "d_values must be 8-byte aligned");
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) { return ingest_single(ctx, b, hid, d_values, n, s); });
}
extern "C" lh_status lh_ingest_keyed_f64_u16(lh_ctx *ctx, const uint16_t *d_ids, const double *d_values, size_t n, void *stream) {
    LH_ENTER(ctx);
    return ingest_keyed<unsigned short, double>(ctx, d_ids, d_values, n, stream);
}
extern "C" lh_status lh_ingest_keyed_f64_u32(lh_ctx *ctx, const uint32_t *d_ids, const double *d_values, size_t n, void *stream) {
    LH_ENTER(ctx);
    return ingest_keyed<unsigned int, double>(ctx, d_ids, d_values, n, stream);
}
extern "C" lh_status lh_ingest_keyed_i64ns_u16(lh_ctx *ctx, const uint16_t *d_ids, const int64_t *d_nanos, size_t n, void *stream) {
    LH_ENTER(ctx);
    return ingest_keyed<unsigned short, long long>(ctx, d_ids, reinterpret_cast<const long long *>(d_nanos), n, stream);
}
extern "C" lh_status lh_ingest_keyed_pair_u16(lh_ctx *ctx, const uint16_t *d_ids_f64, const double *d_values, size_t n_f64,
                                              const uint16_t *d_ids_ns, const int64_t *d_nanos, size_t n_ns, void *stream) {
    LH_ENTER(ctx);
    if (lh_status st = check_pairs(ctx, d_ids_f64, d_values, n_f64); st != LH_OK) return st;
    if (lh_status st = check_pairs(ctx, d_ids_ns, d_nanos, n_ns); st != LH_OK) return st;
    if (n_f64 == 0 && n_ns == 0) return LH_OK;
    cudaStream_t s = pick_stream(ctx, stream);
    const long long *nanos = reinterpret_cast<const long long *>(d_nanos);
    return write_bracket(ctx, s, [&](int b) {
        return launch_keyed_pair<unsigned short>(ctx, b, d_ids_f64, d_values, n_f64, d_ids_ns, nanos, n_ns, s);
    });
}
extern "C" lh_status lh_counter_add_u16(lh_ctx *ctx, const uint16_t *d_ids, const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    if (lh_status st = check_pairs(ctx, d_ids, d_amounts, n); st != LH_OK) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) { return add_counters<unsigned short>(ctx, b, ctx->C, d_ids, d_amounts, n, s, IdIdentity{}); });
}
extern "C" lh_status lh_counter_add_u32(lh_ctx *ctx, const uint32_t *d_ids, const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    if (lh_status st = check_pairs(ctx, d_ids, d_amounts, n); st != LH_OK) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) { return add_counters<unsigned int>(ctx, b, ctx->C, d_ids, d_amounts, n, s, IdIdentity{}); });
}
static_assert(LH_MAP_MAX == LH_MAP_MAX_IDS, "the header and the kernels agree on the map size");
namespace {
// The host map of a mapped call into the parameter block's form; LH_ERR_INVALID / LH_ERR_RANGE as the header says.
lh_status make_map(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, uint32_t limit, IdMap &m) {
    if (k > LH_MAP_MAX) return fail(ctx, LH_ERR_INVALID, "more than 4096 mapped ids");
    if (k && !h_map) return fail(ctx, LH_ERR_INVALID, "h_map is NULL");
    for (uint32_t i = 0; i < k; i++)
        if (h_map[i] != LH_GRAPH_UNBOUND && h_map[i] >= limit) return fail(ctx, LH_ERR_RANGE, "map entry >= max_histograms / max_counters");
    m.k = k;
    m.any_unbound = std::find(h_map, h_map + k, LH_GRAPH_UNBOUND) != h_map + k;
    std::copy(h_map, h_map + k, m.row);
    return LH_OK;
}

template <typename IdT>
lh_status ingest_keyed_mapped(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const IdT *d_ids, const void *d_values,
                              uint32_t kind, size_t n, void *stream) {
    if (lh_status st = check_kind(ctx, kind); st != LH_OK) return st;
    if (lh_status st = check_pairs(ctx, d_ids, d_values, n); st != LH_OK) return st;
    IdMap m;
    lh_status st = make_map(ctx, h_map, k, ctx->H, m);
    if (st != LH_OK || n == 0) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) {
        return kind == LH_VALUES_F64 ? launch_keyed<IdT, double>(ctx, b, d_ids, static_cast<const double *>(d_values), n, s, m)
                                     : launch_keyed<IdT, long long>(ctx, b, d_ids, static_cast<const long long *>(d_values), n, s, m);
    });
}

template <typename IdT>
lh_status counter_add_mapped(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const IdT *d_ids, const uint64_t *d_amounts,
                             size_t n, void *stream) {
    if (lh_status st = check_pairs(ctx, d_ids, d_amounts, n); st != LH_OK) return st;
    IdMap m;
    lh_status st = make_map(ctx, h_map, kc, ctx->C, m);
    if (st != LH_OK || n == 0) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) { return add_counters<IdT>(ctx, b, kc, d_ids, d_amounts, n, s, m); });
}
}  // namespace

extern "C" lh_status lh_ingest_keyed_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint16_t *d_ids,
                                                const void *d_values, uint32_t kind, size_t n, void *stream) {
    LH_ENTER(ctx);
    return ingest_keyed_mapped<unsigned short>(ctx, h_map, k, d_ids, d_values, kind, n, stream);
}
extern "C" lh_status lh_ingest_keyed_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t k, const uint32_t *d_ids,
                                                const void *d_values, uint32_t kind, size_t n, void *stream) {
    LH_ENTER(ctx);
    return ingest_keyed_mapped<unsigned int>(ctx, h_map, k, d_ids, d_values, kind, n, stream);
}
extern "C" lh_status lh_counter_add_mapped_u16(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint16_t *d_ids,
                                               const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    return counter_add_mapped<unsigned short>(ctx, h_map, kc, d_ids, d_amounts, n, stream);
}
extern "C" lh_status lh_counter_add_mapped_u32(lh_ctx *ctx, const uint32_t *h_map, uint32_t kc, const uint32_t *d_ids,
                                               const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    return counter_add_mapped<unsigned int>(ctx, h_map, kc, d_ids, d_amounts, n, stream);
}
extern "C" lh_status lh_ingest_batch(lh_ctx *ctx, const lh_batch_item *h_items, uint32_t n_items, void *stream) {
    LH_ENTER(ctx);
    unsigned long long n = 0;
    lh_status st = check_batch(ctx, h_items, n_items, ctx->H, &n);
    if (st != LH_OK || n == 0) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) {
        lh_status bs = launch_batch(ctx, buffer_target(ctx, b), h_items, n_items, s);
        if (bs == LH_OK) ctx->stats.samples += n;
        return bs;
    });
}

// =========================================================== ingest (host)
// Chunks of staging_bytes go through the slot ring: (memcpy into pinned if the
// source is pageable) -> async H2D -> kernel, all on the ingest stream.
namespace {
enum HostKind { HK_SINGLE, HK_KEYED_U16, HK_COUNTER_U16, HK_KEYED_I64_U16 };

// One staging step: copy n 8-byte items from h_a and, unless kind is HK_SINGLE, n uint16 ids from h_ids (to byte
// ids_off) into the device buffer of slot `sl`, then ingest them in one write bracket.  The copies run on their own
// stream so that chunk k+1's DMA overlaps chunk k's kernel; the bracket opens after the ingest stream has waited for
// them, so the kernel time excludes the copy.  Unless a copy fails, the slot is in flight afterwards.
lh_status staging_step(lh_ctx *ctx, Slot &sl, HostKind kind, uint32_t hid, const void *h_a, const void *h_ids, size_t n,
                       size_t ids_off) {
    cudaStream_t cs = ctx->copy_stream.get(), s = ctx->ingest_stream.get();
    lh_status st = LH_OK;
    if (n) {
        char *d_a = (char *)sl.d.get();
        const unsigned short *d_i = (const unsigned short *)(d_a + ids_off);
        // the device buffer is free again once the kernel that read it last is done (slot_wait_free already waited
        // on the host for a recycled slot, the event wait covers the rest)
        if (sl.seq) LH_CUDA(ctx, cudaStreamWaitEvent(cs, sl.done.get(), 0));
        LH_CUDA(ctx, cudaMemcpyAsync(d_a, h_a, n * 8, cudaMemcpyHostToDevice, cs));
        if (kind != HK_SINGLE) LH_CUDA(ctx, cudaMemcpyAsync(d_a + ids_off, h_ids, n * 2, cudaMemcpyHostToDevice, cs));
        LH_CUDA(ctx, cudaEventRecord(sl.copied.get(), cs));
        LH_CUDA(ctx, cudaStreamWaitEvent(s, sl.copied.get(), 0));
        ctx->stats.h2d_bytes += n * (kind == HK_SINGLE ? 8 : 10);
        st = write_bracket(ctx, s, [&](int b) {
            switch (kind) {
            case HK_SINGLE: return ingest_single(ctx, b, hid, (const double *)d_a, n, s);
            case HK_KEYED_U16: return launch_keyed<unsigned short, double>(ctx, b, d_i, (const double *)d_a, n, s, IdIdentity{});
            case HK_KEYED_I64_U16: return launch_keyed<unsigned short, long long>(ctx, b, d_i, (const long long *)d_a, n, s, IdIdentity{});
            default: return add_counters<unsigned short>(ctx, b, ctx->C, d_i, (const uint64_t *)d_a, n, s, IdIdentity{});   // HK_COUNTER_U16
            }
        });
    }
    LH_CUDA(ctx, cudaEventRecord(sl.done.get(), s));
    sl.state = SLOT_INFLIGHT;
    sl.seq = ++ctx->slot_seq;
    ctx->slot_cv.notify_all();
    return st;
}

lh_status ingest_host(lh_ctx *ctx, std::unique_lock<std::mutex> &lk, HostKind kind, uint32_t hid,
                      const void *h_a /* 8-byte items */, const uint16_t *h_ids, size_t n) {
    const bool pinned = is_pinned_or_managed(h_a) && (!h_ids || is_pinned_or_managed(h_ids));
    const size_t item = (kind == HK_SINGLE) ? 8 : 10;
    size_t per = ctx->staging_bytes / item;
    per &= ~(size_t)15;   // keeps the ids region 16-byte aligned
    if (per == 0) return fail(ctx, LH_ERR_INVALID, "staging_bytes too small");
    size_t done = 0;
    cudaEvent_t last_copied = nullptr;
    while (done < n) {
        size_t m = std::min(per, n - done);
        int si;
        lh_status st = slot_wait_free(ctx, lk, &si);
        if (st != LH_OK) return st;
        Slot &sl = ctx->slots[si];
        const void *src_a = (const char *)h_a + done * 8;
        const void *src_i = h_ids ? (const void *)(h_ids + done) : nullptr;
        if (!pinned) {
            // pageable source: stage through the slot's pinned buffer.  The memcpy (milliseconds per 32 MiB) runs with
            // the context mutex RELEASED -- the slot is parked as SLOT_FILLING so no other thread can take it.
            sl.state = SLOT_FILLING;
            lk.unlock();
            memcpy(sl.h.get(), src_a, m * 8);
            if (h_ids) memcpy((char *)sl.h.get() + per * 8, src_i, m * 2);
            lk.lock();
            src_a = sl.h.get();
            src_i = (char *)sl.h.get() + per * 8;
        }
        st = staging_step(ctx, sl, kind, hid, src_a, src_i, m, per * 8);
        if (st != LH_OK) return st;
        last_copied = sl.copied.get();
        done += m;
    }
    if (pinned && last_copied) {
        // the caller may reuse its buffers on return: the async copies must have READ them (the kernels may still run);
        // waited for with the mutex released
        lk.unlock();
        cudaError_t e = cudaEventSynchronize(last_copied);
        lk.lock();
        if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "cudaEventSynchronize(copied)", e);
    }
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_ingest_f64_host(lh_ctx *ctx, uint32_t hid, const double *h_values, size_t n) {
    LH_ENTER(ctx);
    if (n && !h_values) return fail(ctx, LH_ERR_INVALID, "h_values is NULL");
    if (hid >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram_id >= max_histograms");
    return ingest_host(ctx, _lk, HK_SINGLE, hid, h_values, nullptr, n);
}
extern "C" lh_status lh_ingest_keyed_f64_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const double *h_values, size_t n) {
    LH_ENTER(ctx);
    if (n && (!h_ids || !h_values)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    return ingest_host(ctx, _lk, HK_KEYED_U16, 0, h_values, h_ids, n);
}
extern "C" lh_status lh_ingest_keyed_i64ns_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const int64_t *h_nanos, size_t n) {
    LH_ENTER(ctx);
    if (n && (!h_ids || !h_nanos)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    return ingest_host(ctx, _lk, HK_KEYED_I64_U16, 0, h_nanos, h_ids, n);
}
extern "C" lh_status lh_counter_add_u16_host(lh_ctx *ctx, const uint16_t *h_ids, const uint64_t *h_amounts, size_t n) {
    LH_ENTER(ctx);
    if (n && (!h_ids || !h_amounts)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    return ingest_host(ctx, _lk, HK_COUNTER_U16, 0, h_amounts, h_ids, n);
}

// Merge sparse bucket counts held in host memory (e.g. another process's lh_snapshot_export) into the ACTIVE arrays.
extern "C" lh_status lh_merge_counts_host(lh_ctx *ctx, const uint32_t *h_ids, const int16_t *h_keys, const uint64_t *h_counts, size_t n) {
    LH_ENTER(ctx);
    if (n && (!h_ids || !h_keys || !h_counts)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    if (!n) return LH_OK;
    cudaStream_t s = ctx->ingest_stream.get();
    const int b = ctx->active;
    lh_status st = before_write(ctx, b, s);
    if (st != LH_OK) return st;
    AsyncPtr buf(s);
    const size_t off_keys = n * 4, off_counts = ((n * 6 + 7) / 8) * 8, total = off_counts + n * 8;
    LH_CUDA(ctx, cudaMallocAsync((void **)buf.out(), total, s));
    char *d = buf.get();
    cudaError_t e = cudaMemcpyAsync(d, h_ids, n * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + off_keys, h_keys, n * 2, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + off_counts, h_counts, n * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        int grid = grid_1d(ctx, n, 256, 1, 8);
        k_merge_sparse<<<grid, 256, 0, s>>>((const uint32_t *)d, (const short *)(d + off_keys), (const unsigned long long *)(d + off_counts),
                                            n, ctx->H, ctx->buf[b].d_buckets.get(), ctx->buf[b].d_flags.get(), ctx->d_dropped.get(), ctx->pc.win);
        e = cudaGetLastError();
    }
    buf.reset();
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_merge_counts_host", e);
    ctx->stats.kernel_launches++;
    ctx->stats.h2d_bytes += n * 14;
    LH_CUDA(ctx, cudaStreamSynchronize(s));   // the host arrays may be pageable: they have been read by now
    return after_write(ctx, b, s);
}

// =========================================================== staging ring
extern "C" lh_status lh_staging_acquire(lh_ctx *ctx, lh_staging *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    int si;
    lh_status st = slot_wait_free(ctx, _lk, &si);
    if (st != LH_OK) return st;
    ctx->slots[si].state = SLOT_ACQUIRED;
    out->host = ctx->slots[si].h.get();
    out->bytes = ctx->staging_bytes;
    out->slot = (uint32_t)si;
    out->reserved = 0;
    return LH_OK;
}

namespace {
lh_status staging_commit(lh_ctx *ctx, const lh_staging *sg, HostKind kind, uint32_t hid, size_t n, uint64_t ids_offset) {
    if (!sg || sg->slot >= ctx->slots.size()) return fail(ctx, LH_ERR_INVALID, "bad staging handle");
    Slot &sl = ctx->slots[sg->slot];
    if (sl.state != SLOT_ACQUIRED) return fail(ctx, LH_ERR_STATE, "staging slot was not acquired");
    const size_t item_bytes = n * 8;
    if (kind == HK_SINGLE) {
        if (item_bytes > ctx->staging_bytes) return fail(ctx, LH_ERR_RANGE, "n exceeds the staging slot");
    } else {
        if ((ids_offset & 15u) || ids_offset < item_bytes || ids_offset + n * 2 > ctx->staging_bytes)
            return fail(ctx, LH_ERR_RANGE, "ids_offset / n do not fit the staging slot");
    }
    return staging_step(ctx, sl, kind, hid, sl.h.get(), (char *)sl.h.get() + ids_offset, n, ids_offset);
}
}  // namespace

extern "C" lh_status lh_staging_commit_f64(lh_ctx *ctx, const lh_staging *s, uint32_t hid, size_t n) {
    LH_ENTER(ctx);
    if (hid >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram_id >= max_histograms");
    return staging_commit(ctx, s, HK_SINGLE, hid, n, 0);
}
extern "C" lh_status lh_staging_commit_keyed_f64_u16(lh_ctx *ctx, const lh_staging *s, size_t n, uint64_t ids_offset) {
    LH_ENTER(ctx);
    return staging_commit(ctx, s, HK_KEYED_U16, 0, n, ids_offset);
}
extern "C" lh_status lh_staging_commit_counter_u16(lh_ctx *ctx, const lh_staging *s, size_t n, uint64_t ids_offset) {
    LH_ENTER(ctx);
    return staging_commit(ctx, s, HK_COUNTER_U16, 0, n, ids_offset);
}
extern "C" lh_status lh_staging_abandon(lh_ctx *ctx, const lh_staging *s) {
    LH_ENTER(ctx);
    if (!s || s->slot >= ctx->slots.size()) return fail(ctx, LH_ERR_INVALID, "bad staging handle");
    if (ctx->slots[s->slot].state != SLOT_ACQUIRED) return fail(ctx, LH_ERR_STATE, "staging slot was not acquired");
    ctx->slots[s->slot].state = SLOT_FREE;
    ctx->slot_cv.notify_all();
    return LH_OK;
}

// =========================================================== record scopes
extern "C" lh_status lh_record_begin(lh_ctx *ctx, void *stream, lh_recorder *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    cudaStream_t s = pick_stream(ctx, stream);
    const int b = ctx->active;
    lh_status st = before_write(ctx, b, s);
    if (st != LH_OK) return st;
    *out = buffer_target(ctx, b);
    out->block_smem_bytes = subhist_words(ctx->pc.win) * 4u;
    out->scope = ctx->next_scope++;
    ctx->scopes.push_back(Scope{out->scope, b, s, std::this_thread::get_id()});
    return LH_OK;
}

extern "C" lh_status lh_record_end(lh_ctx *ctx, const lh_recorder *rec) {
    LH_ENTER(ctx);
    if (!rec) return fail(ctx, LH_ERR_INVALID, "rec is NULL");
    for (size_t i = 0; i < ctx->scopes.size(); i++) {
        if (ctx->scopes[i].ticket != rec->scope) continue;
        const Scope sc = ctx->scopes[i];
        ctx->scopes.erase(ctx->scopes.begin() + (long)i);
        ctx->scope_cv.notify_all();
        return after_write(ctx, sc.buf, sc.stream);
    }
    return fail(ctx, LH_ERR_INVALID, "unknown or already ended record scope");
}

// =========================================================== graph recorders
namespace {
// handle = context tag (16 bits) | serial (48 bits)
uint64_t graph_handle(const lh_ctx *ctx, uint64_t serial) {
    return (ctx->ctx_id % 0xFFFFu + 1u) << 48 | (serial & 0xFFFFFFFFFFFFull);
}

// the live recorder a handle names (its rows must match too), or nullptr
GraphRec *graph_of(lh_ctx *ctx, const lh_graph_recorder *g) {
    if (!g) return nullptr;
    for (auto &gr : ctx->graphs)
        if (gr.handle == g->handle && gr.rec.d_buckets == g->rec.d_buckets) return &gr;
    return nullptr;
}

// target ids: each < limit or LH_GRAPH_UNBOUND
bool ids_ok(const uint32_t *ids, uint32_t n, uint32_t limit) {
    for (uint32_t i = 0; ids && i < n; i++)
        if (ids[i] >= limit && ids[i] != LH_GRAPH_UNBOUND) return false;
    return true;
}
}  // namespace

extern "C" lh_status lh_graph_recorder_create(lh_ctx *ctx, uint32_t k, uint32_t kc, const uint32_t *hist_ids,
                                              const uint32_t *counter_ids, lh_graph_recorder *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    if (k == 0 && kc == 0) return fail(ctx, LH_ERR_INVALID, "a graph recorder needs a histogram or a counter");
    if (k > ctx->H || kc > ctx->C) return fail(ctx, LH_ERR_RANGE, "more rows than max_histograms / max_counters");
    if (!ids_ok(hist_ids, k, ctx->H) || !ids_ok(counter_ids, kc, ctx->C))
        return fail(ctx, LH_ERR_RANGE, "target id >= max_histograms / max_counters");
    if (!ctx->graph_drained.get()) LH_CUDA(ctx, cudaEventCreateWithFlags(ctx->graph_drained.out(), cudaEventDisableTiming));
    // one allocation: rows [k][65536], counters [kc], timer marks [k], flags [k]
    const size_t row_bytes = (size_t)k * 65536u * 8u, mark_off = row_bytes + (size_t)kc * 8u, flag_off = mark_off + (size_t)k * 8u;
    const size_t bytes = flag_off + (size_t)k * 4u;
    cudaStream_t s = ctx->snap_stream.get();
    AsyncPtr mem(s);
    LH_CUDA(ctx, cudaMallocAsync((void **)mem.out(), bytes, s));
    char *base = mem.get();
    cudaError_t e = cudaMemsetAsync(base, 0, bytes, s);
    static_assert(kTimerNeverStarted == ~0ull, "marks are set bytewise");
    if (e == cudaSuccess) e = cudaMemsetAsync(base + mark_off, 0xFF, (size_t)k * 8u, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_graph_recorder_create", e);
    GraphRec gr;
    gr.mem = std::move(mem);
    gr.handle = graph_handle(ctx, ctx->next_graph++);
    memset(&gr.rec, 0, sizeof gr.rec);
    gr.rec.d_buckets = reinterpret_cast<uint64_t *>(base);
    gr.rec.d_counters = reinterpret_cast<uint64_t *>(base + row_bytes);
    gr.rec.d_flags = reinterpret_cast<uint32_t *>(base + flag_off);
    gr.d_marks = reinterpret_cast<unsigned long long *>(base + mark_off);
    gr.rec.d_dropped = reinterpret_cast<uint64_t *>(ctx->d_dropped.get());
    gr.rec.max_histograms = k;
    gr.rec.max_counters = kc;
    gr.rec.block_smem_bytes = subhist_words(ctx->pc.win) * 4u;
    gr.rec.scope = 0;   // never a scope ticket: lh_record_end refuses it
    memcpy(gr.rec.prec, &ctx->pc, sizeof ctx->pc);
    gr.hid.assign(k, LH_GRAPH_UNBOUND);
    gr.cid.assign(kc, LH_GRAPH_UNBOUND);
    if (hist_ids) gr.hid.assign(hist_ids, hist_ids + k);
    if (counter_ids) gr.cid.assign(counter_ids, counter_ids + kc);
    out->handle = gr.handle;
    out->rec = gr.rec;
    ctx->graphs.push_back(std::move(gr));
    return LH_OK;
}

extern "C" lh_status lh_graph_recorder_bind(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *hist_ids,
                                            const uint32_t *counter_ids) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    if (!ids_ok(hist_ids, gr->rec.max_histograms, ctx->H) || !ids_ok(counter_ids, gr->rec.max_counters, ctx->C))
        return fail(ctx, LH_ERR_RANGE, "target id >= max_histograms / max_counters");
    if (hist_ids) gr->hid.assign(hist_ids, hist_ids + gr->rec.max_histograms);
    if (counter_ids) gr->cid.assign(counter_ids, counter_ids + gr->rec.max_counters);
    return LH_OK;
}

extern "C" lh_status lh_graph_recorder_ingest(lh_ctx *ctx, const lh_graph_recorder *g, const lh_batch_item *h_items,
                                              uint32_t n_items, void *stream) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    unsigned long long n = 0;
    lh_status st = check_batch(ctx, h_items, n_items, gr->rec.max_histograms, &n);
    if (st != LH_OK || n == 0) return st;
    return launch_batch(ctx, gr->rec, h_items, n_items, pick_stream(ctx, stream));
}

namespace {
template <typename IdT>
lh_status graph_keyed(lh_ctx *ctx, const lh_graph_recorder *g, const IdT *d_ids, const void *d_values, uint32_t kind, size_t n,
                      void *stream) {
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    if (lh_status st = check_kind(ctx, kind); st != LH_OK) return st;
    if (lh_status st = check_pairs(ctx, d_ids, d_values, n); st != LH_OK) return st;
    if (n == 0) return LH_OK;
    return launch_keyed_graph<IdT>(ctx, gr->rec, d_ids, static_cast<const unsigned long long *>(d_values), n,
                                   kind == LH_VALUES_I64NS, pick_stream(ctx, stream));
}

template <typename IdT>
lh_status graph_counters(lh_ctx *ctx, const lh_graph_recorder *g, const IdT *d_ids, const uint64_t *d_amounts, size_t n,
                         void *stream) {
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    if (lh_status st = check_pairs(ctx, d_ids, d_amounts, n); st != LH_OK) return st;
    if (n == 0) return LH_OK;
    return launch_counter<IdT>(ctx, reinterpret_cast<unsigned long long *>(gr->rec.d_counters), gr->rec.max_counters, d_ids,
                               d_amounts, n, pick_stream(ctx, stream), IdIdentity{});
}
}  // namespace

extern "C" lh_status lh_graph_recorder_ingest_keyed_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                        const void *d_values, uint32_t kind, size_t n, void *stream) {
    LH_ENTER(ctx);
    return graph_keyed<unsigned short>(ctx, g, d_ids, d_values, kind, n, stream);
}
extern "C" lh_status lh_graph_recorder_ingest_keyed_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                        const void *d_values, uint32_t kind, size_t n, void *stream) {
    LH_ENTER(ctx);
    return graph_keyed<unsigned int>(ctx, g, d_ids, d_values, kind, n, stream);
}
extern "C" lh_status lh_graph_recorder_counter_add_u16(lh_ctx *ctx, const lh_graph_recorder *g, const uint16_t *d_ids,
                                                       const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    return graph_counters<unsigned short>(ctx, g, d_ids, d_amounts, n, stream);
}
extern "C" lh_status lh_graph_recorder_counter_add_u32(lh_ctx *ctx, const lh_graph_recorder *g, const uint32_t *d_ids,
                                                       const uint64_t *d_amounts, size_t n, void *stream) {
    LH_ENTER(ctx);
    return graph_counters<unsigned int>(ctx, g, d_ids, d_amounts, n, stream);
}

// A span of the recorder's local histogram: the start writes the row's mark, the stop records now - mark into the row.
// No event or host state, so both may be captured; the caller orders them (see the header).
extern "C" lh_status lh_graph_recorder_timer_start(lh_ctx *ctx, const lh_graph_recorder *g, uint32_t histogram, void *stream) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    if (histogram >= gr->rec.max_histograms) return fail(ctx, LH_ERR_RANGE, "histogram >= the recorder's histograms");
    k_gpu_timer_mark<<<1, 1, 0, pick_stream(ctx, stream)>>>(gr->d_marks + histogram);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return LH_OK;
}

extern "C" lh_status lh_graph_recorder_timer_stop(lh_ctx *ctx, const lh_graph_recorder *g, uint32_t histogram, void *stream,
                                                  int64_t *d_duration_ns) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    if (histogram >= gr->rec.max_histograms) return fail(ctx, LH_ERR_RANGE, "histogram >= the recorder's histograms");
    if (((uintptr_t)d_duration_ns & 7u) != 0) return fail(ctx, LH_ERR_INVALID, "d_duration_ns must be 8-byte aligned");
    k_gpu_timer_stop<<<1, 1, 0, pick_stream(ctx, stream)>>>(
        gr->d_marks + histogram, reinterpret_cast<unsigned long long *>(gr->rec.d_buckets) + (size_t)histogram * 65536u,
        gr->rec.d_flags + histogram, reinterpret_cast<long long *>(d_duration_ns), ctx->d_dropped.get(), ctx->pc);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return LH_OK;
}

extern "C" lh_status lh_graph_recorder_destroy(lh_ctx *ctx, const lh_graph_recorder *g, void *stream) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    cudaStream_t s = pick_stream(ctx, stream);
    // after every collection drain issued so far, then the final drain, then the free: all stream-ordered on s
    LH_CUDA(ctx, cudaStreamWaitEvent(s, ctx->graph_drained.get(), 0));
    lh_status st = write_bracket(ctx, s, [&](int b) { return drain_graphs(ctx, gr, 1, b, s); });
    if (st != LH_OK) return st;
    LH_CUDA(ctx, gr->mem.reset(s));
    ctx->graphs.erase(ctx->graphs.begin() + (gr - ctx->graphs.data()));
    return LH_OK;
}

// =========================================================== GPU timers
namespace {
// handle = context tag (16 bits) | generation (28 bits) | slot (20 bits)
constexpr int kTimerSlotBits = 20, kTimerGenBits = 28;

uint64_t timer_handle(const lh_ctx *ctx, uint32_t slot, uint32_t gen) {
    const uint64_t tag = ctx->ctx_id % 0xFFFFu + 1u;   // 1 ... 65535, so no handle is 0
    return tag << (kTimerSlotBits + kTimerGenBits) | (uint64_t)(gen & ((1u << kTimerGenBits) - 1u)) << kTimerSlotBits | slot;
}

// the held slot a handle names, or nullptr for a released, stale, foreign or malformed handle
TimerSlot *timer_slot(lh_ctx *ctx, const lh_gpu_timer *t) {
    if (!t) return nullptr;
    const uint32_t k = (uint32_t)(t->handle & ((1u << kTimerSlotBits) - 1u));
    if (k >= ctx->timer_slots.size()) return nullptr;
    TimerSlot &ts = ctx->timer_slots[k];
    if (ts.state != TIMER_HELD || t->handle != timer_handle(ctx, k, ts.gen)) return nullptr;
    return &ts;
}

// A mark enqueued during capture would run only at replay, against a slot that may belong to another token by then.
lh_status refuse_capture(lh_ctx *ctx, cudaStream_t s) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    LH_CUDA(ctx, cudaStreamIsCapturing(s, &cs));
    if (cs != cudaStreamCaptureStatusNone) return fail(ctx, LH_ERR_STATE, "GPU timers cannot be captured into a CUDA graph");
    return LH_OK;
}

// every kernel that read or wrote the slot has completed (queried, never waited for)
bool timer_slot_idle(const TimerSlot &ts) {
    bool idle = cudaEventQuery(ts.started.get()) == cudaSuccess;
    for (const auto &w : ts.stops) idle = idle && cudaEventQuery(w.ev.get()) == cudaSuccess;
    cudaGetLastError();   // cudaErrorNotReady is not an error
    return idle;
}

// A slot for a new token: the oldest released slot if its kernels are done, else a fresh one, else any released slot
// whose kernels are done.
lh_status timer_take(lh_ctx *ctx, uint32_t *out) {
    if (!ctx->d_timer_marks.get()) {
        DevPtr<unsigned long long> marks;
        LH_CUDA(ctx, cudaMalloc(marks.out(), (size_t)ctx->timer_slots_n * sizeof(unsigned long long)));
        ctx->timer_slots.resize(ctx->timer_slots_n);
        ctx->d_timer_marks = std::move(marks);
    }
    const bool fresh = ctx->timer_fresh < ctx->timer_slots_n;
    const size_t scan = fresh ? std::min<size_t>(1, ctx->timer_released.size()) : ctx->timer_released.size();
    for (size_t i = 0; i < scan; i++) {
        const uint32_t k = ctx->timer_released[i];
        TimerSlot &ts = ctx->timer_slots[k];
        if (!timer_slot_idle(ts)) continue;
        ctx->timer_released.erase(ctx->timer_released.begin() + (long)i);
        for (auto &w : ts.stops) ctx->timer_spare_events.push_back(std::move(w.ev));
        ts.stops.clear();
        *out = k;
        return LH_OK;
    }
    if (fresh) { *out = ctx->timer_fresh++; return LH_OK; }
    return fail(ctx, LH_ERR_RANGE, "every GPU timer slot is held or still in use on the device");
}
}  // namespace

extern "C" lh_status lh_gpu_timer_start(lh_ctx *ctx, void *stream, lh_gpu_timer *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    cudaStream_t s = pick_stream(ctx, stream);
    lh_status st = refuse_capture(ctx, s);
    if (st != LH_OK) return st;
    uint32_t k = 0;
    st = timer_take(ctx, &k);
    if (st != LH_OK) return st;
    TimerSlot &ts = ctx->timer_slots[k];
    cudaError_t e = ts.started.get() ? cudaSuccess : cudaEventCreateWithFlags(ts.started.out(), cudaEventDisableTiming);
    if (e == cudaSuccess) {
        k_gpu_timer_mark<<<1, 1, 0, s>>>(ctx->d_timer_marks.get() + k);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(ts.started.get(), s);
    if (e != cudaSuccess) {   // back to the pool, behind whatever may have been enqueued
        ts.state = TIMER_RELEASED;
        ctx->timer_released.push_back(k);
        return fail(ctx, LH_ERR_CUDA, "lh_gpu_timer_start", e);
    }
    ctx->stats.kernel_launches++;
    ts.state = TIMER_HELD;
    ts.start_stream = s;
    out->handle = timer_handle(ctx, k, ts.gen);
    return LH_OK;
}

extern "C" lh_status lh_gpu_timer_stop(lh_ctx *ctx, const lh_gpu_timer *t, uint32_t hid, void *stream, int64_t *d_out) {
    LH_ENTER(ctx);
    cudaStream_t s = pick_stream(ctx, stream);
    lh_status st = refuse_capture(ctx, s);
    if (st != LH_OK) return st;
    if (hid >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram_id >= max_histograms");
    TimerSlot *ts = timer_slot(ctx, t);
    if (!ts) return fail(ctx, LH_ERR_INVALID, "released, stale or foreign GPU timer handle");
    if (((uintptr_t)d_out & 7u) != 0) return fail(ctx, LH_ERR_INVALID, "d_duration_ns must be 8-byte aligned");
    if (s != ts->start_stream) LH_CUDA(ctx, cudaStreamWaitEvent(s, ts->started.get(), 0));
    const unsigned long long *mark = ctx->d_timer_marks.get() + (ts - ctx->timer_slots.data());
    st = write_bracket(ctx, s, [&](int b) -> lh_status {
        k_gpu_timer_stop<<<1, 1, 0, s>>>(mark, ctx->buf[b].d_buckets.get() + (size_t)hid * 65536u, ctx->buf[b].d_flags.get() + hid,
                                         reinterpret_cast<long long *>(d_out), ctx->d_dropped.get(), ctx->pc);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        ctx->stats.samples++;
        return LH_OK;
    });
    if (st != LH_OK) return st;
    // the slot is not handed out again before this stop has run (one event per stream that stopped the token)
    for (auto &w : ts->stops)
        if (w.stream == s) { LH_CUDA(ctx, cudaEventRecord(w.ev.get(), s)); return LH_OK; }
    WriterEvent w{s, {}};
    if (!ctx->timer_spare_events.empty()) {
        w.ev = std::move(ctx->timer_spare_events.back());
        ctx->timer_spare_events.pop_back();
    } else {
        LH_CUDA(ctx, cudaEventCreateWithFlags(w.ev.out(), cudaEventDisableTiming));
    }
    ts->stops.push_back(std::move(w));
    LH_CUDA(ctx, cudaEventRecord(ts->stops.back().ev.get(), s));
    return LH_OK;
}

extern "C" lh_status lh_gpu_timer_release(lh_ctx *ctx, const lh_gpu_timer *t) {
    LH_ENTER(ctx);
    TimerSlot *ts = timer_slot(ctx, t);
    if (!ts) return fail(ctx, LH_ERR_INVALID, "released, stale or foreign GPU timer handle");
    ts->state = TIMER_RELEASED;
    ts->gen++;
    ctx->timer_released.push_back((uint32_t)(ts - ctx->timer_slots.data()));
    return LH_OK;
}

// =========================================================== snapshot
extern "C" lh_status lh_snapshot_begin(lh_ctx *ctx) {
    LH_ENTER(ctx);
    if (ctx->frozen) return fail(ctx, LH_ERR_STATE, "previous snapshot not ended");
    if (ctx->freezing) return fail(ctx, LH_ERR_STATE, "another snapshot is waiting for record scopes");
    const int f = ctx->active;
    if (!ctx->scopes.empty()) {
        // device code is still writing the interval: make the spare arrays active first, so that scopes and ingest
        // calls from now on go to the next interval and cannot starve this one, then wait (mutex released) until
        // every scope on the buffer being frozen has ended.  Every open scope is on `f`: a scope on the other buffer
        // would have been waited for by the snapshot that froze it.
        const std::thread::id me = std::this_thread::get_id();
        for (const Scope &sc : ctx->scopes)
            if (sc.thread == me) return fail(ctx, LH_ERR_STATE, "lh_snapshot_begin from a thread that holds an open record scope");
        ctx->active ^= 1;
        ctx->freezing = true;
        ctx->scope_cv.wait(_lk, [&] {
            for (const Scope &sc : ctx->scopes)
                if (sc.buf == f) return false;
            return true;
        });
        ctx->freezing = false;
    }
    // order the snapshot stream after every ingest launch that wrote the buffer being frozen
    for (auto &w : ctx->buf[f].writers) LH_CUDA(ctx, cudaStreamWaitEvent(ctx->snap_stream.get(), w.ev.get(), 0));
    if (!ctx->graphs.empty()) {   // what graph recorders hold so far joins the interval being frozen
        lh_status st = drain_graphs(ctx, ctx->graphs.data(), ctx->graphs.size(), f, ctx->snap_stream.get());
        if (st != LH_OK) return st;
        LH_CUDA(ctx, cudaEventRecord(ctx->graph_drained.get(), ctx->snap_stream.get()));
    }
    if (ctx->buf[f].hot_pending) {   // drain the keyed path's uint32 window into the uint64 buckets
        lh_status st = fold_hot(ctx, f, ctx->snap_stream.get());
        if (st != LH_OK) return st;
    }
    ctx->active = f ^ 1;
    ctx->frozen = true;
    ctx->rows_read = false;
    ctx->pub_slot = -1;
    ctx->nnz_valid = false;
    ctx->view_reduced = false;
    ctx->view_counters_reduced = false;
    ctx->rows_packed = false;
    ctx->stats.snapshots++;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_device(lh_ctx *ctx, lh_device_view *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    mark_rows_read(ctx);   // the caller may read the rows from here on
    const int f = ctx->active ^ 1;
    out->d_buckets = reinterpret_cast<uint64_t *>(ctx->buf[f].d_buckets.get());
    out->d_counters = reinterpret_cast<uint64_t *>(ctx->buf[f].d_counters.get());
    out->n_bucket_words = (uint64_t)ctx->H * 65536u;
    out->n_counter_words = ctx->C;
    out->stream = ctx->snap_stream.get();
    out->d_flags = ctx->buf[f].d_flags.get();
    out->n_flag_words = ctx->H;
    return LH_OK;
}

namespace {
struct ResLayout { size_t count, sum, avg, pvals, pkeys, total; };
ResLayout res_layout(size_t H, uint32_t np) {
    ResLayout l;
    l.count = 0; l.sum = H * 8; l.avg = H * 16; l.pvals = H * 24; l.pkeys = H * 24 + H * np * 8;
    l.total = l.pkeys + H * np * 4;
    return l;
}

// the arrays the open snapshot's reduction / export read: this rank's frozen buffer, or the sums over all ranks
// once lh_snapshot_allreduce has run
struct View { const unsigned long long *buckets; const uint32_t *flags; const unsigned long long *counters; };
View snapshot_view(lh_ctx *ctx) {
    const int f = ctx->active ^ 1;
    View v;
    v.buckets = ctx->view_reduced ? ctx->d_red_buckets.get() : ctx->buf[f].d_buckets.get();
    v.flags = ctx->view_reduced ? ctx->d_red_flags.get() : ctx->buf[f].d_flags.get();
    v.counters = ctx->view_counters_reduced ? ctx->d_red_counters.get() : ctx->buf[f].d_counters.get();
    return v;
}

// K3 takes the shared-memory window path when the 2*win-1 cells fit comfortably (two CTAs per SM); the dense path
// otherwise (0 cells)
uint32_t k3_smem_cells(uint32_t win) {
    const size_t cells = (size_t)2 * win - 1;
    return cells * 8 <= (size_t)100 * 1024 ? (uint32_t)cells : 0u;
}

// enqueue K3 + one packed D2H for the open snapshot into result slot `slot`
lh_status enqueue_reduce(lh_ctx *ctx, const double *ps, uint32_t np, int slot) {
    mark_rows_read(ctx);
    cudaStream_t s = ctx->snap_stream.get();
    const ResLayout l = res_layout(ctx->H, np);
    const View v = snapshot_view(ctx);
    if (np) {
        LH_CUDA(ctx, cudaMemcpyAsync(ctx->d_ps[slot].get(), ps, np * sizeof(double), cudaMemcpyHostToDevice, s));
    }
    char *d = ctx->d_res[slot].get();
    const uint32_t smem_cells = k3_smem_cells(ctx->pc.win);
    k_reduce<<<ctx->H, K3_THREADS, (size_t)smem_cells * 8, s>>>(v.buckets, v.flags, ctx->pc.win, ctx->d_decomp.get(), ctx->d_ps[slot].get(), (int)np,
                                           (unsigned long long *)(d + l.count), (double *)(d + l.sum), (double *)(d + l.avg),
                                           (int *)(d + l.pkeys), (double *)(d + l.pvals), ctx->d_nnz.get() + (size_t)slot * ctx->H,
                                           smem_cells);
    LH_CUDA(ctx, cudaGetLastError());
    LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_res[slot].get(), d, l.total, cudaMemcpyDeviceToHost, s));
    LH_CUDA(ctx, cudaEventRecord(ctx->res_done[slot].get(), s));
    ctx->stats.kernel_launches++;
    ctx->stats.d2h_bytes += l.total;
    ctx->nnz_valid = true;
    ctx->nnz_slot = slot;
    ctx->res_np[slot] = np;
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_snapshot_reduce_async(lh_ctx *ctx, const double *percentiles, uint32_t np, uint64_t *ticket) {
    LH_ENTER(ctx);
    if (!ticket) return fail(ctx, LH_ERR_INVALID, "ticket is NULL");
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (np > LH_MAX_PERCENTILES || (np && !percentiles)) return fail(ctx, LH_ERR_INVALID, "bad percentile array");
    const uint64_t t = ctx->next_ticket++;
    const int slot = (int)(t & 1);
    // the slot's previous results (ticket t-2) are overwritten: make sure its copy is not still in flight
    // (waited for with the mutex released: ingest threads are not held up)
    if (ctx->res_ticket[slot]) {
        cudaEvent_t ev = ctx->res_done[slot].get();
        _lk.unlock();
        cudaError_t e = cudaEventSynchronize(ev);
        _lk.lock();
        if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "cudaEventSynchronize(result slot)", e);
        if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "snapshot ended while waiting");
    }
    lh_status st = enqueue_reduce(ctx, percentiles, np, slot);
    if (st != LH_OK) return st;
    ctx->pub_slot = slot;
    ctx->res_ticket[slot] = t;
    *ticket = t;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_result(lh_ctx *ctx, uint64_t ticket, uint64_t *counts, double *sums, double *avgs,
                                        int32_t *pkeys, double *pvals) {
    if (!ctx) return LH_ERR_INVALID;
    RelaxedCapture relaxed;
    const int slot = (int)(ticket & 1);
    cudaEvent_t ev;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ticket == 0 || ctx->res_ticket[slot] != ticket) return fail(ctx, LH_ERR_STATE, "ticket expired or unknown");
        ev = ctx->res_done[slot].get();
    }
    // wait outside the lock so ingest threads are not held up by the reaper
    cudaError_t e = cudaEventSynchronize(ev);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "cudaEventSynchronize(result)", e);
    if (ctx->res_ticket[slot] != ticket) return fail(ctx, LH_ERR_STATE, "ticket expired while waiting");
    const size_t H = ctx->H;
    const uint32_t np = ctx->res_np[slot];
    const ResLayout l = res_layout(H, np);
    const char *h = ctx->h_res[slot].get();
    if (counts) memcpy(counts, h + l.count, H * 8);
    if (sums) memcpy(sums, h + l.sum, H * 8);
    if (avgs) memcpy(avgs, h + l.avg, H * 8);
    if (pvals && np) memcpy(pvals, h + l.pvals, H * np * 8);
    if (pkeys && np) memcpy(pkeys, h + l.pkeys, H * np * 4);
    return LH_OK;
}

extern "C" lh_status lh_snapshot_reduce(lh_ctx *ctx, const double *percentiles, uint32_t np, uint64_t *counts,
                                        double *sums, double *avgs, int32_t *pkeys, double *pvals) {
    uint64_t t = 0;
    lh_status st = lh_snapshot_reduce_async(ctx, percentiles, np, &t);
    if (st != LH_OK) return st;
    return lh_snapshot_result(ctx, t, counts, sums, avgs, pkeys, pvals);
}

extern "C" lh_status lh_snapshot_export(lh_ctx *ctx, lh_sparse *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    mark_rows_read(ctx);
    cudaStream_t s = ctx->snap_stream.get();
    const View v = snapshot_view(ctx);
    if (!ctx->nnz_valid) {
        // non-empty bucket counts come out of K3: run it with no percentiles into the scratch result slot, which never
        // carries a ticket (outstanding lh_snapshot_reduce_async tickets keep their documented lifetime)
        lh_status st = enqueue_reduce(ctx, nullptr, 0, 2);
        if (st != LH_OK) return st;
    }
    k_scan_nnz<<<1, 1024, 0, s>>>(ctx->d_nnz.get() + (size_t)ctx->nnz_slot * ctx->H, ctx->H, ctx->d_offsets.get());
    LH_CUDA(ctx, cudaGetLastError());
    LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_offsets.get(), ctx->d_offsets.get(), ((size_t)ctx->H + 1) * 4, cudaMemcpyDeviceToHost, s));
    LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_counter_deltas.get(), v.counters, (size_t)ctx->C * 8, cudaMemcpyDeviceToHost, s));
    LH_CUDA(ctx, cudaStreamSynchronize(s));
    const size_t total = ctx->h_offsets.get()[ctx->H];
    if (total > ctx->x_cap) {
        size_t cap = std::max<size_t>(total, 4096) * 2;
        ctx->d_x_keys.reset(); ctx->d_x_counts.reset(); ctx->h_x_keys.reset(); ctx->h_x_counts.reset(); ctx->x_cap = 0;
        DevPtr<short> d_keys; DevPtr<unsigned long long> d_counts; PinnedPtr<short> h_keys; PinnedPtr<unsigned long long> h_counts;
        LH_CUDA(ctx, cudaMalloc(d_keys.out(), cap * 2));
        LH_CUDA(ctx, cudaMalloc(d_counts.out(), cap * 8));
        LH_CUDA(ctx, cudaMallocHost(h_keys.out(), cap * 2));
        LH_CUDA(ctx, cudaMallocHost(h_counts.out(), cap * 8));
        ctx->d_x_keys = std::move(d_keys); ctx->d_x_counts = std::move(d_counts); ctx->x_cap = cap;
        ctx->h_x_keys = std::move(h_keys); ctx->h_x_counts = std::move(h_counts);
    }
    if (total) {
        k_export<<<ctx->H, K3_THREADS, 0, s>>>(v.buckets, v.flags, ctx->pc.win, ctx->d_offsets.get(), ctx->d_x_keys.get(), ctx->d_x_counts.get());
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches += 2;
        LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_x_keys.get(), ctx->d_x_keys.get(), total * 2, cudaMemcpyDeviceToHost, s));
        LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_x_counts.get(), ctx->d_x_counts.get(), total * 8, cudaMemcpyDeviceToHost, s));
        LH_CUDA(ctx, cudaStreamSynchronize(s));
    }
    ctx->stats.d2h_bytes += total * 10 + ((size_t)ctx->H + 1) * 4 + (size_t)ctx->C * 8;
    out->offsets = ctx->h_offsets.get();
    out->keys = ctx->h_x_keys.get();
    out->counts = reinterpret_cast<const uint64_t *>(ctx->h_x_counts.get());
    out->counter_deltas = reinterpret_cast<const uint64_t *>(ctx->h_counter_deltas.get());
    out->total_entries = total;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_copy_histogram(lh_ctx *ctx, uint32_t hid, uint64_t *h_out) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (hid >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram_id >= max_histograms");
    if (!h_out) return fail(ctx, LH_ERR_INVALID, "h_out is NULL");
    mark_rows_read(ctx);
    const View v = snapshot_view(ctx);
    LH_CUDA(ctx, cudaMemcpyAsync(h_out, v.buckets + (size_t)hid * 65536u, 65536 * 8, cudaMemcpyDeviceToHost, ctx->snap_stream.get()));
    LH_CUDA(ctx, cudaStreamSynchronize(ctx->snap_stream.get()));
    ctx->stats.d2h_bytes += 65536 * 8;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_end(lh_ctx *ctx) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    const int f = ctx->active ^ 1;
    cudaStream_t s = ctx->snap_stream.get();
    // zero only what the interval touched (flags), not the whole uint64[H][65536] array
    k_clear_touched<<<ctx->H, 256, 0, s>>>(ctx->buf[f].d_buckets.get(), ctx->buf[f].d_flags.get(), ctx->pc.win);
    LH_CUDA(ctx, cudaGetLastError());
    if (ctx->view_reduced) {
        k_clear_touched<<<ctx->H, 256, 0, s>>>(ctx->d_red_buckets.get(), ctx->d_red_flags.get(), ctx->pc.win);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
    }
    ctx->stats.kernel_launches++;
    LH_CUDA(ctx, cudaMemsetAsync(ctx->buf[f].d_counters.get(), 0, (size_t)ctx->C * 8u, s));
    LH_CUDA(ctx, cudaEventRecord(ctx->buf[f].cleared.get(), s));
    ctx->frozen = false;
    ctx->pub_slot = -1;
    ctx->view_reduced = false;
    ctx->view_counters_reduced = false;
    ctx->rows_packed = false;
    return LH_OK;
}

// =========================================================== device subscriptions
namespace {
// the image, then the id table of k_board_stage (16-byte aligned)
size_t board_image_bytes(uint32_t k, uint32_t kc) {
    return sizeof(lh_board_header) + (size_t)k * sizeof(lh_board_hist_row) + (size_t)kc * sizeof(lh_board_counter_row);
}
size_t board_table_offset(uint32_t k, uint32_t kc) { return (board_image_bytes(k, kc) + 15u) & ~(size_t)15u; }

// the live board a handle names (its memory must match too), or nullptr
Board *board_of(lh_ctx *ctx, const lh_board *b) {
    if (!b) return nullptr;
    for (auto &x : ctx->boards)
        if (x.b.handle == b->handle && x.b.d_board == b->d_board) return &x;
    return nullptr;
}
}  // namespace

extern "C" lh_status lh_board_create(lh_ctx *ctx, uint32_t k, uint32_t kc, lh_board *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    if (k == 0 && kc == 0) return fail(ctx, LH_ERR_INVALID, "a board needs a histogram or a counter row");
    if (k > ctx->H || kc > ctx->C) return fail(ctx, LH_ERR_RANGE, "more rows than max_histograms / max_counters");
    const size_t bytes = board_table_offset(k, kc) + (size_t)(k + kc) * sizeof(BoardEntry);
    cudaStream_t s = ctx->snap_stream.get();
    Board bd;
    bd.mem = AsyncPtr(s);
    LH_CUDA(ctx, cudaMallocAsync((void **)bd.mem.out(), bytes, s));
    cudaError_t e = cudaMemsetAsync(bd.mem.get(), 0, bytes, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_board_create", e);
    lh_board &b = bd.b;
    b.handle = graph_handle(ctx, ctx->next_board++);
    b.d_board = bd.mem.get();
    b.k = k;
    b.kc = kc;
    b.bytes = board_image_bytes(k, kc);
    *out = b;
    ctx->boards.push_back(std::move(bd));
    return LH_OK;
}

// One k_board_publish on the snapshot stream, after the reduction it reads.  Entries that do not fit its parameter
// block are first copied into the board's table by k_board_stage launches (see lh_kernels.cuh: the word is odd only
// inside the one publish kernel).
extern "C" lh_status lh_snapshot_publish(lh_ctx *ctx, const lh_board *b, const uint32_t *hist_ids,
                                         const uint32_t *counter_ids, const uint64_t *counter_totals) {
    LH_ENTER(ctx);
    Board *bd = board_of(ctx, b);
    if (!bd) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign board");
    if (!ctx->frozen || ctx->pub_slot < 0)
        return fail(ctx, LH_ERR_STATE, "lh_snapshot_publish needs a reduction of the open snapshot");
    if (!ids_ok(hist_ids, bd->b.k, ctx->H) || !ids_ok(counter_ids, bd->b.kc, ctx->C))
        return fail(ctx, LH_ERR_RANGE, "id >= max_histograms / max_counters");
    const int slot = ctx->pub_slot;
    const uint32_t np = ctx->res_np[slot];
    const ResLayout l = res_layout(ctx->H, np);
    const char *d = ctx->d_res[slot].get();
    cudaStream_t s = ctx->snap_stream.get();
    BoardParams &p = ctx->board_prm;
    p.board = (char *)bd->b.d_board;
    p.table = reinterpret_cast<BoardEntry *>(p.board + board_table_offset(bd->b.k, bd->b.kc));
    p.count = (const unsigned long long *)(d + l.count);
    p.sum = (const double *)(d + l.sum);
    p.avg = (const double *)(d + l.avg);
    p.pvals = (const double *)(d + l.pvals);
    p.pkeys = (const int *)(d + l.pkeys);
    p.nnz = ctx->d_nnz.get() + (size_t)slot * ctx->H;
    p.ps = ctx->d_ps[slot].get();
    p.counters = snapshot_view(ctx).counters;
    p.np = np;
    p.k = bd->b.k;
    const uint32_t rows = bd->b.k + bd->b.kc;
    for (uint32_t r0 = 0;; r0 += BP_MAX_ENTRIES) {
        const uint32_t n = std::min<uint32_t>(BP_MAX_ENTRIES, rows - r0);
        p.n_staged = r0;
        p.n = n;
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t row = r0 + i;
            if (row < bd->b.k) {
                p.e[i] = BoardEntry{row, hist_ids ? hist_ids[row] : LH_GRAPH_UNBOUND, 0ull};
            } else {
                const uint32_t c = row - bd->b.k;
                p.e[i] = BoardEntry{row, counter_ids ? counter_ids[c] : LH_GRAPH_UNBOUND,
                                    counter_totals ? (unsigned long long)counter_totals[c] : 0ull};
            }
        }
        if (r0 + n == rows) break;
        k_board_stage<<<1, BP_THREADS, 0, s>>>(p);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
    }
    k_board_publish<<<1, BP_THREADS, 0, s>>>(p);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return LH_OK;
}

extern "C" lh_status lh_board_read(lh_ctx *ctx, const lh_board *b, void *d_out, void *stream) {
    LH_ENTER(ctx);
    Board *bd = board_of(ctx, b);
    if (!bd) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign board");
    if (!d_out || ((uintptr_t)d_out & 7u)) return fail(ctx, LH_ERR_INVALID, "d_out is NULL or not 8-byte aligned");
    k_board_read<<<1, BR_THREADS, 0, pick_stream(ctx, stream)>>>((const unsigned long long *)bd->b.d_board,
                                                                 (unsigned long long *)d_out, (uint32_t)(bd->b.bytes / 8u));
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return LH_OK;
}

extern "C" lh_status lh_board_destroy(lh_ctx *ctx, const lh_board *b) {
    LH_ENTER(ctx);
    Board *bd = board_of(ctx, b);
    if (!bd) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign board");
    LH_CUDA(ctx, bd->mem.reset());   // after every publish issued (all on this stream)
    ctx->boards.erase(ctx->boards.begin() + (bd - ctx->boards.data()));
    return LH_OK;
}

// =========================================================== raw device subscriptions
namespace {
// headers, the k rows of cells, then the id table of k_raw_stage
size_t raw_table_offset(uint32_t k) { return LH_RAW_CELLS_OFFSET(k) + (size_t)k * 65536u * 8u; }
// A window board continues, 256-byte aligned, with its k sum rows, the slot counts [k][2] and the slot levels
// [k][window] (zeroed at creation: every slot empty), then its k * window slots.
size_t raw_window_offset(uint32_t k) { return (raw_table_offset(k) + (size_t)k * 4u + 255u) & ~(size_t)255u; }
size_t raw_nlevel_offset(uint32_t k) { return raw_window_offset(k) + (size_t)k * 65536u * 8u; }
size_t raw_levels_offset(uint32_t k) { return raw_nlevel_offset(k) + (size_t)k * 8u; }
size_t raw_slots_offset(uint32_t k, uint32_t w) { return (raw_levels_offset(k) + (size_t)k * w + 255u) & ~(size_t)255u; }

// the live raw board a handle names (its memory must match too), or nullptr
RawBoard *raw_board_of(lh_ctx *ctx, const lh_raw_board *b) {
    if (!b) return nullptr;
    for (auto &x : ctx->raw_boards)
        if (x.b.handle == b->handle && x.b.d_rows == b->d_rows) return &x;
    return nullptr;
}

// non-NULL and a-byte aligned
bool arg_ok(const void *p, uintptr_t a) { return p && ((uintptr_t)p & (a - 1u)) == 0; }

// lh_raw_board_create (window 1) and lh_raw_board_create_window, with ctx->mu held.  One allocation holds the whole
// board, so that a failure leaves nothing allocated and lh_raw_board_destroy frees everything at once.
lh_status raw_board_create(lh_ctx *ctx, uint32_t k, uint32_t window, lh_raw_board *out) {
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    if (k == 0) return fail(ctx, LH_ERR_INVALID, "a raw board needs a row");
    if (window == 0) return fail(ctx, LH_ERR_INVALID, "a window of 0 publishes");
    if (k > ctx->H) return fail(ctx, LH_ERR_RANGE, "more rows than max_histograms");
    if (window > LH_RAW_MAX_WINDOW) return fail(ctx, LH_ERR_RANGE, "window > LH_RAW_MAX_WINDOW");
    const size_t bytes = window == 1 ? raw_table_offset(k) + (size_t)k * 4u
                                     : raw_slots_offset(k, window) + (size_t)k * window * 65536u * 8u;
    cudaStream_t s = ctx->snap_stream.get();
    RawBoard rb;
    rb.mem = AsyncPtr(s);
    cudaError_t e = cudaMallocAsync((void **)rb.mem.out(), bytes, s);
    char *base = rb.mem.get();
    if (e != cudaSuccess)
        return fail(ctx, e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA, "allocating a raw board", e);
    // only the headers, each an empty row (publish 0, total 0, key_lo > key_hi): a row's cells are read only inside
    // the key range its latest publish wrote, so the cells of a row never published are never read.  A window board's
    // sums, slot counts and levels start at 0; its slots are read only inside the range of the level they record.
    std::vector<lh_raw_row_header> empty(k);
    for (auto &h : empty) { h.key_lo = 0; h.key_hi = -1; }
    e = cudaMemcpyAsync(base, empty.data(), (size_t)k * sizeof(lh_raw_row_header), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && window > 1)
        e = cudaMemsetAsync(base + raw_window_offset(k), 0, raw_levels_offset(k) + (size_t)k * window - raw_window_offset(k), s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_raw_board_create", e);
    rb.b.handle = graph_handle(ctx, ctx->next_raw_board++);
    rb.b.d_rows = base;
    rb.b.d_decomp = ctx->d_decomp.get();
    rb.b.k = k;
    memcpy(rb.b.prec, &ctx->pc, sizeof(Prec));
    rb.window = window;
    *out = rb.b;
    ctx->raw_boards.push_back(std::move(rb));
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_raw_board_create(lh_ctx *ctx, uint32_t k, lh_raw_board *out) {
    LH_ENTER(ctx);
    return raw_board_create(ctx, k, 1, out);
}

extern "C" lh_status lh_raw_board_create_window(lh_ctx *ctx, uint32_t k, uint32_t window, lh_raw_board *out) {
    LH_ENTER(ctx);
    return raw_board_create(ctx, k, window, out);
}

// One k_raw_publish (a CTA per row) on the snapshot stream, after whatever wrote the snapshot view it reads, or one
// k_raw_publish_window for a window board.  Ids that do not fit its parameter block are first copied into the board's
// table by k_raw_stage launches (see lh_kernels.cuh: a row's word is odd only inside the CTA that writes the row).
extern "C" lh_status lh_snapshot_publish_raw(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *hist_ids) {
    LH_ENTER(ctx);
    RawBoard *rb = raw_board_of(ctx, b);
    if (!rb) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign raw board");
    const lh_raw_board *bd = &rb->b;
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "lh_snapshot_publish_raw needs an open snapshot");
    if (!ids_ok(hist_ids, bd->k, ctx->H)) return fail(ctx, LH_ERR_RANGE, "id >= max_histograms");
    const bool windowed = rb->window > 1;
    if (windowed && rb->snapshot == ctx->stats.snapshots)   // the interval would be counted twice
        return fail(ctx, LH_ERR_STATE, "a window board takes one publish per snapshot");
    mark_rows_read(ctx);
    const View v = snapshot_view(ctx);
    cudaStream_t s = ctx->snap_stream.get();
    RawPublishParams &p = ctx->raw_prm;
    p.rows = (char *)bd->d_rows;
    p.cells = reinterpret_cast<unsigned long long *>(p.rows + LH_RAW_CELLS_OFFSET(bd->k));
    p.table = reinterpret_cast<uint32_t *>(p.rows + raw_table_offset(bd->k));
    p.buckets = v.buckets;
    p.flags = v.flags;
    p.win = ctx->pc.win;
    p.sums = windowed ? reinterpret_cast<unsigned long long *>(p.rows + raw_window_offset(bd->k)) : nullptr;
    p.nlevel = windowed ? reinterpret_cast<uint32_t *>(p.rows + raw_nlevel_offset(bd->k)) : nullptr;
    p.levels = windowed ? reinterpret_cast<uint8_t *>(p.rows + raw_levels_offset(bd->k)) : nullptr;
    p.slots = windowed ? reinterpret_cast<unsigned long long *>(p.rows + raw_slots_offset(bd->k, rb->window)) : nullptr;
    p.window = rb->window;
    p.slot = (uint32_t)(rb->published % rb->window);
    for (uint32_t r0 = 0;; r0 += RP_MAX_IDS) {
        const uint32_t n = std::min<uint32_t>(RP_MAX_IDS, bd->k - r0);
        p.n_staged = r0;
        p.n = n;
        for (uint32_t i = 0; i < n; i++) p.ids[i] = hist_ids ? hist_ids[r0 + i] : LH_GRAPH_UNBOUND;
        if (r0 + n == bd->k) break;
        k_raw_stage<<<1, RP_THREADS, 0, s>>>(p);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
    }
    if (windowed) k_raw_publish_window<<<bd->k, RP_THREADS, 0, s>>>(p);
    else k_raw_publish<<<bd->k, RP_THREADS, 0, s>>>(p);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    rb->published++;
    rb->snapshot = ctx->stats.snapshots;
    return LH_OK;
}

namespace {
// One k_raw_percentiles / k_raw_ranks over n queries (rows == nullptr: the grid form, m inputs per row), every
// argument checked before it is enqueued.
lh_status raw_query(lh_ctx *ctx, const lh_raw_board *b, bool pct, const uint32_t *d_rows, const double *d_x,
                    uint64_t n, uint32_t m, void *d_out1, void *d_out2, uint64_t *d_publish, void *stream) {
    const RawBoard *rb = raw_board_of(ctx, b);
    if (!rb) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign raw board");
    const lh_raw_board *bd = &rb->b;
    if (n == 0) return LH_OK;
    if (n > UINT32_MAX) return fail(ctx, LH_ERR_RANGE, "more than 2^32 - 1 queries");
    const bool grid = m != 0;
    if ((!grid && !arg_ok(d_rows, 4)) || !arg_ok(d_x, 8) || !arg_ok(d_out1, pct ? 4 : 8) || !arg_ok(d_out2, 8) ||
        !arg_ok(d_publish, 8))
        return fail(ctx, LH_ERR_INVALID, "a query array is NULL or not naturally aligned");
    const uint32_t blocks = (uint32_t)((n + RQ_THREADS - 1) / RQ_THREADS);
    cudaStream_t s = pick_stream(ctx, stream);
    if (pct)
        k_raw_percentiles<<<blocks, RQ_THREADS, 0, s>>>(*bd, grid ? nullptr : d_rows, d_x, (uint32_t)n, m, (int32_t *)d_out1,
                                                         (double *)d_out2, (unsigned long long *)d_publish);
    else
        k_raw_ranks<<<blocks, RQ_THREADS, 0, s>>>(*bd, grid ? nullptr : d_rows, d_x, (uint32_t)n, m,
                                                   (unsigned long long *)d_out1, (unsigned long long *)d_out2,
                                                   (unsigned long long *)d_publish);
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_raw_percentiles(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_ps,
                                        uint32_t n, int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream) {
    LH_ENTER(ctx);
    return raw_query(ctx, b, true, d_rows, d_ps, n, 0, d_keys, d_vals, d_publish, stream);
}

extern "C" lh_status lh_raw_ranks(lh_ctx *ctx, const lh_raw_board *b, const uint32_t *d_rows, const double *d_values,
                                  uint32_t n, uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream) {
    LH_ENTER(ctx);
    return raw_query(ctx, b, false, d_rows, d_values, n, 0, d_ranks, d_totals, d_publish, stream);
}

extern "C" lh_status lh_raw_percentiles_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_ps, uint32_t m,
                                             int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream) {
    LH_ENTER(ctx);
    const RawBoard *rb = raw_board_of(ctx, b);
    return raw_query(ctx, b, true, nullptr, d_ps, rb ? (uint64_t)rb->b.k * m : 0, m, d_keys, d_vals, d_publish, stream);
}

extern "C" lh_status lh_raw_ranks_grid(lh_ctx *ctx, const lh_raw_board *b, const double *d_values, uint32_t m,
                                       uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish, void *stream) {
    LH_ENTER(ctx);
    const RawBoard *rb = raw_board_of(ctx, b);
    return raw_query(ctx, b, false, nullptr, d_values, rb ? (uint64_t)rb->b.k * m : 0, m, d_ranks, d_totals, d_publish,
                     stream);
}

extern "C" lh_status lh_raw_board_destroy(lh_ctx *ctx, const lh_raw_board *b) {
    LH_ENTER(ctx);
    RawBoard *rb = raw_board_of(ctx, b);
    if (!rb) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign raw board");
    LH_CUDA(ctx, rb->mem.reset());   // after every publish issued (all on this stream)
    ctx->raw_boards.erase(ctx->raw_boards.begin() + (rb - ctx->raw_boards.data()));
    return LH_OK;
}

// =========================================================== device gauges
namespace {
constexpr uint32_t kGaugeBytes[] = {8, 4, 2, 2, 8, 4, 8};   // by LH_GAUGE_*
static_assert(sizeof(GaugeEntry) == sizeof(lh_gauge_src), "one table entry per lh_gauge_src");

constexpr uint32_t kGaugeKinds = sizeof kGaugeBytes / sizeof kGaugeBytes[0];

// LH_OK when k_gauge_read may load the entry: a known dtype, a naturally aligned address in device or managed memory of
// the context's device.  Anything else could fault the kernel, so it is refused before any launch.  `kind` and i name
// the entry in the error ("gauge 3", "array 3").
lh_status check_gauge(lh_ctx *ctx, const char *kind, uint32_t i, const lh_gauge_src &s) {
    char what[160];
    if (s.dtype >= kGaugeKinds || s.reserved) {
        snprintf(what, sizeof what, "%s %u: unknown dtype %u or non-zero reserved", kind, i, s.dtype);
        return fail(ctx, LH_ERR_INVALID, what);
    }
    if (!s.d_value || ((uintptr_t)s.d_value & (kGaugeBytes[s.dtype] - 1u))) {
        snprintf(what, sizeof what, "%s %u: address is NULL or not %u-byte aligned", kind, i, kGaugeBytes[s.dtype]);
        return fail(ctx, LH_ERR_INVALID, what);
    }
    cudaPointerAttributes a{};
    const cudaError_t e = cudaPointerGetAttributes(&a, s.d_value);
    if (e != cudaSuccess) cudaGetLastError();
    if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != ctx->device) {
        snprintf(what, sizeof what, "%s %u: address is not device or managed memory of device %d", kind, i, ctx->device);
        return fail(ctx, LH_ERR_INVALID, what);
    }
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_gauges_read(lh_ctx *ctx, const lh_gauge_src *h_srcs, uint32_t n, double *h_out) {
    if (!ctx) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> one_read(ctx->gauge_mu);
    LH_ENTER(ctx);
    if (n && (!h_srcs || !h_out)) return fail(ctx, LH_ERR_INVALID, "h_srcs / h_out is NULL");
    for (uint32_t i = 0; i < n; i++)
        if (lh_status st = check_gauge(ctx, "gauge", i, h_srcs[i]); st != LH_OK) return st;
    if (n == 0) return LH_OK;
    if (n > ctx->gauge_cap) {
        const uint32_t cap = std::max<uint32_t>(n, 4096);
        ctx->h_gauges.reset();   // no read is in flight: every call waits for its launches
        ctx->d_gauges = nullptr;
        ctx->gauge_cap = 0;
        PinnedPtr<double> h; double *d = nullptr;
        LH_CUDA(ctx, cudaHostAlloc((void **)h.out(), (size_t)cap * 8u, cudaHostAllocMapped));
        LH_CUDA(ctx, cudaHostGetDevicePointer((void **)&d, h.get(), 0));
        ctx->h_gauges = std::move(h); ctx->d_gauges = d; ctx->gauge_cap = cap;
    }
    if (!ctx->gauge_done.get()) LH_CUDA(ctx, cudaEventCreateWithFlags(ctx->gauge_done.out(), cudaEventDisableTiming));
    cudaStream_t s = ctx->snap_stream.get();
    GaugeParams &p = ctx->gauge_prm;
    for (uint32_t i0 = 0; i0 < n; i0 += GR_MAX_ENTRIES) {
        const uint32_t m = std::min<uint32_t>(GR_MAX_ENTRIES, n - i0);
        p.out = ctx->d_gauges + i0;
        p.n = m;
        for (uint32_t j = 0; j < m; j++) p.e[j] = GaugeEntry{h_srcs[i0 + j].d_value, h_srcs[i0 + j].dtype, 0u};
        k_gauge_read<<<(m + GR_THREADS - 1) / GR_THREADS, GR_THREADS, 0, s>>>(p);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
    }
    LH_CUDA(ctx, cudaEventRecord(ctx->gauge_done.get(), s));
    // wait outside the lock so ingest threads are not held up; gauge_mu keeps the buffer ours
    cudaEvent_t ev = ctx->gauge_done.get();
    _lk.unlock();
    const cudaError_t e = cudaEventSynchronize(ev);
    _lk.lock();
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "cudaEventSynchronize(gauges)", e);
    memcpy(h_out, ctx->h_gauges.get(), (size_t)n * 8u);
    return LH_OK;
}

// =========================================================== distribution gauges
namespace {
static_assert(sizeof(ArraySeg) == 16, "k_ingest_arrays' table entry");
using MemGetAddressRange = CUresult (*)(CUdeviceptr *, size_t *, CUdeviceptr);

// cuMemGetAddressRange of the driver the runtime uses (the library does not link libcuda); nullptr when it has none
MemGetAddressRange mem_get_address_range() {
    static const MemGetAddressRange fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            return (MemGetAddressRange) nullptr;
        }
        return reinterpret_cast<MemGetAddressRange>(p);
    }();
    return fn;
}

// LH_OK when k_ingest_arrays may load every element of the entry: a known dtype and, when it has elements, check_gauge's
// checks on its first element, an id below max_histograms, and all n elements inside the allocation that holds the
// first one.  A base address alone would let the kernel read past the end of its allocation.
lh_status check_array(lh_ctx *ctx, uint32_t i, const lh_array_src &a) {
    char what[192];
    if (a.dtype >= kGaugeKinds) {
        snprintf(what, sizeof what, "array %u: unknown dtype %u", i, a.dtype);
        return fail(ctx, LH_ERR_INVALID, what);
    }
    if (a.n == 0) return LH_OK;
    if (lh_status st = check_gauge(ctx, "array", i, lh_gauge_src{a.d_values, a.dtype, 0u}); st != LH_OK) return st;
    if (a.histogram_id >= ctx->H) {
        snprintf(what, sizeof what, "array %u: histogram_id %u >= max_histograms", i, a.histogram_id);
        return fail(ctx, LH_ERR_RANGE, what);
    }
    const MemGetAddressRange range = mem_get_address_range();
    const CUdeviceptr p = (CUdeviceptr)(uintptr_t)a.d_values;
    CUdeviceptr base = 0;
    size_t bytes = 0;
    if (!range || range(&base, &bytes, p) != CUDA_SUCCESS || p < base ||
        a.n > (uint64_t)(base + bytes - p) / kGaugeBytes[a.dtype]) {
        snprintf(what, sizeof what, "array %u: its %llu elements of %u bytes do not lie inside one allocation", i,
                 (unsigned long long)a.n, kGaugeBytes[a.dtype]);
        return fail(ctx, LH_ERR_INVALID, what);
    }
    return LH_OK;
}

// lh_ingest_arrays routing (launch_arrays<gauge::Streaming>): an item at least this long goes to K1 in the form of its
// dtype, float64 ones from kBatchK1Min as in lh_ingest_batch; shorter ones, and every int64 / uint64 item, go to
// k_ingest_arrays.  Both narrow thresholds are kBatchK1Min's value, not measured for these forms: at 2^28 samples the
// 4-byte form runs 750 G samples/s and the 16-bit form 830 G (H100 80GB HBM3, 700 W; DESIGN.md section 5.1).
constexpr size_t kArraysK1Min4 = 1024 * 1024;   // float32, int32: the 4-byte form
constexpr size_t kArraysK1Min2 = 1024 * 1024;   // float16, bfloat16: the 16-bit form
size_t arrays_k1_min(uint32_t dtype) {
    if (dtype == LH_GAUGE_F64) return kBatchK1Min;
    const int f = k1n_index(dtype);
    return f < 0 ? SIZE_MAX : g_k1_narrow[f].bytes == 4 ? kArraysK1Min4 : kArraysK1Min2;
}

// Validated arrays into the rows of `target` on s: as few launches of k_ingest_arrays<Ld> as the parameter block and
// the uint32 table counts allow (launch_batch's packing); an array that does not fit the launch being filled is split
// across launches.  With Ld = gauge::Streaming (lh_ingest_arrays, stream-ordered) long items go to K1 instead, by
// arrays_k1_min; gauge::Relaxed (distribution gauges) takes every item through k_ingest_arrays.  Kernels only (the
// graph recorder's form is captured); the caller counts the samples in stats.
template <typename Ld>
lh_status launch_arrays(lh_ctx *ctx, const lh_recorder &target, const lh_array_src *srcs, uint32_t n_srcs, cudaStream_t s) {
    ArrayParams &prm = ctx->array_prm;
    prm.rec = target;
    const int grid_max = batch_grid_max(ctx);
    const unsigned long long cap = launch_cap(grid_max);
    uint32_t k = 0;
    unsigned long long total = 0;
    auto launch = [&]() -> lh_status {
        if (!k) return LH_OK;
        prm.n_items = k;
        const unsigned long long pieces = (total + BI_PIECE - 1) / BI_PIECE;
        const int grid = (int)std::min<unsigned long long>((unsigned long long)grid_max, pieces);
        k_ingest_arrays<Ld><<<grid, BI_THREADS, BlockRecorder::smem_bytes(BI_TABLE_ENTRIES), s>>>(prm);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        k = 0;
        total = 0;
        return LH_OK;
    };
    for (uint32_t i = 0; i < n_srcs; i++) {
        const lh_array_src &a = srcs[i];
        if (std::is_same<Ld, gauge::Streaming>::value && a.n >= arrays_k1_min(a.dtype)) {
            unsigned long long *row = reinterpret_cast<unsigned long long *>(target.d_buckets) + (size_t)a.histogram_id * 65536u;
            uint32_t *flag = target.d_flags + a.histogram_id;
            const int f = k1n_index(a.dtype);
            lh_status st = f < 0 ? launch_single(ctx, row, flag, (const double *)a.d_values, (size_t)a.n, s)
                                 : launch_narrow_single(ctx, f, row, flag, a.d_values, (size_t)a.n, s);
            if (st != LH_OK) return st;
            continue;
        }
        const char *p = (const char *)a.d_values;
        unsigned long long left = a.n;
        while (left) {
            if (k == (uint32_t)BI_MAX_ITEMS || total == cap) {
                lh_status st = launch();
                if (st != LH_OK) return st;
            }
            const unsigned long long m = std::min(left, cap - total);
            prm.seg[k] = ArraySeg{p, a.histogram_id, a.dtype};
            prm.start[k] = total;
            total += m;
            prm.start[k + 1] = total;
            k++;
            p += m * kGaugeBytes[a.dtype];
            left -= m;
        }
    }
    return launch();
}
}  // namespace

extern "C" lh_status lh_snapshot_ingest_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs) {
    LH_ENTER(ctx);
    if (n_srcs && !h_srcs) return fail(ctx, LH_ERR_INVALID, "h_srcs is NULL");
    unsigned long long total = 0;
    for (uint32_t i = 0; i < n_srcs; i++) {
        if (lh_status st = check_array(ctx, i, h_srcs[i]); st != LH_OK) return st;
        total += h_srcs[i].n;
    }
    if (!ctx->frozen || ctx->rows_read)
        return fail(ctx, LH_ERR_STATE, "lh_snapshot_ingest_arrays needs an open snapshot whose rows nothing has read yet");
    if (total == 0) return LH_OK;
    // after lh_snapshot_begin's writer waits, graph drain and hot-window fold, all on the snapshot stream
    lh_status st = launch_arrays<gauge::Relaxed>(ctx, buffer_target(ctx, ctx->active ^ 1), h_srcs, n_srcs, ctx->snap_stream.get());
    if (st != LH_OK) return st;
    ctx->stats.samples += total;
    return LH_OK;
}

namespace {
// Validation of lh_ingest_arrays / lh_graph_recorder_ingest_arrays against `limit` histogram ids (check_batch's, by
// dtype); the samples of the call.  The arrays are read in stream order, like lh_ingest_batch's, so unlike
// lh_snapshot_ingest_arrays the memory kind and the allocation range are the caller's to get right.
lh_status check_stream_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs, uint32_t limit,
                              unsigned long long *n_out) {
    if (n_srcs && !h_srcs) return fail(ctx, LH_ERR_INVALID, "h_srcs is NULL");
    char what[160];
    unsigned long long n = 0;
    for (uint32_t i = 0; i < n_srcs; i++) {
        const lh_array_src &a = h_srcs[i];
        if (a.dtype >= kGaugeKinds) {
            snprintf(what, sizeof what, "array %u: unknown dtype %u", i, a.dtype);
            return fail(ctx, LH_ERR_INVALID, what);
        }
        if (a.n == 0) continue;
        if (!a.d_values || ((uintptr_t)a.d_values & (kGaugeBytes[a.dtype] - 1u))) {
            snprintf(what, sizeof what, "array %u: d_values is NULL or not %u-byte aligned", i, kGaugeBytes[a.dtype]);
            return fail(ctx, LH_ERR_INVALID, what);
        }
        if (a.histogram_id >= limit) {
            snprintf(what, sizeof what, "array %u: histogram_id %u >= max_histograms", i, a.histogram_id);
            return fail(ctx, LH_ERR_RANGE, what);
        }
        n += a.n;
    }
    *n_out = n;
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_ingest_arrays(lh_ctx *ctx, const lh_array_src *h_srcs, uint32_t n_srcs, void *stream) {
    LH_ENTER(ctx);
    unsigned long long n = 0;
    lh_status st = check_stream_arrays(ctx, h_srcs, n_srcs, ctx->H, &n);
    if (st != LH_OK || n == 0) return st;
    cudaStream_t s = pick_stream(ctx, stream);
    return write_bracket(ctx, s, [&](int b) {
        lh_status bs = launch_arrays<gauge::Streaming>(ctx, buffer_target(ctx, b), h_srcs, n_srcs, s);
        if (bs == LH_OK) ctx->stats.samples += n;
        return bs;
    });
}

extern "C" lh_status lh_graph_recorder_ingest_arrays(lh_ctx *ctx, const lh_graph_recorder *g, const lh_array_src *h_srcs,
                                                     uint32_t n_srcs, void *stream) {
    LH_ENTER(ctx);
    GraphRec *gr = graph_of(ctx, g);
    if (!gr) return fail(ctx, LH_ERR_INVALID, "destroyed or foreign graph recorder");
    unsigned long long n = 0;
    lh_status st = check_stream_arrays(ctx, h_srcs, n_srcs, gr->rec.max_histograms, &n);
    if (st != LH_OK || n == 0) return st;
    return launch_arrays<gauge::Streaming>(ctx, gr->rec, h_srcs, n_srcs, pick_stream(ctx, stream));
}

// =========================================================== reduce caller-supplied sparse histograms
namespace {
// The device part of lh_reduce_sparse_host, rs_mu held: one H2D of the input, per batch of K6_BATCH segments scatter
// + K3 + epilogue + clear into the call's own result buffer, one D2H of the packed results into h_res.
cudaError_t reduce_sparse_device(lh_ctx *ctx, uint32_t n, const uint32_t *h_offsets, const int16_t *h_keys,
                                 const uint64_t *h_counts, const double *ps, uint32_t np, char *h_res, const char **what) {
#define RS_CUDA(call)                                                    \
    do {                                                                 \
        cudaError_t _e = (call);                                         \
        if (_e != cudaSuccess) { *what = #call; return _e; }             \
    } while (0)
    RS_CUDA(cudaSetDevice(ctx->device));
    if (!ctx->rs_stream.get()) RS_CUDA(cudaStreamCreateWithFlags(ctx->rs_stream.out(), cudaStreamNonBlocking));
    cudaStream_t s = ctx->rs_stream.get();
    const size_t row_bytes = (size_t)K6_BATCH * 65536u * 8u;
    if (!ctx->d_rs_rows.get()) {
        DevPtr<uint32_t> flags, nnz; DevPtr<unsigned long long> rows;
        RS_CUDA(cudaMalloc(flags.out(), K6_BATCH * 4));
        RS_CUDA(cudaMalloc(nnz.out(), K6_BATCH * 4));
        RS_CUDA(cudaMalloc(rows.out(), row_bytes));
        ctx->d_rs_flags = std::move(flags); ctx->d_rs_nnz = std::move(nnz); ctx->d_rs_rows = std::move(rows);
        ctx->rs_dirty = true;
    }
    if (ctx->rs_dirty) {
        RS_CUDA(cudaMemsetAsync(ctx->d_rs_rows.get(), 0, row_bytes, s));
        RS_CUDA(cudaMemsetAsync(ctx->d_rs_flags.get(), 0, K6_BATCH * 4, s));
    }
    ctx->rs_dirty = true;                        // until the last clear of this call has run

    const uint32_t base = h_offsets[0];
    const size_t ne = (size_t)h_offsets[n] - base;
    const ResLayout l = res_layout(n, np);
    const size_t off_keys = ((size_t)n + 1) * 4, off_counts = (off_keys + ne * 2 + 7) & ~(size_t)7;
    const size_t off_ps = off_counts + ne * 8, off_res = off_ps + LH_MAX_PERCENTILES * 8;
    AsyncPtr buf(s);   // released on every return path
    RS_CUDA(cudaMallocAsync((void **)buf.out(), off_res + l.total, s));
    char *d = buf.get();
    RS_CUDA(cudaMemcpyAsync(d, h_offsets, off_keys, cudaMemcpyHostToDevice, s));
    if (ne) {
        RS_CUDA(cudaMemcpyAsync(d + off_keys, h_keys + base, ne * 2, cudaMemcpyHostToDevice, s));
        RS_CUDA(cudaMemcpyAsync(d + off_counts, h_counts + base, ne * 8, cudaMemcpyHostToDevice, s));
    }
    if (np) RS_CUDA(cudaMemcpyAsync(d + off_ps, ps, np * sizeof(double), cudaMemcpyHostToDevice, s));
    const uint32_t *d_off = (const uint32_t *)d;
    const short *d_keys = (const short *)(d + off_keys);
    const unsigned long long *d_counts = (const unsigned long long *)(d + off_counts);
    const double *d_ps = (const double *)(d + off_ps);
    char *r = d + off_res;
    unsigned long long *r_count = (unsigned long long *)(r + l.count);
    double *r_sum = (double *)(r + l.sum), *r_avg = (double *)(r + l.avg), *r_pvals = (double *)(r + l.pvals);
    int *r_pkeys = (int *)(r + l.pkeys);
    const uint32_t win = ctx->pc.win, smem_cells = k3_smem_cells(win);
    for (uint32_t b0 = 0; b0 < n; b0 += K6_BATCH) {
        const uint32_t nb = std::min<uint32_t>(K6_BATCH, n - b0);
        const size_t m = (size_t)h_offsets[b0 + nb] - h_offsets[b0];
        const size_t po = (size_t)b0 * np;
        if (m) {
            const int grid = (int)std::min<size_t>((m + 255) / 256, (size_t)ctx->sm_count * 8);
            k_scatter_segments<<<grid, 256, 0, s>>>(d_off + b0, nb, base, d_keys, d_counts, ctx->d_rs_rows.get(), ctx->d_rs_flags.get(), win);
        }
        k_reduce<<<nb, K3_THREADS, (size_t)smem_cells * 8, s>>>(ctx->d_rs_rows.get(), ctx->d_rs_flags.get(), win, ctx->d_decomp.get(), d_ps, (int)np,
                                                                 r_count + b0, r_sum + b0, r_avg + b0, r_pkeys + po, r_pvals + po,
                                                                 ctx->d_rs_nnz.get(), smem_cells);
        k_sparse_epilogue<<<nb, 256, 0, s>>>(d_off + b0, base, d_keys, ctx->d_rs_rows.get(), ctx->d_decomp.get(), d_ps, (int)np,
                                             r_count + b0, r_sum + b0, r_avg + b0, r_pkeys + po, r_pvals + po);
        k_clear_touched<<<nb, 256, 0, s>>>(ctx->d_rs_rows.get(), ctx->d_rs_flags.get(), win);
        RS_CUDA(cudaGetLastError());
    }
    RS_CUDA(cudaMemcpyAsync(h_res, r, l.total, cudaMemcpyDeviceToHost, s));
    RS_CUDA(cudaStreamSynchronize(s));
    ctx->rs_dirty = false;
    return cudaSuccess;
#undef RS_CUDA
}
}  // namespace

// processHistograms + percentile over caller-supplied sparse histograms.  Never takes the context mutex while work is
// in flight (only to record an error or the stats), and touches none of the snapshot / ingest state.
extern "C" lh_status lh_reduce_sparse_host(lh_ctx *ctx, uint32_t n, const uint32_t *h_offsets, const int16_t *h_keys,
                                           const uint64_t *h_counts, const double *percentiles, uint32_t np,
                                           uint64_t *counts, double *sums, double *avgs, int32_t *pkeys, double *pvals) {
    if (!ctx) return LH_ERR_INVALID;
    auto bad = [ctx](lh_status st, const char *what, cudaError_t e = cudaSuccess) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        return fail(ctx, st, what, e);
    };
    if (n == 0) return LH_OK;
    if (!h_offsets) return bad(LH_ERR_INVALID, "offsets is NULL");
    if (np > LH_MAX_PERCENTILES || (np && !percentiles)) return bad(LH_ERR_INVALID, "bad percentile array");
    for (uint32_t i = 0; i < n; i++)
        if (h_offsets[i + 1] < h_offsets[i]) return bad(LH_ERR_INVALID, "offsets decrease");
    const size_t ne = (size_t)h_offsets[n] - h_offsets[0];
    if (ne && (!h_keys || !h_counts)) return bad(LH_ERR_INVALID, "keys / counts NULL with entries");
    const ResLayout l = res_layout(n, np);
    std::vector<char> h_res(l.total);
    {
        std::lock_guard<std::mutex> rs(ctx->rs_mu);
        const char *what = "";
        const cudaError_t e = reduce_sparse_device(ctx, n, h_offsets, h_keys, h_counts, percentiles, np, h_res.data(), &what);
        if (e != cudaSuccess) return bad(e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA, what, e);
    }
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->stats.kernel_launches += 4 * (((size_t)n + K6_BATCH - 1) / K6_BATCH);
        ctx->stats.h2d_bytes += ((size_t)n + 1) * 4 + ne * 10 + np * 8;
        ctx->stats.d2h_bytes += l.total;
    }
    const char *h = h_res.data();
    if (counts) memcpy(counts, h + l.count, (size_t)n * 8);
    if (sums) memcpy(sums, h + l.sum, (size_t)n * 8);
    if (avgs) memcpy(avgs, h + l.avg, (size_t)n * 8);
    if (pvals && np) memcpy(pvals, h + l.pvals, (size_t)n * np * 8);
    if (pkeys && np) memcpy(pkeys, h + l.pkeys, (size_t)n * np * 4);
    return LH_OK;
}

// =========================================================== multi-GPU (peer memory)
extern "C" lh_status lh_comm_export(lh_ctx *ctx, lh_peer_handle *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    PeerWire w{};
    w.magic = kPeerMagic; w.abi = LH_ABI_VERSION; w.H = ctx->H; w.C = ctx->C;
    w.precision = (uint32_t)ctx->pc.precision; w.device = (uint32_t)ctx->device;
    w.pid = (int64_t)getpid(); w.ctx_id = ctx->ctx_id;
    for (int b = 0; b < 2; b++) {
        w.ptr_buckets[b] = (uint64_t)(uintptr_t)ctx->buf[b].d_buckets.get();
        w.ptr_flags[b] = (uint64_t)(uintptr_t)ctx->buf[b].d_flags.get();
        w.ptr_counters[b] = (uint64_t)(uintptr_t)ctx->buf[b].d_counters.get();
        LH_CUDA(ctx, cudaIpcGetMemHandle(&w.ipc_buckets[b], ctx->buf[b].d_buckets.get()));
        LH_CUDA(ctx, cudaIpcGetMemHandle(&w.ipc_flags[b], ctx->buf[b].d_flags.get()));
        LH_CUDA(ctx, cudaIpcGetMemHandle(&w.ipc_counters[b], ctx->buf[b].d_counters.get()));
    }
    w.ptr_comm = (uint64_t)(uintptr_t)ctx->d_comm.get();
    LH_CUDA(ctx, cudaIpcGetMemHandle(&w.ipc_comm, ctx->d_comm.get()));
    if (lh_status st = comm_alloc_reduced(ctx)) return st;
    w.ptr_red = (uint64_t)(uintptr_t)ctx->d_red_buckets.get();
    LH_CUDA(ctx, cudaIpcGetMemHandle(&w.ipc_red, ctx->d_red_buckets.get()));
    memset(out, 0, sizeof *out);
    memcpy(out->bytes, &w, sizeof w);
    return LH_OK;
}

extern "C" lh_status lh_comm_import(lh_ctx *ctx, uint32_t rank, uint32_t world, const lh_peer_handle *all) {
    LH_ENTER(ctx);
    if (!all || world < 1 || world > (uint32_t)kMaxRanks || rank >= world) return fail(ctx, LH_ERR_INVALID, "bad rank / world / handles");
    if (ctx->frozen) return fail(ctx, LH_ERR_STATE, "lh_comm_import during a snapshot");
    comm_unmap(ctx);
    const int64_t my_pid = (int64_t)getpid();
    for (uint32_t r = 0; r < world; r++) {
        PeerWire w;
        memcpy(&w, all[r].bytes, sizeof w);
        if (w.magic != kPeerMagic || w.abi != LH_ABI_VERSION) return fail(ctx, LH_ERR_INVALID, "peer handle is not from this library version");
        if (w.H != ctx->H || w.C != ctx->C || w.precision != (uint32_t)ctx->pc.precision)
            return fail(ctx, LH_ERR_INVALID, "peer context has a different shape (max_histograms / max_counters / precision)");
        PeerMap &pm = ctx->peers[r];
        if (r == rank) {
            if (w.ctx_id != ctx->ctx_id || w.pid != my_pid) return fail(ctx, LH_ERR_INVALID, "handles[rank] is not this context's own handle");
            for (int b = 0; b < 2; b++) { pm.buckets[b] = ctx->buf[b].d_buckets.get(); pm.flags[b] = ctx->buf[b].d_flags.get(); pm.counters[b] = ctx->buf[b].d_counters.get(); }
            pm.comm = ctx->d_comm.get();
            if (lh_status st = comm_alloc_reduced(ctx)) return st;
            pm.red = ctx->d_red_buckets.get();
            continue;
        }
        if (w.pid == my_pid) {
            // same process (one thread per GPU): plain peer access on the raw pointers
            if ((int)w.device != ctx->device) {
                int can = 0;
                LH_CUDA(ctx, cudaDeviceCanAccessPeer(&can, ctx->device, (int)w.device));
                if (!can) return fail(ctx, LH_ERR_NO_DEVICE, "no peer access between the two devices");
                cudaError_t e = cudaDeviceEnablePeerAccess((int)w.device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(ctx, LH_ERR_CUDA, "cudaDeviceEnablePeerAccess", e);
                cudaGetLastError();
            }
            for (int b = 0; b < 2; b++) {
                pm.buckets[b] = (unsigned long long *)(uintptr_t)w.ptr_buckets[b];
                pm.flags[b] = (uint32_t *)(uintptr_t)w.ptr_flags[b];
                pm.counters[b] = (unsigned long long *)(uintptr_t)w.ptr_counters[b];
            }
            pm.comm = (unsigned long long *)(uintptr_t)w.ptr_comm;
            pm.red = (unsigned long long *)(uintptr_t)w.ptr_red;
        } else {
            // another process on this node: CUDA IPC mappings (NVLink peer-to-peer underneath)
            pm.ipc = true;
            for (int b = 0; b < 2; b++) {
                LH_CUDA(ctx, cudaIpcOpenMemHandle((void **)&pm.buckets[b], w.ipc_buckets[b], cudaIpcMemLazyEnablePeerAccess));
                LH_CUDA(ctx, cudaIpcOpenMemHandle((void **)&pm.flags[b], w.ipc_flags[b], cudaIpcMemLazyEnablePeerAccess));
                LH_CUDA(ctx, cudaIpcOpenMemHandle((void **)&pm.counters[b], w.ipc_counters[b], cudaIpcMemLazyEnablePeerAccess));
            }
            LH_CUDA(ctx, cudaIpcOpenMemHandle((void **)&pm.comm, w.ipc_comm, cudaIpcMemLazyEnablePeerAccess));
            LH_CUDA(ctx, cudaIpcOpenMemHandle((void **)&pm.red, w.ipc_red, cudaIpcMemLazyEnablePeerAccess));
        }
    }
    if (lh_status st = comm_alloc_row_maps(ctx)) return st;
    ctx->comm_rank = rank;
    ctx->comm_world = world;
    return LH_OK;
}

namespace {
// The launches of one all-reduce (both forms), with ctx->mu held and every argument checked.  frozen[r]: the buffer
// rank r froze; n_rows: the histogram rows in play (H for the identity form), which set the payload and the grid.
void k5_launch(int grid, size_t smem, cudaStream_t s, const PeerParams &p, RowIdentity) { k_peer_allreduce<<<grid, K5_THREADS, smem, s>>>(p); }
void k5_launch(int grid, size_t smem, cudaStream_t s, const PeerParams &p, const RowMap &m) { k_peer_allreduce_rows<<<grid, K5_THREADS, smem, s>>>(p, m); }

template <typename Rows>
lh_status launch_allreduce(lh_ctx *ctx, uint64_t seq, const uint32_t *frozen, uint32_t n_rows, uint32_t include_counters,
                           Rows rows, uint64_t *seq_out) {
    mark_rows_read(ctx);
    const int f = ctx->active ^ 1;
    cudaStream_t s = ctx->snap_stream.get();
    // status and cells describe this all-reduce only: zeroed behind the previous one on the same stream
    LH_CUDA(ctx, cudaMemsetAsync(ctx->d_comm_aux.get() + 1, 0, 12, s));
    PeerParams p{};
    p.rank = ctx->comm_rank; p.world = ctx->comm_world; p.H = ctx->H; p.C = ctx->C; p.win = ctx->pc.win;
    p.do_counters = include_counters ? 1u : 0u; p.frozen = (uint32_t)f;
    p.seq = seq;
    ctx->comm_seq = seq;
    p.timeout_ns = 10ull * 1000ull * 1000ull * 1000ull;
    for (uint32_t r = 0; r < ctx->comm_world; r++) {
        const int fr = frozen ? (int)frozen[r] : f;
        p.buckets[r] = ctx->peers[r].buckets[fr];
        p.flags[r] = ctx->peers[r].flags[fr];
        p.counters[r] = ctx->peers[r].counters[fr];
        p.comm[r] = ctx->peers[r].comm;
    }
    p.out_buckets = ctx->d_red_buckets.get(); p.out_flags = ctx->d_red_flags.get(); p.out_counters = ctx->d_red_counters.get();
    p.block_counter = ctx->d_comm_aux.get(); p.status = ctx->d_comm_aux.get() + 1;
    p.cells = reinterpret_cast<unsigned long long *>(ctx->d_comm_aux.get() + 2);
    for (uint32_t r = 0; r < ctx->comm_world; r++) p.out_peer[r] = ctx->peers[r].red;
    // payload = the window cells of every histogram that can be live; above 1 MiB the reduce-scatter + push form wins
    const size_t payload = (size_t)n_rows * (2u * ctx->pc.win - 1u) * 8u;
    p.two_shot = payload >= (1u << 20) ? 1u : 0u;
    ctx->comm_two_shot = p.two_shot != 0;
    const int ring = (int)(p.seq % lh_ctx::kCommRing);
    // a few CTAs: the kernel shares the GPU with the next interval's ingest (which leaves k1_reserve_sms SMs free);
    // CTAs that are not resident yet simply start later (no CTA waits for another CTA of its own grid before the end)
    const size_t items = (size_t)std::max(1u, n_rows) * (65536u / K5_CHUNK);
    int grid = (int)std::min<size_t>(items, n_rows <= 1 ? 5 : 16);
    LH_CUDA(ctx, cudaEventRecord(ctx->comm_t0[ring].get(), s));
    if (p.two_shot) {
        // An SM sustains only ~4 GB/s of NVLink loads (measured, tools/peer_probe.py: 36 MB take 9.1 / 2.3 / 0.64 / 0.21 ms
        // on 1 / 4 / 16 / 64 SMs), so the large payload cannot hide on the few SMs the ingest kernels leave free.  It goes
        // wide and short instead: one small CTA announces this rank and waits for the peers (it may spin for as long as
        // the ranks are skewed, on one SM), then up to 128 CTAs do the sums in ~0.2 ms; the next ingest kernel's CTAs
        // start as those finish.
        PeerParams pa = p;
        pa.arrive_only = 1;
        k5_launch(1, ctx->H, s, pa, rows);
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
        grid = (int)std::min<size_t>((n_rows + ctx->comm_world - 1) / ctx->comm_world, (size_t)std::max(1, std::min(128, ctx->sm_count - 20)));
    }
    k5_launch(grid, ctx->H, s, p, rows);
    LH_CUDA(ctx, cudaGetLastError());
    LH_CUDA(ctx, cudaEventRecord(ctx->comm_t1[ring].get(), s));
    ctx->stats.kernel_launches++;
    ctx->view_reduced = true;
    ctx->view_counters_reduced = include_counters != 0;
    ctx->nnz_valid = false;
    if (seq_out) *seq_out = p.seq;
    return LH_OK;
}
}  // namespace

extern "C" lh_status lh_snapshot_allreduce(lh_ctx *ctx, uint32_t include_counters, uint64_t *seq_out) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->comm_world < 2) return fail(ctx, LH_ERR_STATE, "lh_comm_import has not been called with world >= 2");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    return launch_allreduce(ctx, ctx->comm_seq + 1, nullptr, ctx->H, include_counters, RowIdentity{}, seq_out);
}

extern "C" lh_status lh_snapshot_rows(lh_ctx *ctx, uint8_t *hist_touched, uint64_t *counter_deltas, uint32_t *frozen) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    mark_rows_read(ctx);
    const int f = ctx->active ^ 1;
    cudaStream_t s = ctx->snap_stream.get();
    if (lh_status st = alloc_rows_staging(ctx)) return st;
    // behind the writer events, the graph drain and the hot-window fold lh_snapshot_begin ordered on this stream
    if (hist_touched) LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_rows_flags.get(), ctx->buf[f].d_flags.get(), (size_t)ctx->H * 4, cudaMemcpyDeviceToHost, s));
    if (counter_deltas) LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_rows_counters.get(), ctx->buf[f].d_counters.get(), (size_t)ctx->C * 8, cudaMemcpyDeviceToHost, s));
    LH_CUDA(ctx, cudaStreamSynchronize(s));
    if (hist_touched)
        for (uint32_t h = 0; h < ctx->H; h++) hist_touched[h] = ctx->h_rows_flags.get()[h] != 0;
    if (counter_deltas) memcpy(counter_deltas, ctx->h_rows_counters.get(), (size_t)ctx->C * 8);
    if (frozen) *frozen = (uint32_t)f;
    ctx->stats.d2h_bytes += (hist_touched ? (size_t)ctx->H * 4 : 0) + (counter_deltas ? (size_t)ctx->C * 8 : 0);
    return LH_OK;
}

extern "C" lh_status lh_snapshot_allreduce_rows(lh_ctx *ctx, uint64_t seq, const uint32_t *frozen, uint32_t n_rows,
                                                const uint32_t *hist_map, uint32_t n_counter_rows,
                                                const uint32_t *counter_map, uint64_t *seq_out) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->comm_world < 2) return fail(ctx, LH_ERR_STATE, "lh_comm_import has not been called with world >= 2");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    const uint32_t W = ctx->comm_world;
    if (!frozen) return fail(ctx, LH_ERR_INVALID, "frozen is NULL");
    for (uint32_t r = 0; r < W; r++)
        if (frozen[r] > 1) return fail(ctx, LH_ERR_INVALID, "frozen[r] is not 0 or 1");
    if (frozen[ctx->comm_rank] != (uint32_t)(ctx->active ^ 1)) return fail(ctx, LH_ERR_INVALID, "frozen[rank] is not the buffer this snapshot froze");
    if (n_rows > ctx->H) return fail(ctx, LH_ERR_INVALID, "n_rows > max_histograms");
    if (n_counter_rows > ctx->C) return fail(ctx, LH_ERR_INVALID, "n_counter_rows > max_counters");
    if ((n_rows && !hist_map) || (n_counter_rows && !counter_map)) return fail(ctx, LH_ERR_INVALID, "map is NULL with rows");
    if (seq <= ctx->comm_seq) return fail(ctx, LH_ERR_INVALID, "seq does not exceed this context's last all-reduce");
    const size_t nh = (size_t)W * n_rows, nc = (size_t)W * n_counter_rows;
    for (size_t i = 0; i < nh; i++)
        if (hist_map[i] != LH_ROW_ABSENT && hist_map[i] >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram map entry >= max_histograms");
    for (size_t i = 0; i < nc; i++)
        if (counter_map[i] != LH_ROW_ABSENT && counter_map[i] >= ctx->C) return fail(ctx, LH_ERR_RANGE, "counter map entry >= max_counters");
    if (lh_status st = comm_alloc_row_maps(ctx)) return st;
    // the staging is rewritten only after the previous upload from it has run
    LH_CUDA(ctx, cudaEventSynchronize(ctx->row_maps_copied.get()));
    if (nh) memcpy(ctx->h_row_maps.get(), hist_map, nh * 4);
    if (nc) memcpy(ctx->h_row_maps.get() + nh, counter_map, nc * 4);
    cudaStream_t s = ctx->snap_stream.get();
    if (nh + nc) {
        LH_CUDA(ctx, cudaMemcpyAsync(ctx->d_row_maps.get(), ctx->h_row_maps.get(), (nh + nc) * 4, cudaMemcpyHostToDevice, s));
        ctx->stats.h2d_bytes += (nh + nc) * 4;
    }
    LH_CUDA(ctx, cudaEventRecord(ctx->row_maps_copied.get(), s));
    RowMap m{};
    m.hist = ctx->d_row_maps.get(); m.ctr = ctx->d_row_maps.get() + nh;
    m.n_rows = n_rows; m.n_counter_rows = n_counter_rows;
    for (uint32_t r = 0; r < W; r++) m.frozen_mask |= frozen[r] << r;
    return launch_allreduce(ctx, seq, frozen, n_rows, 1u, m, seq_out);
}

// =========================================================== multi-GPU (caller's all-reduce)
extern "C" lh_status lh_snapshot_row_levels(lh_ctx *ctx, uint8_t *levels) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    if (!levels) return fail(ctx, LH_ERR_INVALID, "levels is NULL");
    mark_rows_read(ctx);
    if (lh_status st = alloc_rows_staging(ctx)) return st;
    cudaStream_t s = ctx->snap_stream.get();
    LH_CUDA(ctx, cudaMemcpyAsync(ctx->h_rows_flags.get(), ctx->buf[ctx->active ^ 1].d_flags.get(), (size_t)ctx->H * 4, cudaMemcpyDeviceToHost, s));
    LH_CUDA(ctx, cudaStreamSynchronize(s));
    for (uint32_t h = 0; h < ctx->H; h++) {
        const uint32_t fl = ctx->h_rows_flags.get()[h];
        levels[h] = fl == 0 ? 0 : (fl & 2u) ? 3 : 1;
    }
    ctx->stats.d2h_bytes += (size_t)ctx->H * 4;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_pack_rows(lh_ctx *ctx, uint32_t n_rows, const uint32_t *hist_rows, const uint8_t *levels,
                                           uint32_t n_counter_rows, const uint32_t *counter_rows, uint64_t **d_send,
                                           uint64_t **d_recv, uint64_t *n_words, void **stream) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    if (ctx->rows_packed) return fail(ctx, LH_ERR_STATE, "this snapshot has already been packed");
    if (n_rows > ctx->H) return fail(ctx, LH_ERR_INVALID, "n_rows > max_histograms");
    if (n_counter_rows > ctx->C) return fail(ctx, LH_ERR_INVALID, "n_counter_rows > max_counters");
    if ((n_rows && (!hist_rows || !levels)) || (n_counter_rows && !counter_rows))
        return fail(ctx, LH_ERR_INVALID, "map or levels is NULL with rows");
    if (!d_send || !d_recv || !n_words || !stream) return fail(ctx, LH_ERR_INVALID, "an output pointer is NULL");
    for (uint32_t g = 0; g < n_rows; g++)
        if (levels[g] != 0 && levels[g] != 1 && levels[g] != 3) return fail(ctx, LH_ERR_INVALID, "a level is not 0, 1 or 3");
    for (uint32_t g = 0; g < n_rows; g++)
        if (hist_rows[g] != LH_ROW_ABSENT && hist_rows[g] >= ctx->H) return fail(ctx, LH_ERR_RANGE, "histogram row >= max_histograms");
    for (uint32_t g = 0; g < n_counter_rows; g++)
        if (counter_rows[g] != LH_ROW_ABSENT && counter_rows[g] >= ctx->C) return fail(ctx, LH_ERR_RANGE, "counter row >= max_counters");
    mark_rows_read(ctx);
    const size_t table_bytes = (size_t)ctx->H * sizeof(RowsEntry) + (size_t)ctx->C * 4;
    if (!ctx->d_rows_table.get()) {
        DevPtr<unsigned char> d; PinnedPtr<unsigned char> h; Event copied;
        LH_CUDA(ctx, cudaMalloc(d.out(), table_bytes));
        LH_CUDA(ctx, cudaMallocHost(h.out(), table_bytes));
        LH_CUDA(ctx, cudaEventCreateWithFlags(copied.out(), cudaEventDisableTiming));
        ctx->d_rows_table = std::move(d); ctx->h_rows_table = std::move(h); ctx->rows_table_copied = std::move(copied);
    }
    if (lh_status st = comm_alloc_reduced(ctx)) return st;
    // the layout: every rank computes the same offsets from the same levels
    const uint32_t wcells = 2u * ctx->pc.win - 1u;
    // the staging is rewritten only after the previous upload from it has run
    LH_CUDA(ctx, cudaEventSynchronize(ctx->rows_table_copied.get()));
    RowsEntry *tab = reinterpret_cast<RowsEntry *>(ctx->h_rows_table.get());
    uint64_t words = 0;
    for (uint32_t g = 0; g < n_rows; g++) {
        tab[g].row = hist_rows[g]; tab[g].level = levels[g]; tab[g].off = words;
        words += levels[g] == 0 ? 0u : levels[g] == 1 ? wcells : 65536u;
    }
    const uint64_t ctr_off = words;
    words += n_counter_rows;
    uint32_t *tab_ctr = reinterpret_cast<uint32_t *>(ctx->h_rows_table.get() + (size_t)n_rows * sizeof(RowsEntry));
    if (n_counter_rows) memcpy(tab_ctr, counter_rows, (size_t)n_counter_rows * 4);
    if (words > ctx->rows_cap) {
        // even, so that the 16-byte granule of the last word is inside the allocation
        const size_t cap = (words + 1) & ~(size_t)1;
        ctx->d_rows_send.reset(); ctx->d_rows_recv.reset(); ctx->rows_cap = 0;
        DevPtr<unsigned long long> send, recv;
        LH_CUDA(ctx, cudaMalloc(send.out(), cap * 8));
        LH_CUDA(ctx, cudaMalloc(recv.out(), cap * 8));
        ctx->d_rows_send = std::move(send); ctx->d_rows_recv = std::move(recv); ctx->rows_cap = cap;
    }
    cudaStream_t s = ctx->snap_stream.get();
    const size_t up = (size_t)n_rows * sizeof(RowsEntry) + (size_t)n_counter_rows * 4;
    if (up) {
        LH_CUDA(ctx, cudaMemcpyAsync(ctx->d_rows_table.get(), ctx->h_rows_table.get(), up, cudaMemcpyHostToDevice, s));
        ctx->stats.h2d_bytes += up;
    }
    LH_CUDA(ctx, cudaEventRecord(ctx->rows_table_copied.get(), s));
    if (words) {
        const int f = ctx->active ^ 1;
        const size_t items = (size_t)n_rows * ROWS_PER_ROW + (n_counter_rows ? 1 : 0);
        const int grid = (int)std::min<size_t>(items, (size_t)ctx->sm_count * 8);
        const RowsEntry *dtab = reinterpret_cast<const RowsEntry *>(ctx->d_rows_table.get());
        k_rows_pack<<<grid, ROWS_THREADS, 0, s>>>(dtab, n_rows, ctx->pc.win, ctx->buf[f].d_buckets.get(),
                                                   reinterpret_cast<const uint32_t *>(dtab + n_rows), n_counter_rows,
                                                   ctx->buf[f].d_counters.get(), ctr_off, ctx->d_rows_send.get());
        LH_CUDA(ctx, cudaGetLastError());
        ctx->stats.kernel_launches++;
    }
    ctx->rows_packed = true;
    ctx->rows_n = n_rows; ctx->rows_nc = n_counter_rows; ctx->rows_words = words;
    *d_send = reinterpret_cast<uint64_t *>(ctx->d_rows_send.get());
    *d_recv = reinterpret_cast<uint64_t *>(ctx->d_rows_recv.get());
    *n_words = words;
    *stream = s;
    return LH_OK;
}

extern "C" lh_status lh_snapshot_unpack_rows(lh_ctx *ctx, uint32_t summed) {
    LH_ENTER(ctx);
    if (!ctx->frozen) return fail(ctx, LH_ERR_STATE, "no snapshot in progress");
    if (ctx->view_reduced) return fail(ctx, LH_ERR_STATE, "this snapshot has already been all-reduced");
    if (!ctx->rows_packed) return fail(ctx, LH_ERR_STATE, "this snapshot has not been packed");
    cudaStream_t s = ctx->snap_stream.get();
    const uint32_t n_rows = ctx->rows_n;
    const uint64_t ctr_off = ctx->rows_words - ctx->rows_nc;
    const size_t items = std::max<size_t>((size_t)n_rows * ROWS_PER_ROW, 1);
    const int grid = (int)std::min<size_t>(items, (size_t)ctx->sm_count * 8);
    k_rows_unpack<<<grid, ROWS_THREADS, 0, s>>>(reinterpret_cast<const RowsEntry *>(ctx->d_rows_table.get()), n_rows,
                                                ctx->pc.win, summed ? ctx->d_rows_recv.get() : ctx->d_rows_send.get(),
                                                ctx->rows_nc, ctx->C, ctr_off, ctx->d_red_buckets.get(),
                                                ctx->d_red_flags.get(), ctx->d_red_counters.get());
    LH_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches++;
    ctx->view_reduced = true;
    ctx->view_counters_reduced = true;
    ctx->nnz_valid = false;
    return LH_OK;
}

extern "C" lh_status lh_comm_allreduce_ms(lh_ctx *ctx, uint64_t seq, float *ms) {
    if (!ctx || !ms) return LH_ERR_INVALID;
    cudaEvent_t e0, e1;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (seq == 0 || seq > ctx->comm_seq || ctx->comm_seq - seq >= (uint64_t)lh_ctx::kCommRing)
            return fail(ctx, LH_ERR_STATE, "that all-reduce is unknown or its events were recycled");
        const int ring = (int)(seq % lh_ctx::kCommRing);
        e0 = ctx->comm_t0[ring].get(); e1 = ctx->comm_t1[ring].get();
    }
    cudaError_t e = cudaEventSynchronize(e1);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_comm_allreduce_ms", e);
    return LH_OK;
}

extern "C" lh_status lh_comm_info(lh_ctx *ctx, lh_comm_stats *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    memset(out, 0, sizeof *out);
    out->rank = ctx->comm_rank; out->world = ctx->comm_world; out->allreduces = ctx->comm_seq;
    if (ctx->comm_world >= 2) {
        unsigned int aux[2] = {0, 0};
        LH_CUDA(ctx, cudaMemcpy(aux, ctx->d_comm_aux.get(), 8, cudaMemcpyDeviceToHost));
        out->status = aux[1];
        // bytes this rank read from its peers in the last all-reduce: window (or dense) cells of every touched histogram
        unsigned long long cells = 0;
        LH_CUDA(ctx, cudaMemcpy(&cells, ctx->d_comm_aux.get() + 2, 8, cudaMemcpyDeviceToHost));
        // one-shot: every cell from every peer; two-shot: this rank's 1/world of the cells from every peer (and as much pushed back)
        out->last_bytes_from_peers = ctx->comm_two_shot ? cells * 8u * (ctx->comm_world - 1) / ctx->comm_world : cells * 8u * (ctx->comm_world - 1);
    }
    return LH_OK;
}

extern "C" const char *lh_keyed_kernel_name(lh_ctx *ctx) { return ctx ? ctx->keyed_kernel : ""; }

// =========================================================== probes
extern "C" lh_status lh_compress_f64(lh_ctx *ctx, const double *d_values, size_t n, int16_t *d_out, int mode, void *stream) {
    LH_ENTER(ctx);
    if (n && (!d_values || !d_out)) return fail(ctx, LH_ERR_INVALID, "NULL input");
    if (!n) return LH_OK;
    cudaStream_t s = pick_stream(ctx, stream);
    k_compress_probe<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_values, n, d_out, mode, ctx->pc);
    LH_CUDA(ctx, cudaGetLastError());
    return LH_OK;
}

extern "C" lh_status lh_decompress_table(lh_ctx *ctx, double *h_out) {
    LH_ENTER(ctx);
    if (!h_out) return fail(ctx, LH_ERR_INVALID, "h_out is NULL");
    LH_CUDA(ctx, cudaMemcpy(h_out, ctx->d_decomp.get(), 65536 * sizeof(double), cudaMemcpyDeviceToHost));
    return LH_OK;
}

extern "C" lh_status lh_fastpath_margin(lh_ctx *ctx, const double *d_values, size_t n, double *h_max_err, uint64_t *h_n_slow, void *stream) {
    LH_ENTER(ctx);
    if (n && !d_values) return fail(ctx, LH_ERR_INVALID, "NULL input");
    cudaStream_t s = pick_stream(ctx, stream);
    DevPtr<unsigned long long> d;
    LH_CUDA(ctx, cudaMalloc(d.out(), 24));
    LH_CUDA(ctx, cudaMemsetAsync(d.get(), 0, 24, s));
    if (n) k_fastpath_margin<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_values, n, d.get(), ctx->pc);
    unsigned long long h[3];
    cudaError_t e = cudaMemcpyAsync(h, d.get(), 24, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_fastpath_margin", e);
    // the larger of the two estimators' errors (positive doubles order like their bit patterns)
    const unsigned long long worst = std::max(h[0], h[2]);
    if (h_max_err) memcpy(h_max_err, &worst, 8);
    if (h_n_slow) *h_n_slow = h[1];
    ctx->last_margin[0] = h[0]; ctx->last_margin[1] = h[2];
    return LH_OK;
}

// the two estimators' errors of the last lh_fastpath_margin call, separately (bucket units)
extern "C" lh_status lh_fastpath_margin_detail(lh_ctx *ctx, double *h_err_estimator1, double *h_err_estimator2) {
    LH_ENTER(ctx);
    if (h_err_estimator1) memcpy(h_err_estimator1, &ctx->last_margin[0], 8);
    if (h_err_estimator2) memcpy(h_err_estimator2, &ctx->last_margin[1], 8);
    return LH_OK;
}

// every cell of the fast window at every precision of [p_lo, p_hi], one launch of k_fastpath_certify per precision
extern "C" lh_status lh_fastpath_certify(lh_ctx *ctx, uint32_t p_lo, uint32_t p_hi, lh_certify_form *h_out) {
    LH_ENTER(ctx);
    static_assert(sizeof(lh_certify_form) == FC_FIELDS * 8, "lh_certify_form mirrors the FC_* words");
    if (!h_out) return fail(ctx, LH_ERR_INVALID, "h_out is NULL");
    if (p_lo < 1 || p_hi > LH_MAX_PRECISION || p_lo > p_hi) return fail(ctx, LH_ERR_RANGE, "precisions must satisfy 1 <= p_lo <= p_hi <= 250");
    const size_t rows = (size_t)(p_hi - p_lo + 1) * FC_FORMS;
    std::vector<unsigned long long> h(rows * FC_FIELDS, 0ull);
    for (size_t r = 0; r < rows; r++) h[r * FC_FIELDS + FC_MIN_MARGIN] = 0x7FF0000000000000ull;   // +Inf
    cudaStream_t s = ctx->ingest_stream.get();
    DevPtr<unsigned long long> d;
    LH_CUDA(ctx, cudaMalloc(d.out(), h.size() * 8));
    cudaError_t e = cudaMemcpyAsync(d.get(), h.data(), h.size() * 8, cudaMemcpyHostToDevice, s);
    for (uint32_t p = p_lo; p <= p_hi && e == cudaSuccess; p++) {
        k_fastpath_certify<<<ctx->sm_count * 8, FC_THREADS, 0, s>>>(d.get() + (size_t)(p - p_lo) * FC_FORMS * FC_FIELDS, make_prec(p));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h.data(), d.get(), h.size() * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_fastpath_certify", e);
    memcpy(h_out, h.data(), h.size() * 8);
    return LH_OK;
}

// =========================================================== streams
extern "C" lh_status lh_gen_stream_f64(lh_ctx *ctx, int kind, uint64_t seed, uint64_t start, size_t n, double *d_out, void *stream) {
    LH_ENTER(ctx);
    if (n && !d_out) return fail(ctx, LH_ERR_INVALID, "d_out is NULL");
    if (!n) return LH_OK;
    k_gen_stream<<<ctx->sm_count * 8, 256, 0, pick_stream(ctx, stream)>>>(kind, seed, start, n, d_out);
    LH_CUDA(ctx, cudaGetLastError());
    return LH_OK;
}
extern "C" lh_status lh_gen_ids_u16(lh_ctx *ctx, int kind, uint64_t seed, uint64_t start, size_t n, uint32_t n_ids, uint16_t *d_out, void *stream) {
    LH_ENTER(ctx);
    if (n && !d_out) return fail(ctx, LH_ERR_INVALID, "d_out is NULL");
    if (n_ids == 0 || n_ids > 65536) return fail(ctx, LH_ERR_RANGE, "n_ids must be in 1..65536");
    if (!n) return LH_OK;
    k_gen_ids_u16<<<ctx->sm_count * 8, 256, 0, pick_stream(ctx, stream)>>>(kind, seed, start, n, n_ids, d_out);
    LH_CUDA(ctx, cudaGetLastError());
    return LH_OK;
}

// =========================================================== misc
extern "C" lh_status lh_get_stats(lh_ctx *ctx, lh_stats *out) {
    LH_ENTER(ctx);
    if (!out) return fail(ctx, LH_ERR_INVALID, "out is NULL");
    unsigned long long dropped = 0;
    LH_CUDA(ctx, cudaMemcpy(&dropped, ctx->d_dropped.get(), 8, cudaMemcpyDeviceToHost));
    ctx->stats.dropped = dropped;
    *out = ctx->stats;
    return LH_OK;
}
extern "C" lh_status lh_sync(lh_ctx *ctx) {
    LH_ENTER(ctx);
    // this context's work only (its three streams and every caller stream that carried an ingest), not the whole
    // device: another context on the same GPU may be inside a collective that waits for THIS caller's next step
    std::vector<cudaStream_t> streams = {ctx->ingest_stream.get(), ctx->copy_stream.get(), ctx->snap_stream.get()};
    for (int b = 0; b < 2; b++)
        for (auto &w : ctx->buf[b].writers)
            if (std::find(streams.begin(), streams.end(), w.stream) == streams.end()) streams.push_back(w.stream);
    _lk.unlock();
    cudaError_t e = cudaSuccess;
    for (cudaStream_t st : streams) { cudaError_t x = cudaStreamSynchronize(st); if (e == cudaSuccess) e = x; }
    _lk.lock();
    if (e != cudaSuccess) return fail(ctx, LH_ERR_CUDA, "lh_sync", e);
    for (auto &sl : ctx->slots)
        if (sl.state == SLOT_INFLIGHT && cudaEventQuery(sl.done.get()) == cudaSuccess) sl.state = SLOT_FREE;
    cudaGetLastError();
    return LH_OK;
}
extern "C" void *lh_ingest_stream(lh_ctx *ctx) { return ctx ? (void *)ctx->ingest_stream.get() : nullptr; }

extern "C" lh_status lh_device_alloc(lh_ctx *ctx, size_t bytes, void **d_out) {
    LH_ENTER(ctx);
    if (!d_out) return fail(ctx, LH_ERR_INVALID, "d_out is NULL");
    cudaError_t e = cudaMalloc(d_out, bytes ? bytes : 1);
    if (e != cudaSuccess) return fail(ctx, e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA, "cudaMalloc", e);
    return LH_OK;
}
extern "C" lh_status lh_device_free(lh_ctx *ctx, void *d_ptr) {
    LH_ENTER(ctx);
    LH_CUDA(ctx, cudaFree(d_ptr));
    return LH_OK;
}
extern "C" lh_status lh_host_alloc_pinned(lh_ctx *ctx, size_t bytes, void **h_out) {
    LH_ENTER(ctx);
    if (!h_out) return fail(ctx, LH_ERR_INVALID, "h_out is NULL");
    cudaError_t e = cudaMallocHost(h_out, bytes ? bytes : 1);
    if (e != cudaSuccess) return fail(ctx, e == cudaErrorMemoryAllocation ? LH_ERR_NOMEM : LH_ERR_CUDA, "cudaMallocHost", e);
    return LH_OK;
}
extern "C" lh_status lh_host_free_pinned(lh_ctx *ctx, void *h_ptr) {
    LH_ENTER(ctx);
    LH_CUDA(ctx, cudaFreeHost(h_ptr));
    return LH_OK;
}
extern "C" lh_status lh_memcpy_h2d(lh_ctx *ctx, void *d_dst, const void *h_src, size_t bytes) {
    LH_ENTER(ctx);
    LH_CUDA(ctx, cudaMemcpy(d_dst, h_src, bytes, cudaMemcpyHostToDevice));
    // From pageable memory cudaMemcpy may return once the source is staged, before the DMA has reached d_dst, and it
    // runs on the legacy stream, which the context's (and torch's) non-blocking streams are not ordered after: wait
    // for the DMA, so that a kernel on any stream may read d_dst as soon as this returns.
    LH_CUDA(ctx, cudaStreamSynchronize(cudaStreamLegacy));
    return LH_OK;
}
extern "C" lh_status lh_memcpy_d2h(lh_ctx *ctx, void *h_dst, const void *d_src, size_t bytes) {
    LH_ENTER(ctx);
    LH_CUDA(ctx, cudaMemcpy(h_dst, d_src, bytes, cudaMemcpyDeviceToHost));
    return LH_OK;
}

extern "C" lh_status lh_tune(lh_ctx *ctx, const char *key, int64_t value) {
    LH_ENTER(ctx);
    if (!key) return fail(ctx, LH_ERR_INVALID, "key is NULL");
    if (!strcmp(key, "k1")) {
        if (value < 0 || value >= kNumK1Variants) return fail(ctx, LH_ERR_RANGE, "unknown k1 variant");
        ctx->k1_variant = (int)value;
        return LH_OK;
    }
    if (!strcmp(key, "k1_grid_mult")) {
        if (value < 1 || value > 64) return fail(ctx, LH_ERR_RANGE, "k1_grid_mult out of range");
        ctx->k1_grid_mult = (int)value;
        return LH_OK;
    }
    if (!strcmp(key, "k1_reserve_sms")) {
        if (value < 0 || value >= ctx->sm_count) return fail(ctx, LH_ERR_RANGE, "k1_reserve_sms out of range");
        ctx->k1_reserve_sms = (int)value;
        return LH_OK;
    }
    if (!strcmp(key, "keyed_mode")) {
        if (value < 0 || value > 2) return fail(ctx, LH_ERR_RANGE, "keyed_mode is 0 (auto), 1 (L2 atomics) or 2 (owner-partitioned, write-combining)");
        ctx->keyed_mode = (int)value;
        return LH_OK;
    }
    if (!strcmp(key, "wc_pf")) {
        if (value < 0 || value > 8) return fail(ctx, LH_ERR_RANGE, "wc_pf is 0 ... 8 tiles");
        ctx->wc_pf_tiles = (uint32_t)value;
        return LH_OK;
    }
    if (!strcmp(key, "wc_flush")) {
        if (value < 4096 || value > 65536) return fail(ctx, LH_ERR_RANGE, "wc_flush is 4096 ... 65536 samples");
        ctx->wc_flush_samples = (uint32_t)value;
        return LH_OK;
    }
    if (!strcmp(key, "wc_spt")) {
        if (value != 4 && value != 6 && value != 3 && value != 8)
            return fail(ctx, LH_ERR_RANGE, "wc_spt is a shape code: 6 (896 threads x 4 samples), 4 (1024 x 4), 3 (768 x 4) or 8 (512 x 8)");
        ctx->wc_spt = (int)value;
        return LH_OK;
    }
    if (!strcmp(key, "kp_chunk")) {
        if (value < (1 << 16) || value > ((int64_t)1 << 28)) return fail(ctx, LH_ERR_RANGE, "kp_chunk out of range");
        ctx->kp_chunk = value;
        return LH_OK;
    }
    if (!strcmp(key, "gpu_timer_slots")) {
        if (value < 1 || value > (1 << 20)) return fail(ctx, LH_ERR_RANGE, "gpu_timer_slots is 1 ... 2^20");
        if (ctx->d_timer_marks.get()) return fail(ctx, LH_ERR_STATE, "gpu_timer_slots is set before the first lh_gpu_timer_start");
        ctx->timer_slots_n = (uint32_t)value;
        return LH_OK;
    }
    if (!strcmp(key, "keyed_blocks_per_sm")) {
        if (value < 1 || value > 32) return fail(ctx, LH_ERR_RANGE, "keyed_blocks_per_sm out of range");
        ctx->keyed_blocks_per_sm = (int)value;
        return LH_OK;
    }
    return fail(ctx, LH_ERR_INVALID, "unknown tuning key");
}

extern "C" int32_t lh_k1_variant_count(void) { return kNumK1Variants; }
extern "C" int32_t lh_k1_variant_current(lh_ctx *ctx) { return ctx ? ctx->k1_variant : -1; }
extern "C" const char *lh_k1_variant_name(lh_ctx *ctx, int32_t i) {
    if (!ctx || i < 0 || i >= kNumK1Variants) return "";
    return ctx->k1[i].name;
}

extern "C" uint64_t lh_ingest_seq(lh_ctx *ctx) {
    if (!ctx) return 0;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return ctx->ingest_seq;
}

extern "C" lh_status lh_kernel_ms(lh_ctx *ctx, uint64_t seq, float *ms) {
    LH_ENTER(ctx);
    if (!ms) return fail(ctx, LH_ERR_INVALID, "ms is NULL");
    if (seq == 0 || seq > ctx->ingest_seq || ctx->ingest_seq - seq >= (uint64_t)lh_ctx::kTimingRing)
        return fail(ctx, LH_ERR_STATE, "that ingest launch is unknown or its events were recycled");
    const int i = (int)((seq - 1) % lh_ctx::kTimingRing);
    LH_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1s[i].get()));
    LH_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev_t0s[i].get(), ctx->ev_t1s[i].get()));
    return LH_OK;
}

extern "C" lh_status lh_last_kernel_ms(lh_ctx *ctx, float *ms) {
    LH_ENTER(ctx);
    if (!ms) return fail(ctx, LH_ERR_INVALID, "ms is NULL");
    if (!ctx->timing_valid) return fail(ctx, LH_ERR_STATE, "no ingest kernel has been launched");
    LH_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1));
    LH_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev_t0, ctx->ev_t1));
    return LH_OK;
}
