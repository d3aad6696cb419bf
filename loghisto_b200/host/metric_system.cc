// metric_system.cc -- see metric_system.h.  Host glue only: interning, batching into the pinned staging
// ring, rebuilding RawMetricSet / ProcessedMetricSet from what the device returns.
#include "metric_system.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <sys/syscall.h>
#include <unistd.h>
#include <cstring>
#include <limits>
#include <stdexcept>

#include "../../include/loghisto_b200.h"

// Bound weakly, so that the mirror still loads over a build of the C ABI without this entry point (an older
// libloghisto_b200.so, or a stand-in that implements only the snapshot path); processMetrics then refuses the
// histograms of sets this system did not collect instead of failing to load.
#pragma weak lh_reduce_sparse_host
// Likewise for record scopes: over a build without them, BeginRecording throws.
#pragma weak lh_record_begin
#pragma weak lh_record_end
#pragma weak lh_ingest_f64
#pragma weak lh_ingest_batch
// And for GPU timers: over a build without them, StartGpuTimer hands out tokens whose Stop drops and counts.
#pragma weak lh_gpu_timer_start
#pragma weak lh_gpu_timer_stop
#pragma weak lh_gpu_timer_release
// And for graph recorders: over a build without them, NewGraphRecorder throws.
#pragma weak lh_graph_recorder_create
#pragma weak lh_graph_recorder_bind
#pragma weak lh_graph_recorder_ingest
#pragma weak lh_graph_recorder_destroy
// The later graph recorder calls: over a build without them, the GraphRecorder method that needs one throws.
#pragma weak lh_graph_recorder_ingest_keyed_u16
#pragma weak lh_graph_recorder_ingest_keyed_u32
#pragma weak lh_graph_recorder_counter_add_u16
#pragma weak lh_graph_recorder_counter_add_u32
#pragma weak lh_graph_recorder_timer_start
#pragma weak lh_graph_recorder_timer_stop
// Arrays of any gauge dtype: over a build without them, RecordScope::Arrays / GraphRecorder::Arrays throw.
#pragma weak lh_ingest_arrays
#pragma weak lh_graph_recorder_ingest_arrays

#pragma weak lh_ingest_keyed_mapped_u16
#pragma weak lh_ingest_keyed_mapped_u32
#pragma weak lh_counter_add_mapped_u16
#pragma weak lh_counter_add_mapped_u32
// And for device subscriptions: over a build without them, NewDeviceSubscription throws.
#pragma weak lh_board_create
#pragma weak lh_snapshot_publish
#pragma weak lh_board_read
#pragma weak lh_board_destroy
// And for raw device subscriptions: over a build without them, NewRawDeviceSubscription throws.
#pragma weak lh_raw_board_create
#pragma weak lh_snapshot_publish_raw
#pragma weak lh_raw_percentiles_grid
#pragma weak lh_raw_ranks_grid
#pragma weak lh_raw_board_destroy
#pragma weak lh_raw_board_create_window   // window boards: over a build without them, a window other than 1 throws
// And for device gauges: over a build without them, RegisterDeviceGauge throws.
#pragma weak lh_gauges_read
// And for joined ranks: over a build without them, JoinRanks throws.
#pragma weak lh_comm_export
#pragma weak lh_comm_import
#pragma weak lh_comm_info
#pragma weak lh_snapshot_copy_histogram
#pragma weak lh_snapshot_rows
#pragma weak lh_snapshot_allreduce_rows
// And for joined ranks through the caller's all-reduce: over a build without them, that JoinRanks throws.
#pragma weak lh_snapshot_row_levels
#pragma weak lh_snapshot_pack_rows
#pragma weak lh_snapshot_unpack_rows
// And for distribution gauges: over a build without them, RegisterDeviceDistribution throws.
#pragma weak lh_snapshot_ingest_arrays

namespace loghisto {

// an open graph recorder, shared by its GraphRecorder and the system's list of open recorders
struct GraphRecorder::State {
    MetricSystem *ms;                   // nullptr once closed (or once the system is gone)
    lh_graph_recorder g{};
    std::vector<std::string> hnames, cnames;
};

// an open device subscription, shared by its DeviceSubscription and the system's list of open subscriptions
struct DeviceSubscription::State {
    MetricSystem *ms;                   // nullptr once closed (or once the system is gone)
    lh_board b{};
    std::vector<std::string> hnames, cnames;
};

// an open raw device subscription, shared like DeviceSubscription::State
struct RawDeviceSubscription::State {
    MetricSystem *ms;                   // nullptr once closed (or once the system is gone)
    lh_raw_board b{};
    std::vector<std::string> hnames;
    uint32_t window = 1;
};

namespace {

std::string format_label(const std::string &label, const std::string &name) {   // fmt.Sprintf(label, name), one %s
    size_t p = label.find("%s");
    if (p == std::string::npos) return label;
    return label.substr(0, p) + name + label.substr(p + 2);
}

// uint64(float64) as the Go compiler lowers it on amd64 (metrics.go:374): CVTTSD2SQ below 2^63
// (negative values wrap two's-complement), subtract-2^63 path above.
uint64_t go_f64_to_u64(double x) {
    if (x < 9223372036854775808.0) {
        if (!(x > -9223372036854777856.0)) return 0x8000000000000000ull;
        return (uint64_t)(int64_t)x;
    }
    if (!(x < 18446744073709551616.0)) return 0;
    return (uint64_t)(int64_t)(x - 9223372036854775808.0) ^ 0x8000000000000000ull;
}

void check(lh_ctx *ctx, lh_status st, const char *what) {
    if (st != LH_OK) {
        std::string msg = std::string(what) + ": " + lh_strerror(st);
        if (ctx) msg += std::string(" (") + lh_last_error(ctx) + ")";
        throw std::runtime_error(msg);
    }
}

// ---- asymmetric owner / reaper exclusion ------------------------------------------------------------------
// A staging shard that belongs to ONE thread is entered by that thread with plain stores (no locked instruction on
// the per-call path: on x86 a locked RMW waits for every store in flight, i.e. for the cache misses of the pinned
// buffer it just wrote).  The reaper, which needs the shard once per interval, raises `reaper_wants`, forces a full
// barrier on every thread of the process with membarrier(PRIVATE_EXPEDITED), and then waits for `owner_busy` to
// drop: the Dekker handshake with the expensive half moved to the side that runs once per interval.  Where the
// syscall is unavailable (or LOGHISTO_B200_SHARD_LOCK=1) every shard falls back to its spinlock.
constexpr int kMembarrierQuery = 0, kMembarrierPrivateExpedited = 1 << 3, kMembarrierRegisterPrivateExpedited = 1 << 4;
bool asym_available() {
    if (const char *e = getenv("LOGHISTO_B200_SHARD_LOCK")) if (e[0] == '1') return false;   // read per system: A/B runs in one process
    static const bool ok = [] {
#ifdef __NR_membarrier
        const long q = syscall(__NR_membarrier, kMembarrierQuery, 0);
        if (q < 0 || !(q & kMembarrierPrivateExpedited)) return false;
        return syscall(__NR_membarrier, kMembarrierRegisterPrivateExpedited, 0) == 0;
#else
        return false;
#endif
    }();
    return ok;
}
void asym_barrier() {
#ifdef __NR_membarrier
    syscall(__NR_membarrier, kMembarrierPrivateExpedited, 0);
#endif
}

// live systems by id: a thread that ends (or moves to another system) hands its exclusive shard back through this
std::mutex g_reg_mu;
std::unordered_map<uint64_t, MetricSystem *> g_systems;

size_t next_thread_slot() {
    static std::atomic<size_t> next{0};
    return next.fetch_add(1);
}

// ---- per-thread name -> id cache --------------------------------------------------------------------------
// The reference pays an RWMutex RLock/RUnlock (two atomic RMWs on ONE shared cache line) plus two string-hashed
// map lookups per sample (metrics.go:275-279); that line ping-pongs between cores and caps multi-core ingest.
// Here the steady-state lookup touches only thread-local memory: a direct-mapped cache keyed by the hash of the
// name's bytes, verified byte for byte (a collision can never send a sample to the wrong histogram).  A miss falls
// back to the shared intern table (the reference's RLock / double-checked Lock idiom, metrics.go:275-294).
// Fixed-size loads only: a memcpy of a run-time length is a library call, and it was most of the cost of a lookup.
inline uint64_t load8(const char *p) { uint64_t w; memcpy(&w, p, 8); return w; }
inline uint64_t load_1to7(const char *p, size_t n) {        // n in 1..7, reads only p[0..n)
    if (n >= 4) {
        uint32_t a, b;
        memcpy(&a, p, 4);
        memcpy(&b, p + n - 4, 4);
        return (uint64_t)a | ((uint64_t)b << 32);
    }
    return (uint64_t)(uint8_t)p[0] | ((uint64_t)(uint8_t)p[n >> 1] << 8) | ((uint64_t)(uint8_t)p[n - 1] << 16);
}
// the (at most) 16 bytes of a short name as two words that determine them given the length
inline void short_words(const char *p, size_t n, uint64_t *w0, uint64_t *w1) {
    if (n >= 8) { *w0 = load8(p); *w1 = load8(p + n - 8); }
    else { *w0 = n ? load_1to7(p, n) : 0; *w1 = 0; }
}
inline uint64_t hash_bytes(const char *p, size_t n) {
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (n * 0xFF51AFD7ED558CCDull);
    const char *q = p;
    size_t m = n;
    while (m >= 8) {
        h = (h ^ load8(q)) * 0xC2B2AE3D27D4EB4Full;
        h ^= h >> 29;
        q += 8; m -= 8;
    }
    if (m) {                                                 // the tail: an overlapping 8-byte load when the name allows it
        const uint64_t w = n >= 8 ? load8(p + n - 8) : load_1to7(q, m);
        h = (h ^ w) * 0xC2B2AE3D27D4EB4Full;
        h ^= h >> 29;
    }
    // full avalanche: the table index is the LOW bits, and the bytes that tell "histogram7" from "histogram1023" sit in
    // the high half of the overlapping tail word
    h ^= h >> 33;
    h *= 0xFF51AFD7ED558CCDull;
    h ^= h >> 33;
    return h;
}

struct NameCache {
    // open addressing, linear probing, load factor <= 1/2: a name that was interned once is found without ever going
    // back to the shared table (a direct-mapped cache thrashes as soon as two hot names collide).  Entries are 48
    // bytes; the names' bytes live in an append-only arena owned by the cache.  An entry holds the id's generation
    // too: the append re-checks it, and refreshes the entry through put() when the id was retired since.
    struct Entry {                               // id_plus1 == 0: empty
        uint64_t hash; const char *name; uint32_t len; uint32_t id_plus1;
        uint64_t w0, w1;                         // short_words() of a name of at most 16 bytes: it never touches the arena
        uint32_t gen;
        bool matches(uint64_t h, const char *p, size_t n) const {
            if (hash != h || len != n) return false;
            if (n <= 16) {
                uint64_t a0, a1;
                short_words(p, n, &a0, &a1);
                return a0 == w0 && a1 == w1;
            }
            return memcmp(name, p, n) == 0;
        }
    };
    std::vector<Entry> e;
    std::vector<std::unique_ptr<char[]>> arena;
    size_t arena_left = 0;
    char *arena_next = nullptr;
    size_t count = 0;
    const Entry *last = nullptr;                 // most recently found entry: a thread that repeats one name skips the hash
    bool find_last(const char *p, size_t n, uint32_t *id, uint32_t *gen) const {
        const Entry *x = last;
        if (x && x->len == n) {
            bool same;
            if (n <= 16) { uint64_t a0, a1; short_words(p, n, &a0, &a1); same = a0 == x->w0 && a1 == x->w1; }
            else same = memcmp(x->name, p, n) == 0;
            if (same) { *id = x->id_plus1 - 1; *gen = x->gen; return true; }
        }
        return false;
    }
    Entry *probe(uint64_t h, const char *p, size_t n) {
        if (e.empty()) return nullptr;
        const size_t mask = e.size() - 1;
        for (size_t i = h & mask;; i = (i + 1) & mask) {
            Entry &x = e[i];
            if (!x.id_plus1) return nullptr;
            if (x.matches(h, p, n)) return &x;
        }
    }
    bool find(uint64_t h, const char *p, size_t n, uint32_t *id, uint32_t *gen) {
        const Entry *x = probe(h, p, n);
        if (!x) return false;
        *id = x->id_plus1 - 1; *gen = x->gen; last = x;
        return true;
    }
    void insert_raw(const Entry &en) {
        const size_t mask = e.size() - 1;
        size_t i = en.hash & mask;
        while (e[i].id_plus1) i = (i + 1) & mask;
        e[i] = en;
    }
    void put(uint64_t h, const char *p, size_t n, uint32_t id, uint32_t gen) {
        if (Entry *x = probe(h, p, n)) { x->id_plus1 = id + 1; x->gen = gen; return; }   // refresh in place
        if (e.empty()) e.assign(256, Entry{});
        last = nullptr;
        if ((count + 1) * 2 > e.size()) {        // grow and rehash
            std::vector<Entry> old(e.size() * 2, Entry{});
            old.swap(e);
            for (const Entry &x : old) if (x.id_plus1) insert_raw(x);
        }
        if (n > arena_left) {
            const size_t block = std::max<size_t>(n, 16384);
            arena.emplace_back(new char[block]);
            arena_next = arena.back().get();
            arena_left = block;
        }
        memcpy(arena_next, p, n);
        Entry en{};
        en.hash = h; en.name = arena_next; en.len = (uint32_t)n; en.id_plus1 = id + 1; en.gen = gen;
        if (n <= 16) short_words(p, n, &en.w0, &en.w1);
        insert_raw(en);
        arena_next += n; arena_left -= n;
        count++;
    }
    void reset() { last = nullptr; e.clear(); arena.clear(); arena_left = 0; arena_next = nullptr; count = 0; }
};

// Everything a thread needs on the per-call path, reached through ONE thread-local pointer (a plain pointer has no
// initialisation guard; the object behind it is created on the thread's first call and freed when the thread ends).
struct ThreadState {
    uint64_t system_id = 0;                      // which MetricSystem `shard` and the caches belong to
    void *shard = nullptr;                       // MetricSystem::Shard * of this thread
    bool exclusive = false;                      // the shard is this thread's alone (handed back when the thread ends)
    size_t slot = 0;                             // process-wide thread number
    NameCache h, c;
};
void release_thread_shard(ThreadState *ts) {
    if (!ts->shard || !ts->exclusive) return;
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_systems.find(ts->system_id);
    if (it != g_systems.end()) it->second->release_shard(ts->shard);
    ts->shard = nullptr;
    ts->exclusive = false;
}
thread_local ThreadState *tl_state = nullptr;
struct ThreadStateOwner {                        // destroyed at thread exit
    ThreadState *p = nullptr;
    ~ThreadStateOwner() {
        if (p) release_thread_shard(p);
        delete p;
        p = nullptr;
        tl_state = nullptr;                      // a later thread-local destructor that still records a sample starts over
    }
};
thread_local ThreadStateOwner tl_owner;
ThreadState *make_thread_state() {
    tl_owner.p = new ThreadState();
    tl_owner.p->slot = next_thread_slot();
    tl_state = tl_owner.p;
    return tl_state;
}

std::atomic<uint64_t> g_system_ids{1};

}  // namespace

// One staging shard: a pinned staging slot for (id, value) samples and one for (id, amount) counter ops, filled
// with plain stores.  Threads map onto shards round-robin (one shard per hardware thread by default), so in the
// steady state a shard has ONE writer and its spinlock is uncontended (an exchange and a store, ~10 ns); the reaper
// takes it once per interval to commit whatever is open.
struct alignas(128) MetricSystem::Shard {     // its own cache-line pair: nothing else on the heap shares the lines its owner writes on every call
    // exclusive shards (one owner thread): asymmetric handshake, see asym_available()
    std::atomic<uint32_t> owner_busy{0};     // written by the owner with plain stores
    std::atomic<uint32_t> reaper_wants{0};   // raised by a collecting thread
    bool exclusive = false;
    // shared shards (more threads than shards, or no membarrier): a spinlock
    std::atomic_flag busy = ATOMIC_FLAG_INIT;
    void lock() { while (busy.test_and_set(std::memory_order_acquire)) { __builtin_ia32_pause(); } }
    void unlock() { busy.clear(std::memory_order_release); }
    // histogram / timer samples
    lh_staging hs{};
    bool h_open = false;
    size_t h_n = 0, h_cap = 0;
    double *h_vals = nullptr;
    uint16_t *h_ids = nullptr;
    // counter ops
    lh_staging cs{};
    bool c_open = false;
    size_t c_n = 0, c_cap = 0;
    uint64_t *c_amounts = nullptr;
    uint16_t *c_ids = nullptr;
    std::vector<uint8_t> c_touched;      // [max_counters] Counter(name, x) was called this interval, even with x == 0
    bool c_any_touched = false;
    std::atomic<uint64_t> dropped{0};    // samples lost to a failed staging call (never silent: dropped_samples())
    char pad[128];                       // keep neighbouring shards (and the adjacent-line prefetcher) off this one's cache lines
};

namespace {
struct ShardGuard {                      // the calling thread's OWN shard (or a shared one)
    MetricSystem::Shard &s;
    explicit ShardGuard(MetricSystem::Shard &sh) : s(sh) {
        if (!s.exclusive) { s.lock(); return; }
        for (;;) {
            s.owner_busy.store(1, std::memory_order_relaxed);
            std::atomic_signal_fence(std::memory_order_seq_cst);             // compiler only; the reaper's membarrier supplies the fence
            if (__builtin_expect(s.reaper_wants.load(std::memory_order_acquire) == 0, 1)) return;
            s.owner_busy.store(0, std::memory_order_release);                // a collect is flushing this shard (microseconds)
            while (s.reaper_wants.load(std::memory_order_acquire)) __builtin_ia32_pause();
        }
    }
    ~ShardGuard() {
        if (s.exclusive) s.owner_busy.store(0, std::memory_order_release);
        else s.unlock();
    }
};
struct ForeignGuard {                    // another thread's shard, after reaper_wants was raised and asym_barrier() ran
    MetricSystem::Shard &s;
    explicit ForeignGuard(MetricSystem::Shard &sh) : s(sh) {
        if (!s.exclusive) { s.lock(); return; }
        while (s.owner_busy.load(std::memory_order_acquire)) __builtin_ia32_pause();
    }
    ~ForeignGuard() {
        if (s.exclusive) s.reaper_wants.store(0, std::memory_order_release);
        else s.unlock();
    }
};
void log_once(std::atomic<bool> &flag, lh_ctx *ctx, lh_status st, const char *what) {
    if (!flag.exchange(true))
        fprintf(stderr, "loghisto: %s failed: %s (%s); samples are being dropped and counted\n", what, lh_strerror(st),
                ctx ? lh_last_error(ctx) : "");
}
std::atomic<bool> g_logged_staging{false};
}  // namespace

std::chrono::nanoseconds TimerToken::Stop() {
    auto d = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - Start);
    if (id_valid) System->histogram_id(Name, id, gen, (double)d.count());   // float64(duration.Nanoseconds()); name interned by StartTimer
    else System->Histogram(Name, (double)d.count());
    return d;
}

MetricSystem::MetricSystem(std::chrono::nanoseconds interval, bool /*sysStats*/, const Options &opt)
    : interval_(interval.count() > 0 ? interval : std::chrono::nanoseconds(1)), opt_(opt) {
    percentiles_ = {{"%s_min", 0.0}, {"%s_50", .5}, {"%s_75", .75}, {"%s_90", .9}, {"%s_95", .95},
                    {"%s_99", .99}, {"%s_99.9", .999}, {"%s_99.99", .9999}, {"%s_max", 1.0}};   // metrics.go:145-155
    // one shard per hardware thread: goroutines of print_benchmark.go:59-67 become OS threads here, each with its own
    // operational overrides (no recompile): LOGHISTO_B200_SHARDS, LOGHISTO_B200_STAGING_BYTES
    if (const char *e = getenv("LOGHISTO_B200_SHARDS")) { long v = atol(e); if (v > 0 && v <= 4096) opt_.shards = (uint32_t)v; }
    if (const char *e = getenv("LOGHISTO_B200_STAGING_BYTES")) { long long v = atoll(e); if (v >= 4096) opt_.staging_bytes = (uint64_t)v; }
    uint32_t nshards = opt_.shards ? opt_.shards : std::min<uint32_t>(std::max(1u, std::thread::hardware_concurrency()), 256u);
    system_id_ = g_system_ids.fetch_add(1);
    lh_config cfg{};
    cfg.struct_size = sizeof(cfg);
    cfg.device = opt.device;
    cfg.max_histograms = opt.max_histograms;
    cfg.max_counters = opt.max_counters;
    cfg.staging_bytes = opt_.staging_bytes;
    // exclusive shards for the first `nshards` live threads; a few shared, spin-locked ones for the threads beyond that
    asym_ = asym_available();
    const uint32_t nshared = asym_ ? 8u : 0u;
    cfg.staging_slots = 2 * (nshards + nshared) + 2;   // every shard may hold one histogram and one counter slot (memory is allocated on first use)
    cfg.precision = opt.precision;
    lh_status st = lh_create(&cfg, &ctx_);
    if (st != LH_OK) throw std::runtime_error(std::string("lh_create: ") + lh_strerror(st));
    for (auto *t : {&histos_, &counters_}) {
        t->capacity = std::min<uint32_t>(t == &histos_ ? opt.max_histograms : opt.max_counters, 65536u);   // u16 ids
        t->gen.reset(new std::atomic<uint32_t>[t->capacity]);
        for (uint32_t i = 0; i < t->capacity; i++) t->gen[i].store(0, std::memory_order_relaxed);
    }
    for (uint32_t i = 0; i < nshards + nshared; i++) {
        shards_.emplace_back(new Shard());
        shards_.back()->c_touched.assign(opt.max_counters, 0);
        if (asym_ && i < nshards) {
            shards_.back()->exclusive = true;
            free_exclusive_.push_back(shards_.back().get());
        } else {
            shared_.push_back(shards_.back().get());
        }
    }
    std::lock_guard<std::mutex> lk(g_reg_mu);
    g_systems[system_id_] = this;
}

// the calling thread's shard: an exclusive one while any is free, otherwise one of the shared ones (round-robin)
void *MetricSystem::assign_shard(size_t thread_slot, bool *exclusive) {
    {
        std::lock_guard<std::mutex> lk(assign_mu_);
        if (!free_exclusive_.empty()) {
            Shard *s = free_exclusive_.back();
            free_exclusive_.pop_back();
            *exclusive = true;
            return s;
        }
    }
    *exclusive = false;
    return shared_[thread_slot % shared_.size()];
}
void MetricSystem::release_shard(void *shard) {
    std::lock_guard<std::mutex> lk(assign_mu_);
    free_exclusive_.push_back(static_cast<Shard *>(shard));   // whatever it still holds is committed by the next collect
}

MetricSystem::~MetricSystem() {
    {
        std::lock_guard<std::mutex> lk(g_reg_mu);
        g_systems.erase(system_id_);
    }
    try { Stop(); } catch (...) {}
    if (reaper_thread_.joinable()) reaper_thread_.join();
    {   // recorders left open are freed by lh_destroy; their objects only forget the system
        std::lock_guard<std::mutex> lk(graph_mu_);
        for (auto &g : graphs_) g->ms = nullptr;
    }
    {   // likewise for subscriptions' boards
        std::lock_guard<std::mutex> lk(sub_mu_);
        for (auto &d : subs_) d->ms = nullptr;
        for (auto &d : raw_subs_) d->ms = nullptr;
    }
    lh_destroy(ctx_);
}

void MetricSystem::SpecifyPercentiles(const std::map<std::string, double> &percentiles) {
    std::lock_guard<std::mutex> lk(percentiles_mu_);
    percentiles_.assign(percentiles.begin(), percentiles.end());
    if (percentiles_.size() > LH_MAX_PERCENTILES) percentiles_.resize(LH_MAX_PERCENTILES);
}

// name -> (id, generation); false when no id is free (the caller drops and counts the sample).  A retiring name is
// revived, a new one takes a free id; both count as a use of the name in this interval (NameTable).
bool MetricSystem::intern(NameTable &t, const char *p, size_t n, uint32_t *id, uint32_t *gen) {
    const std::string name(p, n);
    {   // read-lock fast path, then write-lock and re-check: the idiom of metrics.go:275-294
        std::shared_lock<std::shared_mutex> rl(t.mu);
        auto it = t.ids.find(name);
        if (it != t.ids.end() && t.state[it->second] == kLive) {
            *id = it->second;
            *gen = t.gen[*id].load(std::memory_order_relaxed);   // only changes under the write lock
            return true;
        }
    }
    std::unique_lock<std::shared_mutex> wl(t.mu);
    *id = intern_locked(t, name);
    if (*id == RecordScope::kUnbound) return false;
    *gen = t.gen[*id].load(std::memory_order_relaxed);
    return true;
}

// The write-locked half of intern: the name's id, revived or taken from the free ids, live and used this interval;
// RecordScope::kUnbound when no id is free.
uint32_t MetricSystem::intern_locked(NameTable &t, const std::string &name) {
    uint32_t id;
    auto it = t.ids.find(name);
    if (it != t.ids.end()) {
        id = it->second;
    } else {
        if (!t.free_ids.empty()) {
            id = t.free_ids.back();
            t.free_ids.pop_back();
            t.names[id] = name;
        } else if (t.names.size() < t.capacity) {
            id = (uint32_t)t.names.size();
            t.names.push_back(name);
            t.state.push_back(kFree);
            t.used.push_back(0);
        } else {
            return RecordScope::kUnbound;
        }
        t.ids.emplace(name, id);
    }
    t.state[id] = kLive;
    t.used[id] = 1;
    return id;
}

// The id lifecycle step of collectRawMetrics, with t.mu held for writing (NameTable).  touched[id]: a sample or
// counter op of the id landed in the interval just collected.
void MetricSystem::recycle(NameTable &t, const std::vector<uint8_t> &touched) {
    for (uint32_t id = 0; id < (uint32_t)t.names.size(); id++) {
        const bool live_now = touched[id] || t.used[id];
        t.used[id] = 0;
        if (t.state[id] == kRetiring && !live_now) {
            t.ids.erase(t.names[id]);
            t.names[id].clear();
            t.state[id] = kFree;
            t.free_ids.push_back(id);
        } else if (t.state[id] == kLive && !live_now) {
            t.state[id] = kRetiring;
            t.gen[id].store(t.gen[id].load(std::memory_order_relaxed) + 1, std::memory_order_release);
        } else if (t.state[id] == kRetiring) {
            t.state[id] = kLive;
        }
    }
}

// The calling thread's state for THIS system (a thread that moves to another MetricSystem starts over).
static inline ThreadState *thread_state(MetricSystem &ms, uint64_t system_id) {
    ThreadState *ts = tl_state;
    if (__builtin_expect(ts == nullptr, 0)) ts = make_thread_state();
    if (__builtin_expect(ts->system_id != system_id, 0)) {
        release_thread_shard(ts);                // a shard of the system this thread used before
        ts->system_id = system_id;
        ts->shard = ms.assign_shard(ts->slot, &ts->exclusive);
        ts->h.reset();
        ts->c.reset();
    }
    return ts;
}

// name -> (id, generation) from the intern table, refreshing the calling thread's cache (after a miss, or after the
// append found the cached generation stale); false when no id is free (sample dropped, counted).  Names come and go,
// so a cache that has collected twice as many names as the table holds starts over instead of growing for ever.
static inline void cache_put(NameCache &c, uint32_t capacity, const char *p, size_t n, uint32_t id, uint32_t gen) {
    if (c.count >= 2 * (size_t)capacity + 64) c.reset();
    c.put(hash_bytes(p, n), p, n, id, gen);
}
bool MetricSystem::lookup_histogram(const char *p, size_t n, uint32_t *id, uint32_t *gen) {
    ThreadState *ts = thread_state(*this, system_id_);
    if (!intern(histos_, p, n, id, gen)) { dropped_over_limit_.fetch_add(1, std::memory_order_relaxed); return false; }
    cache_put(ts->h, histos_.capacity, p, n, *id, *gen);
    return true;
}
bool MetricSystem::lookup_counter(const char *p, size_t n, uint32_t *id, uint32_t *gen) {
    ThreadState *ts = thread_state(*this, system_id_);
    if (!intern(counters_, p, n, id, gen)) { dropped_over_limit_.fetch_add(1, std::memory_order_relaxed); return false; }
    cache_put(ts->c, counters_.capacity, p, n, *id, *gen);
    return true;
}

// Ingest never fails the caller and never throws (metrics.go:570-573, 632-636: problems are logged and data is
// dropped): a staging call that fails resets the shard, counts the samples it held as dropped and logs once.
// The append re-checks `gen` inside the critical section, on purpose (NameTable).  If the id was retired since the
// caller looked `name` up, it appends nothing, leaves the section and retries through the intern table (which
// revives the name or gives it a free id); that retry cannot find a stale generation again unless another collection
// retires the name in between, which its own revival prevents.
void MetricSystem::append_histogram(Shard &s, uint32_t id, uint32_t gen, double value, const char *name, size_t len) noexcept {
    {
        ShardGuard g(s);
        if (__builtin_expect(histos_.gen[id].load(std::memory_order_acquire) == gen, 1)) {
            if (!s.h_open) {
                lh_status st = lh_staging_acquire(ctx_, &s.hs);
                if (st != LH_OK) { s.dropped.fetch_add(1, std::memory_order_relaxed); log_once(g_logged_staging, ctx_, st, "lh_staging_acquire"); return; }
                s.h_cap = ((size_t)s.hs.bytes / 10) & ~(size_t)15;
                s.h_vals = reinterpret_cast<double *>(s.hs.host);
                s.h_ids = reinterpret_cast<uint16_t *>(reinterpret_cast<char *>(s.hs.host) + s.h_cap * 8);
                s.h_n = 0;
                s.h_open = true;
            }
            s.h_vals[s.h_n] = value;
            s.h_ids[s.h_n] = (uint16_t)id;
            if (++s.h_n == s.h_cap) commit_histograms(s);
            return;
        }
    }
    retry_histogram(s, value, name, len);
}
void MetricSystem::retry_histogram(Shard &s, double value, const char *name, size_t len) noexcept {
    uint32_t id, gen;
    if (lookup_histogram(name, len, &id, &gen)) append_histogram(s, id, gen, value, name, len);   // else dropped, counted
}
void MetricSystem::histogram_id(const std::string &name, uint32_t id, uint32_t gen, double value) noexcept {
    append_histogram(*static_cast<Shard *>(thread_state(*this, system_id_)->shard), id, gen, value, name.data(), name.size());
}

void MetricSystem::commit_histograms(Shard &s) noexcept {
    if (!s.h_open) return;
    lh_status st = lh_staging_commit_keyed_f64_u16(ctx_, &s.hs, s.h_n, s.h_cap * 8);
    if (st != LH_OK) {
        s.dropped.fetch_add(s.h_n, std::memory_order_relaxed);
        log_once(g_logged_staging, ctx_, st, "lh_staging_commit_keyed_f64_u16");
        lh_staging_abandon(ctx_, &s.hs);      // harmless if the commit already recycled the slot
    }
    s.h_open = false;
    s.h_n = 0;
}

void MetricSystem::commit_counters(Shard &s) noexcept {
    if (!s.c_open) return;
    lh_status st = lh_staging_commit_counter_u16(ctx_, &s.cs, s.c_n, s.c_cap * 8);
    if (st != LH_OK) {
        s.dropped.fetch_add(s.c_n, std::memory_order_relaxed);
        log_once(g_logged_staging, ctx_, st, "lh_staging_commit_counter_u16");
        lh_staging_abandon(ctx_, &s.cs);
    }
    s.c_open = false;
    s.c_n = 0;
}

void MetricSystem::Histogram(const std::string &name, double value) noexcept { Histogram(name.data(), name.size(), value); }
void MetricSystem::Histogram(const char *name, size_t len, double value) noexcept {
    // steady state: one thread-local pointer, one hash of the name's bytes, one probe of this thread's name cache, one
    // uncontended spinlock, two stores into pinned memory
    ThreadState *ts = thread_state(*this, system_id_);
    uint32_t id, gen;
    if (!ts->h.find_last(name, len, &id, &gen) && __builtin_expect(!ts->h.find(hash_bytes(name, len), name, len, &id, &gen), 0)) {
        if (!lookup_histogram(name, len, &id, &gen)) return;        // no free id: dropped and counted
    }
    append_histogram(*static_cast<Shard *>(ts->shard), id, gen, value, name, len);
}

void MetricSystem::Counter(const std::string &name, uint64_t amount) noexcept {
    ThreadState *ts = thread_state(*this, system_id_);
    uint32_t id, gen;
    if (!ts->c.find_last(name.data(), name.size(), &id, &gen) &&
        __builtin_expect(!ts->c.find(hash_bytes(name.data(), name.size()), name.data(), name.size(), &id, &gen), 0)) {
        if (!lookup_counter(name.data(), name.size(), &id, &gen)) return;   // no free id: dropped and counted
    }
    append_counter(*static_cast<Shard *>(ts->shard), id, gen, amount, name.data(), name.size());
}

// as append_histogram: the generation is checked inside the critical section, a stale one retried by name
void MetricSystem::append_counter(Shard &s, uint32_t id, uint32_t gen, uint64_t amount, const char *name, size_t len) noexcept {
    {
        ShardGuard g(s);
        if (__builtin_expect(counters_.gen[id].load(std::memory_order_acquire) == gen, 1)) {
            s.c_touched[id] = 1;            // Counter(name, 0) still makes the name appear in Rates (metrics.go:430-433)
            s.c_any_touched = true;
            if (amount == 0) return;        // nothing to add on the device
            if (!s.c_open) {
                lh_status st = lh_staging_acquire(ctx_, &s.cs);
                if (st != LH_OK) { s.dropped.fetch_add(1, std::memory_order_relaxed); log_once(g_logged_staging, ctx_, st, "lh_staging_acquire"); return; }
                s.c_cap = ((size_t)s.cs.bytes / 10) & ~(size_t)15;
                s.c_amounts = reinterpret_cast<uint64_t *>(s.cs.host);
                s.c_ids = reinterpret_cast<uint16_t *>(reinterpret_cast<char *>(s.cs.host) + s.c_cap * 8);
                s.c_n = 0;
                s.c_open = true;
            }
            s.c_amounts[s.c_n] = amount;
            s.c_ids[s.c_n] = (uint16_t)id;
            if (++s.c_n == s.c_cap) commit_counters(s);
            return;
        }
    }
    retry_counter(s, amount, name, len);
}
void MetricSystem::retry_counter(Shard &s, uint64_t amount, const char *name, size_t len) noexcept {
    uint32_t id, gen;
    if (lookup_counter(name, len, &id, &gen)) append_counter(s, id, gen, amount, name, len);   // else dropped, counted
}

TimerToken MetricSystem::StartTimer(const std::string &name) {
    TimerToken t;
    t.Name = name;
    t.System = this;
    // interned once here; Stop() skips the lookup unless the id was retired in between
    ThreadState *ts = thread_state(*this, system_id_);
    t.id_valid = ts->h.find(hash_bytes(name.data(), name.size()), name.data(), name.size(), &t.id, &t.gen) ||
                 lookup_histogram(name.data(), name.size(), &t.id, &t.gen);
    t.Start = std::chrono::steady_clock::now();
    return t;
}

// ---- record scopes bound to names ---------------------------------------------------------------------------
// BeginRecording hands ids to device code, which cannot re-check a generation per record as the append does.  So the
// ids are pinned for the scope instead:
//   1. intern every name (a retiring name is revived, a new one takes a free id) and note each id's generation;
//   2. lh_record_begin;
//   3. under each table's write lock, re-read the generations; if any changed, end the empty scope and start over;
//      otherwise mark every bound id used in the current interval.
// Why this is enough: lh_snapshot_begin does not return while the scope is open, so the collection X that labels the
// scope's records (the first to freeze after step 2) labels them after step 3.  An unchanged generation at step 3
// means no collection retired the id since step 1, so it is still live under this name, and the used mark of step 3
// keeps it live through the next recycle step; a later one can only retire it (the id and its name stay), and only
// the one after that can free it.  The recycle steps that can run between step 3 and the labelling of the interval
// after X are at most two: the one of a collection already past lh_snapshot_begin at step 2, and X's.  So device
// records (interval of X) and ingest calls through the scope (interval of X, or the next one when X froze first) are
// labelled with this name.  A collection between steps 1 and 3 that retired the id changed its generation, so the
// retry catches every other case.
void MetricSystem::bind_names(NameTable &t, const std::vector<std::string> &names, std::vector<uint32_t> &ids,
                              std::vector<uint32_t> &gens) {
    ids.assign(names.size(), RecordScope::kUnbound);
    gens.assign(names.size(), 0);
    for (size_t i = 0; i < names.size(); i++)
        if (!intern(t, names[i].data(), names[i].size(), &ids[i], &gens[i])) ids[i] = RecordScope::kUnbound;
}
bool MetricSystem::pin_names(NameTable &t, const std::vector<uint32_t> &ids, const std::vector<uint32_t> &gens) {
    std::unique_lock<std::shared_mutex> wl(t.mu);
    for (size_t i = 0; i < ids.size(); i++)
        if (ids[i] != RecordScope::kUnbound && t.gen[ids[i]].load(std::memory_order_acquire) != gens[i]) return false;
    for (uint32_t id : ids)
        if (id != RecordScope::kUnbound) t.used[id] = 1;
    return true;
}

RecordScope MetricSystem::BeginRecording(void *stream, const std::vector<std::string> &histograms,
                                         const std::vector<std::string> &counters) {
    if (!lh_record_begin || !lh_record_end || !lh_ingest_f64)
        throw std::runtime_error("BeginRecording: this libloghisto_b200 has no record scopes");
    RecordScope s;
    std::vector<uint32_t> hgen, cgen;
    for (;;) {
        bind_names(histos_, histograms, s.hids_, hgen);
        bind_names(counters_, counters, s.cids_, cgen);
        check(ctx_, lh_record_begin(ctx_, stream, &s.rec_), "lh_record_begin");
        if (pin_names(histos_, s.hids_, hgen) && pin_names(counters_, s.cids_, cgen)) break;
        lh_record_end(ctx_, &s.rec_);   // nothing was enqueued under the stale ids
    }
    s.ms_ = this;
    s.stream_ = stream;
    s.owner_ = std::this_thread::get_id();
    std::lock_guard<std::mutex> lk(scope_mu_);
    scope_threads_[s.owner_]++;
    return s;
}

void MetricSystem::refuse_in_scope(const char *what) {
    std::lock_guard<std::mutex> lk(scope_mu_);
    if (scope_threads_.count(std::this_thread::get_id()))
        throw std::runtime_error(std::string(what) + " from a thread that holds an open record scope");
}

void MetricSystem::end_scope(RecordScope &s) {
    const lh_status st = lh_record_end(ctx_, &s.rec_);
    {
        std::lock_guard<std::mutex> lk(scope_mu_);
        auto it = scope_threads_.find(s.owner_);
        if (it != scope_threads_.end() && --it->second == 0) scope_threads_.erase(it);
    }
    s.ms_ = nullptr;
    check(ctx_, st, "lh_record_end");
}

RecordScope &RecordScope::operator=(RecordScope &&o) noexcept {
    if (this != &o) {
        try { End(); } catch (...) {}
        ms_ = o.ms_; stream_ = o.stream_; owner_ = o.owner_;
        hids_ = std::move(o.hids_); cids_ = std::move(o.cids_); rec_ = o.rec_;
        o.ms_ = nullptr;
    }
    return *this;
}
RecordScope::~RecordScope() {
    try { End(); } catch (...) {}
}
void RecordScope::End() {
    if (ms_) ms_->end_scope(*this);
}
void RecordScope::Histogram(size_t i, const double *d_values, size_t n) {
    const uint32_t id = hids_.at(i);
    if (!ms_) throw std::runtime_error("RecordScope::Histogram after End()");
    if (id == kUnbound) { ms_->dropped_over_limit_.fetch_add(n, std::memory_order_relaxed); return; }
    check(ms_->ctx_, lh_ingest_f64(ms_->ctx_, id, d_values, n, stream_), "lh_ingest_f64");
}
void RecordScope::Histograms(const std::vector<Item> &items) {
    if (!ms_) throw std::runtime_error("RecordScope::Histograms after End()");
    for (const Item &it : items) (void)hids_.at(it.name);   // std::out_of_range before anything is issued
    if (!lh_ingest_batch) throw std::runtime_error("lh_ingest_batch: not in this build of the library");
    std::vector<lh_batch_item> batch;
    batch.reserve(items.size());
    uint64_t unbound = 0;
    for (const Item &it : items) {
        const uint32_t id = hids_[it.name];
        if (id == kUnbound) { unbound += it.n; continue; }
        batch.push_back(lh_batch_item{it.d_values, (uint64_t)it.n, id, it.kind});
    }
    check(ms_->ctx_, lh_ingest_batch(ms_->ctx_, batch.data(), (uint32_t)batch.size(), stream_), "lh_ingest_batch");
    ms_->dropped_over_limit_.fetch_add(unbound, std::memory_order_relaxed);
}
void RecordScope::Arrays(const std::vector<ArrayItem> &items) {
    if (!ms_) throw std::runtime_error("RecordScope::Arrays after End()");
    for (const ArrayItem &it : items) (void)hids_.at(it.name);   // std::out_of_range before anything is issued
    if (!lh_ingest_arrays) throw std::runtime_error("lh_ingest_arrays: not in this build of the library");
    std::vector<lh_array_src> srcs;
    srcs.reserve(items.size());
    uint64_t unbound = 0;
    for (const ArrayItem &it : items) {
        const uint32_t id = hids_[it.name];
        if (id == kUnbound) { unbound += it.n; continue; }
        srcs.push_back(lh_array_src{it.d_values, (uint64_t)it.n, it.dtype, id});
    }
    check(ms_->ctx_, lh_ingest_arrays(ms_->ctx_, srcs.data(), (uint32_t)srcs.size(), stream_), "lh_ingest_arrays");
    ms_->dropped_over_limit_.fetch_add(unbound, std::memory_order_relaxed);
}
void RecordScope::Keyed(const void *d_ids, size_t id_bytes, const void *d_values, uint32_t kind, size_t n) {
    if (!ms_) throw std::runtime_error("RecordScope::Keyed after End()");
    if (id_bytes != 2 && id_bytes != 4) throw std::invalid_argument("RecordScope::Keyed: id_bytes must be 2 or 4");
    auto fn16 = lh_ingest_keyed_mapped_u16;
    auto fn32 = lh_ingest_keyed_mapped_u32;
    if (id_bytes == 2 ? !fn16 : !fn32) throw std::runtime_error("RecordScope::Keyed: this libloghisto_b200 has no mapped keyed ingest");
    const uint32_t k = (uint32_t)hids_.size();
    lh_status st = id_bytes == 2 ? fn16(ms_->ctx_, hids_.data(), k, static_cast<const uint16_t *>(d_ids), d_values, kind, n, stream_)
                                 : fn32(ms_->ctx_, hids_.data(), k, static_cast<const uint32_t *>(d_ids), d_values, kind, n, stream_);
    check(ms_->ctx_, st, "lh_ingest_keyed_mapped");
}
void RecordScope::Counters(const void *d_ids, size_t id_bytes, const uint64_t *d_amounts, size_t n) {
    if (!ms_) throw std::runtime_error("RecordScope::Counters after End()");
    if (id_bytes != 2 && id_bytes != 4) throw std::invalid_argument("RecordScope::Counters: id_bytes must be 2 or 4");
    auto fn16 = lh_counter_add_mapped_u16;
    auto fn32 = lh_counter_add_mapped_u32;
    if (id_bytes == 2 ? !fn16 : !fn32) throw std::runtime_error("RecordScope::Counters: this libloghisto_b200 has no mapped counter adds");
    const uint32_t kc = (uint32_t)cids_.size();
    lh_status st = id_bytes == 2 ? fn16(ms_->ctx_, cids_.data(), kc, static_cast<const uint16_t *>(d_ids), d_amounts, n, stream_)
                                 : fn32(ms_->ctx_, cids_.data(), kc, static_cast<const uint32_t *>(d_ids), d_amounts, n, stream_);
    check(ms_->ctx_, st, "lh_counter_add_mapped");
}

// ---- graph recorders -------------------------------------------------------------------------------------------
// Interns (or revives) every name of an open recorder, marking it used in this interval so that it keeps its id while
// the recorder is open, and binds the rows to the ids; with graph_mu_ held.  Each drain (lh_snapshot_begin of
// collectRawMetrics, lh_graph_recorder_destroy of Close) follows a call of this in the same collection or Close, so the
// ids it drains into are live in the interval it drains into, and that interval's collection labels them with these
// names.
void MetricSystem::bind_graph(GraphRecorder::State &g) {
    std::vector<uint32_t> hids(g.hnames.size()), cids(g.cnames.size());
    {
        std::unique_lock<std::shared_mutex> wl(histos_.mu);
        for (size_t i = 0; i < hids.size(); i++) hids[i] = intern_locked(histos_, g.hnames[i]);
    }
    {
        std::unique_lock<std::shared_mutex> wl(counters_.mu);
        for (size_t i = 0; i < cids.size(); i++) cids[i] = intern_locked(counters_, g.cnames[i]);
    }
    if (g.g.handle)
        check(ctx_, lh_graph_recorder_bind(ctx_, &g.g, hids.data(), cids.data()), "lh_graph_recorder_bind");
    else
        check(ctx_, lh_graph_recorder_create(ctx_, (uint32_t)hids.size(), (uint32_t)cids.size(), hids.data(), cids.data(), &g.g),
              "lh_graph_recorder_create");
}

GraphRecorder MetricSystem::NewGraphRecorder(const std::vector<std::string> &histograms, const std::vector<std::string> &counters) {
    if (!lh_graph_recorder_create || !lh_graph_recorder_bind || !lh_graph_recorder_ingest || !lh_graph_recorder_destroy)
        throw std::runtime_error("NewGraphRecorder: this libloghisto_b200 has no graph recorders");
    auto st = std::make_shared<GraphRecorder::State>();
    st->ms = this;
    st->hnames = histograms;
    st->cnames = counters;
    std::lock_guard<std::mutex> lk(graph_mu_);
    bind_graph(*st);
    graphs_.push_back(st);
    GraphRecorder g;
    g.st_ = std::move(st);
    return g;
}

const lh_recorder &GraphRecorder::recorder() const {
    if (!st_) throw std::runtime_error("GraphRecorder::recorder of a closed recorder");
    return st_->g.rec;
}

void GraphRecorder::Histograms(const std::vector<Item> &items, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::Histograms of a closed recorder");
    std::vector<lh_batch_item> batch;
    batch.reserve(items.size());
    for (const Item &it : items) {
        if (it.name >= st_->hnames.size()) throw std::out_of_range("GraphRecorder::Histograms: no such histogram name");
        batch.push_back(lh_batch_item{it.d_values, (uint64_t)it.n, (uint32_t)it.name, it.kind});
    }
    MetricSystem *ms = st_->ms;
    check(ms->ctx_, lh_graph_recorder_ingest(ms->ctx_, &st_->g, batch.data(), (uint32_t)batch.size(), stream),
          "lh_graph_recorder_ingest");
}

void GraphRecorder::Arrays(const std::vector<ArrayItem> &items, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::Arrays of a closed recorder");
    std::vector<lh_array_src> srcs;
    srcs.reserve(items.size());
    for (const ArrayItem &it : items) {
        if (it.name >= st_->hnames.size()) throw std::out_of_range("GraphRecorder::Arrays: no such histogram name");
        srcs.push_back(lh_array_src{it.d_values, (uint64_t)it.n, it.dtype, (uint32_t)it.name});
    }
    if (!lh_graph_recorder_ingest_arrays) throw std::runtime_error("lh_graph_recorder_ingest_arrays: not in this build of the library");
    MetricSystem *ms = st_->ms;
    check(ms->ctx_, lh_graph_recorder_ingest_arrays(ms->ctx_, &st_->g, srcs.data(), (uint32_t)srcs.size(), stream),
          "lh_graph_recorder_ingest_arrays");
}

void GraphRecorder::Keyed(const void *d_ids, size_t id_bytes, const void *d_values, uint32_t kind, size_t n, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::Keyed of a closed recorder");
    MetricSystem *ms = st_->ms;
    if (id_bytes != 2 && id_bytes != 4) throw std::invalid_argument("GraphRecorder::Keyed: id_bytes must be 2 or 4");
    auto fn16 = lh_graph_recorder_ingest_keyed_u16;
    auto fn32 = lh_graph_recorder_ingest_keyed_u32;
    if (id_bytes == 2 ? !fn16 : !fn32) throw std::runtime_error("GraphRecorder::Keyed: this libloghisto_b200 has no captured keyed ingest");
    lh_status st = id_bytes == 2 ? fn16(ms->ctx_, &st_->g, static_cast<const uint16_t *>(d_ids), d_values, kind, n, stream)
                                 : fn32(ms->ctx_, &st_->g, static_cast<const uint32_t *>(d_ids), d_values, kind, n, stream);
    check(ms->ctx_, st, "lh_graph_recorder_ingest_keyed");
}

void GraphRecorder::Counters(const void *d_ids, size_t id_bytes, const uint64_t *d_amounts, size_t n, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::Counters of a closed recorder");
    MetricSystem *ms = st_->ms;
    if (id_bytes != 2 && id_bytes != 4) throw std::invalid_argument("GraphRecorder::Counters: id_bytes must be 2 or 4");
    auto fn16 = lh_graph_recorder_counter_add_u16;
    auto fn32 = lh_graph_recorder_counter_add_u32;
    if (id_bytes == 2 ? !fn16 : !fn32) throw std::runtime_error("GraphRecorder::Counters: this libloghisto_b200 has no captured counter adds");
    lh_status st = id_bytes == 2 ? fn16(ms->ctx_, &st_->g, static_cast<const uint16_t *>(d_ids), d_amounts, n, stream)
                                 : fn32(ms->ctx_, &st_->g, static_cast<const uint32_t *>(d_ids), d_amounts, n, stream);
    check(ms->ctx_, st, "lh_graph_recorder_counter_add");
}

void GraphRecorder::StartTimer(size_t name, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::StartTimer of a closed recorder");
    MetricSystem *ms = st_->ms;
    if (name >= st_->hnames.size()) throw std::out_of_range("GraphRecorder::StartTimer: no such histogram name");
    if (!lh_graph_recorder_timer_start) throw std::runtime_error("GraphRecorder::StartTimer: this libloghisto_b200 has no graph timers");
    check(ms->ctx_, lh_graph_recorder_timer_start(ms->ctx_, &st_->g, (uint32_t)name, stream), "lh_graph_recorder_timer_start");
}

void GraphRecorder::StopTimer(size_t name, void *stream, int64_t *d_duration_ns) {
    if (!st_ || !st_->ms) throw std::runtime_error("GraphRecorder::StopTimer of a closed recorder");
    MetricSystem *ms = st_->ms;
    if (name >= st_->hnames.size()) throw std::out_of_range("GraphRecorder::StopTimer: no such histogram name");
    if (!lh_graph_recorder_timer_stop) throw std::runtime_error("GraphRecorder::StopTimer: this libloghisto_b200 has no graph timers");
    check(ms->ctx_, lh_graph_recorder_timer_stop(ms->ctx_, &st_->g, (uint32_t)name, stream, d_duration_ns),
          "lh_graph_recorder_timer_stop");
}

void GraphRecorder::Close(void *stream) {
    if (!st_) return;
    std::shared_ptr<State> st = std::move(st_);
    MetricSystem *ms = st->ms;
    if (!ms) return;
    std::lock_guard<std::mutex> lk(ms->graph_mu_);
    auto &v = ms->graphs_;
    v.erase(std::remove(v.begin(), v.end(), st), v.end());
    st->ms = nullptr;
    ms->bind_graph(*st);   // the final drain's ids are used in the interval it drains into
    check(ms->ctx_, lh_graph_recorder_destroy(ms->ctx_, &st->g, stream), "lh_graph_recorder_destroy");
}

GraphRecorder &GraphRecorder::operator=(GraphRecorder &&o) noexcept {
    if (this != &o) {
        try { Close(); } catch (...) {}
        st_ = std::move(o.st_);
    }
    return *this;
}
GraphRecorder::~GraphRecorder() {
    try { Close(); } catch (...) {}
}

// ---- device subscriptions ----------------------------------------------------------------------------------------
DeviceSubscription MetricSystem::NewDeviceSubscription(const std::vector<std::string> &histograms,
                                                       const std::vector<std::string> &counters) {
    if (!lh_board_create || !lh_snapshot_publish || !lh_board_read || !lh_board_destroy)
        throw std::runtime_error("NewDeviceSubscription: this libloghisto_b200 has no device subscriptions");
    auto st = std::make_shared<DeviceSubscription::State>();
    st->ms = this;
    st->hnames = histograms;
    st->cnames = counters;
    check(ctx_, lh_board_create(ctx_, (uint32_t)histograms.size(), (uint32_t)counters.size(), &st->b), "lh_board_create");
    std::lock_guard<std::mutex> lk(sub_mu_);
    subs_.push_back(st);
    DeviceSubscription d;
    d.st_ = std::move(st);
    return d;
}

namespace {
// the id each name carries in this collection's labels (id_of: the names of Histograms / Rates), or LH_GRAPH_UNBOUND
std::vector<uint32_t> bind_rows(const std::vector<std::string> &names, const std::unordered_map<std::string, uint32_t> &id_of) {
    std::vector<uint32_t> ids(names.size());
    for (size_t i = 0; i < ids.size(); i++) {
        auto it = id_of.find(names[i]);
        ids[i] = it == id_of.end() ? LH_GRAPH_UNBOUND : it->second;
    }
    return ids;
}
}  // namespace

// With sub_mu_ held, between the reduction of collectRawMetrics and lh_snapshot_end: row i of every open subscription
// is bound to the id that carries its name in this collection's labels, if the name is in Histograms (hid_of) or
// Rates (cid_of); totals are the Counters values.  The first failure is returned; the other boards still publish.
lh_status MetricSystem::publish_subscriptions(const RawMetricSet &raw, const std::unordered_map<std::string, uint32_t> &hid_of,
                                              const std::unordered_map<std::string, uint32_t> &cid_of) {
    lh_status first = LH_OK;
    for (auto &d : subs_) {
        const std::vector<uint32_t> hids = bind_rows(d->hnames, hid_of), cids = bind_rows(d->cnames, cid_of);
        std::vector<uint64_t> totals(d->cnames.size());
        for (size_t i = 0; i < totals.size(); i++) {
            auto t = raw.Counters.find(d->cnames[i]);
            totals[i] = t == raw.Counters.end() ? 0 : t->second;
        }
        const lh_status st = lh_snapshot_publish(ctx_, &d->b, hids.data(), cids.data(), totals.data());
        if (st != LH_OK && first == LH_OK) first = st;
    }
    return first;
}

const lh_board &DeviceSubscription::board() const {
    if (!st_) throw std::runtime_error("DeviceSubscription::board of a closed subscription");
    return st_->b;
}

void DeviceSubscription::Read(void *d_out, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("DeviceSubscription::Read of a closed subscription");
    MetricSystem *ms = st_->ms;
    check(ms->ctx_, lh_board_read(ms->ctx_, &st_->b, d_out, stream), "lh_board_read");
}

void DeviceSubscription::Close() {
    if (!st_) return;
    std::shared_ptr<State> st = std::move(st_);
    MetricSystem *ms = st->ms;
    if (!ms) return;
    std::lock_guard<std::mutex> lk(ms->sub_mu_);   // not during a collection's publish
    auto &v = ms->subs_;
    v.erase(std::remove(v.begin(), v.end(), st), v.end());
    st->ms = nullptr;
    check(ms->ctx_, lh_board_destroy(ms->ctx_, &st->b), "lh_board_destroy");
}

DeviceSubscription &DeviceSubscription::operator=(DeviceSubscription &&o) noexcept {
    if (this != &o) {
        try { Close(); } catch (...) {}
        st_ = std::move(o.st_);
    }
    return *this;
}
DeviceSubscription::~DeviceSubscription() {
    try { Close(); } catch (...) {}
}

// ---- raw device subscriptions --------------------------------------------------------------------------------------
RawDeviceSubscription MetricSystem::NewRawDeviceSubscription(const std::vector<std::string> &histograms,
                                                             uint32_t window) {
    if (!lh_raw_board_create || !lh_snapshot_publish_raw || !lh_raw_percentiles_grid || !lh_raw_ranks_grid ||
        !lh_raw_board_destroy)
        throw std::runtime_error("NewRawDeviceSubscription: this libloghisto_b200 has no raw device subscriptions");
    if (window != 1 && !lh_raw_board_create_window)
        throw std::runtime_error("NewRawDeviceSubscription: this libloghisto_b200 has no window boards");
    auto st = std::make_shared<RawDeviceSubscription::State>();
    st->ms = this;
    st->hnames = histograms;
    st->window = window;
    if (window == 1)
        check(ctx_, lh_raw_board_create(ctx_, (uint32_t)histograms.size(), &st->b), "lh_raw_board_create");
    else
        check(ctx_, lh_raw_board_create_window(ctx_, (uint32_t)histograms.size(), window, &st->b),
              "lh_raw_board_create_window");
    std::lock_guard<std::mutex> lk(sub_mu_);
    raw_subs_.push_back(st);
    RawDeviceSubscription d;
    d.st_ = std::move(st);
    return d;
}

// With sub_mu_ held, before lh_snapshot_end: row i of every open raw subscription is bound as publish_subscriptions
// binds histogram rows.  The first failure is returned; the other boards still publish.
lh_status MetricSystem::publish_raw_subscriptions(const std::unordered_map<std::string, uint32_t> &hid_of) {
    lh_status first = LH_OK;
    for (auto &d : raw_subs_) {
        const std::vector<uint32_t> hids = bind_rows(d->hnames, hid_of);
        const lh_status st = lh_snapshot_publish_raw(ctx_, &d->b, hids.data());
        if (st != LH_OK && first == LH_OK) first = st;
    }
    return first;
}

const lh_raw_board &RawDeviceSubscription::board() const {
    if (!st_) throw std::runtime_error("RawDeviceSubscription::board of a closed subscription");
    return st_->b;
}

uint32_t RawDeviceSubscription::window() const { return st_ ? st_->window : 1u; }

void RawDeviceSubscription::Percentiles(const double *d_ps, uint32_t m, int32_t *d_keys, double *d_vals,
                                        uint64_t *d_publish, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("RawDeviceSubscription::Percentiles of a closed subscription");
    MetricSystem *ms = st_->ms;
    check(ms->ctx_, lh_raw_percentiles_grid(ms->ctx_, &st_->b, d_ps, m, d_keys, d_vals, d_publish, stream),
          "lh_raw_percentiles_grid");
}

void RawDeviceSubscription::Ranks(const double *d_values, uint32_t m, uint64_t *d_ranks, uint64_t *d_totals,
                                  uint64_t *d_publish, void *stream) {
    if (!st_ || !st_->ms) throw std::runtime_error("RawDeviceSubscription::Ranks of a closed subscription");
    MetricSystem *ms = st_->ms;
    check(ms->ctx_, lh_raw_ranks_grid(ms->ctx_, &st_->b, d_values, m, d_ranks, d_totals, d_publish, stream),
          "lh_raw_ranks_grid");
}

void RawDeviceSubscription::Close() {
    if (!st_) return;
    std::shared_ptr<State> st = std::move(st_);
    MetricSystem *ms = st->ms;
    if (!ms) return;
    std::lock_guard<std::mutex> lk(ms->sub_mu_);   // not during a collection's publish
    auto &v = ms->raw_subs_;
    v.erase(std::remove(v.begin(), v.end(), st), v.end());
    st->ms = nullptr;
    check(ms->ctx_, lh_raw_board_destroy(ms->ctx_, &st->b), "lh_raw_board_destroy");
}

RawDeviceSubscription &RawDeviceSubscription::operator=(RawDeviceSubscription &&o) noexcept {
    if (this != &o) {
        try { Close(); } catch (...) {}
        st_ = std::move(o.st_);
    }
    return *this;
}
RawDeviceSubscription::~RawDeviceSubscription() {
    try { Close(); } catch (...) {}
}

// ---- GPU timers ------------------------------------------------------------------------------------------------
void *const GpuTimerToken::kStartStream = reinterpret_cast<void *>(~(uintptr_t)0);

GpuTimerToken MetricSystem::StartGpuTimer(const std::string &name, void *stream) {
    GpuTimerToken t;
    t.ms_ = this;
    t.name_ = name;
    t.stream_ = stream;
    if (!lh_gpu_timer_start || !lh_gpu_timer_stop || !lh_gpu_timer_release) return t;
    const lh_status st = lh_gpu_timer_start(ctx_, stream, &t.t_);
    if (st == LH_ERR_RANGE) return t;   // every slot is in use: as StartTimer, this does not fail; Stop drops and counts
    check(ctx_, st, "lh_gpu_timer_start");
    t.held_ = true;
    return t;
}

// The name is bound at stop time through a record scope on the stop's stream, so the id the sample lands on keeps
// the name until the interval is collected (see bind_names), however long the token was held.
void GpuTimerToken::Stop(void *stream, int64_t *d_duration_ns) {
    if (!ms_) throw std::runtime_error("GpuTimerToken::Stop on an empty token");
    if (stream == kStartStream) stream = stream_;
    if (!held_) { ms_->dropped_over_limit_.fetch_add(1, std::memory_order_relaxed); return; }
    RecordScope s = ms_->BeginRecording(stream, {name_}, {});
    const uint32_t id = s.histogram_id(0);
    if (id == RecordScope::kUnbound) { ms_->dropped_over_limit_.fetch_add(1, std::memory_order_relaxed); return; }
    const lh_status st = lh_gpu_timer_stop(ms_->ctx_, &t_, id, stream, d_duration_ns);
    s.End();
    check(ms_->ctx_, st, "lh_gpu_timer_stop");
}

GpuTimerToken &GpuTimerToken::operator=(GpuTimerToken &&o) noexcept {
    if (this != &o) {
        if (held_ && ms_) lh_gpu_timer_release(ms_->ctx_, &t_);
        ms_ = o.ms_; name_ = std::move(o.name_); stream_ = o.stream_; t_ = o.t_; held_ = o.held_;
        o.ms_ = nullptr;
        o.held_ = false;
    }
    return *this;
}
GpuTimerToken::~GpuTimerToken() {
    if (held_ && ms_) lh_gpu_timer_release(ms_->ctx_, &t_);
}

void MetricSystem::RegisterGaugeFunc(const std::string &name, std::function<double()> f) {
    std::lock_guard<std::mutex> lk(gauge_mu_);
    device_gauges_.erase(name);
    gauge_funcs_[name] = std::move(f);
}
void MetricSystem::RegisterDeviceGauge(const std::string &name, const void *d_value, uint32_t dtype) {
    if (!lh_gauges_read) throw std::runtime_error("RegisterDeviceGauge: this libloghisto_b200 has no device gauges");
    const lh_gauge_src src{d_value, dtype, 0u};
    double v = 0;
    const lh_status st = lh_gauges_read(ctx_, &src, 1, &v);
    if (st == LH_ERR_INVALID)
        throw std::invalid_argument(std::string("RegisterDeviceGauge(") + name + "): " + lh_last_error(ctx_));
    check(ctx_, st, "lh_gauges_read");
    std::lock_guard<std::mutex> lk(gauge_mu_);
    gauge_funcs_.erase(name);
    device_gauges_[name] = src;
}
void MetricSystem::DeregisterGaugeFunc(const std::string &name) {
    std::lock_guard<std::mutex> lk(gauge_mu_);
    gauge_funcs_.erase(name);
    device_gauges_.erase(name);
}
void MetricSystem::RegisterDeviceDistribution(const std::string &name, const void *d_values, uint64_t n, uint32_t dtype) {
    if (!lh_snapshot_ingest_arrays || !lh_gauges_read)
        throw std::runtime_error("RegisterDeviceDistribution: this libloghisto_b200 has no distribution gauges");
    if (dtype > LH_GAUGE_U64)
        throw std::invalid_argument("RegisterDeviceDistribution(" + name + "): unknown dtype " + std::to_string(dtype));
    if (n) {   // the first element, as RegisterDeviceGauge checks a gauge; the range is checked at every collection
        const lh_gauge_src src{d_values, dtype, 0u};
        double v = 0;
        const lh_status st = lh_gauges_read(ctx_, &src, 1, &v);
        if (st == LH_ERR_INVALID)
            throw std::invalid_argument("RegisterDeviceDistribution(" + name + "): " + lh_last_error(ctx_));
        check(ctx_, st, "lh_gauges_read");
    }
    refuse_in_scope("RegisterDeviceDistribution");   // before dist_mu_, which a collection holds across its scope wait
    std::lock_guard<std::mutex> lk(dist_mu_);
    device_dists_[name] = lh_array_src{d_values, n, dtype, 0u};
}
void MetricSystem::DeregisterDeviceDistribution(const std::string &name) {
    refuse_in_scope("DeregisterDeviceDistribution");
    std::lock_guard<std::mutex> lk(dist_mu_);
    device_dists_.erase(name);
}

// commit whatever the shard holds and hand over (and clear) its touched-counter marks
void MetricSystem::flush_shard(Shard &s, std::vector<uint8_t> *touched) {
    ForeignGuard g(s);
    commit_histograms(s);
    commit_counters(s);
    if (s.c_any_touched) {
        for (size_t i = 0; i < s.c_touched.size(); i++)
            if (s.c_touched[i]) { (*touched)[i] = 1; s.c_touched[i] = 0; }
        s.c_any_touched = false;
    }
}

uint64_t MetricSystem::dropped_samples() {
    lh_stats st{};
    lh_get_stats(ctx_, &st);
    uint64_t d = st.dropped + dropped_over_limit_.load();
    for (auto &s : shards_) d += s->dropped.load(std::memory_order_relaxed);
    return d;
}

// ---- joined ranks ------------------------------------------------------------------------------------------------
namespace {
void put_u32(std::string &b, uint32_t v) { b.append(reinterpret_cast<const char *>(&v), 4); }
void put_u64(std::string &b, uint64_t v) { b.append(reinterpret_cast<const char *>(&v), 8); }
struct Reader {
    const std::string &b;
    size_t at = 0;
    void need(size_t n) {
        if (b.size() - at < n) throw std::runtime_error("truncated rank payload");
    }
    uint32_t u32() { need(4); uint32_t v; memcpy(&v, b.data() + at, 4); at += 4; return v; }
    uint64_t u64() { need(8); uint64_t v; memcpy(&v, b.data() + at, 8); at += 8; return v; }
    std::string str() { const uint32_t n = u32(); need(n); std::string v = b.substr(at, n); at += n; return v; }
};
constexpr uint32_t kJoinMagic = 0x4C48524Bu;   // first exchange: handle + shape
constexpr uint32_t kRowsMagic = 0x4C485253u;   // per collection: sequence, frozen half, touched names (and levels)
}  // namespace

void MetricSystem::JoinRanks(uint32_t rank, uint32_t world, AllGather allgather) {
    if (!lh_comm_export || !lh_comm_import || !lh_comm_info || !lh_snapshot_copy_histogram || !lh_snapshot_rows ||
        !lh_snapshot_allreduce_rows)
        throw std::runtime_error("JoinRanks: this libloghisto_b200 has no row-mapped all-reduce");
    join(rank, world, std::move(allgather), nullptr);
}

void MetricSystem::JoinRanks(uint32_t rank, uint32_t world, AllGather allgather, AllReduce allreduce) {
    if (!lh_snapshot_copy_histogram || !lh_snapshot_rows || !lh_snapshot_row_levels || !lh_snapshot_pack_rows ||
        !lh_snapshot_unpack_rows)
        throw std::runtime_error("JoinRanks: this libloghisto_b200 has no lh_snapshot_pack_rows");
    if (!allreduce) throw std::invalid_argument("JoinRanks: allreduce is empty");
    join(rank, world, std::move(allgather), std::move(allreduce));
}

// The join of both transports: the configuration and the transport are exchanged and checked on every rank alike;
// the peer transport (allreduce empty) then maps every rank's arrays.
void MetricSystem::join(uint32_t rank, uint32_t world, AllGather allgather, AllReduce allreduce) {
    if (world < 2 || world > LH_MAX_RANKS || rank >= world)
        throw std::invalid_argument("JoinRanks: need 2 <= world <= LH_MAX_RANKS and rank < world");
    if (!allgather) throw std::invalid_argument("JoinRanks: allgather is empty");
    std::lock_guard<std::mutex> snap(snapshot_mu_);
    if (collected_) throw std::runtime_error("JoinRanks on a system that has collected already");
    if (allgather_) throw std::runtime_error("JoinRanks on a system that has joined already");
    const uint32_t transport = allreduce ? 1u : 0u;   // 0 peer memory, 1 the caller's all-reduce
    lh_peer_handle mine{};
    if (!allreduce) check(ctx_, lh_comm_export(ctx_, &mine), "lh_comm_export");
    std::string b;
    put_u32(b, kJoinMagic);
    put_u32(b, opt_.max_histograms); put_u32(b, opt_.max_counters); put_u32(b, opt_.precision);
    put_u32(b, transport);
    b.append(reinterpret_cast<const char *>(mine.bytes), sizeof mine.bytes);
    const std::vector<std::string> all = allgather(b);
    if (all.size() != world) throw std::runtime_error("JoinRanks: allgather returned a list of the wrong size");
    std::vector<lh_peer_handle> handles(world);
    for (uint32_t r = 0; r < world; r++) {   // every rank checks the same payloads: all refuse alike
        if (all[r].size() != b.size()) throw std::invalid_argument("JoinRanks: a rank's payload is malformed");
        Reader rd{all[r]};
        if (rd.u32() != kJoinMagic) throw std::invalid_argument("JoinRanks: a rank's payload is malformed");
        const uint32_t h = rd.u32(), c = rd.u32(), p = rd.u32(), t = rd.u32();
        if (h != opt_.max_histograms || c != opt_.max_counters || p != opt_.precision)
            throw std::invalid_argument("JoinRanks: the ranks differ in max_histograms, max_counters or precision");
        if (t != transport)
            throw std::invalid_argument("JoinRanks: the ranks differ in transport (some pass an allreduce, some not)");
        memcpy(handles[r].bytes, all[r].data() + rd.at, sizeof handles[r].bytes);
    }
    if (!allreduce) check(ctx_, lh_comm_import(ctx_, rank, world, handles.data()), "lh_comm_import");
    allgather_ = std::move(allgather);
    allreduce_ = std::move(allreduce);
    std::lock_guard<std::mutex> lk(ranks_mu_);
    ranks_.rank = rank;
    ranks_.world = world;
}

MetricSystem::RanksState MetricSystem::RanksInfo() {
    std::lock_guard<std::mutex> lk(ranks_mu_);
    return ranks_;
}

// What the exchange of one collection decided: the job-wide rows and, for recycling, this rank's own interval.
struct MetricSystem::JobRows {
    std::vector<uint8_t> hist_touched;          // [H] this rank's frozen rows with data
    std::vector<uint64_t> counter_deltas;       // [C] this rank's frozen counter deltas
    std::vector<std::string> hnames, cnames;    // job-wide row g -> name
};

// Steps between lh_snapshot_begin and the reduction of a joined system's collection: lh_snapshot_rows, one exchange,
// the unions, the maps, lh_snapshot_allreduce_rows (or sum_rows through the caller's all-reduce, with each touched
// row's level in the exchange).  False when the exchange failed (nothing was launched: the collection is this rank's
// own).  counter_touched: the host's touched marks (Counter(name, 0) is in Rates).
bool MetricSystem::join_collection(JobRows &j, const std::vector<uint8_t> &counter_touched) {
    const uint32_t H = opt_.max_histograms, Cn = opt_.max_counters;
    const uint32_t rank = ranks_.rank, world = ranks_.world;
    const bool by_allreduce = static_cast<bool>(allreduce_);
    j.hist_touched.assign(H, 0);
    j.counter_deltas.assign(Cn, 0);
    uint32_t frozen = 0;
    std::vector<uint8_t> my_levels;
    lh_comm_stats cs{};
    if (by_allreduce) {
        my_levels.assign(H, 0);
        check(ctx_, lh_snapshot_rows(ctx_, nullptr, j.counter_deltas.data(), &frozen), "lh_snapshot_rows");
        check(ctx_, lh_snapshot_row_levels(ctx_, my_levels.data()), "lh_snapshot_row_levels");
        for (uint32_t h = 0; h < H; h++) j.hist_touched[h] = my_levels[h] != 0;
    } else {
        check(ctx_, lh_snapshot_rows(ctx_, j.hist_touched.data(), j.counter_deltas.data(), &frozen), "lh_snapshot_rows");
        check(ctx_, lh_comm_info(ctx_, &cs), "lh_comm_info");
    }
    std::vector<std::pair<uint32_t, std::string>> mine_h, mine_c;
    {
        std::shared_lock<std::shared_mutex> rl(histos_.mu);
        for (uint32_t h = 0; h < H && h < histos_.names.size(); h++)
            if (j.hist_touched[h]) mine_h.emplace_back(h, histos_.names[h]);
    }
    {
        std::shared_lock<std::shared_mutex> rl(counters_.mu);
        for (uint32_t c = 0; c < Cn && c < counters_.names.size(); c++)
            if (j.counter_deltas[c] || counter_touched[c]) mine_c.emplace_back(c, counters_.names[c]);
    }
    std::string b;
    put_u32(b, kRowsMagic);
    put_u64(b, cs.allreduces);
    put_u32(b, frozen);
    put_u32(b, (uint32_t)mine_h.size());
    for (auto &e : mine_h) {
        put_u32(b, e.first); put_u32(b, (uint32_t)e.second.size()); b += e.second;
        if (by_allreduce) put_u32(b, my_levels[e.first]);
    }
    put_u32(b, (uint32_t)mine_c.size());
    for (auto &e : mine_c) { put_u32(b, e.first); put_u32(b, (uint32_t)e.second.size()); b += e.second; }

    std::vector<uint64_t> seqs(world);
    std::vector<uint32_t> frozens(world);
    std::vector<std::vector<std::pair<uint32_t, std::string>>> hs(world), cs_(world);
    std::vector<std::vector<uint32_t>> hlevels(world);   // by_allreduce: the level of each entry of hs[r]
    try {
        const std::vector<std::string> all = allgather_(b);
        if (all.size() != world) throw std::runtime_error("allgather returned a list of the wrong size");
        for (uint32_t r = 0; r < world; r++) {
            Reader rd{all[r]};
            if (rd.u32() != kRowsMagic) throw std::runtime_error("a rank's payload is malformed");
            seqs[r] = rd.u64();
            frozens[r] = rd.u32();
            if (frozens[r] > 1) throw std::runtime_error("a rank's payload is malformed");
            for (auto *list : {&hs[r], &cs_[r]}) {
                const uint32_t n = rd.u32();
                const uint32_t bound = list == &hs[r] ? H : Cn;
                for (uint32_t i = 0; i < n; i++) {
                    const uint32_t id = rd.u32();
                    if (id >= bound) throw std::runtime_error("a rank's payload is malformed");
                    list->emplace_back(id, rd.str());
                    if (by_allreduce && list == &hs[r]) {
                        const uint32_t lv = rd.u32();
                        if (lv != 1 && lv != 3) throw std::runtime_error("a rank's payload is malformed");
                        hlevels[r].push_back(lv);
                    }
                }
            }
        }
    } catch (const std::exception &e) {
        std::lock_guard<std::mutex> lk(ranks_mu_);
        ranks_.status = 3;
        ranks_.bytes_from_peers = 0;
        if (!exchange_logged_) {
            exchange_logged_ = true;
            fprintf(stderr, "loghisto: rank %u: the collection's exchange failed (%s); collecting this rank alone\n",
                    rank, e.what());
        }
        return false;
    }
    // job-wide rows: the byte-sorted union of each list, cut at the bound
    auto unite = [&](const std::vector<std::vector<std::pair<uint32_t, std::string>>> &per, uint32_t bound,
                     std::vector<std::string> &names, std::vector<uint32_t> &map) {
        std::vector<std::string> u;
        for (auto &l : per) for (auto &e : l) u.push_back(e.second);
        std::sort(u.begin(), u.end());
        u.erase(std::unique(u.begin(), u.end()), u.end());
        const uint64_t dropped_names = u.size() > bound ? u.size() - bound : 0;
        if (u.size() > bound) u.resize(bound);
        std::unordered_map<std::string, uint32_t> row;
        for (uint32_t g = 0; g < u.size(); g++) row.emplace(u[g], g);
        map.assign((size_t)world * u.size(), LH_ROW_ABSENT);
        for (uint32_t r = 0; r < world; r++)
            for (auto &e : per[r]) {
                auto it = row.find(e.second);
                if (it != row.end()) map[(size_t)r * u.size() + it->second] = e.first;
            }
        names = std::move(u);
        return dropped_names;
    };
    std::vector<uint32_t> hmap, cmap;
    const uint64_t dropped_names = unite(hs, H, j.hnames, hmap) + unite(cs_, Cn, j.cnames, cmap);
    if (dropped_names) {   // count what this rank recorded under the names left out (rare: the union is over the bound)
        std::unordered_map<std::string, uint32_t> kept;
        for (auto &n : j.hnames) kept.emplace(n, 0);
        std::vector<uint64_t> row(65536);
        for (auto &e : mine_h)
            if (!kept.count(e.second)) {
                check(ctx_, lh_snapshot_copy_histogram(ctx_, e.first, row.data()), "lh_snapshot_copy_histogram");
                uint64_t n = 0;
                for (uint64_t v : row) n += v;
                dropped_over_limit_.fetch_add(n, std::memory_order_relaxed);
            }
        kept.clear();
        for (auto &n : j.cnames) kept.emplace(n, 0);
        for (auto &e : mine_c)
            if (!kept.count(e.second)) dropped_over_limit_.fetch_add(j.counter_deltas[e.first], std::memory_order_relaxed);
    }
    if (by_allreduce) {
        {
            std::lock_guard<std::mutex> lk(ranks_mu_);
            ranks_.names_dropped += dropped_names;
        }
        // the agreed level of row g: the largest any rank froze it at
        std::unordered_map<std::string, uint32_t> row;
        for (uint32_t g = 0; g < j.hnames.size(); g++) row.emplace(j.hnames[g], g);
        std::vector<uint8_t> levels(j.hnames.size(), 0);
        for (uint32_t r = 0; r < world; r++)
            for (size_t i = 0; i < hs[r].size(); i++) {
                auto it = row.find(hs[r][i].second);
                if (it != row.end()) levels[it->second] = std::max<uint8_t>(levels[it->second], (uint8_t)hlevels[r][i]);
            }
        const size_t nh = j.hnames.size(), nc = j.cnames.size();
        sum_rows(std::vector<uint32_t>(hmap.begin() + rank * nh, hmap.begin() + (rank + 1) * nh), levels,
                 std::vector<uint32_t>(cmap.begin() + rank * nc, cmap.begin() + (rank + 1) * nc));
        return true;
    }
    const uint64_t seq = *std::max_element(seqs.begin(), seqs.end()) + 1;
    check(ctx_, lh_snapshot_allreduce_rows(ctx_, seq, frozens.data(), (uint32_t)j.hnames.size(), hmap.data(),
                                           (uint32_t)j.cnames.size(), cmap.data(), nullptr),
          "lh_snapshot_allreduce_rows");
    std::lock_guard<std::mutex> lk(ranks_mu_);
    ranks_.names_dropped += dropped_names;
    return true;
}

// The job-wide rows through the caller's all-reduce: pack this rank's column of the maps at the agreed levels, sum,
// unpack.  Every rank derives n_words from the same exchange, so every rank calls allreduce_ with the same size, or
// none does.  An allreduce_ that throws leaves this rank's own counts under the job-wide rows (status 4).
void MetricSystem::sum_rows(const std::vector<uint32_t> &hmap, const std::vector<uint8_t> &levels,
                            const std::vector<uint32_t> &cmap) {
    uint64_t *send = nullptr, *recv = nullptr, n_words = 0;
    void *stream = nullptr;
    check(ctx_, lh_snapshot_pack_rows(ctx_, (uint32_t)hmap.size(), hmap.data(), levels.data(), (uint32_t)cmap.size(),
                                      cmap.data(), &send, &recv, &n_words, &stream),
          "lh_snapshot_pack_rows");
    uint32_t status = 0;
    try {
        if (n_words) allreduce_(send, recv, (size_t)n_words, stream);
    } catch (const std::exception &e) {
        status = 4;
        if (!allreduce_logged_) {
            allreduce_logged_ = true;
            fprintf(stderr, "loghisto: rank %u: the collection's allreduce failed (%s); this rank's own counts under the "
                    "job-wide names\n", ranks_.rank, e.what());
        }
    }
    check(ctx_, lh_snapshot_unpack_rows(ctx_, status == 0 ? 1u : 0u), "lh_snapshot_unpack_rows");
    std::lock_guard<std::mutex> lk(ranks_mu_);
    ranks_.status = status;
    ranks_.bytes_from_peers = status == 0 ? 8 * n_words : 0;
    if (status == 0) ranks_.summed++;
}

// collectRawMetrics, metrics.go:420-479.
std::shared_ptr<RawMetricSet> MetricSystem::collectRawMetrics() {
    // lh_snapshot_begin would refuse the call after the flush below; refuse it before anything moves
    refuse_in_scope("collectRawMetrics");
    std::lock_guard<std::mutex> snap(snapshot_mu_);
    collected_ = true;
    auto raw = std::make_shared<RawMetricSet>();
    const int64_t now = std::chrono::duration_cast<std::chrono::nanoseconds>(
                            std::chrono::system_clock::now().time_since_epoch()).count();
    const int64_t iv = interval_.count();
    raw->Time = TimePoint(std::chrono::duration_cast<TimePoint::duration>(std::chrono::nanoseconds(now / iv * iv)));   // :421-423
    raw->origin = this;
    {
        std::lock_guard<std::mutex> lk(percentiles_mu_);
        raw->percentile_labels = percentiles_;
    }

    std::vector<uint8_t> touched(opt_.max_counters, 0);
    // exclusive shards: announce, one process-wide barrier, then every shard is entered as soon as its owner is out
    if (asym_) {
        for (auto &s : shards_) if (s->exclusive) s->reaper_wants.store(1, std::memory_order_seq_cst);
        asym_barrier();
    }
    for (auto &s : shards_) flush_shard(*s, &touched);
    for (size_t c = 0; c < carried_touched_.size(); c++) touched[c] |= carried_touched_[c];
    carried_touched_.clear();
    {   // the drain in lh_snapshot_begin moves graph recorders' counts under the ids their names have now
        std::lock_guard<std::mutex> lk(graph_mu_);
        for (auto &g : graphs_) bind_graph(*g);
    }
    // distribution gauges: every registered name interned (or revived) and used in this interval, so it keeps its id;
    // a name with no free id has its samples dropped and counted.  dist_mu_ stays held until the reduction below has
    // run after the arrays' kernels on the snapshot stream.
    std::unique_lock<std::mutex> dists_held(dist_mu_);
    std::vector<lh_array_src> dists;
    if (!device_dists_.empty()) {
        std::unique_lock<std::shared_mutex> wl(histos_.mu);
        for (auto &d : device_dists_) {
            const uint32_t id = intern_locked(histos_, d.first);
            if (id == RecordScope::kUnbound) { dropped_over_limit_.fetch_add(d.second.n, std::memory_order_relaxed); continue; }
            dists.push_back(d.second);
            dists.back().histogram_id = id;
        }
    }
    if (const lh_status st = lh_snapshot_begin(ctx_); st != LH_OK) {   // the marks stay for the next collection
        carried_touched_ = std::move(touched);
        check(ctx_, st, "lh_snapshot_begin");
    }
    // every array's current values join the interval just frozen, before anything reads it
    if (!dists.empty() && lh_snapshot_ingest_arrays(ctx_, dists.data(), (uint32_t)dists.size()) != LH_OK)
        fprintf(stderr, "loghisto: lh_snapshot_ingest_arrays failed: %s\n", lh_last_error(ctx_));   // the set is still delivered
    // the cache swaps of :425-428 and :460-463 happened in lh_snapshot_begin

    const uint32_t H = opt_.max_histograms, np = (uint32_t)raw->percentile_labels.size();
    std::vector<double> ps(np);
    for (uint32_t j = 0; j < np; j++) ps[j] = raw->percentile_labels[j].second;
    std::vector<uint64_t> counts(H);
    std::vector<double> sums(H), avgs(H), pvals((size_t)H * np);
    std::vector<int32_t> pkeys((size_t)H * np);
    lh_sparse sp{};
    JobRows job;
    bool joined = false;
    try {
        if (allgather_) {
            joined = join_collection(job, touched);
        }
        check(ctx_, lh_snapshot_reduce(ctx_, ps.data(), np, counts.data(), sums.data(), avgs.data(), pkeys.data(), pvals.data()),
              "lh_snapshot_reduce");
        dists_held.unlock();
        check(ctx_, lh_snapshot_export(ctx_, &sp), "lh_snapshot_export");
        if (joined && !allreduce_) {
            lh_comm_stats cs{};
            check(ctx_, lh_comm_info(ctx_, &cs), "lh_comm_info");
            std::lock_guard<std::mutex> lk(ranks_mu_);
            ranks_.status = cs.status;
            ranks_.bytes_from_peers = cs.last_bytes_from_peers;
            if (cs.status == 0) ranks_.summed++;
        }
    } catch (...) {
        lh_snapshot_end(ctx_);
        throw;
    }
    // Label the export with the id -> name tables as they stand (retiring ids included), then step every id's
    // lifecycle (NameTable), each under its table's write lock.  A name interned since lh_snapshot_begin has no data
    // in this export.  Joined, the export's rows are the job-wide ones, and each id's lifecycle follows this rank's
    // own interval (lh_snapshot_rows).
    std::vector<std::string> hnames, cnames;
    {
        std::unique_lock<std::shared_mutex> wl(histos_.mu);
        hnames = joined ? job.hnames : histos_.names;
        std::vector<uint8_t> landed(histos_.names.size());
        for (size_t h = 0; h < landed.size(); h++)
            landed[h] = joined ? job.hist_touched[h] != 0 : sp.offsets[h] != sp.offsets[h + 1];
        recycle(histos_, landed);
    }
    {
        std::unique_lock<std::shared_mutex> wl(counters_.mu);
        cnames = joined ? job.cnames : counters_.names;
        std::vector<uint8_t> landed(counters_.names.size());
        for (size_t c = 0; c < landed.size(); c++)
            landed[c] = (joined ? job.counter_deltas[c] : sp.counter_deltas[c]) != 0 || touched[c];
        recycle(counters_, landed);
    }
    if (joined) touched.assign(cnames.size(), 1);   // every job-wide counter row was touched on some rank
    // histograms: present only when touched this interval (the swapped-out cache only holds touched names)
    for (size_t h = 0; h < hnames.size(); h++) {
        if (sp.offsets[h] == sp.offsets[h + 1]) continue;
        auto &m = raw->Histograms[hnames[h]];
        for (uint32_t i = sp.offsets[h]; i < sp.offsets[h + 1]; i++) m[sp.keys[i]] = sp.counts[i];
        ReducedHistogram r;
        r.count = counts[h]; r.sum = sums[h]; r.avg = avgs[h];
        r.pkeys.assign(pkeys.begin() + h * np, pkeys.begin() + (h + 1) * np);
        r.pvals.assign(pvals.begin() + h * np, pvals.begin() + (h + 1) * np);
        raw->reduced[hnames[h]] = std::move(r);
    }
    // counters: Rates = interval deltas of the names touched (:430-433); Counters = cumulative store (:435-458).
    // "Touched" is tracked on the host (a name appears in Rates even when only Counter(name, 0) was called, or when
    // its amounts wrapped to a zero delta); the deltas themselves come from the device.
    {
        std::lock_guard<std::mutex> lk(counter_store_mu_);
        for (size_t c = 0; c < cnames.size(); c++) {
            uint64_t d = sp.counter_deltas[c];
            if (d || touched[c]) {
                raw->Rates[cnames[c]] = d;
                counter_store_[cnames[c]] += d;
            }
        }
        raw->Counters = counter_store_;
    }
    {   // device subscriptions: this collection's rows, from the reduction above, before the snapshot ends
        std::lock_guard<std::mutex> lk(sub_mu_);
        if (!subs_.empty() || !raw_subs_.empty()) {
            std::unordered_map<std::string, uint32_t> hid_of, cid_of;   // names of Histograms / Rates -> their ids
            for (size_t h = 0; h < hnames.size(); h++)
                if (sp.offsets[h] != sp.offsets[h + 1]) hid_of.emplace(hnames[h], (uint32_t)h);
            for (size_t c = 0; c < cnames.size(); c++)
                if (sp.counter_deltas[c] || touched[c]) cid_of.emplace(cnames[c], (uint32_t)c);
            if (publish_subscriptions(*raw, hid_of, cid_of) != LH_OK)   // the host's metric set is still delivered
                fprintf(stderr, "loghisto: lh_snapshot_publish failed: %s\n", lh_last_error(ctx_));
            if (publish_raw_subscriptions(hid_of) != LH_OK)
                fprintf(stderr, "loghisto: lh_snapshot_publish_raw failed: %s\n", lh_last_error(ctx_));
        }
    }
    check(ctx_, lh_snapshot_end(ctx_), "lh_snapshot_end");
    {
        std::lock_guard<std::mutex> lk(gauge_mu_);
        for (auto &g : gauge_funcs_) raw->Gauges[g.first] = g.second();   // :465-470
        if (!device_gauges_.empty()) {   // every device gauge in one read; none at all when it fails
            std::vector<lh_gauge_src> srcs;
            srcs.reserve(device_gauges_.size());
            for (auto &g : device_gauges_) srcs.push_back(g.second);
            std::vector<double> vals(srcs.size());
            if (lh_gauges_read(ctx_, srcs.data(), (uint32_t)srcs.size(), vals.data()) == LH_OK) {
                size_t i = 0;
                for (auto &g : device_gauges_) raw->Gauges[g.first] = vals[i++];
            } else {   // the host's metric set is still delivered
                fprintf(stderr, "loghisto: lh_gauges_read failed: %s\n", lh_last_error(ctx_));
            }
        }
    }
    return raw;
}

// processMetrics + processHistograms, metrics.go:483-506 and :336-387.  A histogram of a set this system collected
// uses the reduction the device made for that snapshot (parked in raw.reduced); every other histogram (hand-built or
// deserialised sets, unions of several hosts' sets, another system's sets) is reduced from its map by one
// lh_reduce_sparse_host call, with the percentile labels configured now, as processHistograms reads ms.percentiles.
std::shared_ptr<ProcessedMetricSet> MetricSystem::processMetrics(const RawMetricSet &raw) {
    auto out = std::make_shared<ProcessedMetricSet>();
    out->Time = raw.Time;
    auto &m = out->Metrics;
    for (auto &c : raw.Counters) m[c.first] = (double)c.second;
    for (auto &r : raw.Rates) m[r.first + "_rate"] = (double)r.second;

    auto emit = [&](const std::string &name, const ReducedHistogram &r,
                    const std::vector<std::pair<std::string, double>> &labels) {
        const std::string sumName = name + "_sum", countName = name + "_count", avgName = name + "_avg";
        m[countName] = (double)r.count;
        m[sumName] = r.sum;
        m[avgName] = r.avg;
        {   // aggregate store, :359-376
            std::lock_guard<std::mutex> lk(histogram_count_mu_);
            histogram_count_store_[sumName] += go_f64_to_u64(r.sum);
            histogram_count_store_[countName] += r.count;
        }
        for (size_t j = 0; j < labels.size(); j++) {
            if (r.pkeys[j] == std::numeric_limits<int32_t>::min()) {   // percentile() error: logged, key omitted (:380-382)
                fprintf(stderr, "loghisto: unable to calculate percentile: Invalid percentile.  Should be between 0 and 1.\n");
                continue;
            }
            m[format_label(labels[j].first, name)] = r.pvals[j];
        }
    };

    // histograms without a parked reduction, as one CSR
    std::vector<const std::string *> names;
    std::vector<uint32_t> offsets{0};
    std::vector<int16_t> keys;
    std::vector<uint64_t> counts;
    for (auto &h : raw.Histograms) {
        if (raw.origin == this) {
            auto it = raw.reduced.find(h.first);
            if (it != raw.reduced.end()) {
                emit(h.first, it->second, raw.percentile_labels);
                continue;
            }
        }
        names.push_back(&h.first);
        for (auto &b : h.second) { keys.push_back(b.first); counts.push_back(b.second); }
        offsets.push_back((uint32_t)keys.size());
    }
    if (!names.empty()) {
        std::vector<std::pair<std::string, double>> labels;
        {
            std::lock_guard<std::mutex> lk(percentiles_mu_);
            labels = percentiles_;
        }
        const uint32_t n = (uint32_t)names.size(), np = (uint32_t)labels.size();
        std::vector<double> ps(np);
        for (uint32_t j = 0; j < np; j++) ps[j] = labels[j].second;
        std::vector<uint64_t> rc(n);
        std::vector<double> sums(n), avgs(n), pvals((size_t)n * np);
        std::vector<int32_t> pkeys((size_t)n * np);
        if (!lh_reduce_sparse_host)
            throw std::runtime_error("processMetrics: this libloghisto_b200 has no lh_reduce_sparse_host, so only sets this "
                                     "MetricSystem collected can be processed");
        check(ctx_, lh_reduce_sparse_host(ctx_, n, offsets.data(), keys.data(), counts.data(), ps.data(), np, rc.data(),
                                          sums.data(), avgs.data(), pkeys.data(), pvals.data()),
              "lh_reduce_sparse_host");
        for (uint32_t i = 0; i < n; i++) {
            ReducedHistogram r;
            r.count = rc[i]; r.sum = sums[i]; r.avg = avgs[i];
            r.pkeys.assign(pkeys.begin() + (size_t)i * np, pkeys.begin() + (size_t)(i + 1) * np);
            r.pvals.assign(pvals.begin() + (size_t)i * np, pvals.begin() + (size_t)(i + 1) * np);
            emit(*names[i], r, labels);
        }
    }
    for (auto &g : raw.Gauges) m[g.first] = g.second;
    return out;
}

// the reaper's "add aggregate mean" step, metrics.go:590-608 (integer division)
void MetricSystem::add_aggregates(const RawMetricSet &raw, ProcessedMetricSet &out) {
    for (auto &h : raw.Histograms) {
        uint64_t aggCount = 0, aggSum = 0;
        bool countPresent, sumPresent;
        {
            std::lock_guard<std::mutex> lk(histogram_count_mu_);
            auto c = histogram_count_store_.find(h.first + "_count");
            auto s = histogram_count_store_.find(h.first + "_sum");
            countPresent = c != histogram_count_store_.end();
            sumPresent = s != histogram_count_store_.end();
            if (countPresent) aggCount = c->second;
            if (sumPresent) aggSum = s->second;
        }
        if (countPresent && sumPresent && aggCount > 0) {
            out.Metrics[h.first + "_agg_avg"] = (double)(aggSum / aggCount);
            out.Metrics[h.first + "_agg_count"] = (double)aggCount;
            out.Metrics[h.first + "_agg_sum"] = (double)aggSum;
        }
    }
}

void MetricSystem::SubscribeToRawMetrics(std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>> ch) {
    std::lock_guard<std::mutex> lk(subscribers_mu_);
    raw_subscribers_.push_back(std::move(ch));
}
void MetricSystem::UnsubscribeFromRawMetrics(std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>> ch) {
    std::lock_guard<std::mutex> lk(subscribers_mu_);
    raw_subscribers_.erase(std::remove(raw_subscribers_.begin(), raw_subscribers_.end(), ch), raw_subscribers_.end());
    raw_bad_.erase(ch.get());
}
void MetricSystem::SubscribeToProcessedMetrics(std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>> ch) {
    std::lock_guard<std::mutex> lk(subscribers_mu_);
    processed_subscribers_.push_back(std::move(ch));
}
void MetricSystem::UnsubscribeFromProcessedMetrics(std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>> ch) {
    std::lock_guard<std::mutex> lk(subscribers_mu_);
    processed_subscribers_.erase(std::remove(processed_subscribers_.begin(), processed_subscribers_.end(), ch),
                                 processed_subscribers_.end());
    processed_bad_.erase(ch.get());
}

// reaper, metrics.go:530-639: wake at wall-clock multiples of the interval, collect, broadcast raw,
// process, add aggregates, broadcast processed; never block on a subscriber, close one that misses twice.
void MetricSystem::reaper() {
    for (;;) {
        const int64_t iv = interval_.count();
        const int64_t now = std::chrono::duration_cast<std::chrono::nanoseconds>(
                                std::chrono::system_clock::now().time_since_epoch()).count();
        const int64_t tts = iv - (now % iv);
        {
            std::unique_lock<std::mutex> lk(run_mu_);
            if (run_cv_.wait_for(lk, std::chrono::nanoseconds(tts), [&] { return shutdown_; })) {
                reaping_ = false;
                return;
            }
        }
        std::shared_ptr<RawMetricSet> raw;
        try {
            raw = collectRawMetrics();
        } catch (const std::exception &e) {
            fprintf(stderr, "loghisto: collectRawMetrics failed: %s\n", e.what());
            continue;
        }
        {
            std::lock_guard<std::mutex> lk(subscribers_mu_);
            for (size_t i = 0; i < raw_subscribers_.size();) {
                auto &ch = raw_subscribers_[i];
                if (ch->TrySend(raw)) { raw_bad_.erase(ch.get()); i++; continue; }
                fprintf(stderr, "loghisto: a raw subscriber has allowed their channel to fill up. dropping their metrics on the floor rather than blocking.\n");
                if (++raw_bad_[ch.get()] >= 2) {
                    ch->Close();
                    raw_bad_.erase(ch.get());
                    raw_subscribers_.erase(raw_subscribers_.begin() + i);
                } else {
                    i++;
                }
            }
        }
        std::shared_ptr<ProcessedMetricSet> processed;
        try {
            processed = processMetrics(*raw);
        } catch (const std::exception &e) {
            fprintf(stderr, "loghisto: processMetrics failed: %s\n", e.what());
            continue;
        }
        add_aggregates(*raw, *processed);
        {
            std::lock_guard<std::mutex> lk(subscribers_mu_);
            for (size_t i = 0; i < processed_subscribers_.size();) {
                auto &ch = processed_subscribers_[i];
                if (ch->TrySend(processed)) { processed_bad_.erase(ch.get()); i++; continue; }
                fprintf(stderr, "loghisto: a subscriber has allowed their channel to fill up. dropping their metrics on the floor rather than blocking.\n");
                if (++processed_bad_[ch.get()] >= 2) {
                    ch->Close();
                    processed_bad_.erase(ch.get());
                    processed_subscribers_.erase(processed_subscribers_.begin() + i);
                } else {
                    i++;
                }
            }
        }
    }
}

void MetricSystem::Start() {
    std::lock_guard<std::mutex> lk(run_mu_);
    if (reaping_ || shutdown_) return;
    reaping_ = true;
    reaper_thread_ = std::thread([this] { reaper(); });
}

void MetricSystem::Stop() {   // idempotent, unlike the reference's double close (metrics.go:652)
    {
        std::lock_guard<std::mutex> lk(run_mu_);
        shutdown_ = true;
    }
    run_cv_.notify_all();
    if (reaper_thread_.joinable() && std::this_thread::get_id() != reaper_thread_.get_id()) reaper_thread_.join();
}

}  // namespace loghisto

// ---------------------------------------------------------------------------------------------
// C shim so that ctypes tests can replay the reference's metrics_test.go against the C++ mirror.
using namespace loghisto;

extern "C" {
#define LHMS_API __attribute__((visibility("default")))
typedef void (*lhms_emit_fn)(void *ctx, int kind, const char *name, int key, uint64_t u, double f);

LHMS_API void *lhms_new(int64_t interval_ns, int device, uint32_t max_histograms, uint32_t max_counters, char *err, int errlen) {
    try {
        Options o;
        o.device = device;
        o.max_histograms = max_histograms;
        o.max_counters = max_counters;
        return new MetricSystem(std::chrono::nanoseconds(interval_ns), false, o);
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return nullptr;
    }
}
// as lhms_new, at a bucket precision other than the reference's 100 (Options.precision)
LHMS_API void *lhms_new_precision(int64_t interval_ns, int device, uint32_t max_histograms, uint32_t max_counters,
                                  uint32_t precision, char *err, int errlen) {
    try {
        Options o;
        o.device = device;
        o.max_histograms = max_histograms;
        o.max_counters = max_counters;
        o.precision = precision;
        return new MetricSystem(std::chrono::nanoseconds(interval_ns), false, o);
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return nullptr;
    }
}
static void end_scopes_of(void *ms);
LHMS_API void lhms_free(void *ms) {
    end_scopes_of(ms);   // scopes the caller left open end before their system goes
    delete static_cast<MetricSystem *>(ms);
}
// Nothing may unwind through these C entry points (ctypes / cgo callers): the ingest methods are noexcept, the
// remaining allocations are guarded.
LHMS_API void lhms_histogram(void *ms, const char *name, double v) {
    if (!ms || !name) return;
    static_cast<MetricSystem *>(ms)->Histogram(name, strlen(name), v);
}
LHMS_API void lhms_counter(void *ms, const char *name, uint64_t a) {
    if (!ms || !name) return;
    try { static_cast<MetricSystem *>(ms)->Counter(std::string(name), a); } catch (...) {}
}
LHMS_API void lhms_histogram_many(void *ms, const char *name, const double *v, size_t n) {
    if (!ms || !name) return;
    auto *m = static_cast<MetricSystem *>(ms);
    const size_t len = strlen(name);
    for (size_t i = 0; i < n; i++) m->Histogram(name, len, v[i]);
}
LHMS_API void *lhms_start_timer(void *ms, const char *name) {
    if (!ms || !name) return nullptr;
    try { return new TimerToken(static_cast<MetricSystem *>(ms)->StartTimer(name)); } catch (...) { return nullptr; }
}
// consumes the token; a NULL token (failed start, or a second stop through a cleared handle) returns 0
LHMS_API int64_t lhms_timer_stop(void *token) {
    if (!token) return 0;
    auto *t = static_cast<TimerToken *>(token);
    int64_t ns = t->Stop().count();
    delete t;
    return ns;
}
LHMS_API void lhms_timer_free(void *token) { delete static_cast<TimerToken *>(token); }
LHMS_API void lhms_specify_percentiles(void *ms, int n, const char *const *labels, const double *ps) {
    std::map<std::string, double> m;
    for (int i = 0; i < n; i++) m[labels[i]] = ps[i];
    static_cast<MetricSystem *>(ms)->SpecifyPercentiles(m);
}
LHMS_API void lhms_register_constant_gauge(void *ms, const char *name, double v) {
    static_cast<MetricSystem *>(ms)->RegisterGaugeFunc(name, [v] { return v; });
}
// RegisterDeviceGauge: LH_OK, LH_ERR_INVALID when the address or dtype is refused, LH_ERR_STATE for any other failure.
LHMS_API int lhms_register_device_gauge(void *ms, const char *name, const void *d_value, uint32_t dtype) {
    if (!ms || !name) return LH_ERR_INVALID;
    try {
        static_cast<MetricSystem *>(ms)->RegisterDeviceGauge(name, d_value, dtype);
        return LH_OK;
    } catch (const std::invalid_argument &) {
        return LH_ERR_INVALID;
    } catch (const std::exception &) {
        return LH_ERR_STATE;
    }
}
// DeregisterGaugeFunc: removes a gauge function or a device gauge
LHMS_API void lhms_deregister_gauge(void *ms, const char *name) {
    static_cast<MetricSystem *>(ms)->DeregisterGaugeFunc(name);
}
// RegisterDeviceDistribution: LH_OK, LH_ERR_INVALID when the dtype or the first element's address is refused,
// LH_ERR_STATE for any other failure (a thread that holds an open record scope among them).
LHMS_API int lhms_register_device_distribution(void *ms, const char *name, const void *d_values, uint64_t n, uint32_t dtype) {
    if (!ms || !name) return LH_ERR_INVALID;
    try {
        static_cast<MetricSystem *>(ms)->RegisterDeviceDistribution(name, d_values, n, dtype);
        return LH_OK;
    } catch (const std::invalid_argument &) {
        return LH_ERR_INVALID;
    } catch (const std::exception &) {
        return LH_ERR_STATE;
    }
}
// DeregisterDeviceDistribution: LH_OK, or LH_ERR_STATE from a thread that holds an open record scope.
LHMS_API int lhms_deregister_device_distribution(void *ms, const char *name) {
    if (!ms || !name) return LH_ERR_INVALID;
    try {
        static_cast<MetricSystem *>(ms)->DeregisterDeviceDistribution(name);
        return LH_OK;
    } catch (const std::exception &) {
        return LH_ERR_STATE;
    }
}
// lh_get_stats of the system's context (e.g. the kernel launches a collection issues)
LHMS_API int lhms_stats(void *ms, lh_stats *out) {
    return lh_get_stats(static_cast<MetricSystem *>(ms)->context(), out);
}

static void emit_raw(const RawMetricSet &raw, lhms_emit_fn emit, void *ctx) {
    for (auto &c : raw.Counters) emit(ctx, 0, c.first.c_str(), 0, c.second, 0);
    for (auto &r : raw.Rates) emit(ctx, 1, r.first.c_str(), 0, r.second, 0);
    for (auto &h : raw.Histograms)
        for (auto &b : h.second) emit(ctx, 2, h.first.c_str(), b.first, b.second, 0);
    for (auto &g : raw.Gauges) emit(ctx, 4, g.first.c_str(), 0, 0, g.second);
}
static void emit_processed(const ProcessedMetricSet &p, lhms_emit_fn emit, void *ctx) {
    for (auto &m : p.Metrics) emit(ctx, 3, m.first.c_str(), 0, 0, m.second);
}

// processMetrics(collectRawMetrics()), as metrics_test.go:195 does.  Returns 0, or -1 with err filled.
LHMS_API int lhms_collect_and_process(void *ms, lhms_emit_fn emit, void *ctx, char *err, int errlen) {
    try {
        auto *m = static_cast<MetricSystem *>(ms);
        auto raw = m->collectRawMetrics();
        auto p = m->processMetrics(*raw);
        emit_raw(*raw, emit, ctx);
        emit_processed(*p, emit, ctx);
        return 0;
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -1;
    }
}
// MetricSystem::JoinRanks with a C all-gather: allgather(user, mine, len, sink, sink_ctx) calls sink(sink_ctx, r, p,
// len) once for every rank r with that rank's bytes (the library copies them during the call) and returns 0, or
// nonzero on failure.  It is called on the collecting thread.  Returns 0, -1 with err filled, or -2 with err filled
// when the arguments or the ranks' configurations do not fit (std::invalid_argument).
typedef void (*lhms_ranks_sink_fn)(void *sink_ctx, uint32_t rank, const void *p, uint64_t len);
typedef int (*lhms_ranks_allgather_fn)(void *user, const void *mine, uint64_t len, lhms_ranks_sink_fn sink, void *sink_ctx);
namespace {
struct GatherSink {
    std::vector<std::string> parts;
    std::vector<uint8_t> seen;
};
void gather_sink(void *sink_ctx, uint32_t rank, const void *p, uint64_t len) {
    auto *g = static_cast<GatherSink *>(sink_ctx);
    if (rank >= g->parts.size() || (len && !p)) return;
    g->parts[rank].assign(static_cast<const char *>(p), (size_t)len);
    g->seen[rank] = 1;
}
MetricSystem::AllGather c_allgather(lhms_ranks_allgather_fn allgather, void *user, uint32_t world) {
    return [allgather, user, world](const std::string &mine) {
        GatherSink g;
        g.parts.resize(world);
        g.seen.assign(world, 0);
        if (allgather(user, mine.data(), mine.size(), gather_sink, &g) != 0)
            throw std::runtime_error("the all-gather callback failed");
        for (uint32_t r = 0; r < world; r++)
            if (!g.seen[r]) throw std::runtime_error("the all-gather callback left a rank out");
        return g.parts;
    };
}
}  // namespace
LHMS_API int lhms_ranks_join(void *ms, uint32_t rank, uint32_t world, lhms_ranks_allgather_fn allgather, void *user,
                             char *err, int errlen) {
    try {
        if (!ms || !allgather) throw std::invalid_argument("lhms_ranks_join: NULL system or allgather");
        static_cast<MetricSystem *>(ms)->JoinRanks(rank, world, c_allgather(allgather, user, world));
        return 0;
    } catch (const std::invalid_argument &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -2;
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -1;
    }
}
// MetricSystem::JoinRanks over the caller's all-reduce: allgather as for lhms_ranks_join, and allreduce(user, d_send,
// d_recv, n_words, stream), which leaves in d_recv the wrapping uint64 sum over ranks of d_send (enqueued on stream, or
// completed when it returns) and returns 0, or nonzero on failure.  Both are called on the collecting thread.  Returns
// as lhms_ranks_join.
typedef int (*lhms_ranks_allreduce_fn)(void *user, const uint64_t *d_send, uint64_t *d_recv, uint64_t n_words, void *stream);
LHMS_API int
lhms_ranks_join_allreduce(void *ms, uint32_t rank, uint32_t world, lhms_ranks_allgather_fn allgather,
                          lhms_ranks_allreduce_fn allreduce, void *user, char *err, int errlen) {
    try {
        if (!ms || !allgather || !allreduce) throw std::invalid_argument("lhms_ranks_join_allreduce: NULL system or callback");
        auto reduce = [allreduce, user](const uint64_t *d_send, uint64_t *d_recv, size_t n_words, void *stream) {
            if (allreduce(user, d_send, d_recv, n_words, stream) != 0) throw std::runtime_error("the all-reduce callback failed");
        };
        static_cast<MetricSystem *>(ms)->JoinRanks(rank, world, c_allgather(allgather, user, world), reduce);
        return 0;
    } catch (const std::invalid_argument &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -2;
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -1;
    }
}
// MetricSystem::RanksInfo: out[0..5] = rank, world, status, collections summed, bytes from peers, names dropped.
LHMS_API void lhms_ranks_info(void *ms, uint64_t *out) {
    if (!ms || !out) return;
    const MetricSystem::RanksState r = static_cast<MetricSystem *>(ms)->RanksInfo();
    out[0] = r.rank; out[1] = r.world; out[2] = r.status; out[3] = r.summed; out[4] = r.bytes_from_peers;
    out[5] = r.names_dropped;
}
// processMetrics(raw) for a RawMetricSet built from flat arrays (a set this system did not collect): histogram i is
// entries [offsets[i], offsets[i+1]) of keys / counts (repeated keys are summed).  Emits the processed metrics.
// aggregates != 0 adds the reaper's _agg_* metrics as well (metrics.go:590-608).  Returns 0, or -1 with err filled.
LHMS_API int lhms_process_metrics(void *ms, int64_t time_ns, int aggregates,
                                  uint32_t n_counters, const char *const *counter_names, const uint64_t *counter_values,
                                  uint32_t n_rates, const char *const *rate_names, const uint64_t *rate_values,
                                  uint32_t n_hist, const char *const *hist_names, const uint32_t *offsets,
                                  const int16_t *keys, const uint64_t *counts,
                                  uint32_t n_gauges, const char *const *gauge_names, const double *gauge_values,
                                  lhms_emit_fn emit, void *ctx, char *err, int errlen) {
    try {
        RawMetricSet raw;
        raw.Time = TimePoint(std::chrono::duration_cast<TimePoint::duration>(std::chrono::nanoseconds(time_ns)));
        for (uint32_t i = 0; i < n_counters; i++) raw.Counters[counter_names[i]] = counter_values[i];
        for (uint32_t i = 0; i < n_rates; i++) raw.Rates[rate_names[i]] = rate_values[i];
        for (uint32_t i = 0; i < n_hist; i++) {
            auto &m = raw.Histograms[hist_names[i]];
            for (uint32_t e = offsets[i]; e < offsets[i + 1]; e++) m[keys[e]] += counts[e];
        }
        for (uint32_t i = 0; i < n_gauges; i++) raw.Gauges[gauge_names[i]] = gauge_values[i];
        auto *m = static_cast<MetricSystem *>(ms);
        auto p = m->processMetrics(raw);
        if (aggregates) m->add_aggregates(raw, *p);
        emit_processed(*p, emit, ctx);
        return 0;
    } catch (const std::exception &e) {
        if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", e.what());
        return -1;
    }
}
// Record scopes bound to names (MetricSystem::BeginRecording), kept here by (system, lh_recorder.scope).  h_ids /
// c_ids receive one id per name (0xFFFFFFFF: no free id, records dropped and counted).  Return an lh_status.
static std::mutex g_scopes_mu;
static std::map<std::pair<void *, uint64_t>, RecordScope> g_scopes;
static lh_status scope_status(const std::exception &e) {
    return dynamic_cast<const std::out_of_range *>(&e) ? LH_ERR_RANGE : LH_ERR_STATE;
}
LHMS_API int lhms_record_begin(void *ms, void *stream, uint32_t n_h, const char *const *h_names, uint32_t n_c,
                               const char *const *c_names, lh_recorder *out, uint32_t *h_ids, uint32_t *c_ids) {
    if (!ms || !out || (n_h && (!h_names || !h_ids)) || (n_c && (!c_names || !c_ids))) return LH_ERR_INVALID;
    try {
        std::vector<std::string> hs(h_names, h_names + n_h), cs(c_names, c_names + n_c);
        RecordScope s = static_cast<MetricSystem *>(ms)->BeginRecording(stream, hs, cs);
        *out = s.recorder();
        for (uint32_t i = 0; i < n_h; i++) h_ids[i] = s.histogram_id(i);
        for (uint32_t i = 0; i < n_c; i++) c_ids[i] = s.counter_id(i);
        std::lock_guard<std::mutex> lk(g_scopes_mu);
        g_scopes.emplace(std::make_pair(ms, out->scope), std::move(s));
        return LH_OK;
    } catch (const std::exception &e) {
        return scope_status(e);
    }
}
static void end_scopes_of(void *ms) {
    std::vector<RecordScope> left;
    {
        std::lock_guard<std::mutex> lk(g_scopes_mu);
        for (auto it = g_scopes.begin(); it != g_scopes.end();) {
            if (it->first.first != ms) { ++it; continue; }
            left.push_back(std::move(it->second));
            it = g_scopes.erase(it);
        }
    }
}   // `left` ends them
LHMS_API int lhms_record_end(void *ms, const lh_recorder *rec) {
    if (!ms || !rec) return LH_ERR_INVALID;
    RecordScope s;
    {
        std::lock_guard<std::mutex> lk(g_scopes_mu);
        auto it = g_scopes.find(std::make_pair(ms, rec->scope));
        if (it == g_scopes.end()) return LH_ERR_INVALID;
        s = std::move(it->second);
        g_scopes.erase(it);
    }
    try { s.End(); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_record_ingest_f64(void *ms, const lh_recorder *rec, uint32_t name_index, const double *d_values, size_t n) {
    if (!ms || !rec) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g_scopes_mu);
    auto it = g_scopes.find(std::make_pair(ms, rec->scope));
    if (it == g_scopes.end()) return LH_ERR_INVALID;
    try { it->second.Histogram(name_index, d_values, n); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
// RecordScope::Histograms: item i is n[i] samples of kind kinds[i] (LH_VALUES_*) at d_values[i] under histogram name
// name_index[i] of the scope.
LHMS_API int lhms_scope_histograms(void *ms, const lh_recorder *rec, const uint32_t *name_index,
                                      const void *const *d_values, const uint64_t *n, const uint32_t *kinds,
                                      uint32_t n_items) {
    if (!ms || !rec || (n_items && (!name_index || !d_values || !n || !kinds))) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g_scopes_mu);
    auto it = g_scopes.find(std::make_pair(ms, rec->scope));
    if (it == g_scopes.end()) return LH_ERR_INVALID;
    try {
        std::vector<RecordScope::Item> items(n_items);
        for (uint32_t i = 0; i < n_items; i++) items[i] = RecordScope::Item{name_index[i], d_values[i], (size_t)n[i], kinds[i]};
        it->second.Histograms(items);
        return LH_OK;
    } catch (const std::exception &e) {
        return scope_status(e);
    }
}
// RecordScope::Keyed / Counters (id_bytes 2 or 4: uint16 or uint32 local ids).
LHMS_API int lhms_scoped_keyed(void *ms, const lh_recorder *rec, uint32_t id_bytes, const void *d_ids, const void *d_values,
                               uint32_t kind, size_t n) {
    if (!ms || !rec) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g_scopes_mu);
    auto it = g_scopes.find(std::make_pair(ms, rec->scope));
    if (it == g_scopes.end()) return LH_ERR_INVALID;
    try { it->second.Keyed(d_ids, id_bytes, d_values, kind, n); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_scoped_counters(void *ms, const lh_recorder *rec, uint32_t id_bytes, const void *d_ids,
                                  const uint64_t *d_amounts, size_t n) {
    if (!ms || !rec) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g_scopes_mu);
    auto it = g_scopes.find(std::make_pair(ms, rec->scope));
    if (it == g_scopes.end()) return LH_ERR_INVALID;
    try { it->second.Counters(d_ids, id_bytes, d_amounts, n); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
// GPU timers (MetricSystem::StartGpuTimer).  start returns a token, or NULL with *status set; stop may be called
// repeatedly on `stream` (passed as given: NULL = the context's ingest stream); free releases the token's slot.
LHMS_API void *lhms_gpu_timer_start(void *ms, const char *name, void *stream, int *status) {
    if (!ms || !name || !status) { if (status) *status = LH_ERR_INVALID; return nullptr; }
    try {
        auto *t = new GpuTimerToken(static_cast<MetricSystem *>(ms)->StartGpuTimer(name, stream));
        *status = LH_OK;
        return t;
    } catch (const std::exception &e) {
        *status = scope_status(e);
        return nullptr;
    }
}
LHMS_API int lhms_gpu_timer_stop(void *token, void *stream, int64_t *d_duration_ns) {
    if (!token) return LH_ERR_INVALID;
    try { static_cast<GpuTimerToken *>(token)->Stop(stream, d_duration_ns); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API void lhms_gpu_timer_free(void *token) { delete static_cast<GpuTimerToken *>(token); }
// MetricSystem::NewGraphRecorder: a GraphRecorder handle (NULL with *status set on failure); *out receives its
// recorder.  Free it with lhms_graph_recorder_free, which closes it if lhms_graph_recorder_close has not.
LHMS_API void *lhms_graph_recorder_new(void *ms, uint32_t n_h, const char *const *h_names, uint32_t n_c,
                                       const char *const *c_names, lh_recorder *out, int *status) {
    int dummy;
    if (!status) status = &dummy;
    *status = LH_ERR_INVALID;
    if (!ms || !out || (n_h && !h_names) || (n_c && !c_names)) return nullptr;
    try {
        std::vector<std::string> hs(h_names, h_names + n_h), cs(c_names, c_names + n_c);
        auto *g = new GraphRecorder(static_cast<MetricSystem *>(ms)->NewGraphRecorder(hs, cs));
        *out = g->recorder();
        *status = LH_OK;
        return g;
    } catch (const std::exception &e) {
        *status = scope_status(e);
        return nullptr;
    }
}
// GraphRecorder::Histograms: item i is n[i] samples of kind kinds[i] at d_values[i] under histogram name name_index[i].
LHMS_API int lhms_graph_recorder_histograms(void *g, const uint32_t *name_index, const void *const *d_values,
                                            const uint64_t *n, const uint32_t *kinds, uint32_t n_items, void *stream) {
    if (!g || (n_items && (!name_index || !d_values || !n || !kinds))) return LH_ERR_INVALID;
    try {
        std::vector<GraphRecorder::Item> items(n_items);
        for (uint32_t i = 0; i < n_items; i++) items[i] = GraphRecorder::Item{name_index[i], d_values[i], (size_t)n[i], kinds[i]};
        static_cast<GraphRecorder *>(g)->Histograms(items, stream);
        return LH_OK;
    } catch (const std::exception &e) {
        return scope_status(e);
    }
}
// RecordScope::Arrays of the open scope `rec` and GraphRecorder::Arrays, items as lhms_scope_histograms' with dtypes
// (LH_GAUGE_*) for kinds; statuses as theirs.
LHMS_API int lhms_arrays_scope(void *ms, const lh_recorder *rec, const uint32_t *name_index, const void *const *d_values,
                               const uint64_t *n, const uint32_t *dtypes, uint32_t n_items) {
    if (!ms || !rec || (n_items && (!name_index || !d_values || !n || !dtypes))) return LH_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g_scopes_mu);
    auto it = g_scopes.find(std::make_pair(ms, rec->scope));
    if (it == g_scopes.end()) return LH_ERR_INVALID;
    try {
        std::vector<RecordScope::ArrayItem> items(n_items);
        for (uint32_t i = 0; i < n_items; i++) items[i] = RecordScope::ArrayItem{name_index[i], d_values[i], (size_t)n[i], dtypes[i]};
        it->second.Arrays(items);
        return LH_OK;
    } catch (const std::exception &e) {
        return scope_status(e);
    }
}
LHMS_API int lhms_arrays_graph_recorder(void *g, const uint32_t *name_index, const void *const *d_values, const uint64_t *n,
                                        const uint32_t *dtypes, uint32_t n_items, void *stream) {
    if (!g || (n_items && (!name_index || !d_values || !n || !dtypes))) return LH_ERR_INVALID;
    try {
        std::vector<GraphRecorder::ArrayItem> items(n_items);
        for (uint32_t i = 0; i < n_items; i++) items[i] = GraphRecorder::ArrayItem{name_index[i], d_values[i], (size_t)n[i], dtypes[i]};
        static_cast<GraphRecorder *>(g)->Arrays(items, stream);
        return LH_OK;
    } catch (const std::exception &e) {
        return scope_status(e);
    }
}
// GraphRecorder::Keyed / Counters / StartTimer / StopTimer.
LHMS_API int lhms_graph_keyed(void *g, uint32_t id_bytes, const void *d_ids, const void *d_values, uint32_t kind, size_t n,
                              void *stream) {
    if (!g) return LH_ERR_INVALID;
    try { static_cast<GraphRecorder *>(g)->Keyed(d_ids, id_bytes, d_values, kind, n, stream); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_graph_counters(void *g, uint32_t id_bytes, const void *d_ids, const uint64_t *d_amounts, size_t n, void *stream) {
    if (!g) return LH_ERR_INVALID;
    try { static_cast<GraphRecorder *>(g)->Counters(d_ids, id_bytes, d_amounts, n, stream); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_graph_timer_start(void *g, uint32_t name_index, void *stream) {
    if (!g) return LH_ERR_INVALID;
    try { static_cast<GraphRecorder *>(g)->StartTimer(name_index, stream); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_graph_timer_stop(void *g, uint32_t name_index, void *stream, int64_t *d_duration_ns) {
    if (!g) return LH_ERR_INVALID;
    try { static_cast<GraphRecorder *>(g)->StopTimer(name_index, stream, d_duration_ns); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_graph_recorder_close(void *g, void *stream) {
    if (!g) return LH_ERR_INVALID;
    try { static_cast<GraphRecorder *>(g)->Close(stream); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API void lhms_graph_recorder_free(void *g) { delete static_cast<GraphRecorder *>(g); }
// MetricSystem::NewDeviceSubscription: a DeviceSubscription handle (NULL with *status set on failure); *out receives
// its board.  Free it with lhms_subscription_free, which closes it if lhms_subscription_close has not.
LHMS_API void *lhms_subscription_new(void *ms, uint32_t n_h, const char *const *h_names, uint32_t n_c,
                                     const char *const *c_names, lh_board *out, int *status) {
    int dummy;
    if (!status) status = &dummy;
    *status = LH_ERR_INVALID;
    if (!ms || !out || (n_h && !h_names) || (n_c && !c_names)) return nullptr;
    try {
        std::vector<std::string> hs(h_names, h_names + n_h), cs(c_names, c_names + n_c);
        auto *d = new DeviceSubscription(static_cast<MetricSystem *>(ms)->NewDeviceSubscription(hs, cs));
        *out = d->board();
        *status = LH_OK;
        return d;
    } catch (const std::exception &e) {
        *status = scope_status(e);
        return nullptr;
    }
}
// DeviceSubscription::Read of the board image into d_out on `stream`.
LHMS_API int lhms_subscription_read(void *d, void *d_out, void *stream) {
    if (!d) return LH_ERR_INVALID;
    try { static_cast<DeviceSubscription *>(d)->Read(d_out, stream); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_subscription_close(void *d) {
    if (!d) return LH_ERR_INVALID;
    try { static_cast<DeviceSubscription *>(d)->Close(); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API void lhms_subscription_free(void *d) { delete static_cast<DeviceSubscription *>(d); }
// MetricSystem::NewRawDeviceSubscription: a RawDeviceSubscription handle (NULL with *status set on failure); *out
// receives its board.  Free it with lhms_raw_subscription_free, which closes it if lhms_raw_subscription_close has not.
LHMS_API void *lhms_raw_subscription_new(void *ms, uint32_t n_h, const char *const *h_names, lh_raw_board *out,
                                         int *status) {
    int dummy;
    if (!status) status = &dummy;
    *status = LH_ERR_INVALID;
    if (!ms || !out || (n_h && !h_names)) return nullptr;
    try {
        std::vector<std::string> hs(h_names, h_names + n_h);
        auto *d = new RawDeviceSubscription(static_cast<MetricSystem *>(ms)->NewRawDeviceSubscription(hs));
        *out = d->board();
        *status = LH_OK;
        return d;
    } catch (const std::exception &e) {
        *status = scope_status(e);
        return nullptr;
    }
}
// MetricSystem::NewRawDeviceSubscription with a window: as lhms_raw_subscription_new, each row summed over the last
// `window` collections.
LHMS_API void *lhms_raw_window_subscription_new(void *ms, uint32_t n_h, const char *const *h_names, uint32_t window,
                                                lh_raw_board *out, int *status) {
    int dummy;
    if (!status) status = &dummy;
    *status = LH_ERR_INVALID;
    if (!ms || !out || (n_h && !h_names)) return nullptr;
    try {
        std::vector<std::string> hs(h_names, h_names + n_h);
        auto *d = new RawDeviceSubscription(static_cast<MetricSystem *>(ms)->NewRawDeviceSubscription(hs, window));
        *out = d->board();
        *status = LH_OK;
        return d;
    } catch (const std::exception &e) {
        *status = scope_status(e);
        return nullptr;
    }
}
// RawDeviceSubscription::Percentiles / Ranks on `stream`.
LHMS_API int lhms_raw_subscription_percentiles(void *d, const double *d_ps, uint32_t m, int32_t *d_keys, double *d_vals,
                                               uint64_t *d_publish, void *stream) {
    if (!d) return LH_ERR_INVALID;
    try {
        static_cast<RawDeviceSubscription *>(d)->Percentiles(d_ps, m, d_keys, d_vals, d_publish, stream);
        return LH_OK;
    } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_raw_subscription_ranks(void *d, const double *d_values, uint32_t m, uint64_t *d_ranks,
                                         uint64_t *d_totals, uint64_t *d_publish, void *stream) {
    if (!d) return LH_ERR_INVALID;
    try {
        static_cast<RawDeviceSubscription *>(d)->Ranks(d_values, m, d_ranks, d_totals, d_publish, stream);
        return LH_OK;
    } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API int lhms_raw_subscription_close(void *d) {
    if (!d) return LH_ERR_INVALID;
    try { static_cast<RawDeviceSubscription *>(d)->Close(); return LH_OK; } catch (const std::exception &e) { return scope_status(e); }
}
LHMS_API void lhms_raw_subscription_free(void *d) { delete static_cast<RawDeviceSubscription *>(d); }
LHMS_API void lhms_start(void *ms) { static_cast<MetricSystem *>(ms)->Start(); }
LHMS_API void lhms_stop(void *ms) { static_cast<MetricSystem *>(ms)->Stop(); }
LHMS_API uint64_t lhms_dropped(void *ms) { return static_cast<MetricSystem *>(ms)->dropped_samples(); }

using RawCh = std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>>;
using ProcCh = std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>>;

LHMS_API void *lhms_subscribe_processed(void *ms, int capacity) {
    auto *ch = new ProcCh(std::make_shared<Channel<std::shared_ptr<ProcessedMetricSet>>>((size_t)capacity));
    static_cast<MetricSystem *>(ms)->SubscribeToProcessedMetrics(*ch);
    return ch;
}
LHMS_API void lhms_unsubscribe_processed(void *ms, void *ch) {
    static_cast<MetricSystem *>(ms)->UnsubscribeFromProcessedMetrics(*static_cast<ProcCh *>(ch));
}
// 1 = received, 0 = timeout, -1 = channel closed by the reaper
LHMS_API int lhms_recv_processed(void *ch, int64_t timeout_ns, lhms_emit_fn emit, void *ctx) {
    auto &c = *static_cast<ProcCh *>(ch);
    std::shared_ptr<ProcessedMetricSet> p;
    if (c->Receive(&p, std::chrono::nanoseconds(timeout_ns))) { emit_processed(*p, emit, ctx); return 1; }
    return c->Closed() ? -1 : 0;
}
LHMS_API void lhms_free_processed_channel(void *ch) { delete static_cast<ProcCh *>(ch); }

LHMS_API void *lhms_subscribe_raw(void *ms, int capacity) {
    auto *ch = new RawCh(std::make_shared<Channel<std::shared_ptr<RawMetricSet>>>((size_t)capacity));
    static_cast<MetricSystem *>(ms)->SubscribeToRawMetrics(*ch);
    return ch;
}
LHMS_API void lhms_unsubscribe_raw(void *ms, void *ch) {
    static_cast<MetricSystem *>(ms)->UnsubscribeFromRawMetrics(*static_cast<RawCh *>(ch));
}
LHMS_API int lhms_recv_raw(void *ch, int64_t timeout_ns, lhms_emit_fn emit, void *ctx) {
    auto &c = *static_cast<RawCh *>(ch);
    std::shared_ptr<RawMetricSet> r;
    if (c->Receive(&r, std::chrono::nanoseconds(timeout_ns))) { emit_raw(*r, emit, ctx); return 1; }
    return c->Closed() ? -1 : 0;
}
LHMS_API void lhms_free_raw_channel(void *ch) { delete static_cast<RawCh *>(ch); }
}  // extern "C"
