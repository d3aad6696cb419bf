// metric_system.h -- C++ mirror of loghisto's MetricSystem for the ingest + reduction path.
//
// Same names, argument meaning and error behaviour as the Go type (reference metrics.go:80-653), written in
// C++ because the Go toolchain is absent from the build image (see INTEGRATION.md for the cgo form).
// The bodies of Histogram / Counter / TimerToken::Stop / collectRawMetrics / processMetrics go through the
// C ABI in include/loghisto_b200.h; nothing here computes a bucket, a count or a percentile on the CPU.
//
// Differences from the Go type, all outside the hot path:
//   * sysStats gauges (sys.Alloc, sys.NumGC, ... metrics.go:172-193) are Go-runtime facts and are not provided;
//     RegisterGaugeFunc / DeregisterGaugeFunc work as in the reference, and RegisterDeviceGauge adds gauges whose
//     values live in device memory.
//   * channels are loghisto::Channel<T>: bounded, non-blocking send, closable (Go's `select { case ch <- x: default: }`).
//   * names map to dense ids on the device, and ids of idle names are recycled (NameTable below): max_histograms /
//     max_counters bound the distinct names used in any three consecutive intervals.  The reference has no limit.
//   * processMetrics() accepts any RawMetricSet, as the reference does.  For a set this system's collectRawMetrics()
//     produced, the per-histogram statistics were reduced on the GPU for exactly that snapshot and travel with it;
//     the histograms of any other set are reduced on the GPU from their maps (lh_reduce_sparse_host).
#pragma once

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "loghisto_b200.h"

namespace loghisto {

template <typename T>
class Channel {   // make(chan T, capacity)
 public:
    explicit Channel(size_t capacity) : cap_(capacity) {}
    // non-blocking send: false when the buffer is full or the channel is closed
    bool TrySend(T v) {
        std::lock_guard<std::mutex> lk(mu_);
        if (closed_ || q_.size() >= (cap_ ? cap_ : 1)) return false;
        q_.push_back(std::move(v));
        cv_.notify_one();
        return true;
    }
    // blocking receive with timeout; false on timeout or when closed and drained
    bool Receive(T *out, std::chrono::nanoseconds timeout) {
        std::unique_lock<std::mutex> lk(mu_);
        if (!cv_.wait_for(lk, timeout, [&] { return !q_.empty() || closed_; })) return false;
        if (q_.empty()) return false;
        *out = std::move(q_.front());
        q_.pop_front();
        return true;
    }
    void Close() { std::lock_guard<std::mutex> lk(mu_); closed_ = true; cv_.notify_all(); }
    bool Closed() { std::lock_guard<std::mutex> lk(mu_); return closed_; }
    size_t Len() { std::lock_guard<std::mutex> lk(mu_); return q_.size(); }

 private:
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<T> q_;
    size_t cap_;
    bool closed_ = false;
};

using TimePoint = std::chrono::system_clock::time_point;

// metrics.go:47-50
struct ProcessedMetricSet {
    TimePoint Time;
    std::map<std::string, double> Metrics;
};

struct ReducedHistogram {   // GPU results of processHistograms for one histogram of one snapshot
    uint64_t count = 0;
    double sum = 0, avg = 0;
    std::vector<int32_t> pkeys;   // INT32_MIN: percentile() error, key omitted
    std::vector<double> pvals;
};

// metrics.go:54-60 (map[int16]*uint64 becomes map<int16_t,uint64_t>: the snapshot owns plain values)
struct RawMetricSet {
    TimePoint Time;
    std::map<std::string, uint64_t> Counters;
    std::map<std::string, uint64_t> Rates;
    std::map<std::string, std::map<int16_t, uint64_t>> Histograms;
    std::map<std::string, double> Gauges;
    // travels with the snapshot: what the device reduced for it, and for which percentile labels
    std::map<std::string, ReducedHistogram> reduced;
    std::vector<std::pair<std::string, double>> percentile_labels;
    const void *origin = nullptr;
};

class MetricSystem;

// metrics.go:63-67
struct TimerToken {
    std::string Name;
    std::chrono::steady_clock::time_point Start;
    MetricSystem *System = nullptr;
    uint32_t id = 0;                   // dense histogram id interned by StartTimer (not in the Go type): Stop() skips the lookup
    uint32_t gen = 0;                  // ... while the id still carries this generation (see MetricSystem::NameTable)
    bool id_valid = false;
    std::chrono::nanoseconds Stop();   // metrics.go:242-246
};

// A record scope bound to names (MetricSystem::BeginRecording): the caller's kernels record with lh::record /
// lh::record_ns / lh::stop / lh::count (include/loghisto_b200_device.cuh) under the ids it hands out, and those ids
// keep their names until the interval the scope records into has been collected.
//
//   loghisto::RecordScope s = ms.BeginRecording(stream, {"rpc_latency", "payload_bytes"}, {"requests"});
//   kernel<<<g, b, 0, stream>>>(s.recorder(), s.histogram_id(0), s.histogram_id(1), s.counter_id(0));
//   s.Histogram(0, d_values, n);   // optional: n float64 in device memory under histogram name 0, on the scope's stream
//   s.End();                       // also on destruction; idempotent
//
// Kernels that use the recorder are enqueued on the scope's stream before End().  A name that found no free id is
// bound to kUnbound: every record under it is dropped on the device and counted in dropped_samples().
// A scope holds back the collection of its interval until it ends (the reaper's one included), so keep scopes short:
// open, launch, end.  The thread that opened a scope must end it before it calls collectRawMetrics itself, and every
// scope must end before the MetricSystem is destroyed.
class RecordScope {
 public:
    static constexpr uint32_t kUnbound = 0xFFFFFFFFu;
    RecordScope() = default;
    RecordScope(RecordScope &&o) noexcept { *this = std::move(o); }
    RecordScope &operator=(RecordScope &&o) noexcept;
    RecordScope(const RecordScope &) = delete;
    RecordScope &operator=(const RecordScope &) = delete;
    ~RecordScope();

    const lh_recorder &recorder() const { return rec_; }
    uint32_t histogram_id(size_t i) const { return hids_.at(i); }
    uint32_t counter_id(size_t i) const { return cids_.at(i); }
    // lh_ingest_f64 of n float64 in device memory under histogram name i, on the scope's stream.  Under an unbound
    // name the samples are dropped and counted.  Throws std::out_of_range for a bad index, std::runtime_error when the
    // library refuses the call (e.g. a misaligned pointer) or the scope has ended.
    void Histogram(size_t i, const double *d_values, size_t n);
    // Many device arrays in one lh_ingest_batch on the scope's stream: n samples at d_values (8-byte aligned device
    // memory) under histogram name `name`, of kind LH_VALUES_F64 (float64) or LH_VALUES_I64NS (int64 ns, recorded as
    // float64(ns)).  Names may repeat.  Items under unbound names are dropped and counted; the others are one call.
    // Throws as Histogram does, before anything is issued for a bad index.
    struct Item {
        size_t name;
        const void *d_values;
        size_t n;
        uint32_t kind;
    };
    void Histograms(const std::vector<Item> &items);
    // Many device arrays of any gauge dtype in one lh_ingest_arrays on the scope's stream: n elements at d_values
    // (device memory, naturally aligned) of dtype LH_GAUGE_* under histogram name `name`, each element x recorded as
    // Histogram(name, float64(x)) without a float64 copy.  Names may repeat.  Unbound names, exceptions and a library
    // without the call as in Histograms.
    struct ArrayItem {
        size_t name;
        const void *d_values;
        size_t n;
        uint32_t dtype;
    };
    void Arrays(const std::vector<ArrayItem> &items);
    // (local id, value) pairs in device memory on the scope's stream, local id i being histogram name i
    // (lh_ingest_keyed_mapped_u16 for id_bytes 2, _u32 for 4): values of `kind` as in Histograms.  An id >= the number
    // of names, or under an unbound name, is dropped and counted in dropped_samples().  Names may repeat.
    // Throws before anything is issued: std::invalid_argument for id_bytes other than 2 or 4, std::runtime_error when
    // the scope has ended, the library lacks the call or refuses it (e.g. a misaligned pointer).
    void Keyed(const void *d_ids, size_t id_bytes, const void *d_values, uint32_t kind, size_t n);
    // (local id, amount) pairs, local id i being counter name i (lh_counter_add_mapped_*): wrapping uint64 adds; throws
    // as Keyed.
    void Counters(const void *d_ids, size_t id_bytes, const uint64_t *d_amounts, size_t n);
    void End();
    bool open() const { return ms_ != nullptr; }

 private:
    friend class MetricSystem;
    MetricSystem *ms_ = nullptr;
    void *stream_ = nullptr;
    std::thread::id owner_;
    std::vector<uint32_t> hids_, cids_;
    lh_recorder rec_{};
};

// StartTimer / Stop with both ends on the GPU (MetricSystem::StartGpuTimer): the start and every Stop are stream-ordered
// marks on the device's %globaltimer, and the duration is recorded on the device under the name; nothing synchronises
// with the host.  Use it around CUDA work, where a host timer would measure only the enqueue.
//
//   loghisto::GpuTimerToken t = ms.StartGpuTimer("decode_step", stream);
//   decode<<<g, b, 0, stream>>>(...);
//   t.Stop();                          // on the start's stream; t.Stop(other, d_ns) elsewhere and/or with the duration
//
// Stop binds the name at stop time (BeginRecording), so the sample lands in the interval that is open when Stop is
// called, under the name, however long the token was held.  Like Go's Stop it may be called repeatedly, one sample each
// from the same start.  A name that finds no free id, and every Stop of a token that got no pool slot (the pool of the
// context is exhausted), drop the sample and count it in dropped_samples().  Move-only; the slot goes back to the pool
// on destruction (it is reused only after the token's kernels have run).
class GpuTimerToken {
 public:
    static void *const kStartStream;   // Stop's default: the stream the token was started on
    GpuTimerToken() = default;
    GpuTimerToken(GpuTimerToken &&o) noexcept { *this = std::move(o); }
    GpuTimerToken &operator=(GpuTimerToken &&o) noexcept;
    GpuTimerToken(const GpuTimerToken &) = delete;
    GpuTimerToken &operator=(const GpuTimerToken &) = delete;
    ~GpuTimerToken();

    // Records the duration on the device.  d_duration_ns (device memory, 8-byte aligned, nullable) also receives it as
    // int64.  Throws std::runtime_error when the library refuses the call (e.g. a misaligned d_duration_ns).  These
    // tokens do not time work captured into CUDA graphs; GraphRecorder::StartTimer / StopTimer do.
    void Stop(void *stream = kStartStream, int64_t *d_duration_ns = nullptr);
    bool has_slot() const { return held_; }

 private:
    friend class MetricSystem;
    MetricSystem *ms_ = nullptr;
    std::string name_;
    void *stream_ = nullptr;
    lh_gpu_timer t_{};
    bool held_ = false;
};

// Recording from kernels captured into CUDA graphs, under names (MetricSystem::NewGraphRecorder).  The recorder owns its
// rows (lh_graph_recorder_create), so a captured kernel may be replayed any number of times, in any interval; every
// collection drains what the replays recorded so far into the interval it collects, labelled with the recorder's names.
//
//   loghisto::GraphRecorder g = ms.NewGraphRecorder({"step_latency", "logit_max"}, {"tokens"});
//   cudaStreamBeginCapture(stream, cudaStreamCaptureModeGlobal);
//   kernel<<<grid, block, 0, stream>>>(g.recorder(), /* histogram "step_latency" = local id */ 0, ...);
//   g.Histograms({{1, d_logits, n, LH_VALUES_F64}}, stream);   // optional: device arrays, captured too
//   cudaStreamEndCapture(stream, &graph);  ...  cudaGraphLaunch(exec, stream);   // any number of times
//   g.Close(stream);   // once no replay is pending; also on destruction
//
// The local id of histogram name i is i, and of counter name i is i.  While the recorder is open its names keep their
// ids (they count as used in every interval).  A name that finds no free id at a collection is unbound there: what the
// replays recorded under it since the previous drain is dropped and counted in dropped_samples() (for a counter, its
// amount).  Close the recorder before the MetricSystem is destroyed.
class GraphRecorder {
 public:
    GraphRecorder() = default;
    GraphRecorder(GraphRecorder &&o) noexcept { *this = std::move(o); }
    GraphRecorder &operator=(GraphRecorder &&o) noexcept;
    GraphRecorder(const GraphRecorder &) = delete;
    GraphRecorder &operator=(const GraphRecorder &) = delete;
    ~GraphRecorder();

    const lh_recorder &recorder() const;
    // lh_graph_recorder_ingest on `stream`: n samples at d_values (8-byte aligned device memory) under histogram name
    // `name` (its index), of kind LH_VALUES_F64 or LH_VALUES_I64NS.  Kernels only, so it may be captured.  Throws
    // std::out_of_range for a bad index before anything is issued, std::runtime_error when the library refuses the call
    // or the recorder is closed.
    struct Item {
        size_t name;
        const void *d_values;
        size_t n;
        uint32_t kind;
    };
    void Histograms(const std::vector<Item> &items, void *stream);
    // lh_graph_recorder_ingest_arrays on `stream`: Histograms for arrays of dtype LH_GAUGE_* (RecordScope::Arrays),
    // throwing as Histograms does, and std::runtime_error when the library lacks the call.
    using ArrayItem = RecordScope::ArrayItem;
    void Arrays(const std::vector<ArrayItem> &items, void *stream);
    // Kernels only, like Histograms, so each may be captured; each throws before anything is issued (std::out_of_range
    // for a bad name index, std::invalid_argument for id_bytes other than 2 or 4, std::runtime_error when the library
    // lacks the call or refuses it, or the recorder is closed).
    // lh_graph_recorder_ingest_keyed_u16 (id_bytes 2) / _u32 (4): values[i] of `kind` under local histogram id ids[i]
    // (the index of its name); ids >= the number of names are dropped and counted.
    void Keyed(const void *d_ids, size_t id_bytes, const void *d_values, uint32_t kind, size_t n, void *stream);
    // lh_graph_recorder_counter_add_u16 / _u32: amounts[i] into local counter ids[i] (wrapping uint64).
    void Counters(const void *d_ids, size_t id_bytes, const uint64_t *d_amounts, size_t n, void *stream);
    // lh_graph_recorder_timer_start / _stop: a GPU-timed span of histogram name `name` (its index).  The caller orders
    // the start before the stop; one open span per name and recorder (see the header).  d_duration_ns (nullable, 8-byte
    // aligned device memory) also receives the duration.
    void StartTimer(size_t name, void *stream);
    void StopTimer(size_t name, void *stream, int64_t *d_duration_ns = nullptr);
    // Drains what the recorder still holds into the current interval, on `stream`, and frees it (stream-ordered).
    // Idempotent.
    void Close(void *stream = nullptr);
    bool open() const { return st_ != nullptr; }

    struct State;

 private:
    friend class MetricSystem;
    std::shared_ptr<State> st_;
};

// SubscribeToProcessedMetrics for consumers on the GPU (MetricSystem::NewDeviceSubscription).  Every collection, after
// its reduction, publishes the subscribed names' processed metrics into a board in device memory (lh_board_create,
// lh_snapshot_publish), where kernels and CUDA-graph replays read the latest collection with lh::read_histogram /
// lh::read_counter (include/loghisto_b200_device.cuh) or an lh_board_read copy, with no host call.
//
//   loghisto::DeviceSubscription sub = ms.NewDeviceSubscription({"step_latency"}, {"requests"});
//   shed_load<<<1, 32, 0, stream>>>(sub.board(), /* histogram row of "step_latency" */ 0);   // reads p99 on the device
//   sub.Close();   // once no read of the board is pending; also on destruction
//
// Histogram row i is name histograms[i], counter row i is counters[i].  At a collection a histogram row holds what
// processMetrics emits for that name when the name is in the collection's Histograms (count = <name>_count as uint64,
// sum, avg and every labelled percentile bit for bit; a percentile whose key is INT32_MIN is a label processMetrics
// omits), and present = 0 otherwise.  A counter row holds the name's Rates entry (rate, present = 1) when the name is
// in Rates, and its Counters value as total in any case (0 for a name never counted).  A subscription reads; it does
// not keep its names' ids alive.  Move-only.
class DeviceSubscription {
 public:
    DeviceSubscription() = default;
    DeviceSubscription(DeviceSubscription &&o) noexcept { *this = std::move(o); }
    DeviceSubscription &operator=(DeviceSubscription &&o) noexcept;
    DeviceSubscription(const DeviceSubscription &) = delete;
    DeviceSubscription &operator=(const DeviceSubscription &) = delete;
    ~DeviceSubscription();

    const lh_board &board() const;
    // lh_board_read: one kernel on `stream` copies a consistent image of the board (board().bytes) to d_out.  It may
    // be captured into a CUDA graph.  Throws std::runtime_error when the library refuses the call or it is closed.
    void Read(void *d_out, void *stream);
    // Frees the board, after every publish issued (idempotent); no read of it may be pending.
    void Close();
    bool open() const { return st_ != nullptr; }

    struct State;

 private:
    friend class MetricSystem;
    std::shared_ptr<State> st_;
};

// SubscribeToRawMetrics for consumers on the GPU (MetricSystem::NewRawDeviceSubscription).  Every collection publishes
// the running bucket counts of the subscribed histograms into a raw board in device memory (lh_raw_board_create,
// lh_snapshot_publish_raw), where kernels and CUDA-graph replays answer exact percentile, rank and bucket queries over
// the latest collection with lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count
// (include/loghisto_b200_device.cuh), or Percentiles / Ranks below, with no host call.
//
//   loghisto::RawDeviceSubscription raw = ms.NewRawDeviceSubscription({"step_latency"});
//   admit<<<1, 32, 0, stream>>>(raw.board(), /* row of "step_latency" */ 0, d_budget);   // share under budget, on the GPU
//   raw.Close();   // once no query of the board is pending; also on destruction
//
// Row i is name histograms[i].  At a collection it holds that name's buckets of the collection's RawMetricSet when
// the name is in Histograms, and is empty otherwise (percentiles INT32_MIN / NaN, ranks and totals 0).  A percentile
// query with p equals what processMetrics reports for a label with that p, bit for bit.  A raw subscription reads; it
// does not keep its names' ids alive.  Move-only.
//
// With a window w > 1 (lh_raw_board_create_window), row i answers for the sum of those per-collection histograms over
// the last w collections (fewer before w have run): every collection publishes each open subscription once, a
// collection in which the name is absent, recycled away or unbound enters as an empty interval, and rows follow names,
// not ids.  After JoinRanks each entering interval is the job-wide one, so the window is job-wide too.
class RawDeviceSubscription {
 public:
    RawDeviceSubscription() = default;
    RawDeviceSubscription(RawDeviceSubscription &&o) noexcept { *this = std::move(o); }
    RawDeviceSubscription &operator=(RawDeviceSubscription &&o) noexcept;
    RawDeviceSubscription(const RawDeviceSubscription &) = delete;
    RawDeviceSubscription &operator=(const RawDeviceSubscription &) = delete;
    ~RawDeviceSubscription();

    const lh_raw_board &board() const;
    // publishes summed per row (NewRawDeviceSubscription's window; 1 for a closed subscription)
    uint32_t window() const;
    // lh_raw_percentiles_grid / lh_raw_ranks_grid: one kernel on `stream` answers every row for each of the m device
    // inputs (answers at [row * m + j]; Ranks' d_totals[row] is the total of query (row, 0)).  They may be captured
    // into a CUDA graph.  Throws std::runtime_error when the library refuses the call or the subscription is closed.
    void Percentiles(const double *d_ps, uint32_t m, int32_t *d_keys, double *d_vals, uint64_t *d_publish, void *stream);
    void Ranks(const double *d_values, uint32_t m, uint64_t *d_ranks, uint64_t *d_totals, uint64_t *d_publish,
               void *stream);
    // Frees the board, after every publish issued (idempotent); no query of it may be pending.
    void Close();
    bool open() const { return st_ != nullptr; }

    struct State;

 private:
    friend class MetricSystem;
    std::shared_ptr<State> st_;
};

struct Options {
    int device = 0;
    uint32_t max_histograms = 1024;
    uint32_t max_counters = 1024;
    uint32_t shards = 0;             // staging shards (0 = one per hardware thread, at most 256)
    uint64_t staging_bytes = 4u << 20;
    uint32_t precision = 0;          // compress/decompress precision (0 = the reference's 100, metrics.go:40-43)
};

class MetricSystem {
 public:
    // NewMetricSystem(interval, sysStats), metrics.go:143.  Throws std::runtime_error if no H100 is usable.
    MetricSystem(std::chrono::nanoseconds interval, bool sysStats, const Options &opt = Options());
    ~MetricSystem();
    MetricSystem(const MetricSystem &) = delete;
    MetricSystem &operator=(const MetricSystem &) = delete;

    void SpecifyPercentiles(const std::map<std::string, double> &percentiles);              // :199
    void SubscribeToRawMetrics(std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>> ch);  // :205
    void UnsubscribeFromRawMetrics(std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>> ch);
    void SubscribeToProcessedMetrics(std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>> ch);   // :218
    void UnsubscribeFromProcessedMetrics(std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>> ch);
    TimerToken StartTimer(const std::string &name);                       // :232
    // StartTimer timed on the GPU: enqueues the start mark on `stream` (NULL = the context's ingest stream).  Never
    // fails for want of a pool slot (see GpuTimerToken); throws std::runtime_error when the library refuses the call
    // (e.g. a stream in CUDA-graph capture).
    GpuTimerToken StartGpuTimer(const std::string &name, void *stream);
    // Ingest never throws and never fails the caller (problems are logged, samples dropped and counted).
    void Counter(const std::string &name, uint64_t amount) noexcept;      // :251
    void Histogram(const std::string &name, double value) noexcept;       // :273
    void Histogram(const char *name, size_t len, double value) noexcept;  // same, without building a std::string
    void *assign_shard(size_t thread_slot, bool *exclusive);             // internal: a thread's staging shard (exclusive while any is free)
    void release_shard(void *shard);                                      // internal: a finished thread hands its exclusive shard back
    void histogram_id(const std::string &name, uint32_t id, uint32_t gen, double value) noexcept;   // body of Histogram once the name is interned
    // Opens a record scope on `stream` (NULL = the context's ingest stream) with histogram names and counter names bound
    // to ids for its lifetime (RecordScope).  Throws std::runtime_error only when the library refuses lh_record_begin;
    // a full name table never makes it fail.
    RecordScope BeginRecording(void *stream, const std::vector<std::string> &histograms,
                               const std::vector<std::string> &counters);
    // A recorder for kernels captured into CUDA graphs, with these names (GraphRecorder).  Call it outside any stream
    // capture.  Throws std::runtime_error when the library refuses lh_graph_recorder_create (e.g. more names than
    // max_histograms / max_counters); a full name table never makes it fail.
    GraphRecorder NewGraphRecorder(const std::vector<std::string> &histograms, const std::vector<std::string> &counters);
    // A device subscription to these names (DeviceSubscription): every collection from now on, the reaper's included,
    // publishes into it.  Call it outside any stream capture.  Throws std::runtime_error when the library refuses
    // lh_board_create (e.g. more names than max_histograms / max_counters, or none).
    DeviceSubscription NewDeviceSubscription(const std::vector<std::string> &histograms,
                                             const std::vector<std::string> &counters);
    // A raw device subscription to these histogram names (RawDeviceSubscription): every collection from now on, the
    // reaper's included, publishes their bucket counts into it, each row summed over the last `window` collections.
    // Call it outside any stream capture.  Throws std::runtime_error when the library refuses lh_raw_board_create /
    // lh_raw_board_create_window (more names than max_histograms, or none; window 0 or above LH_RAW_MAX_WINDOW) or has
    // no raw device subscriptions (for window != 1: no window boards).
    RawDeviceSubscription NewRawDeviceSubscription(const std::vector<std::string> &histograms, uint32_t window = 1);
    void RegisterGaugeFunc(const std::string &name, std::function<double()> f);   // :299
    // A gauge whose value lives in device memory: a scalar of type `dtype` (LH_GAUGE_*) at d_value, device or managed
    // memory of this system's device, which must stay allocated while registered.  Every collection reads all device
    // gauges in one lh_gauges_read, which waits for no caller stream, and puts float64(value) in Gauges under `name`,
    // as a RegisterGaugeFunc value.  Gauge functions and device gauges share one name space: registering either kind
    // replaces the other under that name.  Throws std::invalid_argument when lh_gauges_read refuses the address or dtype
    // (checked with one read now, so a bad pointer never reaches a collection), std::runtime_error when this
    // libloghisto_b200 has no device gauges or the read fails otherwise.
    void RegisterDeviceGauge(const std::string &name, const void *d_value, uint32_t dtype);
    void DeregisterGaugeFunc(const std::string &name);                    // :306, device gauges too
    // A distribution gauge: n values of type `dtype` (LH_GAUGE_*) at d_values, device or managed memory of this system's
    // device, which must stay allocated while registered.  At every collection each element x is recorded as
    // Histogram(name, float64(x)) into the interval that collection collects, read on the snapshot stream without
    // waiting for any caller stream (lh_snapshot_ingest_arrays), so Histograms and the processed metrics carry the
    // distribution of the array's current values.  A registered name keeps its id while registered; when no id is free
    // at a collection, its n samples are dropped and counted.  Registering a name again replaces its array.  Throws
    // std::invalid_argument when the dtype, or lh_gauges_read of the first element, is refused (the range is checked at
    // each collection; a refused collection logs and delivers its set without the distributions), std::runtime_error
    // when this libloghisto_b200 has no distribution gauges.
    // Both calls wait for a collection in progress to finish reading the arrays, so an array is never read after
    // DeregisterDeviceDistribution returns and may be freed then.  That collection may itself be waiting for the record
    // scopes of the interval to end, so from a thread that holds an open record scope of this system both throw
    // std::runtime_error instead of waiting, as collectRawMetrics does.
    void RegisterDeviceDistribution(const std::string &name, const void *d_values, uint64_t n, uint32_t dtype);
    void DeregisterDeviceDistribution(const std::string &name);
    void Start();                                                         // :644
    void Stop();                                                          // :651

    // unexported in Go, called directly by metrics_test.go; public here for the same purpose
    std::shared_ptr<RawMetricSet> collectRawMetrics();                                  // :420
    std::shared_ptr<ProcessedMetricSet> processMetrics(const RawMetricSet &raw);        // :483
    void add_aggregates(const RawMetricSet &raw, ProcessedMetricSet &out);              // the reaper's step after it, :590-608

    lh_ctx *context() const { return ctx_; }
    // Samples and counter ops that were not recorded: those of a new name that found no free id (the distinct names
    // used in any three consecutive intervals exceed max_histograms / max_counters, see NameTable), and those lost
    // to a failed staging call.  Never silent.
    uint64_t dropped_samples();

    // Joins the systems of a multi-GPU job (one system per GPU, e.g. one per torchrun rank) so that each collection
    // describes the whole job.  Collective: every rank calls it once, with its rank, the world size (2 ..
    // LH_MAX_RANKS) and an all-gather, before its first collection.  allgather(mine) returns every rank's bytes in rank
    // order and throws on failure; it is the only way the systems talk to each other, so any transport works
    // (torch.distributed, MPI, a barrier between threads).  It runs on the collecting thread (the reaper's, once
    // Start()ed).  Throws std::invalid_argument, on every rank alike and before anything is mapped, when the ranks'
    // max_histograms, max_counters or precision differ, and std::runtime_error when the system has collected already,
    // has joined already, or the library lacks lh_snapshot_rows / lh_snapshot_allreduce_rows.
    //
    // At each collection of a joined system the ranks exchange the names of the histograms and counters their
    // interval touched, agree on the byte-sorted union of each (the first max_histograms / max_counters names of it;
    // samples and counter amounts under the rest are counted in dropped_samples() on the ranks that recorded them),
    // and one peer-memory all-reduce sums every name's rows wherever each rank keeps them.  Then Histograms, Rates,
    // Counters, the aggregates of processMetrics, and processed and raw device subscriptions are job-wide and the same
    // on every rank.  Gauges (functions and device gauges) stay rank-local.  Name ids stay per rank: each rank
    // recycles them from its own interval, exactly as unjoined.  When the exchange fails on a rank, that rank's
    // collection is its own interval alone (RanksInfo().status 3, logged once); ranks whose exchange succeeded give up
    // on it after the all-reduce's 10 s timeout and keep their own counts (status 1).
    using AllGather = std::function<std::vector<std::string>(const std::string &mine)>;
    void JoinRanks(uint32_t rank, uint32_t world, AllGather allgather);

    // JoinRanks over a transport the caller owns, for ranks that cannot map each other's memory (ranks on different
    // hosts: CUDA IPC works only within one).  The collections agree on the same job-wide rows, and the rows are summed
    // by allreduce instead of the peer-memory all-reduce; no peer handle is exported or imported.  At each collection
    // every rank packs its rows into a payload laid out alike on every rank (lh_snapshot_pack_rows) and calls
    // allreduce(d_send, d_recv, n_words, stream) on the collecting thread, with the same n_words on every rank (none
    // when nothing was touched anywhere).  It must leave in d_recv the wrapping uint64 element-wise sum over ranks of
    // d_send, either enqueued on `stream` (the snapshot stream, behind the pack) or completed when it returns, and
    // throw on failure.  A throw gives that rank its own counts under the job-wide rows (RanksInfo().status 4, logged
    // once); the next collection sums again.  The join refuses, on every rank alike (std::invalid_argument), ranks
    // that differ in transport (some with allreduce, some without) as well as in the configuration; std::runtime_error
    // when the library lacks lh_snapshot_pack_rows.  This transport has no timeout of its own: a rank whose exchange
    // failed while others' succeeded leaves those inside the caller's collective until its own timeout.
    using AllReduce = std::function<void(const uint64_t *d_send, uint64_t *d_recv, size_t n_words, void *stream)>;
    void JoinRanks(uint32_t rank, uint32_t world, AllGather allgather, AllReduce allreduce);
    struct RanksState {
        uint32_t rank = 0, world = 0;   // world 0: not joined
        uint32_t status = 0;            // last collection: 0 summed, 1 / 2 as lh_comm_stats, 3 exchange failed,
                                        // 4 the caller's allreduce threw
        uint64_t summed = 0;            // collections summed across the ranks
        uint64_t bytes_from_peers = 0;  // of the last collection's all-reduce (8 x n_words through allreduce)
        uint64_t names_dropped = 0;     // names left out of the job-wide union by the bounds, over all collections
    };
    RanksState RanksInfo();

 public:
    struct Shard;

 private:
    // Name -> dense id, per table (histograms, counters).  Ids are recycled, so the limit bounds the names in use,
    // not every name ever seen.  Each id is free, live or retiring.  A name is live in an interval if a sample or
    // counter op of it landed in that interval (a histogram export segment, a counter delta or touched mark), or if
    // a lookup created or revived it then.  collectRawMetrics, holding `mu`, labels the snapshot with `names`, then:
    //   retiring and not live this interval -> free (name removed from `ids`, id pushed on `free_ids`);
    //   live and not live this interval     -> retiring, gen[id] += 1;
    //   retiring and touched this interval  -> live (a lookup revives a retiring id at once, under the same name).
    // So a name last used in interval k holds its id through k+1 and k+2, and the id is free for k+3.
    //
    // Why this is enough: the name -> (id, gen) lookup runs outside the shard's critical section (thread caches,
    // TimerToken), so a collection may run between the lookup and the append.  The append therefore re-reads
    // gen[id] INSIDE the critical section and, on a mismatch, leaves it, looks the name up again and retries.
    // An append that passed that check before the bump of collection k sits in its shard until collection k+1
    // flushes the shard at the latest (the flush waits for the critical section), so it lands in interval k or
    // k+1 and touches its id there, which keeps the id under the appender's name.  An id is freed only after an
    // interval with neither a touch nor a revival following its bump, so no append validated against an older
    // generation can land on an id that was handed to another name.
    enum : uint8_t { kFree = 0, kLive = 1, kRetiring = 2 };
    struct NameTable {
        std::shared_mutex mu;
        std::unordered_map<std::string, uint32_t> ids;   // live and retiring names
        std::vector<std::string> names;                  // id -> name; ids below names.size() were handed out before
        std::vector<uint8_t> state;                      // per id in names
        std::vector<uint8_t> used;                       // created or revived by a lookup this interval
        std::vector<uint32_t> free_ids;                  // recycled ids, taken before names grows
        std::unique_ptr<std::atomic<uint32_t>[]> gen;    // [capacity], read inside shard critical sections without mu
        uint32_t capacity = 0;
    };
    bool intern(NameTable &t, const char *p, size_t n, uint32_t *id, uint32_t *gen);
    void recycle(NameTable &t, const std::vector<uint8_t> &touched);
    bool lookup_histogram(const char *p, size_t n, uint32_t *id, uint32_t *gen);
    bool lookup_counter(const char *p, size_t n, uint32_t *id, uint32_t *gen);
    void append_histogram(Shard &s, uint32_t id, uint32_t gen, double value, const char *name, size_t len) noexcept;
    void append_counter(Shard &s, uint32_t id, uint32_t gen, uint64_t amount, const char *name, size_t len) noexcept;
    __attribute__((noinline, cold)) void retry_histogram(Shard &s, double value, const char *name, size_t len) noexcept;
    __attribute__((noinline, cold)) void retry_counter(Shard &s, uint64_t amount, const char *name, size_t len) noexcept;
    void commit_histograms(Shard &s) noexcept;
    void commit_counters(Shard &s) noexcept;
    void flush_shard(Shard &s, std::vector<uint8_t> *touched);
    void reaper();
    // record scopes (BeginRecording)
    friend class RecordScope;
    friend class GpuTimerToken;
    void bind_names(NameTable &t, const std::vector<std::string> &names, std::vector<uint32_t> &ids, std::vector<uint32_t> &gens);
    bool pin_names(NameTable &t, const std::vector<uint32_t> &ids, const std::vector<uint32_t> &gens);
    void end_scope(RecordScope &s);
    void refuse_in_scope(const char *what);   // std::runtime_error when the calling thread holds an open record scope
    std::mutex scope_mu_;
    std::unordered_map<std::thread::id, uint32_t> scope_threads_;   // open scopes per opening thread
    std::vector<uint8_t> carried_touched_;   // touched-counter marks of a collection that lh_snapshot_begin refused
    // graph recorders (NewGraphRecorder)
    friend class GraphRecorder;
    uint32_t intern_locked(NameTable &t, const std::string &name);
    void bind_graph(GraphRecorder::State &g);
    std::mutex graph_mu_;
    std::vector<std::shared_ptr<GraphRecorder::State>> graphs_;   // open recorders
    // device subscriptions (NewDeviceSubscription)
    friend class DeviceSubscription;
    std::mutex sub_mu_;
    std::vector<std::shared_ptr<DeviceSubscription::State>> subs_;   // open subscriptions
    lh_status publish_subscriptions(const RawMetricSet &raw, const std::unordered_map<std::string, uint32_t> &hid_of,
                                    const std::unordered_map<std::string, uint32_t> &cid_of);
    // raw device subscriptions (NewRawDeviceSubscription), under sub_mu_ too
    friend class RawDeviceSubscription;
    std::vector<std::shared_ptr<RawDeviceSubscription::State>> raw_subs_;   // open raw subscriptions
    lh_status publish_raw_subscriptions(const std::unordered_map<std::string, uint32_t> &hid_of);

    lh_ctx *ctx_ = nullptr;
    std::chrono::nanoseconds interval_;
    Options opt_;

    std::mutex percentiles_mu_;
    std::vector<std::pair<std::string, double>> percentiles_;   // label (with %s) -> p

    NameTable histos_, counters_;

    std::vector<std::unique_ptr<Shard>> shards_;
    std::mutex assign_mu_;
    std::vector<Shard *> free_exclusive_, shared_;
    bool asym_ = false;             // exclusive shards use the membarrier handshake instead of a lock

    std::mutex counter_store_mu_;
    std::map<std::string, uint64_t> counter_store_;            // metrics.go:111-113
    std::mutex histogram_count_mu_;
    std::map<std::string, uint64_t> histogram_count_store_;    // metrics.go:122-126

    // held across a collection's device read, so a gauge deregistered (and then freed) is never read
    std::mutex gauge_mu_;
    std::map<std::string, std::function<double()>> gauge_funcs_;
    std::map<std::string, lh_gauge_src> device_gauges_;   // no name is in both maps
    // distribution gauges: name -> array (histogram_id unused), held from a collection's binding until its reduction
    // has run, so an array deregistered (and then freed) is never read.  Only threads without an open record scope take
    // it (refuse_in_scope): the collection holding it may wait for the scopes of its interval in lh_snapshot_begin.
    std::mutex dist_mu_;
    std::map<std::string, lh_array_src> device_dists_;

    std::mutex subscribers_mu_;
    std::vector<std::shared_ptr<Channel<std::shared_ptr<RawMetricSet>>>> raw_subscribers_;
    std::vector<std::shared_ptr<Channel<std::shared_ptr<ProcessedMetricSet>>>> processed_subscribers_;
    std::map<void *, int> raw_bad_, processed_bad_;

    std::mutex snapshot_mu_;   // one collectRawMetrics at a time
    std::thread reaper_thread_;
    std::mutex run_mu_;
    std::condition_variable run_cv_;
    bool reaping_ = false, shutdown_ = false;
    std::atomic<uint64_t> dropped_over_limit_{0};
    uint64_t system_id_ = 0;
    // JoinRanks: the exchange and the job-wide rows of a collection (under snapshot_mu_)
    struct JobRows;
    bool join_collection(JobRows &j, const std::vector<uint8_t> &counter_touched);
    void join(uint32_t rank, uint32_t world, AllGather allgather, AllReduce allreduce);
    void sum_rows(const std::vector<uint32_t> &hmap, const std::vector<uint8_t> &levels, const std::vector<uint32_t> &cmap);
    AllGather allgather_;
    AllReduce allreduce_;
    bool allreduce_logged_ = false;
    bool collected_ = false;
    bool exchange_logged_ = false;
    std::mutex ranks_mu_;
    RanksState ranks_;
};

// print_benchmark.go:49: run `op` from `concurrency` threads between StartTimer/Stop and print every interval's
// metrics; returns the last interval's <name>_count after `seconds` (the reference runs forever).
double PrintBenchmark(const std::string &name, unsigned concurrency, std::function<void()> op, double seconds,
                      std::chrono::nanoseconds interval = std::chrono::seconds(1), const Options &opt = Options(),
                      bool print = true);

}  // namespace loghisto
