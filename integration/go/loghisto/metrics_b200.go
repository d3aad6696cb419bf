// Go side of the drop-in: the bodies of MetricSystem.Counter, MetricSystem.Histogram, collectRawMetrics,
// processMetrics and processHistograms (reference metrics.go:251-295, 336-387, 420-506) over the C ABI in
// include/loghisto_b200.h.  Everything else in the package -- the exported API, RawMetricSet / ProcessedMetricSet /
// TimerToken, StartTimer / Stop, the reaper and its subscription bookkeeping, gauges, Submitter, the Graphite and
// OpenTSDB serializers, PrintBenchmark, compress / decompress -- stays the reference's own source, untouched.
//
// STATUS: complete, self-consistent source, but NEVER COMPILED: the build image has no Go toolchain (INTEGRATION.md).
// Every lh_* call below is exercised by the C++ mirror (loghisto_b200/host/) and the ctypes / C clients in tests/.
//
// How it is wired in (INTEGRATION.md has the commands):
//   1. integration/go/split_reference.py moves the five replaced method bodies of metrics.go into metrics_cpu.go
//      under `//go:build !b200` (nothing else changes, a plain `go build` still gives the pure-Go package);
//   2. this file is copied next to it; it is compiled only with `-tags b200`;
//   3. include/loghisto_b200.h and libloghisto_b200.so are made visible through CGO_CFLAGS / CGO_LDFLAGS.

//go:build b200

package loghisto

/*
#include <stdlib.h>
#include <string.h>
#include "loghisto_b200.h"
*/
import "C"

import (
	"fmt"
	"math"
	"runtime"
	"sync"
	"sync/atomic"
	"time"
	"unsafe"

	"github.com/golang/glog"
)

// Limits of one engine.  Ids of idle names are recycled (nameTable), so a limit bounds the distinct names used in
// any three consecutive intervals; a new name that finds no free id is dropped and counted (B200Dropped), never
// silently.
const (
	b200MaxHistograms = 4096
	b200MaxCounters   = 4096
	b200StagingBytes  = 4 << 20 // per pinned staging slot: 419 424 (id, value) pairs
)

// stagingBuf is one C-owned pinned slot being filled: n 8-byte items at offset 0, n uint16 ids at idsOff.
// cgo forbids C code from keeping Go pointers after a call returns, so Go writes into C memory instead.
type stagingBuf struct {
	slot   C.lh_staging
	open   bool
	n, cap int
	items  []uint64 // float64 bits or counter amounts, view of slot.host
	ids    []uint16
	idsOff uint64
}

// b200Shard is what one goroutine at a time appends to.  Goroutines spread over 4*GOMAXPROCS shards by a hash of
// their stack address, so the mutex is almost always uncontended and the slot's cache lines stay on one core.
type b200Shard struct {
	mu      sync.Mutex
	hist    stagingBuf
	counter stagingBuf
	touched []bool // counter ids Counter() was called for this interval, even with amount 0 (metrics.go:430-433)
	anyC    bool
	_       [64]byte
}

// reducedHistogram is what the device computed for one histogram of one snapshot (metrics.go:336-387).
type reducedHistogram struct {
	count    uint64
	sum, avg float64
	pkeys    []int32
	pvals    []float64
}

// reducedSet travels beside a RawMetricSet from collectRawMetrics to processMetrics.
type reducedSet struct {
	labels []string  // percentile labels ("%s_99.9", ...) in the order the device reduced them
	ps     []float64 // the matching percentiles
	byName map[string]*reducedHistogram
}

// Per-table id lifecycle (the same as the C++ mirror's NameTable, loghisto_b200/host/metric_system.h).  Each id is
// free, live or retiring.  A name is live in an interval if a sample or counter op of it landed in that interval (a
// histogram export segment, a counter delta or touched mark), or if intern created or revived it then.
// collectRawMetrics, holding mu, labels the snapshot with names, then:
//   - retiring and not live this interval -> free (name removed from ids, id pushed on freeIDs);
//   - live and not live this interval     -> retiring, gen[id] += 1;
//   - retiring and touched this interval  -> live (intern revives a retiring id at once, under the same name).
// So a name last used in interval k holds its id through k+1 and k+2, and the id is free for k+3.
//
// Why this is enough: intern runs before the shard's mutex is taken, so a collection may run between the two.
// Histogram and Counter therefore re-read gen[id] under s.mu and, on a mismatch, unlock, intern again and retry.
// An append that passed that check before the bump of collection k sits in its shard until collection k+1 flushes
// the shard at the latest (the flush takes s.mu), so it lands in interval k or k+1 and touches its id there, which
// keeps the id under the appender's name.  An id is freed only after an interval with neither a touch nor a revival
// following its bump, so no append validated against an older generation can land on an id handed to another name.
const (
	idFree uint8 = iota
	idLive
	idRetiring
)

type nameTable struct {
	mu      sync.RWMutex // RLock fast path, Lock-and-recheck slow path: the idiom of metrics.go:275-294
	ids     map[string]uint16
	names   []string // id -> name; ids below len(names) were handed out before
	state   []uint8
	used    []bool   // created or revived by intern this interval
	freeIDs []uint16 // recycled ids, taken before names grows
	gen     []uint32 // [limit], read under a shard's mutex with atomic loads
	limit   int
}

func newNameTable(limit int) *nameTable {
	if limit > 65536 {
		limit = 65536 // uint16 ids
	}
	return &nameTable{ids: map[string]uint16{}, gen: make([]uint32, limit), limit: limit}
}

// intern returns the id of name and its generation; ok is false when no id is free.
func (t *nameTable) intern(name string) (id uint16, gen uint32, ok bool) {
	t.mu.RLock()
	id, ok = t.ids[name]
	if ok && t.state[id] == idLive {
		gen = atomic.LoadUint32(&t.gen[id])
		t.mu.RUnlock()
		return id, gen, true
	}
	t.mu.RUnlock()
	t.mu.Lock()
	defer t.mu.Unlock()
	if id, ok = t.ids[name]; ok {
		if t.state[id] == idRetiring {
			t.state[id], t.used[id] = idLive, true
		}
		return id, atomic.LoadUint32(&t.gen[id]), true
	}
	switch {
	case len(t.freeIDs) > 0:
		id = t.freeIDs[len(t.freeIDs)-1]
		t.freeIDs = t.freeIDs[:len(t.freeIDs)-1]
		t.names[id] = name
	case len(t.names) < t.limit:
		id = uint16(len(t.names))
		t.names = append(t.names, name)
		t.state = append(t.state, idFree)
		t.used = append(t.used, false)
	default:
		return 0, 0, false
	}
	t.ids[name] = id
	t.state[id], t.used[id] = idLive, true
	return id, atomic.LoadUint32(&t.gen[id]), true
}

// current reports whether gen is still the generation of id.  Called under the shard's mutex.
func (t *nameTable) current(id uint16, gen uint32) bool {
	return atomic.LoadUint32(&t.gen[id]) == gen
}

// collect returns the id -> name table the snapshot is labelled with (retiring ids included), then steps every id's
// lifecycle; landed(id) reports whether a sample or counter op of id is in the snapshot.
func (t *nameTable) collect(landed func(id int) bool) []string {
	t.mu.Lock()
	defer t.mu.Unlock()
	labels := append([]string(nil), t.names...)
	for id := range t.names {
		liveNow := t.used[id] || landed(id)
		t.used[id] = false
		switch {
		case t.state[id] == idRetiring && !liveNow:
			delete(t.ids, t.names[id])
			t.names[id] = ""
			t.state[id] = idFree
			t.freeIDs = append(t.freeIDs, uint16(id))
		case t.state[id] == idLive && !liveNow:
			t.state[id] = idRetiring
			atomic.StoreUint32(&t.gen[id], t.gen[id]+1)
		case t.state[id] == idRetiring:
			t.state[id] = idLive
		}
	}
	return labels
}

// snapshotNames is the id -> name table without a lifecycle step (a snapshot that failed on the device).
func (t *nameTable) snapshotNames() []string {
	t.mu.RLock()
	defer t.mu.RUnlock()
	return append([]string(nil), t.names...)
}

type b200Engine struct {
	ctx *C.lh_ctx

	histos   *nameTable
	counters *nameTable

	shards  []*b200Shard
	dropped uint64

	snapshotMu sync.Mutex // one collectRawMetrics at a time

	// device reductions waiting for processMetrics: the reaper hands every set to a worker right away
	// (metrics.go:583-587), so a short ring suffices; sets that are never processed (raw-only subscribers) age out
	reducedMu   sync.Mutex
	reducedRing [16]struct {
		raw *RawMetricSet
		red *reducedSet
	}
	reducedNext int
}

func (e *b200Engine) putReduced(raw *RawMetricSet, red *reducedSet) {
	e.reducedMu.Lock()
	e.reducedRing[e.reducedNext].raw, e.reducedRing[e.reducedNext].red = raw, red
	e.reducedNext = (e.reducedNext + 1) % len(e.reducedRing)
	e.reducedMu.Unlock()
}

func (e *b200Engine) takeReduced(raw *RawMetricSet) *reducedSet {
	e.reducedMu.Lock()
	defer e.reducedMu.Unlock()
	for i := range e.reducedRing {
		if e.reducedRing[i].raw == raw {
			red := e.reducedRing[i].red
			e.reducedRing[i].raw, e.reducedRing[i].red = nil, nil
			return red
		}
	}
	return nil
}

var (
	b200Engines   sync.Map // *MetricSystem -> *b200Engine
	b200EnginesMu sync.Mutex
	// B200Device is the CUDA ordinal new engines are created on.
	B200Device = 0
)

func b200Status(st C.lh_status, ctx *C.lh_ctx, what string) error {
	if st == C.LH_OK {
		return nil
	}
	detail := ""
	if ctx != nil {
		detail = C.GoString(C.lh_last_error(ctx))
	}
	return fmt.Errorf("%s: %s (%s)", what, C.GoString(C.lh_strerror(st)), detail)
}

// engineFor returns the engine of a MetricSystem, creating it on first use.  There is no CPU fallback under the
// b200 tag: without a usable H100 the process stops here (build without the tag for the pure-Go package).
func engineFor(ms *MetricSystem) *b200Engine {
	if e, ok := b200Engines.Load(ms); ok {
		return e.(*b200Engine)
	}
	b200EnginesMu.Lock()
	defer b200EnginesMu.Unlock()
	if e, ok := b200Engines.Load(ms); ok {
		return e.(*b200Engine)
	}
	nshards := 4 * runtime.GOMAXPROCS(0)
	var cfg C.lh_config
	cfg.struct_size = C.uint32_t(C.sizeof_lh_config)
	cfg.device = C.int32_t(B200Device)
	cfg.max_histograms = b200MaxHistograms
	cfg.max_counters = b200MaxCounters
	cfg.staging_bytes = b200StagingBytes
	cfg.staging_slots = C.uint32_t(2*nshards + 2) // memory of a slot is allocated on first use
	cfg.precision = C.uint32_t(precision)          // the package constant of metrics.go:40-43
	e := &b200Engine{histos: newNameTable(b200MaxHistograms), counters: newNameTable(b200MaxCounters)}
	if err := b200Status(C.lh_create(&cfg, &e.ctx), nil, "lh_create"); err != nil {
		glog.Fatalf("loghisto (b200 build): %v", err)
	}
	e.shards = make([]*b200Shard, nshards)
	for i := range e.shards {
		e.shards[i] = &b200Shard{touched: make([]bool, b200MaxCounters)}
	}
	runtime.SetFinalizer(e, func(e *b200Engine) { C.lh_destroy(e.ctx) })
	b200Engines.Store(ms, e)
	return e
}

// B200Dropped is the number of samples / counter ops that could not be recorded (name table full, or a staging
// call failed); the reference's philosophy is "log and drop, never block or fail the caller" (metrics.go:570-573).
func (ms *MetricSystem) B200Dropped() uint64 {
	e := engineFor(ms)
	var st C.lh_stats
	C.lh_get_stats(e.ctx, &st)
	return atomic.LoadUint64(&e.dropped) + uint64(st.dropped)
}

func (e *b200Engine) shard() *b200Shard {
	var marker byte
	h := uintptr(unsafe.Pointer(&marker)) // goroutine stacks are disjoint: a cheap, stable per-goroutine hash
	h ^= h >> 17
	return e.shards[(h>>10)%uintptr(len(e.shards))]
}

// openBuf acquires a pinned staging slot for b.  Called with the shard locked.
func (e *b200Engine) openBuf(b *stagingBuf) bool {
	if err := b200Status(C.lh_staging_acquire(e.ctx, &b.slot), e.ctx, "lh_staging_acquire"); err != nil {
		glog.Errorf("loghisto (b200): %v; dropping", err)
		return false
	}
	b.cap = int(uint64(b.slot.bytes)/10) &^ 15
	b.idsOff = uint64(b.cap) * 8
	base := unsafe.Pointer(b.slot.host)
	b.items = unsafe.Slice((*uint64)(base), b.cap)
	b.ids = unsafe.Slice((*uint16)(unsafe.Add(base, uintptr(b.idsOff))), b.cap)
	b.n = 0
	b.open = true
	return true
}

// commitHist / commitCounter hand the slot to the device (async H2D + kernel) and forget it.
func (e *b200Engine) commitHist(b *stagingBuf) {
	if !b.open {
		return
	}
	st := C.lh_staging_commit_keyed_f64_u16(e.ctx, &b.slot, C.size_t(b.n), C.uint64_t(b.idsOff))
	if err := b200Status(st, e.ctx, "lh_staging_commit_keyed_f64_u16"); err != nil {
		glog.Errorf("loghisto (b200): %v; dropping %d samples", err, b.n)
		atomic.AddUint64(&e.dropped, uint64(b.n))
		C.lh_staging_abandon(e.ctx, &b.slot)
	}
	b.open, b.n, b.items, b.ids = false, 0, nil, nil
}

func (e *b200Engine) commitCounter(b *stagingBuf) {
	if !b.open {
		return
	}
	st := C.lh_staging_commit_counter_u16(e.ctx, &b.slot, C.size_t(b.n), C.uint64_t(b.idsOff))
	if err := b200Status(st, e.ctx, "lh_staging_commit_counter_u16"); err != nil {
		glog.Errorf("loghisto (b200): %v; dropping %d counter ops", err, b.n)
		atomic.AddUint64(&e.dropped, uint64(b.n))
		C.lh_staging_abandon(e.ctx, &b.slot)
	}
	b.open, b.n, b.items, b.ids = false, 0, nil, nil
}

// Counter is used for recording a running count of the total occurrences of
// a particular event.  A rate is also exported for the amount that a counter
// has increased during an interval of this MetricSystem.  (metrics.go:251-269)
func (ms *MetricSystem) Counter(name string, amount uint64) {
	e := engineFor(ms)
	for {
		id, gen, ok := e.counters.intern(name)
		if !ok {
			atomic.AddUint64(&e.dropped, 1)
			return
		}
		if e.appendCounter(e.shard(), id, gen, amount) {
			return
		}
		// the id was retired between intern and s.mu: look the name up again
	}
}

// appendCounter reports false, appending nothing, when gen is no longer the generation of id (nameTable).
func (e *b200Engine) appendCounter(s *b200Shard, id uint16, gen uint32, amount uint64) bool {
	s.mu.Lock()
	defer s.mu.Unlock()
	if !e.counters.current(id, gen) {
		return false
	}
	s.touched[id] = true // the name shows up in Rates even when amount == 0
	s.anyC = true
	if amount == 0 {
		return true
	}
	b := &s.counter
	if !b.open && !e.openBuf(b) {
		atomic.AddUint64(&e.dropped, 1)
		return true
	}
	b.items[b.n] = amount
	b.ids[b.n] = id
	b.n++
	if b.n == b.cap {
		e.commitCounter(b)
	}
	return true
}

// Histogram is used for generating rich metrics, such as percentiles, from
// periodically occurring continuous values.  (metrics.go:273-295; compress() runs on the device, bit-exactly)
func (ms *MetricSystem) Histogram(name string, value float64) {
	e := engineFor(ms)
	for {
		id, gen, ok := e.histos.intern(name)
		if !ok {
			atomic.AddUint64(&e.dropped, 1)
			return
		}
		if e.appendHist(e.shard(), id, gen, value) {
			return
		}
		// the id was retired between intern and s.mu: look the name up again
	}
}

// appendHist reports false, appending nothing, when gen is no longer the generation of id (nameTable).
func (e *b200Engine) appendHist(s *b200Shard, id uint16, gen uint32, value float64) bool {
	s.mu.Lock()
	defer s.mu.Unlock()
	if !e.histos.current(id, gen) {
		return false
	}
	b := &s.hist
	if !b.open && !e.openBuf(b) {
		atomic.AddUint64(&e.dropped, 1)
		return true
	}
	b.items[b.n] = math.Float64bits(value)
	b.ids[b.n] = id
	b.n++
	if b.n == b.cap {
		e.commitHist(b)
	}
	return true
}

// collectRawMetrics, metrics.go:420-479: the cache swaps become lh_snapshot_begin (double-buffered device arrays),
// the maps are rebuilt from the sparse export, and the percentile statistics the device reduced for exactly this
// snapshot are parked beside the returned set for processMetrics.
func (ms *MetricSystem) collectRawMetrics() *RawMetricSet {
	e := engineFor(ms)
	e.snapshotMu.Lock()
	defer e.snapshotMu.Unlock()

	normalizedInterval := time.Unix(0, time.Now().UnixNano()/
		ms.interval.Nanoseconds()*
		ms.interval.Nanoseconds())

	// everything the shards hold goes to the device before the swap
	touched := make([]bool, b200MaxCounters)
	for _, s := range e.shards {
		s.mu.Lock()
		e.commitHist(&s.hist)
		e.commitCounter(&s.counter)
		if s.anyC {
			for i, t := range s.touched {
				if t {
					touched[i] = true
					s.touched[i] = false
				}
			}
			s.anyC = false
		}
		s.mu.Unlock()
	}

	// percentile labels in one fixed order for this snapshot (map iteration order is random in Go)
	red := &reducedSet{byName: map[string]*reducedHistogram{}}
	for label, p := range ms.percentiles {
		if len(red.labels) == C.LH_MAX_PERCENTILES {
			glog.Errorf("loghisto (b200): more than %d percentiles configured; %q ignored", C.LH_MAX_PERCENTILES, label)
			continue
		}
		red.labels = append(red.labels, label)
		red.ps = append(red.ps, p)
	}
	np := len(red.ps)

	histograms := make(map[string]map[int16]*uint64)
	rates := make(map[string]uint64)
	deltas := make([]uint64, b200MaxCounters)
	var cnames []string

	if err := b200Status(C.lh_snapshot_begin(e.ctx), e.ctx, "lh_snapshot_begin"); err != nil {
		glog.Errorf("loghisto (b200): %v; this interval's histograms and rates are lost", err)
	} else {
		const H = b200MaxHistograms
		counts := make([]uint64, H)
		sums := make([]float64, H)
		avgs := make([]float64, H)
		pkeys := make([]int32, H*np+1)
		pvals := make([]float64, H*np+1)
		var psPtr *C.double
		if np > 0 {
			psPtr = (*C.double)(unsafe.Pointer(&red.ps[0]))
		}
		st := C.lh_snapshot_reduce(e.ctx, psPtr, C.uint32_t(np),
			(*C.uint64_t)(unsafe.Pointer(&counts[0])), (*C.double)(unsafe.Pointer(&sums[0])),
			(*C.double)(unsafe.Pointer(&avgs[0])), (*C.int32_t)(unsafe.Pointer(&pkeys[0])),
			(*C.double)(unsafe.Pointer(&pvals[0])))
		var sp C.lh_sparse
		if err := b200Status(st, e.ctx, "lh_snapshot_reduce"); err != nil {
			glog.Errorf("loghisto (b200): %v", err)
		} else if err := b200Status(C.lh_snapshot_export(e.ctx, &sp), e.ctx, "lh_snapshot_export"); err != nil {
			glog.Errorf("loghisto (b200): %v", err)
		} else {
			// the pointers in sp are library-owned host memory, valid until the next export
			offsets := unsafe.Slice((*uint32)(unsafe.Pointer(sp.offsets)), H+1)
			total := int(sp.total_entries)
			var keys []int16
			var cnts []uint64
			if total > 0 {
				keys = unsafe.Slice((*int16)(unsafe.Pointer(sp.keys)), total)
				cnts = unsafe.Slice((*uint64)(unsafe.Pointer(sp.counts)), total)
			}
			cd := unsafe.Slice((*uint64)(unsafe.Pointer(sp.counter_deltas)), b200MaxCounters)
			copy(deltas, cd)
			// label the export with the id -> name tables as they stand, then step every id's lifecycle (nameTable);
			// a name interned since lh_snapshot_begin has no data in this export
			hnames := e.histos.collect(func(id int) bool { return offsets[id] != offsets[id+1] })
			cnames = e.counters.collect(func(id int) bool { return deltas[id] != 0 || touched[id] })
			for h, name := range hnames {
				a, b := int(offsets[h]), int(offsets[h+1])
				if a == b {
					continue // untouched this interval: absent, like a name missing from the swapped-out cache
				}
				backing := make([]uint64, b-a) // the RawMetricSet owns its counts forever (metrics.go:427, 462)
				copy(backing, cnts[a:b])
				m := make(map[int16]*uint64, b-a)
				for i := a; i < b; i++ {
					m[keys[i]] = &backing[i-a]
				}
				histograms[name] = m
				red.byName[name] = &reducedHistogram{
					count: counts[h], sum: sums[h], avg: avgs[h],
					pkeys: append([]int32(nil), pkeys[h*np:(h+1)*np]...),
					pvals: append([]float64(nil), pvals[h*np:(h+1)*np]...),
				}
			}
		}
		if err := b200Status(C.lh_snapshot_end(e.ctx), e.ctx, "lh_snapshot_end"); err != nil {
			glog.Errorf("loghisto (b200): %v", err)
		}
	}
	if cnames == nil { // no export: rates from the touched marks alone, and no lifecycle step this time
		cnames = e.counters.snapshotNames()
	}

	// Rates = this interval's deltas of the counters touched (metrics.go:430-433); Counters = cumulative store,
	// including counters not touched this interval (metrics.go:435-458).  The store is the reference's own field.
	counters := make(map[string]uint64)
	ms.counterStoreMu.Lock()
	for c, name := range cnames {
		if deltas[c] == 0 && !touched[c] {
			continue
		}
		rates[name] = deltas[c]
		p, exists := ms.counterStore[name]
		if !exists {
			var z uint64
			p = &z
			ms.counterStore[name] = p
		}
		atomic.AddUint64(p, deltas[c])
	}
	for name, count := range ms.counterStore {
		counters[name] = *count
	}
	ms.counterStoreMu.Unlock()

	ms.gaugeFuncsMu.Lock()
	gauges := make(map[string]float64)
	for name, f := range ms.gaugeFuncs {
		gauges[name] = f()
	}
	ms.gaugeFuncsMu.Unlock()

	raw := &RawMetricSet{
		Time:       normalizedInterval,
		Counters:   counters,
		Rates:      rates,
		Histograms: histograms,
		Gauges:     gauges,
	}
	e.putReduced(raw, red)
	return raw
}

// processHistograms, metrics.go:336-387, for one histogram of a snapshot the device reduced: interval count / sum /
// avg, the aggregate store update (uint64(totalSum) truncation included) and one value per percentile label.
func (ms *MetricSystem) processHistograms(name string, r *reducedHistogram, labels []string) map[string]float64 {
	output := make(map[string]float64)
	sumName := fmt.Sprintf("%s_sum", name)
	countName := fmt.Sprintf("%s_count", name)
	avgName := fmt.Sprintf("%s_avg", name)

	output[countName] = float64(r.count)
	output[sumName] = r.sum
	output[avgName] = r.avg

	ms.histogramCountMu.Lock()
	if _, present := ms.histogramCountStore[sumName]; !present {
		var x, z uint64
		ms.histogramCountStore[sumName] = &x
		ms.histogramCountStore[countName] = &z
	}
	atomic.AddUint64(ms.histogramCountStore[sumName], uint64(r.sum))
	atomic.AddUint64(ms.histogramCountStore[countName], r.count)
	ms.histogramCountMu.Unlock()

	for j, label := range labels {
		if r.pkeys[j] == math.MinInt32 { // percentile() returned its error (p > 1 or NaN): logged, key omitted
			glog.Errorf("unable to calculate percentile: %s", "Invalid percentile.  Should be between 0 and 1.")
			continue
		}
		output[fmt.Sprintf(label, name)] = r.pvals[j]
	}
	return output
}

// reduceSparse reduces the maps of `names` on the device (lh_reduce_sparse_host) with the percentiles configured
// now, as processHistograms reads ms.percentiles: one CSR of every map, one call.  Keys with a count of 0 are passed
// as entries like any other; the device keeps Go's answer for them.
func (ms *MetricSystem) reduceSparse(e *b200Engine, hists map[string]map[int16]*uint64, names []string) *reducedSet {
	red := &reducedSet{byName: map[string]*reducedHistogram{}}
	for label, p := range ms.percentiles {
		if len(red.labels) == C.LH_MAX_PERCENTILES {
			glog.Errorf("loghisto (b200): more than %d percentiles configured; %q ignored", C.LH_MAX_PERCENTILES, label)
			continue
		}
		red.labels = append(red.labels, label)
		red.ps = append(red.ps, p)
	}
	np, n := len(red.ps), len(names)
	// plain Go slices without Go pointers in them: cgo lets C read them for the duration of the call
	total := 0
	for _, name := range names {
		total += len(hists[name])
	}
	offsets := make([]uint32, n+1)
	keys := make([]int16, total+1)
	cnts := make([]uint64, total+1)
	pos := 0
	for i, name := range names {
		offsets[i] = uint32(pos)
		for k, c := range hists[name] {
			keys[pos], cnts[pos] = k, *c
			pos++
		}
	}
	offsets[n] = uint32(pos)
	counts := make([]uint64, n)
	sums := make([]float64, n)
	avgs := make([]float64, n)
	pkeys := make([]int32, n*np+1)
	pvals := make([]float64, n*np+1)
	var psPtr *C.double
	if np > 0 {
		psPtr = (*C.double)(unsafe.Pointer(&red.ps[0]))
	}
	st := C.lh_reduce_sparse_host(e.ctx, C.uint32_t(n), (*C.uint32_t)(unsafe.Pointer(&offsets[0])),
		(*C.int16_t)(unsafe.Pointer(&keys[0])), (*C.uint64_t)(unsafe.Pointer(&cnts[0])), psPtr, C.uint32_t(np),
		(*C.uint64_t)(unsafe.Pointer(&counts[0])), (*C.double)(unsafe.Pointer(&sums[0])),
		(*C.double)(unsafe.Pointer(&avgs[0])), (*C.int32_t)(unsafe.Pointer(&pkeys[0])),
		(*C.double)(unsafe.Pointer(&pvals[0])))
	if err := b200Status(st, e.ctx, "lh_reduce_sparse_host"); err != nil {
		glog.Errorf("loghisto (b200): %v; the histograms of this RawMetricSet are lost", err)
		return red
	}
	for i, name := range names {
		red.byName[name] = &reducedHistogram{
			count: counts[i], sum: sums[i], avg: avgs[i],
			pkeys: append([]int32(nil), pkeys[i*np:(i+1)*np]...),
			pvals: append([]float64(nil), pvals[i*np:(i+1)*np]...),
		}
	}
	return red
}

// processMetrics, metrics.go:483-506, for any RawMetricSet.  A set collectRawMetrics produced is processed with the
// reduction the device made for its snapshot (parked beside it, consumed here); the histograms of every other set --
// hand-built or deserialised sets, unions of several hosts' sets, a set processed a second time or after it aged out
// of the ring -- are gathered into one CSR and reduced on the device by one lh_reduce_sparse_host call.
func (ms *MetricSystem) processMetrics(rawMetrics *RawMetricSet) *ProcessedMetricSet {
	e := engineFor(ms)
	metrics := make(map[string]float64)

	for name, count := range rawMetrics.Counters {
		metrics[name] = float64(count)
	}

	for name, count := range rawMetrics.Rates {
		metrics[fmt.Sprintf("%s_rate", name)] = float64(count)
	}

	red := e.takeReduced(rawMetrics)
	var missing []string
	for name := range rawMetrics.Histograms {
		if red == nil || red.byName[name] == nil {
			missing = append(missing, name)
			continue
		}
		for histoName, histoValue := range ms.processHistograms(name, red.byName[name], red.labels) {
			metrics[histoName] = histoValue
		}
	}
	if len(missing) > 0 {
		fresh := ms.reduceSparse(e, rawMetrics.Histograms, missing)
		for _, name := range missing {
			if r := fresh.byName[name]; r != nil {
				for histoName, histoValue := range ms.processHistograms(name, r, fresh.labels) {
					metrics[histoName] = histoValue
				}
			}
		}
	}

	for name, value := range rawMetrics.Gauges {
		metrics[name] = value
	}

	return &ProcessedMetricSet{Time: rawMetrics.Time, Metrics: metrics}
}
