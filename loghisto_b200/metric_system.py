"""Python face of the C++ MetricSystem mirror (loghisto_b200/host/metric_system.{h,cc}).

Method names follow the Go type (reference metrics.go) so the tests read like metrics_test.go.  All work
happens in the C++ layer and, below it, in the CUDA library; this module only marshals.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import sys

from . import _lib as _L
from . import build as _build
from .engine import (_batch_array, _capture_stream, _stream, _timer_stream, array_src, board_out, board_views, gauge_src,
                     graph_counter_args, graph_duration_out, graph_keyed_args, raw_percentiles, raw_ranks,
                     check_window)

_EMIT = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.c_uint64, C.c_double)
_RANKS_SINK = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64)
_RANKS_ALLGATHER = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, _RANKS_SINK, C.c_void_p)
_RANKS_ALLREDUCE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p)
_lib = None


def _load():
    global _lib
    if _lib is not None:
        return _lib
    if _build.needs_build() or _build.needs_build_host():
        _build.build_host()
    _lib = _bind(C.CDLL(_build.HOST_LIB))
    return _lib


def _bind(L):
    """Declare the lhms_* signatures on a loaded host library."""
    vp = C.c_void_p
    L.lhms_new.restype = vp
    L.lhms_new.argtypes = [C.c_int64, C.c_int, C.c_uint32, C.c_uint32, C.c_char_p, C.c_int]
    L.lhms_new_precision.restype = vp
    L.lhms_new_precision.argtypes = [C.c_int64, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_int]
    L.lhms_free.argtypes = [vp]
    L.lhms_histogram.argtypes = [vp, C.c_char_p, C.c_double]
    L.lhms_counter.argtypes = [vp, C.c_char_p, C.c_uint64]
    L.lhms_histogram_many.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    L.lhms_start_timer.restype = vp
    L.lhms_start_timer.argtypes = [vp, C.c_char_p]
    L.lhms_timer_stop.restype = C.c_int64
    L.lhms_timer_stop.argtypes = [vp]
    L.lhms_specify_percentiles.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double)]
    L.lhms_register_constant_gauge.argtypes = [vp, C.c_char_p, C.c_double]
    L.lhms_register_device_gauge.restype = C.c_int
    L.lhms_register_device_gauge.argtypes = [vp, C.c_char_p, vp, C.c_uint32]
    L.lhms_deregister_gauge.argtypes = [vp, C.c_char_p]
    L.lhms_register_device_distribution.restype = C.c_int
    L.lhms_register_device_distribution.argtypes = [vp, C.c_char_p, vp, C.c_uint64, C.c_uint32]
    L.lhms_deregister_device_distribution.restype = C.c_int
    L.lhms_deregister_device_distribution.argtypes = [vp, C.c_char_p]
    L.lhms_stats.restype = C.c_int
    L.lhms_stats.argtypes = [vp, C.POINTER(_L.lh_stats)]
    L.lhms_collect_and_process.restype = C.c_int
    L.lhms_collect_and_process.argtypes = [vp, _EMIT, vp, C.c_char_p, C.c_int]
    names, u64p = C.POINTER(C.c_char_p), C.POINTER(C.c_uint64)
    L.lhms_process_metrics.restype = C.c_int
    L.lhms_process_metrics.argtypes = [vp, C.c_int64, C.c_int, C.c_uint32, names, u64p, C.c_uint32, names, u64p,
                                       C.c_uint32, names, C.POINTER(C.c_uint32), C.POINTER(C.c_int16), u64p,
                                       C.c_uint32, names, C.POINTER(C.c_double), _EMIT, vp, C.c_char_p, C.c_int]
    L.lhms_start.argtypes = [vp]
    L.lhms_stop.argtypes = [vp]
    L.lhms_dropped.restype = C.c_uint64
    L.lhms_dropped.argtypes = [vp]
    L.lhms_timer_free.argtypes = [vp]
    L.lhms_histogram_stream.restype = C.c_double
    L.lhms_histogram_stream.argtypes = [vp, C.POINTER(C.c_char_p), C.c_uint32, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint]
    L.lhms_histogram_stream2.restype = C.c_double
    L.lhms_histogram_stream2.argtypes = [vp, C.POINTER(C.c_char_p), C.c_uint32, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint,
                                         C.c_int, C.POINTER(C.c_double)]
    L.lhms_timer_loop.restype = C.c_double
    L.lhms_timer_loop.argtypes = [C.c_char_p, C.c_uint, C.c_double, C.c_int64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
    L.lhms_print_benchmark.restype = C.c_double
    L.lhms_print_benchmark.argtypes = [C.c_char_p, C.c_uint, C.c_double, C.c_int64, C.c_int, C.c_int]
    rec, u32p = C.POINTER(_L.lh_recorder), C.POINTER(C.c_uint32)
    L.lhms_record_begin.restype = C.c_int
    L.lhms_record_begin.argtypes = [vp, vp, C.c_uint32, names, C.c_uint32, names, rec, u32p, u32p]
    L.lhms_record_end.restype = C.c_int
    L.lhms_record_end.argtypes = [vp, rec]
    L.lhms_record_ingest_f64.restype = C.c_int
    L.lhms_record_ingest_f64.argtypes = [vp, rec, C.c_uint32, vp, C.c_size_t]
    L.lhms_scope_histograms.restype = C.c_int
    L.lhms_scope_histograms.argtypes = [vp, rec, u32p, C.POINTER(vp), C.POINTER(C.c_uint64), u32p, C.c_uint32]
    L.lhms_scoped_keyed.restype = C.c_int
    L.lhms_scoped_keyed.argtypes = [vp, rec, C.c_uint32, vp, vp, C.c_uint32, C.c_size_t]
    L.lhms_scoped_counters.restype = C.c_int
    L.lhms_scoped_counters.argtypes = [vp, rec, C.c_uint32, vp, vp, C.c_size_t]
    L.lhms_gpu_timer_start.restype = vp
    L.lhms_gpu_timer_start.argtypes = [vp, C.c_char_p, vp, C.POINTER(C.c_int)]
    L.lhms_gpu_timer_stop.restype = C.c_int
    L.lhms_gpu_timer_stop.argtypes = [vp, vp, vp]
    L.lhms_gpu_timer_free.argtypes = [vp]
    L.lhms_graph_recorder_new.restype = vp
    L.lhms_graph_recorder_new.argtypes = [vp, C.c_uint32, names, C.c_uint32, names, rec, C.POINTER(C.c_int)]
    L.lhms_graph_recorder_histograms.restype = C.c_int
    L.lhms_graph_recorder_histograms.argtypes = [vp, u32p, C.POINTER(vp), C.POINTER(C.c_uint64), u32p, C.c_uint32, vp]
    L.lhms_arrays_scope.restype = C.c_int
    L.lhms_arrays_scope.argtypes = [vp, rec, u32p, C.POINTER(vp), C.POINTER(C.c_uint64), u32p, C.c_uint32]
    L.lhms_arrays_graph_recorder.restype = C.c_int
    L.lhms_arrays_graph_recorder.argtypes = [vp, u32p, C.POINTER(vp), C.POINTER(C.c_uint64), u32p, C.c_uint32, vp]
    L.lhms_graph_recorder_close.restype = C.c_int
    L.lhms_graph_recorder_close.argtypes = [vp, vp]
    L.lhms_graph_recorder_free.argtypes = [vp]
    L.lhms_graph_keyed.restype = C.c_int
    L.lhms_graph_keyed.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_size_t, vp]
    L.lhms_graph_counters.restype = C.c_int
    L.lhms_graph_counters.argtypes = [vp, C.c_uint32, vp, vp, C.c_size_t, vp]
    L.lhms_graph_timer_start.restype = C.c_int
    L.lhms_graph_timer_start.argtypes = [vp, C.c_uint32, vp]
    L.lhms_graph_timer_stop.restype = C.c_int
    L.lhms_graph_timer_stop.argtypes = [vp, C.c_uint32, vp, vp]
    L.lhms_subscription_new.restype = vp
    L.lhms_subscription_new.argtypes = [vp, C.c_uint32, names, C.c_uint32, names, C.POINTER(_L.lh_board), C.POINTER(C.c_int)]
    L.lhms_subscription_read.restype = C.c_int
    L.lhms_subscription_read.argtypes = [vp, vp, vp]
    L.lhms_subscription_close.restype = C.c_int
    L.lhms_subscription_close.argtypes = [vp]
    L.lhms_subscription_free.argtypes = [vp]
    L.lhms_raw_subscription_new.restype = vp
    L.lhms_raw_subscription_new.argtypes = [vp, C.c_uint32, names, C.POINTER(_L.lh_raw_board), C.POINTER(C.c_int)]
    L.lhms_raw_window_subscription_new.restype = vp
    L.lhms_raw_window_subscription_new.argtypes = [vp, C.c_uint32, names, C.c_uint32, C.POINTER(_L.lh_raw_board),
                                                   C.POINTER(C.c_int)]
    for q in ("percentiles", "ranks"):
        getattr(L, "lhms_raw_subscription_" + q).restype = C.c_int
        getattr(L, "lhms_raw_subscription_" + q).argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
    L.lhms_raw_subscription_close.restype = C.c_int
    L.lhms_raw_subscription_close.argtypes = [vp]
    L.lhms_raw_subscription_free.argtypes = [vp]
    for kind in ("processed", "raw"):
        getattr(L, "lhms_subscribe_" + kind).restype = vp
        getattr(L, "lhms_subscribe_" + kind).argtypes = [vp, C.c_int]
        getattr(L, "lhms_unsubscribe_" + kind).argtypes = [vp, vp]
        getattr(L, "lhms_recv_" + kind).restype = C.c_int
        getattr(L, "lhms_recv_" + kind).argtypes = [vp, C.c_int64, _EMIT, vp]
        getattr(L, "lhms_free_%s_channel" % kind).argtypes = [vp]
    L.lhms_ranks_join.restype = C.c_int
    L.lhms_ranks_join.argtypes = [vp, C.c_uint32, C.c_uint32, _RANKS_ALLGATHER, vp, C.c_char_p, C.c_int]
    L.lhms_ranks_info.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.lhms_ranks_join_allreduce.restype = C.c_int
    L.lhms_ranks_join_allreduce.argtypes = [vp, C.c_uint32, C.c_uint32, _RANKS_ALLGATHER, _RANKS_ALLREDUCE, vp,
                                            C.c_char_p, C.c_int]
    return L


class _Collector:
    def __init__(self):
        self.raw = {"Counters": {}, "Rates": {}, "Histograms": {}, "Gauges": {}}
        self.metrics = {}

        def emit(_ctx, kind, name, key, u, f):
            name = name.decode()
            if kind == 0:
                self.raw["Counters"][name] = int(u)
            elif kind == 1:
                self.raw["Rates"][name] = int(u)
            elif kind == 2:
                self.raw["Histograms"].setdefault(name, {})[int(key)] = int(u)
            elif kind == 4:
                self.raw["Gauges"][name] = float(f)
            else:
                self.metrics[name] = float(f)

        self.cb = _EMIT(emit)


class TimerToken:
    def __init__(self, lib, handle):
        self._lib, self._h = lib, handle

    def Stop(self) -> int:
        """Submits the duration as a histogram sample and returns it in nanoseconds (metrics.go:242-246).  The Go token
        may be stopped repeatedly (one sample each time); this handle is consumed by the first Stop, later calls
        return 0 without submitting anything."""
        if self._h is None:
            return 0
        ns = self._lib.lhms_timer_stop(self._h)
        self._h = None
        return int(ns)

    def __del__(self):
        try:
            if self._h is not None:      # never stopped: release the C++ token
                self._lib.lhms_timer_free(self._h)
                self._h = None
        except Exception:
            pass


class GpuTimerToken:
    """A timer whose start and stop are marks on the GPU's clock (MetricSystem.StartGpuTimer)."""

    def __init__(self, ms, handle, stream: int):
        self._ms, self._h, self._stream = ms, handle, stream

    def Stop(self, stream=None, out=None):
        """Records the duration on the device under the token's name; nothing is returned to the host.  `stream`:
        None = the stream the timer was started on, else an int handle or a torch.cuda.Stream.  `out`: an optional
        contiguous int64 CUDA tensor whose first element receives the duration in ns.  Consumed by the first call, as
        TimerToken: later calls do nothing."""
        if self._h is None:
            return
        ptr = 0
        if out is not None:
            if not (out.is_cuda and str(out.dtype) == "torch.int64" and out.is_contiguous() and out.numel() >= 1):
                raise TypeError("out must be a contiguous int64 CUDA tensor")
            ptr = out.data_ptr()
        st = self._ms._lib.lhms_gpu_timer_stop(self._h, self._stream if stream is None else _timer_stream(stream), ptr)
        self._free()
        if st != 0:
            raise RuntimeError("lhms_gpu_timer_stop failed (status %d)" % st)

    def _free(self):
        if self._h is not None and self._ms._h:   # a closed MetricSystem already freed the pool
            self._ms._lib.lhms_gpu_timer_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass


class RecordScope:
    """An open record scope of a MetricSystem (MetricSystem.recording).  `recorder` is the lh_recorder to pass by value
    to kernels enqueued on the scope's stream; `histogram_ids` / `counter_ids` map each bound name to the id those
    kernels record under (0xFFFFFFFF when the name found no free id: its records are dropped and counted)."""
    UNBOUND = 0xFFFFFFFF

    def __init__(self, ms, stream, histograms, counters):
        self._ms = ms
        self._hnames, cnames = [str(x) for x in histograms], [str(x) for x in counters]
        self.recorder = _L.lh_recorder()
        hids = (C.c_uint32 * max(len(self._hnames), 1))()
        cids = (C.c_uint32 * max(len(cnames), 1))()
        hn = (C.c_char_p * max(len(self._hnames), 1))(*[x.encode() for x in self._hnames])
        cn = (C.c_char_p * max(len(cnames), 1))(*[x.encode() for x in cnames])
        st = ms._lib.lhms_record_begin(ms._h, _stream(stream), len(self._hnames), hn, len(cnames), cn,
                                       C.byref(self.recorder), hids, cids)
        if st != 0:
            raise RuntimeError("lhms_record_begin failed (status %d)" % st)
        self.histogram_ids = {nm: int(hids[i]) for i, nm in enumerate(self._hnames)}
        self.counter_ids = {nm: int(cids[i]) for i, nm in enumerate(cnames)}
        self._open = True

    def histogram(self, name: str, values):
        """Histogram(name, v) for every element of a contiguous float64 CUDA tensor, on the scope's stream."""
        if not (values.is_cuda and str(values.dtype) == "torch.float64" and values.is_contiguous()):
            raise TypeError("values must be a contiguous float64 CUDA tensor")
        st = self._ms._lib.lhms_record_ingest_f64(self._ms._h, C.byref(self.recorder), self._hnames.index(name),
                                                  values.data_ptr(), values.numel())
        if st != 0:
            raise RuntimeError("lhms_record_ingest_f64 failed (status %d)" % st)

    def histograms(self, arrays):
        """Histogram(name, v) for every element of several device arrays in one call (lh_ingest_batch), on the scope's
        stream: `arrays` is {name: array} or a list of (name, array) pairs, names among the scope's histograms and
        possibly repeated.  An array is a contiguous CUDA tensor (or DeviceArray / __cuda_array_interface__ object):
        float64 values, or int64 nanoseconds recorded as float64(ns) like a Timer's Stop.  TypeError for any other
        array and KeyError for a name the scope was not opened with, before anything is issued."""
        pairs = list(arrays.items()) if isinstance(arrays, dict) else list(arrays)
        k = max(len(pairs), 1)
        idx, ptrs, ns, kinds = (C.c_uint32 * k)(), (C.c_void_p * k)(), (C.c_uint64 * k)(), (C.c_uint32 * k)()
        for i, (name, a) in enumerate(pairs):
            if name not in self._hnames:
                raise KeyError("%r is not a histogram of this scope" % (name,))
            idx[i] = self._hnames.index(name)
            ptrs[i], ns[i], kinds[i] = _batch_array(a)
        st = self._ms._lib.lhms_scope_histograms(self._ms._h, C.byref(self.recorder), idx, ptrs, ns, kinds, len(pairs))
        if st != 0:
            raise RuntimeError("lhms_scope_histograms failed (status %d)" % st)

    def arrays(self, arrays):
        """Histogram(name, float64(x)) for every element x of several device tensors in one call (lh_ingest_arrays),
        on the scope's stream, without a float64 copy: `arrays` as histograms() takes them, each tensor contiguous, on
        the system's device, of any shape, float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64.  TypeError
        for any other array and KeyError for a name the scope was not opened with, before anything is issued."""
        pairs = list(arrays.items()) if isinstance(arrays, dict) else list(arrays)
        idx, ptrs, ns, dts = _array_table(pairs, lambda name: self._hnames.index(name) if name in self._hnames else None,
                                          "scope", self._ms._device)
        st = self._ms._lib.lhms_arrays_scope(self._ms._h, C.byref(self.recorder), idx, ptrs, ns, dts, len(pairs))
        if st != 0:
            raise RuntimeError("lhms_arrays_scope failed (status %d)" % st)

    def keyed(self, ids, values):
        """Histogram(name, values[i]) with name the scope's histogram at position ids[i], for every i, in one call on
        the scope's stream (lh_ingest_keyed_mapped_*).  ids and values as GraphRecorder.keyed takes them (uint16, int32
        or uint32 ids; float64 values, or int64 nanoseconds recorded as float64(ns)); TypeError / ValueError before
        anything is issued.  An id past the names, or under an unbound name, is dropped and counted."""
        id_bytes, ip, vp, kind, n = graph_keyed_args(ids, values)
        st = self._ms._lib.lhms_scoped_keyed(self._ms._h, C.byref(self.recorder), id_bytes, ip, vp, kind, n)
        if st != 0:
            raise RuntimeError("lhms_scoped_keyed failed (status %d)" % st)

    def counters(self, ids, amounts):
        """Counter(name, amounts[i]) with name the scope's counter at position ids[i] (lh_counter_add_mapped_*): ids
        as keyed() takes them, amounts int64 or uint64 (added as uint64 bits, wrapping)."""
        id_bytes, ip, ap, n = graph_counter_args(ids, amounts)
        st = self._ms._lib.lhms_scoped_counters(self._ms._h, C.byref(self.recorder), id_bytes, ip, ap, n)
        if st != 0:
            raise RuntimeError("lhms_scoped_counters failed (status %d)" % st)

    def end(self):
        if self._open:
            self._open = False
            st = self._ms._lib.lhms_record_end(self._ms._h, C.byref(self.recorder))
            if st != 0:
                raise RuntimeError("lhms_record_end failed (status %d)" % st)


def _array_table(pairs, index_of, owner, device):
    """(name indices, addresses, lengths, LH_GAUGE_* dtypes) of (name, tensor) pairs for lhms_arrays_scope /
    lhms_arrays_graph_recorder; KeyError for a name index_of does not know, TypeError for a tensor array_src refuses."""
    k = max(len(pairs), 1)
    idx, ptrs, ns, dts = (C.c_uint32 * k)(), (C.c_void_p * k)(), (C.c_uint64 * k)(), (C.c_uint32 * k)()
    for i, (name, t) in enumerate(pairs):
        j = index_of(name)
        if j is None:
            raise KeyError("%r is not a histogram of this %s" % (name, owner))
        src = array_src(t, device, 0, "an ingested array")
        idx[i], ptrs[i], ns[i], dts[i] = j, src.d_values, src.n, src.dtype
    return idx, ptrs, ns, dts


class GraphRecorder:
    """A graph recorder of a MetricSystem (MetricSystem.graph_recorder).  `recorder` is the lh_recorder to pass by value
    to kernels captured into CUDA graphs; `histogram_ids` / `counter_ids` map each name to the local id those kernels
    record under (its position in the list).  Every collection drains what the replays recorded so far into the
    interval it collects, under the names."""

    def __init__(self, ms, histograms, counters):
        self._ms = ms
        self._hnames, cnames = [str(x) for x in histograms], [str(x) for x in counters]
        self.recorder = _L.lh_recorder()
        hn = (C.c_char_p * max(len(self._hnames), 1))(*[x.encode() for x in self._hnames])
        cn = (C.c_char_p * max(len(cnames), 1))(*[x.encode() for x in cnames])
        st = C.c_int()
        self._h = ms._lib.lhms_graph_recorder_new(ms._h, len(self._hnames), hn, len(cnames), cn,
                                                 C.byref(self.recorder), C.byref(st))
        if not self._h:
            raise RuntimeError("lhms_graph_recorder_new failed (status %d)" % st.value)
        self.histogram_ids = {nm: i for i, nm in enumerate(self._hnames)}
        self.counter_ids = {nm: i for i, nm in enumerate(cnames)}

    def histograms(self, arrays, stream=None):
        """Histogram(name, v) for every element of several device arrays (lh_graph_recorder_ingest): `arrays` as
        RecordScope.histograms takes them.  Kernels only, on `stream` (None = torch's current stream), so inside
        torch.cuda.graph the call is captured and every replay records the arrays' contents at that time."""
        pairs = list(arrays.items()) if isinstance(arrays, dict) else list(arrays)
        k = max(len(pairs), 1)
        idx, ptrs, ns, kinds = (C.c_uint32 * k)(), (C.c_void_p * k)(), (C.c_uint64 * k)(), (C.c_uint32 * k)()
        for i, (name, a) in enumerate(pairs):
            if name not in self.histogram_ids:
                raise KeyError("%r is not a histogram of this recorder" % (name,))
            idx[i] = self.histogram_ids[name]
            ptrs[i], ns[i], kinds[i] = _batch_array(a)
        if self._h is None:
            raise RuntimeError("the graph recorder is closed")
        st = self._ms._lib.lhms_graph_recorder_histograms(self._h, idx, ptrs, ns, kinds, len(pairs), _capture_stream(stream))
        if st != 0:
            raise RuntimeError("lhms_graph_recorder_histograms failed (status %d)" % st)

    def arrays(self, arrays, stream=None):
        """Histogram(name, float64(x)) for every element x of several device tensors (lh_graph_recorder_ingest_arrays):
        `arrays` as RecordScope.arrays takes them.  Kernels only, on `stream` (None = torch's current stream), so inside
        torch.cuda.graph the call is captured and every replay records the tensors' contents at that time."""
        pairs = list(arrays.items()) if isinstance(arrays, dict) else list(arrays)
        idx, ptrs, ns, dts = _array_table(pairs, self.histogram_ids.get, "recorder", self._ms._device)
        if self._h is None:
            raise RuntimeError("the graph recorder is closed")
        st = self._ms._lib.lhms_arrays_graph_recorder(self._h, idx, ptrs, ns, dts, len(pairs), _capture_stream(stream))
        if st != 0:
            raise RuntimeError("lhms_arrays_graph_recorder failed (status %d)" % st)

    def _call(self, what, *args):
        if self._h is None:
            raise RuntimeError("the graph recorder is closed")
        st = getattr(self._ms._lib, what)(self._h, *args)
        if st != 0:
            raise RuntimeError("%s failed (status %d)" % (what, st))

    def _name(self, name):
        if name not in self.histogram_ids:
            raise KeyError("%r is not a histogram of this recorder" % (name,))
        return self.histogram_ids[name]

    def keyed(self, ids, values, stream=None):
        """Histogram(name, values[i]) with name the histogram of local id ids[i] (its position in histogram_ids), for
        every i (lh_graph_recorder_ingest_keyed_*).  ids: uint16, int32 or uint32 device array (an id past the names,
        a negative int32 among them, is dropped and counted); values: float64, or int64 nanoseconds recorded as
        float64(ns).  Kernels only, on `stream` (None = torch's current stream), so inside torch.cuda.graph the call
        is captured.  TypeError / ValueError before anything is issued."""
        id_bytes, ip, vp, kind, n = graph_keyed_args(ids, values)
        self._call("lhms_graph_keyed", id_bytes, ip, vp, kind, n, _capture_stream(stream))

    def counters(self, ids, amounts, stream=None):
        """Counter(name, amounts[i]) with name the counter of local id ids[i] (lh_graph_recorder_counter_add_*): ids as
        keyed() takes them, amounts int64 or uint64 (added as uint64 bits, wrapping).  Capturable like keyed()."""
        id_bytes, ip, ap, n = graph_counter_args(ids, amounts)
        self._call("lhms_graph_counters", id_bytes, ip, ap, n, _capture_stream(stream))

    def start_timer(self, name, stream=None):
        """Start a GPU-timed span of histogram `name` on `stream` (lh_graph_recorder_timer_start); capturable.  One open
        span per name: sequential spans are fine, concurrent ones on parallel branches need another recorder."""
        idx = self._name(name)
        self._call("lhms_graph_timer_start", idx, _capture_stream(stream))

    def stop_timer(self, name, stream=None, out=None):
        """Record the span's duration under `name` (lh_graph_recorder_timer_stop), ordered after its start by the
        caller; `out` (an int64 device array) also receives it in ns.  A stop with no start is dropped and counted."""
        idx = self._name(name)
        ptr = graph_duration_out(out)
        self._call("lhms_graph_timer_stop", idx, _capture_stream(stream), ptr)

    @contextlib.contextmanager
    def timer(self, name, stream=None):
        """`with g.timer("layer"):` -- start_timer before the block and stop_timer after it, on one stream."""
        self.start_timer(name, stream)
        yield
        self.stop_timer(name, stream)

    def close(self, stream=None):
        """Drains what the recorder holds into the current interval on `stream` (None = torch's current stream) and
        frees it.  No replay that uses it may be pending.  Idempotent."""
        if self._h is None:
            return
        h, self._h = self._h, None
        st = 0
        if self._ms._h:   # a closed MetricSystem already freed the recorder
            st = self._ms._lib.lhms_graph_recorder_close(h, _capture_stream(stream))
        self._ms._lib.lhms_graph_recorder_free(h)
        if st != 0:
            raise RuntimeError("lhms_graph_recorder_close failed (status %d)" % st)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceSubscription:
    """A device subscription of a MetricSystem (MetricSystem.device_subscription): every collection publishes the
    processed metrics of its names into `board`, an lh_board in device memory that kernels read with
    lh::read_histogram / lh::read_counter (row numbers in histogram_rows / counter_rows), and read() copies on a stream.
    Usable as a context manager; close() (also on exit) frees the board once no read of it is pending."""

    def __init__(self, ms, histograms, counters):
        self._ms = ms
        hnames, cnames = [str(x) for x in histograms], [str(x) for x in counters]
        self.board = _L.lh_board()
        hn = (C.c_char_p * max(len(hnames), 1))(*[x.encode() for x in hnames])
        cn = (C.c_char_p * max(len(cnames), 1))(*[x.encode() for x in cnames])
        st = C.c_int()
        self._h = ms._lib.lhms_subscription_new(ms._h, len(hnames), hn, len(cnames), cn, C.byref(self.board), C.byref(st))
        if not self._h:
            raise RuntimeError("lhms_subscription_new failed (status %d)" % st.value)
        self.histogram_rows = {nm: i for i, nm in enumerate(hnames)}
        self.counter_rows = {nm: i for i, nm in enumerate(cnames)}
        self._device = ms._device

    def read(self, out=None, stream=None) -> dict:
        """One kernel on `stream` (None = torch's current stream, so that it is captured inside torch.cuda.graph)
        copies a consistent image of the latest publish into `out` (a contiguous uint8 CUDA tensor of at least
        board.bytes, or None for a new one); returns torch views of it (engine.board_views: collection, np,
        percentiles, present, count, sum, avg, pvals, pkeys, counter_present, rate, total).  Nothing is synchronised:
        the views are valid once the stream has run the copy.  A graph replay copies the publish latest at its run."""
        if self._h is None:
            raise RuntimeError("the device subscription is closed")
        buf = board_out(out, self.board.bytes, self._device)
        st = self._ms._lib.lhms_subscription_read(self._h, buf.data_ptr(), _capture_stream(stream))
        if st != 0:
            raise RuntimeError("lhms_subscription_read failed (status %d)" % st)
        return board_views(buf, self.board.k, self.board.kc)

    def close(self):
        """Frees the board after every publish issued.  No read of it may be pending.  Idempotent."""
        if self._h is None:
            return
        h, self._h = self._h, None
        st = 0
        if self._ms._h:   # a closed MetricSystem already freed the board
            st = self._ms._lib.lhms_subscription_close(h)
        self._ms._lib.lhms_subscription_free(h)
        if st != 0:
            raise RuntimeError("lhms_subscription_close failed (status %d)" % st)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RawDeviceSubscription:
    """A raw device subscription of a MetricSystem (MetricSystem.raw_device_subscription): every collection publishes
    the bucket counts of its histogram names into `board`, an lh_raw_board in device memory that kernels query with
    lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count (row numbers in `rows`), and percentiles() / ranks()
    query from torch.  Usable as a context manager; close() (also on exit) frees the board once no query of it is
    pending.  With `window` w > 1 every row answers for its name's histograms summed over the last w collections
    (a collection without the name adds nothing)."""

    def __init__(self, ms, histograms, window=1):
        window = check_window(window)
        self._ms = ms
        hnames = [str(x) for x in histograms]
        self.board = _L.lh_raw_board()
        hn = (C.c_char_p * max(len(hnames), 1))(*[x.encode() for x in hnames])
        st = C.c_int()
        if window == 1:
            self._h = ms._lib.lhms_raw_subscription_new(ms._h, len(hnames), hn, C.byref(self.board), C.byref(st))
        else:
            self._h = ms._lib.lhms_raw_window_subscription_new(ms._h, len(hnames), hn, window, C.byref(self.board),
                                                                C.byref(st))
        if not self._h:
            raise RuntimeError("lhms_raw_subscription_new failed (status %d)" % st.value)
        self.window = window
        self.rows = {nm: i for i, nm in enumerate(hnames)}
        self._device = ms._device

    def _call(self, fn, what):
        if self._h is None:
            raise RuntimeError("the raw device subscription is closed")

        def call(*a):
            st = fn(self._h, *a)
            if st != 0:
                raise RuntimeError("%s failed (status %d)" % (what, st))
        return call

    def percentiles(self, ps, stream=None):
        """For every row and each p of `ps` (a float64 CUDA tensor of length m): keys int32 [k, m], values float64
        [k, m] and publish numbers int64 [k, m], bit for bit what processMetrics reports for a label with that p
        (INT32_MIN / NaN where it omits one).  One kernel on `stream` (None = torch's current stream, so that it is
        captured inside torch.cuda.graph) and no synchronisation; a graph replay answers from the publish latest at
        its run."""
        call = self._call(self._ms._lib.lhms_raw_subscription_percentiles, "lhms_raw_subscription_percentiles")
        return raw_percentiles(call, self.board.k, ps, self._device, stream)

    def ranks(self, values, stream=None):
        """For every row and each value of `values` (a float64 CUDA tensor of length m): ranks int64 [k, m] (samples
        whose bucket is at or below the value's), totals int64 [k] (of the publish query (r, 0) read) and publish
        numbers int64 [k, m].  One kernel, as percentiles()."""
        call = self._call(self._ms._lib.lhms_raw_subscription_ranks, "lhms_raw_subscription_ranks")
        return raw_ranks(call, self.board.k, values, self._device, stream)

    def close(self):
        """Frees the board after every publish issued.  No query of it may be pending.  Idempotent."""
        if self._h is None:
            return
        h, self._h = self._h, None
        st = 0
        if self._ms._h:   # a closed MetricSystem already freed the board
            st = self._ms._lib.lhms_raw_subscription_close(h)
        self._ms._lib.lhms_raw_subscription_free(h)
        if st != 0:
            raise RuntimeError("lhms_raw_subscription_close failed (status %d)" % st)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Subscription:
    def __init__(self, ms, kind, capacity):
        self._ms, self._kind = ms, kind
        self._ch = getattr(ms._lib, "lhms_subscribe_" + kind)(ms._h, capacity)

    def receive(self, timeout_s: float):
        """dict of metrics (processed) / raw dict, None on timeout; raises EOFError if the reaper closed the channel."""
        col = _Collector()
        rc = getattr(self._ms._lib, "lhms_recv_" + self._kind)(self._ch, int(timeout_s * 1e9), col.cb, None)
        if rc == 1:
            return col.metrics if self._kind == "processed" else col.raw
        if rc == -1:
            raise EOFError("channel closed by the reaper")
        return None

    def unsubscribe(self):
        if self._ch is not None and self._ms._h:
            getattr(self._ms._lib, "lhms_unsubscribe_" + self._kind)(self._ms._h, self._ch)

    def close(self):
        """Unsubscribe and free the channel (with whatever metric sets are still queued in it)."""
        if self._ch is not None:
            self.unsubscribe()
            getattr(self._ms._lib, "lhms_free_%s_channel" % self._kind)(self._ch)
            self._ch = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MetricSystem:
    """NewMetricSystem(interval, sysStats) -- sysStats (Go runtime gauges) is accepted and ignored."""

    def __init__(self, interval_s: float, sysStats: bool = False, device: int = 0, max_histograms: int = 1024,
                 max_counters: int = 1024, precision: int = 0):
        """precision: bucket precision of compress() (0 = the reference's 100).

        max_histograms / max_counters bound the distinct histogram / counter names used in any three consecutive
        intervals: ids of idle names are recycled, a name last used in interval k keeping its id through k+2.  A new
        name that finds no free id has its samples dropped and counted (dropped()).

        A Channel(capacity=0) is treated as capacity 1 by the C++ mirror (Go's unbuffered rendezvous has no
        equivalent for a non-blocking sender; the reaper never blocks either way, metrics.go:570-573)."""
        self._lib = _load()
        err = C.create_string_buffer(512)
        if precision:
            self._h = self._lib.lhms_new_precision(max(int(interval_s * 1e9), 1), device, max_histograms, max_counters,
                                                   precision, err, 512)
        else:
            self._h = self._lib.lhms_new(max(int(interval_s * 1e9), 1), device, max_histograms, max_counters, err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._device = device
        self._device_gauges = {}   # name -> tensor: keeps the memory of every registered device gauge allocated
        self._device_dists = {}    # name -> tensor: likewise for distribution gauges

    def close(self):
        if self._h:
            self._lib.lhms_free(self._h)
            self._h = None
            self._device_gauges.clear()
            self._device_dists.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def SpecifyPercentiles(self, percentiles: dict):
        labels = (C.c_char_p * len(percentiles))(*[k.encode() for k in percentiles])
        ps = (C.c_double * len(percentiles))(*list(percentiles.values()))
        self._lib.lhms_specify_percentiles(self._h, len(percentiles), labels, ps)

    def Histogram(self, name: str, value: float):
        self._lib.lhms_histogram(self._h, name.encode(), float(value))

    def HistogramMany(self, name: str, values):
        import numpy as np
        values = np.ascontiguousarray(values, dtype=np.float64)
        self._lib.lhms_histogram_many(self._h, name.encode(), values.ctypes.data, values.size)

    def Counter(self, name: str, amount: int):
        self._lib.lhms_counter(self._h, name.encode(), int(amount))

    def StartTimer(self, name: str) -> TimerToken:
        return TimerToken(self._lib, self._lib.lhms_start_timer(self._h, name.encode()))

    def StartGpuTimer(self, name: str, stream=None) -> GpuTimerToken:
        """StartTimer for stream work: the start is a mark on the GPU's clock enqueued on `stream` (None = the
        engine's ingest stream, an int handle, or a torch.cuda.Stream; torch's default stream is timed as itself), and
        Stop() records the span on the device.  Does not fail when the timer pool is exhausted: that token's Stop
        drops the sample and counts it in dropped()."""
        h = _timer_stream(stream)
        st = C.c_int()
        tok = self._lib.lhms_gpu_timer_start(self._h, name.encode(), h, C.byref(st))
        if not tok:
            raise RuntimeError("lhms_gpu_timer_start failed (status %d)" % st.value)
        return GpuTimerToken(self, tok, h)

    @contextlib.contextmanager
    def gpu_timer(self, name: str, stream=None):
        """`with ms.gpu_timer(name, stream):` -- StartGpuTimer before the block, Stop() on the same stream after it:
        records the GPU time of the stream work enqueued in between, plus the launch latency of the two marks."""
        t = self.StartGpuTimer(name, stream)
        try:
            yield t
        finally:
            t.Stop()

    @contextlib.contextmanager
    def recording(self, stream=None, histograms=(), counters=()):
        """`with ms.recording(stream, histograms=[...], counters=[...]) as s:` -- a record scope whose names keep their
        ids until the interval it records into is collected.  Launch kernels that record with s.recorder under
        s.histogram_ids[name] / s.counter_ids[name] on `stream` (None = the engine's ingest stream, an int handle, or a
        torch.cuda.Stream) inside the block.  The collection of the interval waits for the block to end, so keep it
        short; collecting from inside it raises."""
        scope = RecordScope(self, stream, histograms, counters)
        try:
            yield scope
        finally:
            scope.end()

    @contextlib.contextmanager
    def graph_recorder(self, histograms=(), counters=()):
        """`with ms.graph_recorder(histograms=[...], counters=[...]) as g:` -- a recorder for kernels captured into CUDA
        graphs (GraphRecorder), closed on exit (on torch's current stream).  Create it outside the capture; inside, pass
        g.recorder to captured kernels with ids from g.histogram_ids / g.counter_ids, or capture g.histograms(...).
        Leave the block only once no replay that uses it is pending."""
        g = GraphRecorder(self, histograms, counters)
        try:
            yield g
        finally:
            g.close()

    def device_subscription(self, histograms=(), counters=()) -> DeviceSubscription:
        """SubscribeToProcessedMetrics for the GPU: every collection from now on (the reaper's included) publishes the
        processed metrics of these names into device memory, for kernels and captured graphs (DeviceSubscription).
        `with ms.device_subscription(histograms=[...], counters=[...]) as sub:` closes it on exit.  Create it outside
        any stream capture."""
        return DeviceSubscription(self, histograms, counters)

    def raw_device_subscription(self, histograms=(), window=1) -> RawDeviceSubscription:
        """SubscribeToRawMetrics for the GPU: every collection from now on (the reaper's included) publishes the bucket
        counts of these histogram names into device memory, where kernels, captured graphs and torch callers ask exact
        percentile and rank queries (RawDeviceSubscription).  `with ms.raw_device_subscription(histograms=[...]) as
        raw:` closes it on exit.  Create it outside any stream capture.  `window` (an int >= 1): every row answers for
        the sum of its name's histograms over the last `window` collections (TypeError / ValueError otherwise, before
        any call)."""
        return RawDeviceSubscription(self, histograms, window)

    def RegisterConstantGauge(self, name: str, value: float):
        self._lib.lhms_register_constant_gauge(self._h, name.encode(), float(value))
        self._device_gauges.pop(name, None)

    def RegisterDeviceGauge(self, name: str, tensor):
        """A gauge whose value lives on the GPU: `tensor` is a CUDA tensor (or a view such as t[i]) with exactly one
        element, on this system's device, of dtype float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64
        (TypeError otherwise).  Every collection reads all device gauges in one kernel that waits for no stream, and puts
        float64(value) in Gauges under `name`.  Replaces a gauge of either kind under that name.  The system keeps a
        reference to the tensor while it is registered, so its memory is not reused."""
        ptr, dtype = gauge_src(tensor, self._device)
        st = self._lib.lhms_register_device_gauge(self._h, name.encode(), ptr, dtype)
        if st != 0:
            raise (ValueError if st == _L.LH_ERR_INVALID else RuntimeError)(
                "lhms_register_device_gauge refused %r (status %d)" % (name, st))
        self._device_gauges[name] = tensor

    def DeregisterGaugeFunc(self, name: str):
        """Removes the gauge registered under `name`, a function or a device gauge (metrics.go:306)."""
        self._lib.lhms_deregister_gauge(self._h, name.encode())
        self._device_gauges.pop(name, None)

    def RegisterDeviceDistribution(self, name: str, tensor):
        """A distribution gauge: `tensor` is a contiguous CUDA tensor of any shape on this system's device, of dtype
        float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64 (TypeError otherwise).  At every collection
        each element x is recorded as Histogram(name, float64(x)) into the interval collected, read without waiting for
        any stream, so Histograms and the processed metrics carry the distribution of the tensor's current values.
        Replaces the tensor registered under `name`.  The system keeps a reference to the tensor while it is
        registered, so its memory is not reused.  Waits for a collection in progress; from a thread inside
        `ms.recording(...)` it raises RuntimeError instead, since that collection may be waiting for the scope."""
        src = array_src(tensor, self._device)
        st = self._lib.lhms_register_device_distribution(self._h, name.encode(), src.d_values, src.n, src.dtype)
        if st != 0:
            raise (ValueError if st == _L.LH_ERR_INVALID else RuntimeError)(
                "lhms_register_device_distribution refused %r (status %d)" % (name, st))
        self._device_dists[name] = tensor

    def DeregisterDeviceDistribution(self, name: str):
        """Stops recording the distribution gauge registered under `name` (nothing when there is none).  Waits for a
        collection in progress, so the tensor is not read after the call returns; from a thread inside
        `ms.recording(...)` it raises RuntimeError instead."""
        st = self._lib.lhms_deregister_device_distribution(self._h, name.encode())
        if st != 0:
            raise RuntimeError("lhms_deregister_device_distribution refused %r (status %d): the calling thread holds an "
                               "open record scope" % (name, st))
        self._device_dists.pop(name, None)

    def SubscribeToProcessedMetrics(self, capacity: int = 128) -> Subscription:
        return Subscription(self, "processed", capacity)

    def SubscribeToRawMetrics(self, capacity: int = 128) -> Subscription:
        return Subscription(self, "raw", capacity)

    def Start(self):
        self._lib.lhms_start(self._h)

    def Stop(self):
        self._lib.lhms_stop(self._h)

    def collect_and_process(self):
        """processMetrics(collectRawMetrics()) -> (raw dict, metrics dict), as metrics_test.go calls it."""
        col = _Collector()
        err = C.create_string_buffer(512)
        if self._lib.lhms_collect_and_process(self._h, col.cb, None, err, 512) != 0:
            raise RuntimeError(err.value.decode())
        return col.raw, col.metrics

    def processMetrics(self, raw: dict, aggregates: bool = False) -> dict:
        """processMetrics(raw) (metrics.go:483-506) for a raw dict of the shape collect_and_process returns
        ({"Counters", "Rates", "Histograms": {name: {key: count}}, "Gauges"}; missing parts are empty) -> metrics dict.
        Any set is accepted: hand-built, deserialised, the union of several systems' sets, or one collected here.
        aggregates=True also adds the _agg_avg / _agg_count / _agg_sum metrics the reaper adds (metrics.go:590-608)."""
        def named(d, ctype):
            keys = list(d)
            return len(keys), (C.c_char_p * len(keys))(*[k.encode() for k in keys]), (ctype * len(keys))(*d.values())

        nc, cn, cv = named(raw.get("Counters", {}), C.c_uint64)
        nr, rn, rv = named(raw.get("Rates", {}), C.c_uint64)
        ng, gn, gv = named(raw.get("Gauges", {}), C.c_double)
        hists = raw.get("Histograms", {})
        offsets, keys, counts = [0], [], []
        for m in hists.values():
            keys += [int(k) for k in m]
            counts += [int(c) for c in m.values()]
            offsets.append(len(keys))
        hn = (C.c_char_p * len(hists))(*[k.encode() for k in hists])
        col = _Collector()
        err = C.create_string_buffer(512)
        rc = self._lib.lhms_process_metrics(
            self._h, int(raw.get("Time", 0)), 1 if aggregates else 0, nc, cn, cv, nr, rn, rv, len(hists), hn,
            (C.c_uint32 * len(offsets))(*offsets), (C.c_int16 * len(keys))(*keys), (C.c_uint64 * len(counts))(*counts),
            ng, gn, gv, col.cb, None, err, 512)
        if rc != 0:
            raise RuntimeError(err.value.decode())
        return col.metrics

    def join_ranks(self, rank: int, world: int, allgather, allreduce=None):
        """Joins the systems of a multi-GPU job, so that each collection describes the whole job
        (MetricSystem::JoinRanks).  Collective: every rank calls it once, before its first collection, with
        allgather(bytes) -> list[bytes], every rank's bytes in rank order (loghisto_b200.distributed.rank_allgather builds
        one from a process group).  allgather runs on the collecting thread (the reaper's once Start()ed); an exception
        in it fails that collection's exchange on this rank, which then collects its own interval alone.

        Afterwards Histograms, Rates, Counters, the aggregates and device subscriptions are job-wide and identical on
        every rank; gauges stay rank-local.  ValueError for a bad rank / world, or when the ranks differ in
        max_histograms, max_counters or precision (raised on every rank alike); RuntimeError otherwise.

        With allreduce, the rows are summed through it instead of the peer-memory all-reduce, which needs every rank
        on one host (loghisto_b200.distributed.rank_allreduce builds one from a process group).  At each collection
        allreduce(send_ptr, recv_ptr, n_words, stream_ptr) gets plain ints: two device buffers of n_words uint64 and
        the CUDA stream the payload was packed on.  It must leave in recv the wrapping uint64 element-wise sum over
        ranks of send, enqueued on that stream or complete when it returns.  Every rank calls it with the same n_words,
        or none does.  An exception in it is logged once, and that collection gives this rank's own counts under the
        job-wide names (ranks_info()["status"] 4); the next one sums again.  Every rank must pass an allreduce or none
        (ValueError on every rank alike otherwise); TypeError when it is not callable."""
        rank, world = int(rank), int(world)
        if not callable(allgather):
            raise TypeError("allgather must be callable")
        if allreduce is not None and not callable(allreduce):
            raise TypeError("allreduce must be callable")
        if world < 2 or world > _L.LH_MAX_RANKS or not 0 <= rank < world:
            raise ValueError("join_ranks: need 2 <= world <= %d and 0 <= rank < world" % _L.LH_MAX_RANKS)

        logged = []

        def gather(_user, mine, n, sink, sink_ctx):
            try:
                parts = allgather(C.string_at(mine, n) if n else b"")
                if len(parts) != world:
                    raise ValueError("allgather returned %d parts for a world of %d" % (len(parts), world))
                for r, b in enumerate(parts):
                    b = bytes(b)
                    sink(sink_ctx, r, b, len(b))
                return 0
            except Exception as e:   # the collection goes on with this rank alone; say why, once
                if not logged:
                    logged.append(e)
                    sys.stderr.write("loghisto: rank %d: allgather raised %s: %s\n" % (rank, type(e).__name__, e))
                return 1

        cb = _RANKS_ALLGATHER(gather)
        err = C.create_string_buffer(512)
        if allreduce is None:
            rc = self._lib.lhms_ranks_join(self._h, rank, world, cb, None, err, 512)
        else:
            reduce_logged = []

            def reduce(_user, send, recv, n, stream):
                try:
                    allreduce(int(send or 0), int(recv or 0), int(n), int(stream or 0))
                    return 0
                except Exception as e:   # this collection keeps this rank's own counts; say why, once
                    if not reduce_logged:
                        reduce_logged.append(e)
                        sys.stderr.write("loghisto: rank %d: allreduce raised %s: %s\n" % (rank, type(e).__name__, e))
                    return 1
            rcb = _RANKS_ALLREDUCE(reduce)
            rc = self._lib.lhms_ranks_join_allreduce(self._h, rank, world, cb, rcb, None, err, 512)
            if rc == 0:
                self._ranks_reduce_cb = rcb
        if rc != 0:
            raise (ValueError if rc == -2 else RuntimeError)(err.value.decode())
        self._ranks_cb = cb   # called at every collection from now on

    def ranks_info(self) -> dict:
        """MetricSystem::RanksInfo: rank, world (0: not joined), status of the last collection (0 summed, 1 a peer did
        not arrive in time, 2 peers froze different buffers, 3 the exchange failed, 4 the allreduce passed to join_ranks
        raised), collections summed, bytes read from peers by the last all-reduce (8 x n_words through an allreduce),
        and names left out of the job-wide unions by the bounds."""
        out = (C.c_uint64 * 6)()
        self._lib.lhms_ranks_info(self._h, out)
        keys = ("rank", "world", "status", "summed", "bytes_from_peers", "names_dropped")
        return {k: int(v) for k, v in zip(keys, out)}

    def stats(self) -> dict:
        """lh_get_stats of the system's context, as Engine.stats."""
        st = _L.lh_stats()
        if self._lib.lhms_stats(self._h, C.byref(st)) != 0:
            raise RuntimeError("lhms_stats failed")
        return {f: int(getattr(st, f)) for f, _ in _L.lh_stats._fields_}

    def dropped(self) -> int:
        """Samples and counter ops not recorded so far: those of new names that found no free id (more distinct names
        in three consecutive intervals than max_histograms / max_counters), and those lost to a failed staging call."""
        return int(self._lib.lhms_dropped(self._h))

    def histogram_stream(self, names, kind: int, seed: int, start: int, n: int, threads: int) -> float:
        """Per-call load generator: `threads` OS threads call Histogram(names[id_i], value_i) once per sample for the
        samples [start, start + n) of synthetic stream `kind`; returns the seconds the calls took."""
        arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
        return float(self._lib.lhms_histogram_stream(self._h, arr, len(names), kind, seed, start, n, threads))

    def histogram_stream_timed(self, names, kind: int, seed: int, start: int, n: int, threads: int, dry: bool = False):
        """As histogram_stream; returns (wall seconds incl. the synthetic generator, largest per-thread seconds spent
        inside the Histogram() call loops alone).  dry=True runs the generator only."""
        arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
        calls = C.c_double()
        wall = self._lib.lhms_histogram_stream2(self._h, arr, len(names), kind, seed, start, n, threads, 1 if dry else 0, C.byref(calls))
        return float(wall), float(calls.value)


def timer_loop(name: str, threads: int, seconds: float, interval_s: float = 0.1, device: int = 0):
    """print_benchmark.go:59-67 as a measurement: returns (calls per second, total calls, sum of the <name>_count
    values every interval reported)."""
    total = C.c_uint64()
    rep = C.c_double()
    rate = _load().lhms_timer_loop(name.encode(), threads, seconds, int(interval_s * 1e9), device, C.byref(total), C.byref(rep))
    return float(rate), int(total.value), float(rep.value)


def PrintBenchmark(name: str, concurrency: int, seconds: float = 3.0, interval_s: float = 1.0, device: int = 0,
                   print_metrics: bool = False) -> float:
    """print_benchmark.go:49 with an empty op: `concurrency` threads loop StartTimer/Stop for `seconds`; returns the
    last interval's <name>_count (timer samples ingested per interval -- the figure readme.md:34 quotes)."""
    return float(_load().lhms_print_benchmark(name.encode(), concurrency, seconds, int(interval_s * 1e9), device,
                                              1 if print_metrics else 0))
