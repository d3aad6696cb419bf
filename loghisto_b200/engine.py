"""Thin object wrapper over the C ABI (include/loghisto_b200.h).

`Engine` is what the host-side MetricSystem mirror, the tests and bench.py
drive.  It adds no arithmetic of its own: every bucket, count and percentile
comes out of the CUDA kernels behind `lh_*`.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np

from . import _lib as L


class LhError(RuntimeError):
    def __init__(self, status: int, detail: str = ""):
        self.status = status
        msg = L.load().lh_strerror(status).decode()
        super().__init__(f"loghisto_b200: {msg} ({status})" + (f": {detail}" if detail else ""))


def _ptr(x) -> int:
    """Raw address of a device/host buffer: int, DeviceArray, torch tensor, numpy array or CAI object."""
    if x is None:
        return 0
    if isinstance(x, int):
        return x
    if isinstance(x, DeviceArray):
        return x.ptr
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return int(x.data_ptr())
    if hasattr(x, "__cuda_array_interface__"):
        return int(x.__cuda_array_interface__["data"][0])
    raise TypeError(f"cannot take the address of {type(x)!r}")


def _stream(s) -> int:
    if s is None:
        return 0
    if isinstance(s, int):
        return s
    if hasattr(s, "cuda_stream"):   # torch.cuda.Stream
        return int(s.cuda_stream)
    raise TypeError(f"not a stream: {type(s)!r}")


_BATCH_KINDS = {"float64": L.LH_VALUES_F64, "int64": L.LH_VALUES_I64NS}
_TYPESTRS = {t: np.dtype(t) for t in ("<f8", "<i8")}


def _device_array(x, what="batch arrays"):
    """(address, length, dtype name) of a CUDA torch tensor, a DeviceArray or an object with __cuda_array_interface__,
    contiguous ("" for a big-endian dtype).  TypeError otherwise; `what` names the array in the message."""
    if hasattr(x, "is_cuda") and hasattr(x, "data_ptr"):        # torch.Tensor
        if not x.is_cuda:
            raise TypeError(f"{what} must be in device memory, not a CPU tensor")
        if not x.is_contiguous():
            raise TypeError(f"{what} must be contiguous")
        dtype = str(x.dtype).replace("torch.", "")
        ptr, n = int(x.data_ptr()), int(x.numel())
    elif isinstance(x, DeviceArray):
        dtype, ptr, n = x.dtype.name, x.ptr, x.n
    elif hasattr(x, "__cuda_array_interface__"):
        cai = x.__cuda_array_interface__
        dt = _TYPESTRS.get(cai["typestr"]) or np.dtype(cai["typestr"])
        shape = cai["shape"]
        n = math.prod(shape)
        strides = cai.get("strides")
        if strides is not None and n > 1:
            want, step = [], dt.itemsize
            for d in reversed(shape):
                want.append(step)
                step *= d
            if tuple(strides) != tuple(reversed(want)):
                raise TypeError(f"{what} must be contiguous")
        dtype, ptr = dt.name if dt.byteorder in "=<|" else "", int(cai["data"][0])
    else:
        raise TypeError(f"not a device array: {type(x)!r}")
    return ptr, n, dtype


def _batch_array(x):
    """(address, length, LH_VALUES_* kind) of one device array of a batch: a CUDA torch tensor, a DeviceArray or an
    object with __cuda_array_interface__, contiguous, of dtype float64 or int64.  TypeError otherwise."""
    ptr, n, dtype = _device_array(x)
    if dtype not in _BATCH_KINDS:
        raise TypeError(f"batch arrays must be float64 (Histogram) or int64 (Timer nanoseconds), not {dtype or 'big-endian'}")
    return ptr, n, _BATCH_KINDS[dtype]


CUDA_STREAM_LEGACY = 1   # cudaStreamLegacy


def _timer_stream(s) -> int:
    """_stream for the GPU timers.  torch's default stream has cuda_stream == 0, which the C ABI reads as the context's
    ingest stream; a timer given that stream object must time torch's default stream, so it gets cudaStreamLegacy.
    None and plain ints keep their ABI meaning (None / 0 = the ingest stream)."""
    h = _stream(s)
    if h == 0 and s is not None and not isinstance(s, int):
        return CUDA_STREAM_LEGACY
    return h


class DeviceArray:
    """Device memory owned through lh_device_alloc; exposes __cuda_array_interface__."""

    def __init__(self, engine: "Engine", n: int, dtype):
        self.engine = engine
        self.dtype = np.dtype(dtype)
        self.n = int(n)
        self.nbytes = self.n * self.dtype.itemsize
        p = C.c_void_p()
        engine._check(engine.lib.lh_device_alloc(engine.h, max(self.nbytes, 1), C.byref(p)))
        self.ptr = int(p.value)

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.n,), "typestr": self.dtype.str, "data": (self.ptr, False), "version": 3}

    def offset(self, elems: int) -> int:
        return self.ptr + elems * self.dtype.itemsize

    def to_host(self) -> np.ndarray:
        out = np.empty(self.n, dtype=self.dtype)
        if self.nbytes:
            self.engine._check(self.engine.lib.lh_memcpy_d2h(self.engine.h, out.ctypes.data, self.ptr, self.nbytes))
        return out

    def free(self):
        if self.ptr and self.engine.h:
            self.engine.lib.lh_device_free(self.engine.h, self.ptr)
        self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PinnedArray:
    """Pinned host memory from lh_host_alloc_pinned, viewed as a numpy array."""

    def __init__(self, engine: "Engine", n: int, dtype):
        self.engine = engine
        self.dtype = np.dtype(dtype)
        self.n = int(n)
        self.nbytes = self.n * self.dtype.itemsize
        p = C.c_void_p()
        engine._check(engine.lib.lh_host_alloc_pinned(engine.h, max(self.nbytes, 1), C.byref(p)))
        self.ptr = int(p.value)
        buf = (C.c_char * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=self.n)

    def free(self):
        if self.ptr and self.engine.h:
            self.array = None
            self.engine.lib.lh_host_free_pinned(self.engine.h, self.ptr)
        self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


@dataclass
class Reduced:
    counts: np.ndarray   # uint64[H]
    sums: np.ndarray     # float64[H]
    avgs: np.ndarray     # float64[H]
    pkeys: np.ndarray    # int32[H, np]  (INT32_MIN = percentile() error)
    pvals: np.ndarray    # float64[H, np]


@dataclass
class Sparse:
    offsets: np.ndarray        # uint32[H+1]
    keys: np.ndarray           # int16[total]
    counts: np.ndarray         # uint64[total]
    counter_deltas: np.ndarray  # uint64[C]

    def histogram(self, hid: int) -> dict:
        a, b = int(self.offsets[hid]), int(self.offsets[hid + 1])
        return {int(k): int(c) for k, c in zip(self.keys[a:b], self.counts[a:b])}


def _capture_stream(s) -> int:
    """Stream of a graph recorder call: None = torch's current stream (inside torch.cuda.graph, the capturing stream;
    torch's default stream as itself) where torch has CUDA, else the context's ingest stream; otherwise as _timer_stream."""
    if s is None:
        try:
            import torch
        except ImportError:
            return 0
        if not torch.cuda.is_available():
            return 0
        s = torch.cuda.current_stream()
    return _timer_stream(s)


def _batch_items(items, limit_name: str):
    """lh_batch_item array of (id, array) pairs; TypeError / ValueError before any call."""
    items = list(items)
    arr = (L.lh_batch_item * max(len(items), 1))()
    for i, (hid, a) in enumerate(items):
        ptr, n, kind = _batch_array(a)
        if not 0 <= int(hid) < 1 << 32:
            raise ValueError(f"{limit_name} {hid} is not a uint32")
        arr[i] = L.lh_batch_item(ptr, n, int(hid), kind)
    return arr, len(items)


_ID_BYTES = {"uint16": 2, "int32": 4, "uint32": 4}   # a negative int32 id reads as a large uint32: dropped and counted


def graph_keyed_args(ids, values):
    """(id bytes, ids address, values address, LH_VALUES_* kind, n) of keyed samples for a graph recorder: ids uint16,
    int32 or uint32, values float64 or int64 (as batch arrays), of one length.  TypeError / ValueError otherwise."""
    ip, n, idt = _device_array(ids, "ids")
    if idt not in _ID_BYTES:
        raise TypeError(f"ids must be uint16, int32 or uint32, not {idt or 'big-endian'}")
    vp, nv, kind = _batch_array(values)
    if nv != n:
        raise ValueError(f"{n} ids but {nv} values")
    return _ID_BYTES[idt], ip, vp, kind, n


def graph_counter_args(ids, amounts):
    """(id bytes, ids address, amounts address, n) of counter adds for a graph recorder: ids as graph_keyed_args takes
    them, amounts int64 or uint64 (added as uint64 bits), of one length.  TypeError / ValueError otherwise."""
    ip, n, idt = _device_array(ids, "ids")
    if idt not in _ID_BYTES:
        raise TypeError(f"ids must be uint16, int32 or uint32, not {idt or 'big-endian'}")
    ap, na, adt = _device_array(amounts, "amounts")
    if adt not in ("int64", "uint64"):
        raise TypeError(f"amounts must be int64 or uint64, not {adt or 'big-endian'}")
    if na != n:
        raise ValueError(f"{n} ids but {na} amounts")
    return _ID_BYTES[idt], ip, ap, n


def graph_duration_out(out) -> int:
    """Address of the int64 a graph recorder's timer stop writes its duration to (None = 0: not written)."""
    if out is None:
        return 0
    ptr, n, dtype = _device_array(out, "out")
    if dtype != "int64" or n < 1:
        raise TypeError("out must be a device array of at least one int64")
    return ptr


def _ids(ids):
    ids = [int(x) for x in ids]
    return (C.c_uint32 * max(len(ids), 1))(*ids), len(ids)


class GraphRecorder:
    """A graph recorder of an Engine (Engine.graph_recorder): `recorder` is the lh_recorder to pass by value to kernels
    captured into CUDA graphs, recording under local ids 0 .. len(hist_ids) - 1 (counters 0 .. len(counter_ids) - 1)."""

    def __init__(self, engine: "Engine", hist_ids, counter_ids):
        self._eng = engine
        self.g = L.lh_graph_recorder()
        h, k = _ids(hist_ids)
        c, kc = _ids(counter_ids)
        engine._check(engine.lib.lh_graph_recorder_create(engine.h, k, kc, h, c, C.byref(self.g)))
        self.recorder = self.g.rec
        self._open = True

    def bind(self, hist_ids=None, counter_ids=None):
        """Target ids from the next snapshot_begin on (None = unchanged)."""
        h = _ids(hist_ids)[0] if hist_ids is not None else None
        c = _ids(counter_ids)[0] if counter_ids is not None else None
        self._eng._check(self._eng.lib.lh_graph_recorder_bind(self._eng.h, C.byref(self.g), h, c))

    def ingest(self, items, stream=None):
        """lh_graph_recorder_ingest of (local id, array) pairs, arrays as Engine.ingest_batch takes them, on `stream`
        (None = torch's current stream, so that it is captured inside torch.cuda.graph)."""
        arr, n = _batch_items(items, "local histogram id")
        self._eng._check(self._eng.lib.lh_graph_recorder_ingest(self._eng.h, C.byref(self.g), arr, n, _capture_stream(stream)))

    def ingest_arrays(self, items, stream=None):
        """lh_graph_recorder_ingest_arrays of (local id, tensor) pairs, tensors as Engine.ingest_arrays takes them, on
        `stream` (None = torch's current stream, so that it is captured inside torch.cuda.graph)."""
        arr, n = array_items(items, self._eng.device, "local histogram id")
        self._eng._check(self._eng.lib.lh_graph_recorder_ingest_arrays(self._eng.h, C.byref(self.g), arr, n,
                                                                       _capture_stream(stream)))

    def keyed(self, ids, values, stream=None):
        """lh_graph_recorder_ingest_keyed_u16 / _u32: values[i] into local histogram ids[i], on `stream` (None =
        torch's current stream).  ids uint16 (_u16), int32 or uint32 (_u32); values float64 or int64 nanoseconds."""
        id_bytes, ip, vp, kind, n = graph_keyed_args(ids, values)
        fn = self._eng.lib.lh_graph_recorder_ingest_keyed_u16 if id_bytes == 2 else self._eng.lib.lh_graph_recorder_ingest_keyed_u32
        self._eng._check(fn(self._eng.h, C.byref(self.g), ip, vp, kind, n, _capture_stream(stream)))

    def counters(self, ids, amounts, stream=None):
        """lh_graph_recorder_counter_add_u16 / _u32: amounts[i] into local counter ids[i] (wrapping uint64)."""
        id_bytes, ip, ap, n = graph_counter_args(ids, amounts)
        fn = self._eng.lib.lh_graph_recorder_counter_add_u16 if id_bytes == 2 else self._eng.lib.lh_graph_recorder_counter_add_u32
        self._eng._check(fn(self._eng.h, C.byref(self.g), ip, ap, n, _capture_stream(stream)))

    def start_timer(self, histogram: int, stream=None):
        """lh_graph_recorder_timer_start: mark the start of a span of local histogram `histogram` on `stream`."""
        self._eng._check(self._eng.lib.lh_graph_recorder_timer_start(self._eng.h, C.byref(self.g), int(histogram),
                                                                     _capture_stream(stream)))

    def stop_timer(self, histogram: int, stream=None, out=None):
        """lh_graph_recorder_timer_stop: record now - start into local histogram `histogram`; `out` (an int64 device
        array) also receives the duration in ns."""
        ptr = graph_duration_out(out)
        self._eng._check(self._eng.lib.lh_graph_recorder_timer_stop(self._eng.h, C.byref(self.g), int(histogram),
                                                                    _capture_stream(stream), ptr))

    @contextlib.contextmanager
    def timer(self, histogram: int, stream=None):
        """`with g.timer(h):` -- start_timer before the block and stop_timer after it, on one stream."""
        self.start_timer(histogram, stream)
        yield
        self.stop_timer(histogram, stream)

    def close(self, stream=None):
        """Final drain into the current interval on `stream` (None = torch's current stream), then the rows are freed."""
        if self._open:
            self._open = False
            self._eng._check(self._eng.lib.lh_graph_recorder_destroy(self._eng.h, C.byref(self.g), _capture_stream(stream)))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


_BOARD_HDR_WORDS = C.sizeof(L.lh_board_header) // 8        # 36
_BOARD_ROW_WORDS = C.sizeof(L.lh_board_hist_row) // 8      # 52
_BOARD_CTR_WORDS = C.sizeof(L.lh_board_counter_row) // 8   # 3


def board_out(out, nbytes: int, device: int):
    """The uint8 CUDA tensor a board image is read into: `out` checked (contiguous uint8 on the device, at least
    `nbytes` long, 8-byte aligned), or a new one when out is None."""
    import torch
    if out is None:
        return torch.empty(nbytes, dtype=torch.uint8, device=torch.device("cuda", device))
    if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= nbytes
            and out.data_ptr() % 8 == 0):
        raise TypeError("out must be a contiguous 8-byte aligned uint8 CUDA tensor of at least %d bytes" % nbytes)
    return out


def board_views(buf, k: int, kc: int) -> dict:
    """Torch views of the board image in `buf` (layout of include/loghisto_b200.h), no copy and no synchronisation:
      collection       int64 [], the publish number of the image (0: nothing published yet)
      np               int32 [], percentiles of that publish
      percentiles      float64 [LH_MAX_PERCENTILES], NaN from np on
      present          int32 [k]; count int64 [k] (the uint64 bits); sum, avg float64 [k]
      pvals            float64 [k, LH_MAX_PERCENTILES]; pkeys int32 [k, LH_MAX_PERCENTILES] (INT32_MIN = label omitted)
      counter_present  int32 [kc]; rate, total int64 [kc] (the uint64 bits)
    Percentile columns j >= np hold NaN / INT32_MIN."""
    import torch
    nbytes = (_BOARD_HDR_WORDS + _BOARD_ROW_WORDS * k + _BOARD_CTR_WORDS * kc) * 8
    w64 = buf[:nbytes].view(torch.int64)
    f64 = buf[:nbytes].view(torch.float64)
    i32 = buf[:nbytes].view(torch.int32)
    b8, b4 = w64.storage_offset(), i32.storage_offset()
    h, rw, cb = _BOARD_HDR_WORDS, _BOARD_ROW_WORDS, _BOARD_HDR_WORDS + _BOARD_ROW_WORDS * k
    P = L.LH_MAX_PERCENTILES
    return {
        "image": buf[:nbytes],
        "collection": w64.as_strided((), (), b8 + 1),
        "np": i32.as_strided((), (), b4 + 4),
        "percentiles": f64.as_strided((P,), (1,), b8 + 4),
        "count": w64.as_strided((k,), (rw,), b8 + h),
        "sum": f64.as_strided((k,), (rw,), b8 + h + 1),
        "avg": f64.as_strided((k,), (rw,), b8 + h + 2),
        "present": i32.as_strided((k,), (2 * rw,), b4 + 2 * h + 6),
        "pvals": f64.as_strided((k, P), (rw, 1), b8 + h + 4),
        "pkeys": i32.as_strided((k, P), (2 * rw, 1), b4 + 2 * h + 72),
        "rate": w64.as_strided((kc,), (_BOARD_CTR_WORDS,), b8 + cb),
        "total": w64.as_strided((kc,), (_BOARD_CTR_WORDS,), b8 + cb + 1),
        "counter_present": i32.as_strided((kc,), (2 * _BOARD_CTR_WORDS,), b4 + 2 * cb + 4),
    }


_GAUGE_DTYPES = {"torch.float64": L.LH_GAUGE_F64, "torch.float32": L.LH_GAUGE_F32, "torch.float16": L.LH_GAUGE_F16,
                 "torch.bfloat16": L.LH_GAUGE_BF16, "torch.int64": L.LH_GAUGE_I64, "torch.int32": L.LH_GAUGE_I32,
                 "torch.uint64": L.LH_GAUGE_U64}


def gauge_src(t, device: int) -> tuple:
    """(address, LH_GAUGE_* dtype) of a device gauge: a CUDA tensor (or a view such as t[i]) with exactly one element,
    on `device`, of dtype float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64.  TypeError otherwise."""
    if not (hasattr(t, "is_cuda") and hasattr(t, "data_ptr")):
        raise TypeError(f"a device gauge is a CUDA tensor, not {type(t)!r}")
    if not t.is_cuda or t.device.index != device:
        raise TypeError(f"a device gauge must be on cuda:{device}, not {t.device}")
    if t.numel() != 1:
        raise TypeError(f"a device gauge has exactly one element, not {t.numel()}")
    dtype = _GAUGE_DTYPES.get(str(t.dtype))
    if dtype is None:
        raise TypeError(f"a device gauge must be float64/32/16, bfloat16, int64/32 or uint64, not {t.dtype}")
    return int(t.data_ptr()), dtype


def array_src(t, device: int, histogram_id: int = 0, what: str = "a distribution gauge") -> L.lh_array_src:
    """lh_array_src of a distribution gauge (or of an lh_ingest_arrays item; `what` names it in messages): a contiguous
    CUDA tensor of any shape on `device`, of dtype float64 / float32 / float16 / bfloat16 / int64 / int32 / uint64,
    recorded under `histogram_id`.  TypeError otherwise."""
    if not (hasattr(t, "is_cuda") and hasattr(t, "data_ptr")):
        raise TypeError(f"{what} is a CUDA tensor, not {type(t)!r}")
    if not t.is_cuda or t.device.index != device:
        raise TypeError(f"{what} must be on cuda:{device}, not {t.device}")
    if not t.is_contiguous():
        raise TypeError(f"{what} must be a contiguous tensor")
    dtype = _GAUGE_DTYPES.get(str(t.dtype))
    if dtype is None:
        raise TypeError(f"{what} must be float64/32/16, bfloat16, int64/32 or uint64, not {t.dtype}")
    return L.lh_array_src(int(t.data_ptr()), int(t.numel()), dtype, int(histogram_id))


def array_items(items, device: int, limit_name: str):
    """lh_array_src array of (id, tensor) pairs for lh_ingest_arrays / lh_graph_recorder_ingest_arrays, each tensor as
    array_src takes it; TypeError / ValueError before any call."""
    items = list(items)
    arr = (L.lh_array_src * max(len(items), 1))()
    for i, (hid, t) in enumerate(items):
        if not 0 <= int(hid) < 1 << 32:
            raise ValueError(f"{limit_name} {hid} is not a uint32")
        arr[i] = array_src(t, device, int(hid), "an ingested array")
    return arr, len(items)


class Board:
    """A device subscription board of an Engine (Engine.board): `board` is the lh_board to pass by value to kernels,
    which read it with lh::read_histogram / lh::read_counter."""

    def __init__(self, engine: "Engine", k: int, kc: int):
        self._eng = engine
        self.board = L.lh_board()
        engine._check(engine.lib.lh_board_create(engine.h, int(k), int(kc), C.byref(self.board)))
        self.k, self.kc = int(k), int(kc)
        self._open = True

    def publish(self, hist_ids=None, counter_ids=None, totals=None):
        """lh_snapshot_publish: row i from the open snapshot's latest reduction for hist_ids[i] / counter_ids[i]
        (None = every row unbound; L.LH_GRAPH_UNBOUND = that row), with counter totals `totals` (None = 0)."""
        h = _ids(hist_ids)[0] if hist_ids is not None else None
        c = _ids(counter_ids)[0] if counter_ids is not None else None
        t = (C.c_uint64 * max(len(totals), 1))(*[int(x) for x in totals]) if totals is not None else None
        self._eng._check(self._eng.lib.lh_snapshot_publish(self._eng.h, C.byref(self.board), h, c, t))

    def read(self, out=None, stream=None) -> dict:
        """lh_board_read into `out` (None = a new uint8 CUDA tensor) on `stream` (None = torch's current stream, so
        that it is captured inside torch.cuda.graph); returns board_views of it.  Nothing is synchronised."""
        buf = board_out(out, self.board.bytes, self._eng.device)
        self._eng._check(self._eng.lib.lh_board_read(self._eng.h, C.byref(self.board), buf.data_ptr(), _capture_stream(stream)))
        return board_views(buf, self.k, self.kc)

    def close(self):
        """lh_board_destroy (stream-ordered after every publish issued); no read of the board may be pending."""
        if self._open:
            self._open = False
            self._eng._check(self._eng.lib.lh_board_destroy(self._eng.h, C.byref(self.board)))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def _raw_input(x, what: str, device: int):
    """(address, length) of the query inputs of a raw board: a contiguous 1-D float64 CUDA tensor on `device`.
    TypeError otherwise, before anything is issued."""
    import torch
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float64 and x.dim() == 1
            and x.is_contiguous() and x.device.index == device):
        raise TypeError(f"{what} must be a contiguous 1-D float64 CUDA tensor on cuda:{device}")
    return x.data_ptr(), x.numel()


def raw_percentiles(call, k: int, ps, device: int, stream):
    """Every row of a raw board for each p of `ps` (a float64 CUDA tensor of length m), through `call` (the
    lh_raw_percentiles_grid form: d_ps, m, d_keys, d_vals, d_publish, stream): returns keys int32 [k, m], values
    float64 [k, m] and publish numbers int64 [k, m].  One kernel on `stream` (None = torch's current stream), no
    synchronisation: the tensors hold the answers once the stream has run it."""
    import torch
    ptr, m = _raw_input(ps, "ps", device)
    dev = torch.device("cuda", device)
    keys = torch.empty((k, m), dtype=torch.int32, device=dev)
    vals = torch.empty((k, m), dtype=torch.float64, device=dev)
    pub = torch.empty((k, m), dtype=torch.int64, device=dev)
    if m:
        call(ptr, m, keys.data_ptr(), vals.data_ptr(), pub.data_ptr(), _capture_stream(stream))
    return keys, vals, pub


def raw_ranks(call, k: int, values, device: int, stream):
    """Every row of a raw board for each value of `values` (a float64 CUDA tensor of length m), through `call` (the
    lh_raw_ranks_grid form): returns ranks int64 [k, m] (samples at or below each value's bucket), totals int64 [k]
    (row r's total in the publish its query (r, 0) read) and publish numbers int64 [k, m].  Counts are the uint64 bits.
    As raw_percentiles: one kernel, no synchronisation."""
    import torch
    ptr, m = _raw_input(values, "values", device)
    dev = torch.device("cuda", device)
    ranks = torch.empty((k, m), dtype=torch.int64, device=dev)
    pub = torch.empty((k, m), dtype=torch.int64, device=dev)
    if not m:
        return ranks, torch.zeros(k, dtype=torch.int64, device=dev), pub
    totals = torch.empty(k, dtype=torch.int64, device=dev)
    call(ptr, m, ranks.data_ptr(), totals.data_ptr(), pub.data_ptr(), _capture_stream(stream))
    return ranks, totals, pub


def check_window(window) -> int:
    """A raw board's window: an int >= 1 (TypeError / ValueError otherwise)."""
    import numbers
    if isinstance(window, bool) or not isinstance(window, numbers.Integral):
        raise TypeError(f"window must be an int >= 1, not {type(window).__name__}")
    if window < 1:
        raise ValueError(f"window must be >= 1, not {window}")
    return int(window)


class RawBoard:
    """A raw device subscription board of an Engine (Engine.raw_board): `board` is the lh_raw_board to pass by value to
    kernels, which query it with lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count.  With `window` w > 1
    (lh_raw_board_create_window) each row answers for the sum of its last w publishes."""

    def __init__(self, engine: "Engine", k: int, window: int = 1):
        window = check_window(window)
        self._eng = engine
        self.board = L.lh_raw_board()
        if window == 1:
            engine._check(engine.lib.lh_raw_board_create(engine.h, int(k), C.byref(self.board)))
        else:
            engine._check(engine.lib.lh_raw_board_create_window(engine.h, int(k), window, C.byref(self.board)))
        self.k = int(k)
        self.window = window
        self._open = True

    def publish(self, hist_ids=None):
        """lh_snapshot_publish_raw: row i from histogram hist_ids[i] of the open snapshot (None = every row unbound;
        L.LH_GRAPH_UNBOUND = that row)."""
        h = _ids(hist_ids)[0] if hist_ids is not None else None
        self._eng._check(self._eng.lib.lh_snapshot_publish_raw(self._eng.h, C.byref(self.board), h))

    def _pairs(self, fn, rows, x, what, out_dtypes, stream):
        import torch
        ptr, n = _raw_input(x, what, self._eng.device)
        if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype in (torch.int32, torch.uint32)
                and rows.dim() == 1 and rows.is_contiguous() and rows.device.index == self._eng.device):
            raise TypeError(f"rows must be a contiguous 1-D int32 or uint32 CUDA tensor on cuda:{self._eng.device}")
        if rows.numel() != n:
            raise ValueError(f"{rows.numel()} rows but {n} {what}")
        outs = [torch.empty(n, dtype=dt, device=rows.device) for dt in out_dtypes]
        self._eng._check(fn(self._eng.h, C.byref(self.board), rows.data_ptr(), ptr, n,
                            *[o.data_ptr() for o in outs], _capture_stream(stream)))
        return tuple(outs)

    def percentiles(self, ps, rows=None, stream=None):
        """rows None: lh_raw_percentiles_grid, (keys, values, publish) [k, m] for every row and each p of `ps`.
        Otherwise lh_raw_percentiles, one query (rows[i], ps[i]) each: (keys, values, publish) [n]."""
        import torch
        lib, h = self._eng.lib, self._eng.h
        if rows is not None:
            return self._pairs(lib.lh_raw_percentiles, rows, ps, "ps", (torch.int32, torch.float64, torch.int64), stream)
        return raw_percentiles(lambda *a: self._eng._check(lib.lh_raw_percentiles_grid(h, C.byref(self.board), *a)),
                               self.k, ps, self._eng.device, stream)

    def ranks(self, values, rows=None, stream=None):
        """rows None: lh_raw_ranks_grid, (ranks [k, m], totals [k], publish [k, m]).  Otherwise lh_raw_ranks, one query
        (rows[i], values[i]) each: (ranks, totals, publish) [n]."""
        import torch
        lib, h = self._eng.lib, self._eng.h
        if rows is not None:
            return self._pairs(lib.lh_raw_ranks, rows, values, "values", (torch.int64, torch.int64, torch.int64), stream)
        return raw_ranks(lambda *a: self._eng._check(lib.lh_raw_ranks_grid(h, C.byref(self.board), *a)),
                         self.k, values, self._eng.device, stream)

    def close(self):
        """lh_raw_board_destroy (stream-ordered after every publish issued); no query of the board may be pending."""
        if self._open:
            self._open = False
            self._eng._check(self._eng.lib.lh_raw_board_destroy(self._eng.h, C.byref(self.board)))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Engine:
    def __init__(self, device: int = 0, max_histograms: int = 1, max_counters: int = 1,
                 staging_bytes: int = 0, staging_slots: int = 0, precision: int = 0):
        self.lib = L.load()
        self.h = None
        cfg = L.lh_config(C.sizeof(L.lh_config), device, max_histograms, max_counters,
                          staging_bytes, staging_slots, 0, precision)
        h = C.c_void_p()
        st = self.lib.lh_create(C.byref(cfg), C.byref(h))
        if st != L.LH_OK:
            raise LhError(st, "lh_create")
        self.h = h
        self.device = device
        self.H = max_histograms
        self.C = max_counters

    # ---- plumbing
    def _check(self, st: int):
        if st != L.LH_OK:
            raise LhError(st, self.lib.lh_last_error(self.h).decode() if self.h else "")

    def close(self):
        if self.h:
            self.lib.lh_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def alloc(self, n: int, dtype) -> DeviceArray:
        return DeviceArray(self, n, dtype)

    def pinned(self, n: int, dtype) -> PinnedArray:
        return PinnedArray(self, n, dtype)

    def upload(self, arr: np.ndarray) -> DeviceArray:
        arr = np.ascontiguousarray(arr)
        d = DeviceArray(self, arr.size, arr.dtype)
        if arr.nbytes:
            self._check(self.lib.lh_memcpy_h2d(self.h, d.ptr, arr.ctypes.data, arr.nbytes))
        return d

    def sync(self):
        self._check(self.lib.lh_sync(self.h))

    @property
    def ingest_stream(self) -> int:
        return int(self.lib.lh_ingest_stream(self.h) or 0)

    def tune(self, key: str, value: int):
        self._check(self.lib.lh_tune(self.h, key.encode(), int(value)))

    def k1_variants(self) -> list:
        return [self.lib.lh_k1_variant_name(self.h, i).decode() for i in range(self.lib.lh_k1_variant_count())]

    def k1_variant_name(self) -> str:
        return self.lib.lh_k1_variant_name(self.h, self.lib.lh_k1_variant_current(self.h)).decode()

    def keyed_kernel_name(self) -> str:
        """Name of the kernel the most recent keyed ingest dispatched to."""
        return self.lib.lh_keyed_kernel_name(self.h).decode()

    # ---- multi-GPU (peer-memory all-reduce behind the ABI)
    def comm_export(self) -> bytes:
        buf = C.create_string_buffer(L.LH_PEER_HANDLE_BYTES)
        self._check(self.lib.lh_comm_export(self.h, buf))
        return buf.raw

    def comm_import(self, rank: int, world: int, handles: bytes):
        assert len(handles) == world * L.LH_PEER_HANDLE_BYTES
        self._check(self.lib.lh_comm_import(self.h, rank, world, C.c_char_p(handles)))

    def snapshot_allreduce(self, counters: bool = False) -> int:
        seq = C.c_uint64()
        self._check(self.lib.lh_snapshot_allreduce(self.h, 1 if counters else 0, C.byref(seq)))
        return int(seq.value)

    def snapshot_rows(self):
        """lh_snapshot_rows: (touched uint8[H], counter deltas uint64[C], frozen half) of the frozen interval."""
        touched = np.zeros(self.H, np.uint8)
        deltas = np.zeros(self.C, np.uint64)
        frozen = C.c_uint32()
        self._check(self.lib.lh_snapshot_rows(self.h, touched.ctypes.data, deltas.ctypes.data, C.byref(frozen)))
        return touched, deltas, int(frozen.value)

    def snapshot_allreduce_rows(self, seq: int, frozen, hist_map, counter_map) -> int:
        """lh_snapshot_allreduce_rows: hist_map / counter_map are [world][rows] arrays of frozen rows (LH_ROW_ABSENT for
        none), frozen[r] the buffer rank r froze."""
        fr = np.ascontiguousarray(frozen, dtype=np.uint32)
        hm = np.ascontiguousarray(hist_map, dtype=np.uint32)
        cm = np.ascontiguousarray(counter_map, dtype=np.uint32)
        n_rows = hm.shape[1] if hm.ndim == 2 else 0
        n_counter_rows = cm.shape[1] if cm.ndim == 2 else 0
        out = C.c_uint64()
        self._check(self.lib.lh_snapshot_allreduce_rows(self.h, seq, fr.ctypes.data, n_rows, hm.ctypes.data if n_rows else None,
                                                        n_counter_rows, cm.ctypes.data if n_counter_rows else None,
                                                        C.byref(out)))
        return int(out.value)

    def snapshot_row_levels(self):
        """lh_snapshot_row_levels: uint8[H] levels of the frozen rows (0 no data, 1 window only, 3 beyond the window)."""
        levels = np.zeros(self.H, np.uint8)
        self._check(self.lib.lh_snapshot_row_levels(self.h, levels.ctypes.data))
        return levels

    def snapshot_pack_rows(self, hist_rows, levels, counter_rows):
        """lh_snapshot_pack_rows: this rank's column of the maps (LH_ROW_ABSENT for none) and the agreed levels.
        Returns (send_ptr, recv_ptr, n_words, stream_ptr); the payload is enqueued on that stream."""
        hr = np.ascontiguousarray(hist_rows, dtype=np.uint32)
        lv = np.ascontiguousarray(levels, dtype=np.uint8)
        cr = np.ascontiguousarray(counter_rows, dtype=np.uint32)
        if lv.size != hr.size:
            raise ValueError("levels must have one entry per histogram row")
        send, recv, stream, n = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._check(self.lib.lh_snapshot_pack_rows(self.h, hr.size, hr.ctypes.data if hr.size else None,
                                                   lv.ctypes.data if lv.size else None, cr.size,
                                                   cr.ctypes.data if cr.size else None, C.byref(send), C.byref(recv),
                                                   C.byref(n), C.byref(stream)))
        return int(send.value or 0), int(recv.value or 0), int(n.value), int(stream.value or 0)

    def snapshot_unpack_rows(self, summed: bool):
        """lh_snapshot_unpack_rows: the payload's sums (summed) or this rank's own counts into the reduced arrays."""
        self._check(self.lib.lh_snapshot_unpack_rows(self.h, 1 if summed else 0))

    def comm_allreduce_ms(self, seq: int) -> float:
        ms = C.c_float()
        self._check(self.lib.lh_comm_allreduce_ms(self.h, seq, C.byref(ms)))
        return float(ms.value)

    def comm_info(self) -> dict:
        st = L.lh_comm_stats()
        self._check(self.lib.lh_comm_info(self.h, C.byref(st)))
        return {f: int(getattr(st, f)) for f, _ in L.lh_comm_stats._fields_ if f != "reserved"}

    def comm_last_bytes(self) -> int:
        return self.comm_info()["last_bytes_from_peers"]

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        self._check(self.lib.lh_last_kernel_ms(self.h, C.byref(ms)))
        return float(ms.value)

    def ingest_seq(self) -> int:
        return int(self.lib.lh_ingest_seq(self.h))

    def kernel_ms(self, seq: int) -> float:
        ms = C.c_float()
        self._check(self.lib.lh_kernel_ms(self.h, seq, C.byref(ms)))
        return float(ms.value)

    def stats(self) -> dict:
        s = L.lh_stats()
        self._check(self.lib.lh_get_stats(self.h, C.byref(s)))
        return {f: int(getattr(s, f)) for f, _ in L.lh_stats._fields_}

    # ---- ingest, device inputs
    def ingest_f64(self, histogram_id: int, d_values, n: int, stream=None):
        self._check(self.lib.lh_ingest_f64(self.h, histogram_id, _ptr(d_values), n, _stream(stream)))

    def ingest_keyed_f64_u16(self, d_ids, d_values, n: int, stream=None):
        self._check(self.lib.lh_ingest_keyed_f64_u16(self.h, _ptr(d_ids), _ptr(d_values), n, _stream(stream)))

    def ingest_keyed_f64_u32(self, d_ids, d_values, n: int, stream=None):
        self._check(self.lib.lh_ingest_keyed_f64_u32(self.h, _ptr(d_ids), _ptr(d_values), n, _stream(stream)))

    def ingest_keyed_i64ns_u16(self, d_ids, d_nanos, n: int, stream=None):
        self._check(self.lib.lh_ingest_keyed_i64ns_u16(self.h, _ptr(d_ids), _ptr(d_nanos), n, _stream(stream)))

    def ingest_keyed_pair_u16(self, d_ids_f64, d_values, n_f64: int, d_ids_ns, d_nanos, n_ns: int, stream=None):
        """Histogram samples and Timer samples of one batch in one call (one launch of the write-combining kernel)."""
        self._check(self.lib.lh_ingest_keyed_pair_u16(self.h, _ptr(d_ids_f64), _ptr(d_values), n_f64, _ptr(d_ids_ns), _ptr(d_nanos), n_ns,
                                                      _stream(stream)))

    def ingest_batch(self, items, stream=None):
        """Many device arrays, each under its own histogram id, in one call (lh_ingest_batch): `items` is a list of
        (histogram id, array) pairs; the array is a CUDA torch tensor, a DeviceArray or a __cuda_array_interface__
        object, contiguous, float64 (Histogram samples) or int64 (Timer nanoseconds).  TypeError before the call for
        anything else."""
        arr, n = _batch_items(items, "histogram id")
        self._check(self.lib.lh_ingest_batch(self.h, arr, n, _stream(stream)))

    def ingest_arrays(self, items, stream=None):
        """Many device arrays of any gauge dtype, each under its own histogram id, in one call (lh_ingest_arrays):
        `items` is a list of (histogram id, tensor) pairs, each tensor contiguous, on this engine's device, float64 /
        float32 / float16 / bfloat16 / int64 / int32 / uint64, every element x recorded as float64(x).  TypeError or
        ValueError before the call for anything else."""
        arr, n = array_items(items, self.device, "histogram id")
        self._check(self.lib.lh_ingest_arrays(self.h, arr, n, _stream(stream)))

    def counter_add_u16(self, d_ids, d_amounts, n: int, stream=None):
        self._check(self.lib.lh_counter_add_u16(self.h, _ptr(d_ids), _ptr(d_amounts), n, _stream(stream)))

    def counter_add_u32(self, d_ids, d_amounts, n: int, stream=None):
        self._check(self.lib.lh_counter_add_u32(self.h, _ptr(d_ids), _ptr(d_amounts), n, _stream(stream)))

    def ingest_keyed_mapped_u16(self, h_map, d_ids, d_values, kind: int, n: int, stream=None):
        """lh_ingest_keyed_mapped_u16: local id l < len(h_map) is histogram h_map[l] (a list of ids)."""
        m, k = _ids(h_map)
        self._check(self.lib.lh_ingest_keyed_mapped_u16(self.h, m, k, _ptr(d_ids), _ptr(d_values), kind, n, _stream(stream)))

    def ingest_keyed_mapped_u32(self, h_map, d_ids, d_values, kind: int, n: int, stream=None):
        m, k = _ids(h_map)
        self._check(self.lib.lh_ingest_keyed_mapped_u32(self.h, m, k, _ptr(d_ids), _ptr(d_values), kind, n, _stream(stream)))

    def counter_add_mapped_u16(self, h_map, d_ids, d_amounts, n: int, stream=None):
        """lh_counter_add_mapped_u16: local id l < len(h_map) is counter h_map[l]."""
        m, k = _ids(h_map)
        self._check(self.lib.lh_counter_add_mapped_u16(self.h, m, k, _ptr(d_ids), _ptr(d_amounts), n, _stream(stream)))

    def counter_add_mapped_u32(self, h_map, d_ids, d_amounts, n: int, stream=None):
        m, k = _ids(h_map)
        self._check(self.lib.lh_counter_add_mapped_u32(self.h, m, k, _ptr(d_ids), _ptr(d_amounts), n, _stream(stream)))

    # ---- ingest, host inputs
    def ingest_f64_host(self, histogram_id: int, h_values, n: int | None = None):
        if isinstance(h_values, np.ndarray):
            assert h_values.dtype == np.float64 and h_values.flags.c_contiguous
            n = h_values.size if n is None else n
        self._check(self.lib.lh_ingest_f64_host(self.h, histogram_id, _ptr(h_values), n))

    def ingest_keyed_f64_u16_host(self, h_ids, h_values, n: int | None = None):
        if isinstance(h_values, np.ndarray):
            assert h_values.dtype == np.float64 and h_ids.dtype == np.uint16
            n = h_values.size if n is None else n
        self._check(self.lib.lh_ingest_keyed_f64_u16_host(self.h, _ptr(h_ids), _ptr(h_values), n))

    def ingest_keyed_i64ns_u16_host(self, h_ids, h_nanos, n: int | None = None):
        if isinstance(h_nanos, np.ndarray):
            assert h_nanos.dtype == np.int64 and h_ids.dtype == np.uint16
            n = h_nanos.size if n is None else n
        self._check(self.lib.lh_ingest_keyed_i64ns_u16_host(self.h, _ptr(h_ids), _ptr(h_nanos), n))

    def counter_add_u16_host(self, h_ids, h_amounts, n: int | None = None):
        if isinstance(h_amounts, np.ndarray):
            assert h_amounts.dtype == np.uint64 and h_ids.dtype == np.uint16
            n = h_amounts.size if n is None else n
        self._check(self.lib.lh_counter_add_u16_host(self.h, _ptr(h_ids), _ptr(h_amounts), n))

    def merge_counts_host(self, ids, keys, counts):
        """Add sparse (histogram id, int16 key, uint64 count) triples into the active arrays (exact merge)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        keys = np.ascontiguousarray(keys, dtype=np.int16)
        counts = np.ascontiguousarray(counts, dtype=np.uint64)
        assert ids.size == keys.size == counts.size
        self._check(self.lib.lh_merge_counts_host(self.h, ids.ctypes.data, keys.ctypes.data, counts.ctypes.data, ids.size))

    # ---- staging ring
    def staging_acquire(self) -> L.lh_staging:
        s = L.lh_staging()
        self._check(self.lib.lh_staging_acquire(self.h, C.byref(s)))
        return s

    def staging_view(self, s: L.lh_staging, dtype, count: int, byte_offset: int = 0) -> np.ndarray:
        buf = (C.c_char * int(s.bytes)).from_address(s.host)
        return np.frombuffer(buf, dtype=dtype, count=count, offset=byte_offset)

    def staging_commit_f64(self, s, histogram_id: int, n: int):
        self._check(self.lib.lh_staging_commit_f64(self.h, C.byref(s), histogram_id, n))

    def staging_commit_keyed_f64_u16(self, s, n: int, ids_offset: int):
        self._check(self.lib.lh_staging_commit_keyed_f64_u16(self.h, C.byref(s), n, ids_offset))

    def staging_commit_counter_u16(self, s, n: int, ids_offset: int):
        self._check(self.lib.lh_staging_commit_counter_u16(self.h, C.byref(s), n, ids_offset))

    def staging_abandon(self, s):
        self._check(self.lib.lh_staging_abandon(self.h, C.byref(s)))

    # ---- recording from CUDA code (include/loghisto_b200_device.cuh)
    def record_begin(self, stream=None) -> L.lh_recorder:
        """Open a record scope on `stream` (None = the engine's ingest stream).  Pass the returned recorder by value to
        kernels enqueued on that stream, then close the scope with record_end(); a snapshot waits for it."""
        rec = L.lh_recorder()
        self._check(self.lib.lh_record_begin(self.h, _stream(stream), C.byref(rec)))
        return rec

    def record_end(self, rec: L.lh_recorder):
        self._check(self.lib.lh_record_end(self.h, C.byref(rec)))

    @contextlib.contextmanager
    def recording(self, stream=None):
        """`with eng.recording(stream) as rec:` -- record_begin / record_end around the block."""
        rec = self.record_begin(stream)
        try:
            yield rec
        finally:
            self.record_end(rec)

    def graph_recorder(self, hist_ids=(), counter_ids=()) -> "GraphRecorder":
        """A recorder for kernels captured into CUDA graphs (lh_graph_recorder_create): local histogram row i drains
        into histogram id hist_ids[i] of the interval at every snapshot_begin, local counter i into counter_ids[i]
        (LH_GRAPH_UNBOUND: dropped and counted).  Usable as a context manager that closes it on exit."""
        return GraphRecorder(self, hist_ids, counter_ids)

    # ---- GPU timers (StartTimer / Stop with both ends on the device)
    def board(self, k: int = 0, kc: int = 0) -> "Board":
        """A device subscription board of k histogram rows and kc counter rows (lh_board_create)."""
        return Board(self, k, kc)

    def raw_board(self, k: int, window: int = 1) -> "RawBoard":
        """A raw device subscription board of k histogram rows (lh_raw_board_create), each summed over its last
        `window` publishes (lh_raw_board_create_window; an int >= 1)."""
        return RawBoard(self, k, window)

    def read_gauges(self, tensors) -> np.ndarray:
        """lh_gauges_read of one-element CUDA tensors (gauge_src): float64(value) of each, read on the snapshot stream
        without waiting for any other stream."""
        tensors = list(tensors)
        srcs = (L.lh_gauge_src * max(len(tensors), 1))()
        for i, t in enumerate(tensors):
            srcs[i].d_value, srcs[i].dtype = gauge_src(t, self.device)
        out = np.empty(len(tensors), dtype=np.float64)
        self._check(self.lib.lh_gauges_read(self.h, srcs, len(tensors), out.ctypes.data))
        return out

    def gpu_timer_start(self, stream=None) -> L.lh_gpu_timer:
        """Enqueue a start mark on `stream` (None = the ingest stream; torch's default stream is timed as itself)."""
        t = L.lh_gpu_timer()
        self._check(self.lib.lh_gpu_timer_start(self.h, _timer_stream(stream), C.byref(t)))
        return t

    def gpu_timer_stop(self, t: L.lh_gpu_timer, histogram_id: int, stream=None, d_out=None):
        """Record float64(now - start) into `histogram_id` on the device; with `d_out` (8 bytes of device memory) the
        kernel also writes the int64 duration there.  A token may be stopped any number of times."""
        self._check(self.lib.lh_gpu_timer_stop(self.h, C.byref(t), histogram_id, _timer_stream(stream), _ptr(d_out)))

    def gpu_timer_release(self, t: L.lh_gpu_timer):
        self._check(self.lib.lh_gpu_timer_release(self.h, C.byref(t)))

    # ---- snapshot
    def snapshot_begin(self):
        self._check(self.lib.lh_snapshot_begin(self.h))

    def snapshot_ingest_arrays(self, arrays):
        """lh_snapshot_ingest_arrays: every element of each array as a sample of its id, into the open snapshot's
        rows.  `arrays` holds (histogram_id, tensor) pairs (array_src) or lh_array_src entries passed as they are."""
        arrays = [a if isinstance(a, L.lh_array_src) else array_src(a[1], self.device, a[0]) for a in arrays]
        srcs = (L.lh_array_src * max(len(arrays), 1))(*arrays)
        self._check(self.lib.lh_snapshot_ingest_arrays(self.h, srcs, len(arrays)))

    def snapshot_device(self) -> L.lh_device_view:
        v = L.lh_device_view()
        self._check(self.lib.lh_snapshot_device(self.h, C.byref(v)))
        return v

    def snapshot_reduce(self, percentiles) -> Reduced:
        ps = np.ascontiguousarray(percentiles, dtype=np.float64)
        npct = ps.size
        H = self.H
        counts = np.zeros(H, dtype=np.uint64)
        sums = np.zeros(H, dtype=np.float64)
        avgs = np.zeros(H, dtype=np.float64)
        pkeys = np.zeros((H, npct), dtype=np.int32)
        pvals = np.zeros((H, npct), dtype=np.float64)
        self._check(self.lib.lh_snapshot_reduce(self.h, ps.ctypes.data if npct else 0, npct, counts.ctypes.data,
                                                sums.ctypes.data, avgs.ctypes.data, pkeys.ctypes.data,
                                                pvals.ctypes.data))
        return Reduced(counts, sums, avgs, pkeys, pvals)

    def snapshot_reduce_async(self, percentiles) -> tuple:
        """Enqueue the reduction; returns an opaque handle for snapshot_result()."""
        ps = np.ascontiguousarray(percentiles, dtype=np.float64)
        t = C.c_uint64()
        self._check(self.lib.lh_snapshot_reduce_async(self.h, ps.ctypes.data if ps.size else 0, ps.size, C.byref(t)))
        return (int(t.value), ps.size)

    def snapshot_result(self, handle) -> Reduced:
        ticket, npct = handle
        H = self.H
        counts = np.zeros(H, dtype=np.uint64)
        sums = np.zeros(H, dtype=np.float64)
        avgs = np.zeros(H, dtype=np.float64)
        pkeys = np.zeros((H, npct), dtype=np.int32)
        pvals = np.zeros((H, npct), dtype=np.float64)
        self._check(self.lib.lh_snapshot_result(self.h, ticket, counts.ctypes.data, sums.ctypes.data, avgs.ctypes.data,
                                                pkeys.ctypes.data, pvals.ctypes.data))
        return Reduced(counts, sums, avgs, pkeys, pvals)

    def snapshot_export(self) -> Sparse:
        sp = L.lh_sparse()
        self._check(self.lib.lh_snapshot_export(self.h, C.byref(sp)))
        total = int(sp.total_entries)
        offsets = np.ctypeslib.as_array(sp.offsets, shape=(self.H + 1,)).copy()
        keys = np.ctypeslib.as_array(sp.keys, shape=(total,)).copy() if total else np.zeros(0, np.int16)
        counts = np.ctypeslib.as_array(sp.counts, shape=(total,)).copy() if total else np.zeros(0, np.uint64)
        deltas = np.ctypeslib.as_array(sp.counter_deltas, shape=(self.C,)).copy()
        return Sparse(offsets, keys, counts, deltas)

    def snapshot_copy_histogram(self, histogram_id: int) -> np.ndarray:
        out = np.zeros(65536, dtype=np.uint64)
        self._check(self.lib.lh_snapshot_copy_histogram(self.h, histogram_id, out.ctypes.data))
        return out

    def snapshot_end(self):
        self._check(self.lib.lh_snapshot_end(self.h))

    def reduce_sparse(self, offsets, keys=None, counts=None, percentiles=()) -> Reduced:
        """processHistograms + percentile over sparse histograms held by the caller (lh_reduce_sparse_host): histogram i
        is entries [offsets[i], offsets[i+1]) of keys / counts, in any key order, repeats summed.  `offsets` may be a
        `Sparse` (an export, from this engine or another), in which case keys / counts come from it and percentiles
        may be passed as the second argument.  Touches none of the engine's snapshot or ingest state."""
        if isinstance(offsets, Sparse):
            if keys is not None and counts is None:
                percentiles = keys
            offsets, keys, counts = offsets.offsets, offsets.keys, offsets.counts
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        keys = np.ascontiguousarray(keys, dtype=np.int16)
        counts = np.ascontiguousarray(counts, dtype=np.uint64)
        assert offsets.size >= 1 and keys.size == counts.size and int(offsets[-1]) <= keys.size
        ps =np.ascontiguousarray(percentiles, dtype=np.float64)
        n, npct = offsets.size - 1, ps.size
        out_counts = np.zeros(n, dtype=np.uint64)
        sums = np.zeros(n, dtype=np.float64)
        avgs = np.zeros(n, dtype=np.float64)
        pkeys = np.zeros((n, npct), dtype=np.int32)
        pvals = np.zeros((n, npct), dtype=np.float64)
        self._check(self.lib.lh_reduce_sparse_host(self.h, n, offsets.ctypes.data, keys.ctypes.data, counts.ctypes.data,
                                                   ps.ctypes.data if npct else 0, npct, out_counts.ctypes.data,
                                                   sums.ctypes.data, avgs.ctypes.data, pkeys.ctypes.data, pvals.ctypes.data))
        return Reduced(out_counts, sums, avgs, pkeys, pvals)

    def snapshot(self, percentiles, export: bool = True, arrays=None):
        """begin (+ ingest arrays) + reduce (+ export) + end; returns (Reduced, Sparse | None).  `arrays`: what
        snapshot_ingest_arrays takes, recorded into the interval this snapshot freezes."""
        self.snapshot_begin()
        try:
            if arrays is not None:
                self.snapshot_ingest_arrays(arrays)
            red = self.snapshot_reduce(percentiles)
            sp = self.snapshot_export() if export else None
        finally:
            self.snapshot_end()
        return red, sp

    # ---- probes / streams
    def compress(self, values: np.ndarray, mode: int = 0) -> np.ndarray:
        values = np.ascontiguousarray(values, dtype=np.float64)
        d_in = self.upload(values)
        d_out = self.alloc(values.size, np.int16)
        self._check(self.lib.lh_compress_f64(self.h, d_in.ptr, values.size, d_out.ptr, mode, 0))
        self.sync()
        out = d_out.to_host()
        d_in.free()
        d_out.free()
        return out

    def decompress_table(self) -> np.ndarray:
        out = np.zeros(65536, dtype=np.float64)
        self._check(self.lib.lh_decompress_table(self.h, out.ctypes.data))
        return out

    def fastpath_margin(self, d_values, n: int):
        err = C.c_double()
        slow = C.c_uint64()
        self._check(self.lib.lh_fastpath_margin(self.h, _ptr(d_values), n, C.byref(err), C.byref(slow), 0))
        return float(err.value), int(slow.value)

    def fastpath_margin_detail(self):
        a, b = C.c_double(), C.c_double()
        self._check(self.lib.lh_fastpath_margin_detail(self.h, C.byref(a), C.byref(b)))
        return float(a.value), float(b.value)

    def fastpath_certify(self, p_lo: int = 1, p_hi: int = 250) -> np.ndarray:
        """lh_fastpath_certify: a structured array [p_hi - p_lo + 1, 4] (precision, form) with the fields of
        lh_certify_form; row i is precision p_lo + i."""
        out = (L.lh_certify_form * ((p_hi - p_lo + 1) * 4))() if p_hi >= p_lo else None
        self._check(self.lib.lh_fastpath_certify(self.h, p_lo, p_hi, out))
        return np.ctypeslib.as_array(out).reshape(p_hi - p_lo + 1, 4).copy()

    def gen_stream(self, kind: int, n: int, seed: int, start: int = 0, out: DeviceArray | None = None,
                   stream=None) -> DeviceArray:
        if out is None:
            out = self.alloc(n, np.float64)
        self._check(self.lib.lh_gen_stream_f64(self.h, kind, seed, start, n, out.ptr, _stream(stream)))
        return out

    def gen_ids_u16(self, kind: int, n: int, n_ids: int, seed: int, start: int = 0,
                    out: DeviceArray | None = None, stream=None) -> DeviceArray:
        if out is None:
            out = self.alloc(n, np.uint16)
        self._check(self.lib.lh_gen_ids_u16(self.h, kind, seed, start, n, n_ids, out.ptr, _stream(stream)))
        return out
