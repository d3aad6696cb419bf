"""loghisto_b200: H100-native ingest + percentile-reduction engine behind loghisto's MetricSystem API.

The CUDA library (libloghisto_b200.so, C ABI in include/loghisto_b200.h) is the
product; this package only loads it and mirrors the reference's host-side
interface.  There is no CPU fallback.
"""
from .engine import DeviceArray, Engine, LhError, PinnedArray, Reduced, Sparse  # noqa: F401

STREAM_U, STREAM_L, STREAM_S, STREAM_C, STREAM_Z = 0, 1, 2, 3, 4
STREAM_RAW, STREAM_TIMER_NS, STREAM_AMOUNTS = 5, 6, 7   # raw u64 bits / int64 ns / counter amounts 1..16
STREAM_N = 8                                            # stream U with a random sign
DEFAULT_SEED = 0x10C415C0
