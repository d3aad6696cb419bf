"""How far one ingest call advances lh_ingest_seq.  A device-pointer call takes one sequence number whichever kernels it
runs (the keyed pair included, fused or not), a host-fed call one per staging chunk, a staging commit one; the CUDA
events of every number time that number's kernels."""
import math

import numpy as np
import pytest

import _ingest_routes as R

pytestmark = pytest.mark.gpu

SEED = 0xB4AC7E7


@pytest.fixture(scope="module")
def lh():
    import loghisto_b200
    return loghisto_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def advance(e, call):
    """The sequence numbers `call` took, after checking that each one timed a finite, positive device time."""
    before = e.ingest_seq()
    call()
    after = e.ingest_seq()
    for seq in range(before + 1, after + 1):
        ms = e.kernel_ms(seq)
        assert math.isfinite(ms) and ms > 0, (seq, ms)
    return after - before


@pytest.mark.parametrize("H,n,route", [
    (1024, 1 << 20, R.VEC),     # fusing attempted and declined: 2^21 samples in all, below the write-combining minimum
    (1024, 1 << 21, R.WC),      # fused
    (44, 1 << 20, R.SMALL),     # few histograms: never fused, each array through the shared-memory kernel
])
def test_pair_takes_one_sequence_number(lh, sms, H, n, route):
    assert R.pair_route(H, n, n, 100, sms).kernel == route
    with lh.Engine(device=0, max_histograms=H, max_counters=1) as e:
        d_v = e.gen_stream(lh.STREAM_S, n, SEED)
        d_ns = e.gen_stream(lh.STREAM_TIMER_NS, n, SEED, out=e.alloc(n, np.int64))
        d_i = e.gen_ids_u16(0, n, H, SEED)
        e.sync()
        assert advance(e, lambda: e.ingest_keyed_pair_u16(d_i, d_v, n, d_i, d_ns, n)) == 1
        assert e.keyed_kernel_name() == route
        assert e.stats()["samples"] == 2 * n


def test_device_call_takes_one_sequence_number(lh):
    n = 1 << 20
    with lh.Engine(device=0, max_histograms=8, max_counters=8) as e:
        d_v = e.gen_stream(lh.STREAM_S, n, SEED)
        d_ns = e.gen_stream(lh.STREAM_TIMER_NS, n, SEED, out=e.alloc(n, np.int64))
        d_a = e.gen_stream(lh.STREAM_AMOUNTS, n, SEED, out=e.alloc(n, np.uint64))
        d_i = e.gen_ids_u16(0, n, 8, SEED)
        e.sync()
        for name, call in (("f64", lambda: e.ingest_f64(1, d_v, n)),
                           ("keyed_f64_u16", lambda: e.ingest_keyed_f64_u16(d_i, d_v, n)),
                           ("keyed_i64ns_u16", lambda: e.ingest_keyed_i64ns_u16(d_i, d_ns, n)),
                           ("counter_u16", lambda: e.counter_add_u16(d_i, d_a, n))):
            assert advance(e, call) == 1, name


def test_host_fed_call_takes_one_sequence_number_per_chunk(lh):
    n, staging = 500_000, 1 << 20
    rng = np.random.default_rng(SEED)
    vals = rng.random(n) * 1e6
    ns = rng.integers(1, 10 ** 9, n, dtype=np.int64)
    amounts = rng.integers(1, 17, n, dtype=np.uint64)
    ids = rng.integers(0, 8, n).astype(np.uint16)
    with lh.Engine(device=0, max_histograms=8, max_counters=8, staging_bytes=staging, staging_slots=2) as e:
        for name, call, item in (("f64", lambda: e.ingest_f64_host(1, vals), 8),
                                 ("keyed_f64_u16", lambda: e.ingest_keyed_f64_u16_host(ids, vals), 10),
                                 ("keyed_i64ns_u16", lambda: e.ingest_keyed_i64ns_u16_host(ids, ns), 10),
                                 ("counter_u16", lambda: e.counter_add_u16_host(ids, amounts), 10)):
            per = (staging // item) & ~15                 # samples per staging chunk
            chunks = -(-n // per)
            assert 1 < chunks < 16, (name, chunks)       # several chunks, all still in the ring of timing events
            assert advance(e, call) == chunks, name
        m, ids_offset = 1000, 8000
        for name, commit in (("f64", lambda s: e.staging_commit_f64(s, 1, m)),
                             ("keyed_f64_u16", lambda s: e.staging_commit_keyed_f64_u16(s, m, ids_offset)),
                             ("counter_u16", lambda s: e.staging_commit_counter_u16(s, m, ids_offset))):
            s = e.staging_acquire()
            e.staging_view(s, np.float64, m)[:] = vals[:m]
            e.staging_view(s, np.uint16, m, byte_offset=ids_offset)[:] = ids[:m]
            assert advance(e, lambda: commit(s)) == 1, name
