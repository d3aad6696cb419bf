"""Record scopes bound to names (MetricSystem::BeginRecording, loghisto_b200/host/metric_system.cc) on the CPU: the
C++ mirror compiled against the TEST-ONLY oracle-backed stub of the C ABI plus tests/stub_abi/lh_stub_record.c, which
adds record scopes, a one-sample stand-in for lh::record / lh::count, and a hook that runs collections from inside
lh_record_begin, between the binding's lookup and its generation check.  Both shard modes.  Also: the device timer of
include/loghisto_b200_device.cuh compiles for sm_90a with and without -rdc=true, and the lhms_record_* entry points are
bound in loghisto_b200/metric_system.py.  tests/test_gpu_named_recording.py runs the real library."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
INC = os.path.join(ROOT, "include")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
UNBOUND = 0xFFFFFFFF
HOOK = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_uint64)


@pytest.fixture(scope="module")
def stub_libs():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_named.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_named.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", INC,
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub.c"),
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub_reduce_sparse.c"),
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub_record.c"),
                    os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I", INC,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_named", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    from loghisto_b200 import _lib
    s = ctypes.CDLL(stub)
    rp = ctypes.POINTER(_lib.lh_recorder)
    s.lh_stub_record.argtypes = [rp, ctypes.c_uint32, ctypes.c_double]
    s.lh_stub_record.restype = ctypes.c_int
    s.lh_stub_count.argtypes = [rp, ctypes.c_uint32, ctypes.c_uint64]
    s.lh_stub_count.restype = ctypes.c_int
    s.lh_stub_record_hook.argtypes = [HOOK, ctypes.c_void_p]
    s.lh_stub_record_begins.restype = ctypes.c_uint64
    return s, host


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, stub_libs, monkeypatch):
    import loghisto_b200.metric_system as m
    stub, host = stub_libs
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(host)))
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
    made = []

    def make(max_histograms=4, max_counters=4):
        ms = m.MetricSystem(1e-6, False, max_histograms=max_histograms, max_counters=max_counters)
        made.append(ms)
        return ms
    yield make
    stub.lh_stub_record_hook(HOOK(0), None)
    for ms in made:
        ms.close()


@pytest.fixture
def stub(stub_libs):
    return stub_libs[0]


def record(stub, scope, name, v):
    assert stub.lh_stub_record(ctypes.byref(scope.recorder), scope.histogram_ids[name], v) == 0


def count(stub, scope, name, amount):
    assert stub.lh_stub_count(ctypes.byref(scope.recorder), scope.counter_ids[name], amount) == 0


@pytest.mark.parametrize("collections", [1, 2, 3, 4])
def test_binding_survives_collections_between_lookup_and_begin(MS, stub, oracle, collections):
    """The hook runs `collections` collections between the interning of "h" / "c" (new names) and lh_record_begin,
    then records "other" from the host.  One collection leaves the names live: no retry.  A second retires them, so the
    generation check fails and the binding retries once; from the third on their ids are free, and "other" / "oc" take
    them before the retry.  Either way the scope's records are labelled "h" / "c" by the collection of their interval."""
    ms = MS()
    calls = []

    def hook(_arg, call):
        calls.append(call)
        if len(calls) == 1:
            for _ in range(collections):
                ms.collect_and_process()
            ms.Histogram("other", 1000.0)
            ms.Counter("oc", 3)
    cb = HOOK(hook)
    stub.lh_stub_record_hook(cb, None)
    begins = stub.lh_stub_record_begins()
    with ms.recording(histograms=["h"], counters=["c"]) as s:
        stub.lh_stub_record_hook(HOOK(0), None)
        record(stub, s, "h", 7.0)
        record(stub, s, "h", 7.0)
        count(stub, s, "c", 5)
    retries = stub.lh_stub_record_begins() - begins - 1
    assert retries == (0 if collections == 1 else 1)
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"h": {oracle.compress(7.0): 2}, "other": {oracle.compress(1000.0): 1}}
    assert raw["Rates"] == {"c": 5, "oc": 3}
    assert ms.dropped() == 0


def test_retry_rebinds_to_a_new_id_when_the_old_one_was_taken(MS, stub, oracle):
    """Three collections free the id of "h"; the hook's "other" takes it.  The scope must not record under it."""
    ms = MS(max_histograms=2, max_counters=2)
    first = stub.lh_stub_record_begins()
    old = {}

    def hook(_arg, call):
        if call == first:
            with ms.recording(histograms=["h"]) as probe:   # the id "h" would get without the collections
                old["id"] = probe.histogram_ids["h"]
            for _ in range(3):
                ms.collect_and_process()
            ms.Histogram("other", 1000.0)
    cb = HOOK(hook)
    stub.lh_stub_record_hook(cb, None)
    with ms.recording(histograms=["h"]) as s:
        stub.lh_stub_record_hook(HOOK(0), None)
        assert s.histogram_ids["h"] != old["id"]
        record(stub, s, "h", 7.0)
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"h": {oracle.compress(7.0): 1}, "other": {oracle.compress(1000.0): 1}}


def test_full_table_binds_unbound_and_counts_drops(MS, stub, oracle):
    """No free id: the name is bound to 0xFFFFFFFF, opening the scope counts nothing, and every record, counter op
    and ingested sample under it is dropped and counted.  Bound names in the same scope record normally."""
    ms = MS(max_histograms=2, max_counters=2)
    for nm in ("a", "b"):
        ms.Histogram(nm, 1.0)
        ms.Counter(nm, 1)
    ms.collect_and_process()
    before = ms.dropped()
    with ms.recording(histograms=["a", "new"], counters=["b", "newc"]) as s:
        assert s.histogram_ids["new"] == UNBOUND and s.counter_ids["newc"] == UNBOUND
        assert s.histogram_ids["a"] != UNBOUND and s.counter_ids["b"] != UNBOUND
        assert ms.dropped() == before
        for _ in range(3):
            record(stub, s, "new", 2.0)
        count(stub, s, "newc", 9)
        record(stub, s, "a", 2.0)
        count(stub, s, "b", 4)
        vals = np.array([5.0, 6.0, 7.0, 8.0])
        for i in (0, 1):    # "a", then "new": through lhms_record_ingest_f64 (host memory stands in for device memory)
            assert ms._lib.lhms_record_ingest_f64(ms._h, ctypes.byref(s.recorder), i, vals.ctypes.data, vals.size) == 0
        assert ms._lib.lhms_record_ingest_f64(ms._h, ctypes.byref(s.recorder), 2, vals.ctypes.data, vals.size) != 0
    assert ms.dropped() - before == 3 + 1 + 4
    raw, _ = ms.collect_and_process()
    want = {}
    for v in [2.0, 5.0, 6.0, 7.0, 8.0]:
        want[oracle.compress(v)] = want.get(oracle.compress(v), 0) + 1
    assert raw["Histograms"] == {"a": want}
    assert raw["Rates"] == {"b": 4}


def test_collect_while_holding_a_scope_raises_and_loses_nothing(MS, stub, oracle):
    """collectRawMetrics from the thread that holds a scope raises before it flushes anything: the Counter(name, 0)
    mark, the host samples and the scope's records all come out of the next collection, exactly once."""
    ms = MS()
    ms.Counter("zero", 0)
    ms.Histogram("h", 2.0)
    with ms.recording(histograms=["h"], counters=["c"]) as s:
        record(stub, s, "h", 3.0)
        count(stub, s, "c", 0)          # lh::count of 0 leaves the delta at 0: "c" is not in Rates
        with pytest.raises(RuntimeError, match="record scope"):
            ms.collect_and_process()
        ms.Counter("zero2", 0)
    raw, _ = ms.collect_and_process()
    assert raw["Rates"] == {"zero": 0, "zero2": 0}
    assert raw["Histograms"] == {"h": {oracle.compress(2.0): 1, oracle.compress(3.0): 1}}
    raw, _ = ms.collect_and_process()
    assert raw["Rates"] == {} and raw["Histograms"] == {}
    assert ms.dropped() == 0


def test_scope_end_is_idempotent_and_nested_scopes_work(MS, stub, oracle):
    ms = MS()
    with ms.recording(histograms=["x"]) as outer:
        with ms.recording(histograms=["x", "y"]) as inner:
            assert inner.histogram_ids["x"] == outer.histogram_ids["x"]
            record(stub, inner, "y", 1.0)
        inner.end()
        record(stub, outer, "x", 1.0)
    outer.end()
    raw, _ = ms.collect_and_process()
    assert raw["Histograms"] == {"x": {oracle.compress(1.0): 1}, "y": {oracle.compress(1.0): 1}}


def test_record_entry_points_are_bound(stub_libs):
    """Every lhms_record_* entry point of the C shim is declared by metric_system._bind."""
    import loghisto_b200.metric_system as m
    src = open(os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc")).read()
    names = re.findall(r"LHMS_API \w+ (lhms_record_\w+)\(", src)
    assert sorted(names) == ["lhms_record_begin", "lhms_record_end", "lhms_record_ingest_f64"]
    L = m._bind(ctypes.CDLL(stub_libs[1]))
    for nm in names:
        assert getattr(L, nm).argtypes is not None, nm
    assert callable(m.MetricSystem.recording)


TIMER_A = r'''
#include "loghisto_b200_device.cuh"
__global__ void k_start(lh::TimerToken *tok, uint32_t id) { tok[threadIdx.x] = lh::start_timer(id); }
void launch_start(lh::TimerToken *tok) { k_start<<<1, 32>>>(tok, 0); }
'''
TIMER_B = r'''
#include "loghisto_b200_device.cuh"
static_assert(sizeof(lh::TimerToken) == 16, "16 B token");
__global__ void k_stop(lh_recorder rec, const lh::TimerToken *tok, long long *out) {
    lh::TimerToken t = lh::start_timer(1);
    out[threadIdx.x] = lh::stop(rec, tok[threadIdx.x]) + lh::stop(rec, t);
}
void launch_start(lh::TimerToken *tok);
int main() {
    lh_recorder rec = {};
    launch_start(nullptr);
    k_stop<<<1, 32>>>(rec, nullptr, nullptr);
    return 0;
}
'''


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
@pytest.mark.parametrize("rdc", [True, False], ids=["rdc", "whole"])
def test_device_timer_compiles_and_links_from_two_translation_units(tmp_path, rdc):
    (tmp_path / "a.cu").write_text(TIMER_A)
    (tmp_path / "b.cu").write_text(TIMER_B)
    res = subprocess.run([NVCC] + ARCH + ["-std=c++17"] + (["-rdc=true"] if rdc else []) +
                         ["-I", INC, str(tmp_path / "a.cu"), str(tmp_path / "b.cu"), "-o", str(tmp_path / "timer")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_named_record_client_compiles_without_spills(tmp_path):
    res = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-shared", "-I", INC,
                          os.path.join(ROOT, "tests", "named_record_client.cu"), "-o", str(tmp_path / "client.so")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    assert re.findall(r"Compiling entry function '([^']+)'", log)
    assert not any(int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", log)), log
