"""Recycling of name ids in the C++ MetricSystem mirror (loghisto_b200/host/metric_system.h, NameTable), compiled
against the TEST-ONLY oracle-backed stub of the C ABI (as in tests/test_host_logic_cpu.py), in both shard modes: the
exclusive shards with the membarrier handshake, and the spin-locked fallback (LOGHISTO_B200_SHARD_LOCK=1).  The
cases live in tests/_name_recycling_cases.py; tests/test_gpu_name_recycling.py runs them on the real library."""
import ctypes
import importlib.util
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


@pytest.fixture(scope="module")
def stub_host_lib():
    os.makedirs(BUILD, exist_ok=True)
    stub = os.path.join(BUILD, "liblh_stub_recycling.so")
    host = os.path.join(BUILD, "libloghisto_host_stub_recycling.so")
    inc = os.path.join(ROOT, "include")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", inc,
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub.c"),
                    os.path.join(ROOT, "tests", "stub_abi", "lh_stub_reduce_sparse.c"),
                    os.path.join(ROOT, "oracle", "loghisto_oracle.c"), "-o", stub, "-lm", "-lpthread"], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", inc,
                    os.path.join(ROOT, "loghisto_b200", "host", "metric_system.cc"),
                    os.path.join(ROOT, "loghisto_b200", "host", "print_benchmark.cc"), "-o", host,
                    "-L", BUILD, "-llh_stub_recycling", "-Wl,-rpath," + BUILD, "-lpthread"], check=True)
    return host


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, stub_host_lib, monkeypatch):
    import loghisto_b200.metric_system as m
    monkeypatch.setattr(m, "_lib", m._bind(ctypes.CDLL(stub_host_lib)))
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
    made = []

    def make(interval_s=1e-6, **kw):
        ms = m.MetricSystem(interval_s, False, max_histograms=kw.get("max_histograms", 64),
                            max_counters=kw.get("max_counters", 64))
        made.append(ms)
        return ms
    yield make
    for ms in made:
        ms.close()


def _cases():
    spec = importlib.util.spec_from_file_location("name_recycling_cases",
                                                  os.path.join(ROOT, "tests", "_name_recycling_cases.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_churn_matches_oracle(MS, oracle):
    _cases().churn_matches_oracle(MS, oracle)


@pytest.mark.parametrize("kind", ["histogram", "counter"])
def test_bound_is_three_intervals(MS, kind):
    _cases().bound_drops(MS, kind)


@pytest.mark.parametrize("kind", ["histogram", "counter"])
def test_stale_thread_cache(MS, oracle, kind):
    _cases().stale_thread_cache(MS, oracle, kind)


def test_timer_across_collections(MS, oracle):
    _cases().timer_across_collections(MS, oracle)


def test_race(MS, oracle, monkeypatch, tmp_path):
    monkeypatch.setenv("LOGHISTO_B200_SHARDS", "4")            # 4 exclusive shards, the other threads on shared ones
    monkeypatch.setenv("LOGHISTO_B200_STAGING_BYTES", "65536")
    mod = _cases()
    mod.race(MS, oracle, mod.build_race_driver(tmp_path))
