"""Recycling of name ids in the C++ MetricSystem mirror over the real library, in both shard modes (exclusive shards
with the membarrier handshake; LOGHISTO_B200_SHARD_LOCK=1: the spin-locked fallback).  The cases live in
tests/_name_recycling_cases.py; tests/test_name_recycling_cpu.py runs them over the oracle-backed stub."""
import importlib.util
import os

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(params=["0", "1"], ids=["exclusive", "shard_lock"])
def MS(request, monkeypatch):
    from loghisto_b200.metric_system import MetricSystem
    monkeypatch.setenv("LOGHISTO_B200_SHARD_LOCK", request.param)
    made = []

    def make(interval_s=1e-6, **kw):
        m = MetricSystem(interval_s, False, max_histograms=kw.get("max_histograms", 64),
                         max_counters=kw.get("max_counters", 64))
        made.append(m)
        return m
    yield make
    for m in made:
        m.close()


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
