"""The CUDA-graph shape policy of engine.PlanCache (shared by the encoder's and the fused head's plans), driven with a
fake plan builder: direct launches until a key has been seen `graph_after` times, LRU order on hits, avsr_plan_destroy
on eviction and on clear, and a bounded sighting table."""
import types

import pytest


@pytest.fixture
def cache(monkeypatch):
    from auto_avsr_b200 import engine
    destroyed = []
    monkeypatch.setattr(engine, "lib", types.SimpleNamespace(avsr_plan_destroy=destroyed.append))
    c = engine.PlanCache(max_plans=2)
    c.destroyed = destroyed
    yield c
    c._plans.clear()                                        # the fake handles must never reach the real library


def _builder(log):
    def build_for(key):
        def build():
            log.append(key)
            return (f"plan{key}", f"ws{key}")
        return build
    return build_for


def test_threshold_then_plan_then_hits(cache):
    built = []
    b = _builder(built)
    assert cache.get("a", 3, b("a")) is None
    assert cache.get("a", 3, b("a")) is None
    assert cache.get("a", 3, b("a")) == ("plana", "wsa")     # third sighting builds
    assert cache.get("a", 3, b("a")) == ("plana", "wsa")     # then hits, no rebuild
    assert built == ["a"]
    assert cache.get("b", 1, b("b")) == ("planb", "wsb")     # graph_after = 1: capture at first sight
    assert built == ["a", "b"] and cache.destroyed == []


def test_lru_order_on_hits_and_eviction_destroys(cache):
    b = _builder([])
    cache.get("a", 1, b("a"))
    cache.get("b", 1, b("b"))
    cache.get("a", 1, b("a"))                               # hit: "a" becomes the most recently used
    cache.get("c", 1, b("c"))                                # over max_plans = 2: the least recently used ("b") goes
    assert cache.destroyed == ["planb"]
    assert list(cache._plans) == ["a", "c"]
    cache.clear()
    assert sorted(cache.destroyed) == ["plana", "planb", "planc"] and not cache._plans


def test_seen_is_bounded(cache):
    b = _builder([])
    for t in range(1000):                                   # the B = 1 eval loop: a new T per utterance
        assert cache.get(("B1", t), 3, b(t)) is None
    assert len(cache._seen) == 64 * cache.max_plans
    assert ("B1", 999) in cache._seen and ("B1", 0) not in cache._seen
