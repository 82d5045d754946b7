"""CPU: latency-based-routing as the oracle states it (oracle/latency_router.py), on hand-computed cases, and the
`routing_strategy_args` parsing of the config loader."""
import ctypes as C
import random

import pytest

from oracle import router as O
from oracle.latency_router import STRATEGY_LATENCY_BASED, LatencyOracleRouter, LatencySettings


def _router(deps, n_groups=1, seed=0, **settings):
    st = LatencySettings(strategy=STRATEGY_LATENCY_BASED, enable_pre_call_checks=False, **settings)
    return LatencyOracleRouter(deps, n_groups, {}, st, seed=seed)


def _done(orc, dep, latency_us, tokens=1, now=0):
    return orc.process([O.Event(O.EV_DONE, dep, tokens, latency_us, now)])[0]


@pytest.mark.parametrize("seed", [0, 7, 2**40 + 3])
def test_fresh_group_is_random_choice_over_the_eligible(seed):
    """No samples: every mean is 0.0, so the pick is random.choice over the eligible deployments in config order."""
    deps = [O.Deployment(group=0) for _ in range(5)] + [O.Deployment(group=1)]
    orc = _router(deps, n_groups=2, seed=seed)
    ref = random.Random(seed)
    for _ in range(50):
        assert orc.admit(0, 3, 0, 0).deployment == ref.choice([0, 1, 2, 3, 4])
    assert orc.rng.getstate() == ref.getstate()


def test_single_valid_candidate_still_draws():
    orc = _router([O.Deployment(group=0), O.Deployment(group=0)], seed=5)
    _done(orc, 0, 100)
    _done(orc, 1, 50)
    ref = random.Random(5)
    for _ in range(10):
        assert orc.admit(0, 1, 0, 0).deployment == 1
        ref.choice([1])
    assert orc.rng.getstate() == ref.getstate()


def _buffer_router(ppm, seed):
    orc = _router([O.Deployment(group=0) for _ in range(5)], seed=seed, latency_buffer_ppm=ppm)
    for dep, lat in enumerate([120, 100, 150, 120, 151]):       # means 120, 100, 150, 120, 151 us / token
        _done(orc, dep, lat)
    return orc


def test_buffer_zero_picks_the_lowest_mean():
    orc = _buffer_router(0, seed=3)
    assert all(orc.admit(0, 1, 0, 0).deployment == 1 for _ in range(20))


def test_buffer_half_picks_among_means_within_1_5x_in_mean_then_config_order():
    orc = _buffer_router(500_000, seed=11)
    ref = random.Random(11)
    order = [1, 0, 3, 2]            # threshold 150: 151 is out; 0 and 3 tie at 120 and keep config order
    picks = [orc.admit(0, 1, 0, 0).deployment for _ in range(200)]
    assert picks == [order[ref._randbelow(4)] for _ in range(200)]
    assert set(picks) == set(order)


def test_threshold_is_two_roundings():
    """lowest + (buffer * lowest) with buffer = ppm / 1e6: a mean exactly on the threshold is valid."""
    orc = _router([O.Deployment(group=0), O.Deployment(group=0)], latency_buffer_ppm=100_000)
    _done(orc, 0, 3, tokens=10)                                   # 0.3
    thr = 0.3 + (0.1 * 0.3)
    orc.latencies[1] = [thr]
    assert orc._lat_buffer() == 100_000 / 1e6 == 0.1
    assert {orc.admit(0, 1, 0, 0).deployment for _ in range(40)} == {0, 1}


def test_list_rule_freezes_the_first_n_minus_1_samples():
    orc = _router([O.Deployment(group=0)], latency_list_size=3)
    for lat in (1, 2, 3, 100):
        _done(orc, 0, lat)
    assert orc.latencies[0] == [1.0, 2.0, 100.0]
    assert orc.latency_snapshot() == [((1.0 + 2.0 + 100.0) / 3, 3)]
    _done(orc, 0, 7)
    assert orc.latencies[0] == [1.0, 2.0, 7.0]


def test_list_size_one_keeps_only_the_latest():
    orc = _router([O.Deployment(group=0)], latency_list_size=1)
    for lat in (5, 9, 4):
        _done(orc, 0, lat)
    assert orc.latency_snapshot() == [(4.0, 1)]


def test_sample_is_latency_per_output_token_or_raw_latency_without_tokens():
    orc = _router([O.Deployment(group=0), O.Deployment(group=0), O.Deployment(group=0)])
    _done(orc, 0, 500, tokens=0)
    _done(orc, 1, 500, tokens=4)
    _done(orc, 2, 1000, tokens=3)
    assert orc.latencies[0] == [500.0]
    assert orc.latencies[1] == [125.0]
    assert orc.latencies[2] == [1000 / 3]
    _done(orc, 0, 0)                                              # L <= 0: no sample
    _done(orc, 0, -5)
    assert orc.latencies[0] == [500.0]


def test_fail_records_the_penalty_only_for_a_timeout():
    orc = _router([O.Deployment(group=0), O.Deployment(group=0)], allowed_fails=100)
    orc.process([O.Event(O.EV_FAIL, 0, 0, 0, 0), O.Event(O.EV_FAIL, 1, 0, 1, 0), O.Event(O.EV_FAIL, 1, 0, 2, 0)])
    assert orc.latency_snapshot() == [(0.0, 0), (1e9, 1)]
    assert orc.deps[0].fail_count == 1 and orc.deps[1].fail_count == 2
    # the timed-out deployment is avoided afterwards
    assert all(orc.admit(0, 1, 0, 10).deployment == 0 for _ in range(10))


def test_ttl_expires_one_group_and_leaves_the_other():
    deps = [O.Deployment(group=0), O.Deployment(group=0), O.Deployment(group=1)]
    orc = _router(deps, n_groups=2, latency_ttl_ms=30_000)
    _done(orc, 0, 100, now=0)
    _done(orc, 1, 200, now=0)
    _done(orc, 2, 300, now=20_000)
    assert orc.admit(0, 1, 0, 30_000).deployment == 0            # 30 000 - 0 is not > ttl: still measured
    orc.admit(0, 1, 0, 30_001)                                    # expired: both lists of group 0 cleared
    assert orc.latency_snapshot() == [(0.0, 0), (0.0, 0), (300.0, 1)]
    assert orc.lat_stamp == [0, 20_000]                           # clearing is not a write
    _done(orc, 1, 50, now=40_000)                                 # a write clears (again) and stamps
    assert orc.latency_snapshot() == [(0.0, 0), (50.0, 1), (300.0, 1)]
    assert orc.lat_stamp == [40_000, 20_000]
    _done(orc, 2, 10, now=50_001)                                 # group 1 expired at its own write
    assert orc.latency_snapshot()[2] == (10.0, 1)


def test_other_strategies_ignore_latency_fields():
    for strategy in (0, 1, 2, 3, 4):
        a = LatencyOracleRouter([O.Deployment(group=0) for _ in range(3)], 1, {},
                                LatencySettings(strategy=strategy, latency_list_size=3, latency_ttl_ms=1), seed=1)
        b = O.OracleRouter([O.Deployment(group=0) for _ in range(3)], 1, {}, O.Settings(strategy=strategy), seed=1)
        rng = random.Random(strategy)
        for i in range(300):
            t = rng.choice([0, 0, 1, 2])
            tgt = 0 if t == 0 else rng.randrange(3)
            aux = rng.randrange(0, 5000) if t else 0
            ea, eb = O.Event(t, tgt, rng.randrange(0, 9), aux, i * 10), O.Event(t, tgt, 0, 0, i * 10)
            eb.tokens = ea.tokens
            assert a.process([ea]) == b.process([eb])
        assert a.snapshot() == b.snapshot() and a.rng.getstate() == b.rng.getstate()
        assert a.latency_snapshot() == [(0.0, 0)] * 3


# ---------------------------------------------------------------- config
ML = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny"}},
      {"model_name": "chat", "litellm_params": {"model": "b200/small", "gpu": 1}}]


def test_config_defaults_and_values():
    from rr_b200.config import build_config
    cfg = build_config(ML, {"routing_strategy": "latency-based-routing"})
    assert cfg.strategy_id == 5
    assert (cfg.latency_list_size, cfg.latency_buffer_ppm, cfg.latency_ttl_ms) == (10, 0, 3_600_000)
    cfg = build_config(ML, {"routing_strategy": "latency-based-routing", "routing_strategy_args": {
        "lowest_latency_buffer": 0.1, "max_latency_list_size": 32, "ttl": 30}})
    assert (cfg.latency_list_size, cfg.latency_buffer_ppm, cfg.latency_ttl_ms) == (32, 100_000, 30_000)
    cfg = build_config(ML, {"routing_strategy": "latency-based-routing",
                            "routing_strategy_args": {"lowest_latency_buffer": 0.0000015, "ttl": 0.5}})
    assert (cfg.latency_buffer_ppm, cfg.latency_ttl_ms) == (2, 500)


def test_config_example_file_loads():
    from pathlib import Path
    from rr_b200.config import load_config
    cfg = load_config(str(Path(__file__).resolve().parents[1] / "config" / "latency-routing.yaml"))
    assert cfg.routing_strategy == "latency-based-routing" and cfg.strategy_id == 5
    assert len(cfg.groups) >= 1 and len(cfg.deployments) >= 2
    assert (cfg.latency_list_size, cfg.latency_buffer_ppm, cfg.latency_ttl_ms) == (10, 100_000, 300_000)


@pytest.mark.parametrize("args", [
    {"max_latency_list_size": 0}, {"max_latency_list_size": 33}, {"max_latency_list_size": 2.5},
    {"max_latency_list_size": True}, {"lowest_latency_buffer": -0.1}, {"lowest_latency_buffer": "0.1"},
    {"lowest_latency_buffer": float("nan")}, {"lowest_latency_buffer": 5000.0}, {"ttl": 0}, {"ttl": -1},
    {"ttl": 1e9}, {"ttl": float("inf")}, {"lowest_latency_bufer": 0.1}, [1, 2]])
def test_config_rejects_bad_strategy_args(args):
    from rr_b200.config import build_config
    with pytest.raises(ValueError):
        build_config(ML, {"routing_strategy": "latency-based-routing", "routing_strategy_args": args})


def test_usage_based_routing_is_still_rejected():
    from rr_b200.config import build_config
    for s in ("usage-based-routing", "usage-based-routing-v2", "cost-based-routing"):
        with pytest.raises(ValueError):
            build_config(ML, {"routing_strategy": s})


@pytest.mark.parametrize("strategy", ["latency-based-routing", "least-busy"])
def test_router_state_endpoint_reports_latency_only_under_the_strategy(strategy):
    from starlette.testclient import TestClient
    from rr_b200.config import build_config
    from rr_b200.server import create_app

    class _Fake:
        cfg = build_config(ML, {"routing_strategy": strategy})

        def snapshot(self):
            return [{"inflight": 0, "total_admitted": i} for i in range(2)]

        def latency_snapshot(self):
            return [(12.5, 3), (0.0, 0)]

    deps = TestClient(create_app(_Fake())).get("/router/state").json()["deployments"]
    if strategy == "latency-based-routing":
        assert [(d["latency_us_per_token"], d["latency_samples"]) for d in deps] == [(12.5, 3), (0.0, 0)]
    else:
        assert all("latency_us_per_token" not in d and "latency_samples" not in d for d in deps)
    assert [d["total_admitted"] for d in deps] == [0, 1]


def test_router_settings_struct_keeps_its_size():
    from rr_b200 import _lib
    assert C.sizeof(_lib.RouterSettings) == 32 and C.sizeof(_lib.Event) == 24
    assert _lib.RouterSettings.latency_list_size.offset == 20 and _lib.RouterSettings.latency_ttl_ms.offset == 28
    assert hasattr(_lib.lib, "rr_router_latency_snapshot")
