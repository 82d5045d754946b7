"""GPU: latency-based-routing in the admission kernel K1 (csrc/rr_router.cu) against the oracle (oracle/latency_router.py), bit for
bit, in both state variants; the other strategies unchanged by the latency fields; the native gateway feeding measured
engine latencies and timeout penalties into K1, and the hand-off -> settle latencies of its mock replicas."""
import ctypes as C
import random
import time

import pytest

from oracle import router as O
from oracle.latency_router import STRATEGY_LATENCY_BASED, LatencyOracleRouter, LatencySettings

pytestmark = pytest.mark.gpu


class DevRouter:
    def __init__(self, deps, n_groups, fallbacks, settings, seed):
        from rr_b200 import _lib
        self.L = _lib
        arr = (_lib.DeploymentDesc * len(deps))()
        for i, d in enumerate(deps):
            arr[i] = _lib.DeploymentDesc(d.group, d.rpm, d.tpm, d.weight, d.replica, 0)
        offs, flat = [0], []
        for g in range(n_groups):
            flat += fallbacks.get(g, [])
            offs.append(len(flat))
        st = _lib.RouterSettings(settings.strategy, int(settings.enable_pre_call_checks), settings.allowed_fails,
                                 settings.cooldown_ms, 0, settings.latency_list_size, settings.latency_buffer_ppm,
                                 settings.latency_ttl_ms)
        self.h = C.c_void_p()
        self.n = len(deps)
        _lib.check(_lib.lib.rr_router_create(arr, len(deps), n_groups, (C.c_int32 * len(offs))(*offs),
                                             (C.c_int32 * max(1, len(flat)))(*flat), C.byref(st), seed, 0,
                                             C.byref(self.h)), "create")

    def process(self, events):
        L = self.L
        ev = (L.Event * len(events))()
        for i, e in enumerate(events):
            ev[i] = L.Event(e.type, e.target, e.tokens, e.chain_start, e.now_ms)
        out = (L.Decision * len(events))()
        L.check(L.lib.rr_router_process(self.h, ev, len(events), out), "process")
        return [(d.status, d.deployment, d.served_group, d.chain_pos) for d in out]

    def snapshot(self):
        s = (self.L.DeploymentState * self.n)()
        self.L.check(self.L.lib.rr_router_snapshot(self.h, s), "snapshot")
        return [(x.window, x.req_count, x.tok_count, x.fail_window, x.fail_count, x.inflight,
                 x.cooldown_until_ms, x.total_admitted) for x in s]

    def latency_snapshot(self):
        mean, cnt = (C.c_double * self.n)(), (C.c_int32 * self.n)()
        self.L.check(self.L.lib.rr_router_latency_snapshot(self.h, mean, cnt), "latency_snapshot")
        return list(zip(mean, cnt))

    def close(self):
        self.L.lib.rr_router_destroy(self.h)


def _topology(rng):
    """A 32-deployment group plus a few small ones, shuffled config order, random fallback chains."""
    sizes = [32] + [rng.randrange(1, 6) for _ in range(rng.randrange(1, 4))]
    rng.shuffle(sizes)
    deps = [O.Deployment(group=g, rpm=rng.choice([-1, -1, 3, 10, 40]), tpm=rng.choice([-1, -1, 800, 5000]))
            for g, n in enumerate(sizes) for _ in range(n)]
    rng.shuffle(deps)
    ng = len(sizes)
    fbs = {g: rng.sample(range(ng), rng.randrange(0, min(2, ng) + 1)) for g in range(ng)}
    return deps, ng, fbs


LATENCIES = [0, -7, 40, 40, 80, 120, 400, 1000, 3000]          # few distinct values: equal means happen
# clock steps (ms): mostly short, with rare jumps across the 30 s and the 1 h TTL
STEPS, STEP_W = [0, 1, 5, 50, 500, 20_000, 45_000, 4_000_000], [30, 20, 20, 15, 5, 0.3, 0.15, 0.03]


def _trace(rng, n_groups, n_deps, n, now, random_aux=True):
    ev = []
    for _ in range(n):
        now += rng.choices(STEPS, weights=STEP_W)[0]
        t = rng.choices([O.EV_ADMIT, O.EV_DONE, O.EV_FAIL, O.EV_BURST], weights=[10, 8, 2, 1])[0]
        if t == O.EV_ADMIT:
            ev.append(O.Event(t, rng.randrange(-1, n_groups + 1), rng.randrange(0, 300), rng.choice([0, 0, 0, 1]), now))
        elif t == O.EV_BURST:
            ev.append(O.Event(t, rng.randrange(0, n_groups), rng.randrange(0, 40), 0, now))
        elif t == O.EV_DONE:
            ev.append(O.Event(t, rng.randrange(-1, n_deps + 1), rng.choice([0, 1, 2, 4, 8]),
                              rng.choice(LATENCIES) if random_aux else 0, now))
        else:
            ev.append(O.Event(t, rng.randrange(-1, n_deps + 1), 0, rng.choice([0, 1]) if random_aux else 0, now))
    return ev, now


@pytest.mark.parametrize("global_state", [False, True], ids=["smem", "hbm"])
@pytest.mark.parametrize("ttl_ms", [30_000, 3_600_000])
@pytest.mark.parametrize("buffer_ppm", [0, 100_000, 500_000, 3_000_000])
@pytest.mark.parametrize("list_size", [1, 2, 10, 32])
def test_kernel_matches_oracle_on_random_traces(list_size, buffer_ppm, ttl_ms, global_state, monkeypatch):
    if global_state:
        monkeypatch.setenv("RR_ROUTER_GLOBAL_STATE", "1")           # read by rr_router_create
    else:
        monkeypatch.delenv("RR_ROUTER_GLOBAL_STATE", raising=False)
    seed = list_size * 1009 + buffer_ppm // 1000 + ttl_ms // 1000
    rng = random.Random(seed)
    deps, ng, fbs = _topology(rng)
    st = LatencySettings(strategy=STRATEGY_LATENCY_BASED, enable_pre_call_checks=rng.random() < 0.7,
                         allowed_fails=rng.randrange(0, 4), cooldown_ms=rng.choice([1000, 15000]),
                         latency_list_size=list_size, latency_buffer_ppm=buffer_ppm, latency_ttl_ms=ttl_ms)
    orc = LatencyOracleRouter(deps, ng, fbs, st, seed=seed)
    dev = DevRouter(deps, ng, fbs, st, seed)
    try:
        now, draws = 0, 0
        hot = rng.randrange(len(deps))
        for chunk in range(5):                                     # several launches: state + RNG persist
            ev, now = _trace(rng, ng, len(deps), 900, now)
            if chunk == 4:   # more samples than the list holds for one deployment, then picks in its group
                ev += [O.Event(O.EV_DONE, hot, rng.choice([0, 1, 3]), rng.choice(LATENCIES[2:]), now)
                       for _ in range(list_size + 5)]
                ev += [O.Event(O.EV_ADMIT, deps[hot].group, 1, 0, now) for _ in range(40)]
            want = [d.as_tuple() for d in orc.process(ev)]
            got = dev.process(ev)
            assert got == want, next((i, ev[i], g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w)
            assert dev.snapshot() == orc.snapshot()
            assert dev.latency_snapshot() == orc.latency_snapshot()
            draws += sum(1 for e, d in zip(ev, want) if e.type == O.EV_ADMIT and d[0] == O.RR_OK)
        assert draws > 624                                         # the MT19937 twist ran on the device
        assert orc.latency_snapshot()[hot][1] == list_size         # the list rule's replace branch ran
    finally:
        dev.close()


@pytest.mark.parametrize("strategy", [0, 1, 2, 3, 4])
def test_other_strategies_ignore_the_latency_fields(strategy):
    """Random aux values on DONE / FAIL (and non-default latency settings) change nothing for strategies 0-4."""
    rng = random.Random(strategy + 100)
    deps, ng, fbs = _topology(rng)
    for d in deps:
        d.weight = rng.choice([1, 2, 5])
    st = LatencySettings(strategy=strategy, enable_pre_call_checks=True, allowed_fails=1, cooldown_ms=5000,
                         latency_list_size=3, latency_buffer_ppm=250_000, latency_ttl_ms=1000)
    plain = LatencySettings(strategy=strategy, enable_pre_call_checks=True, allowed_fails=1, cooldown_ms=5000)
    orc = O.OracleRouter(deps, ng, fbs, O.Settings(strategy=strategy, enable_pre_call_checks=True, allowed_fails=1,
                                                   cooldown_ms=5000), seed=3)
    with_aux, zeroed = DevRouter(deps, ng, fbs, st, 3), DevRouter(deps, ng, fbs, plain, 3)
    try:
        now = 0
        for _ in range(3):
            ev, now = _trace(rng, ng, len(deps), 800, now)
            ev0 = [O.Event(e.type, e.target, e.tokens, e.chain_start if e.type in (O.EV_ADMIT, O.EV_BURST) else 0,
                           e.now_ms) for e in ev]
            got = with_aux.process(ev)
            assert got == zeroed.process(ev0) == [d.as_tuple() for d in orc.process(ev0)]
            assert with_aux.snapshot() == zeroed.snapshot() == orc.snapshot()
            assert with_aux.latency_snapshot() == [(0.0, 0)] * len(deps)
    finally:
        with_aux.close()
        zeroed.close()


# ---------------------------------------------------------------- native gateway, real engines
def _oracle_for(r, seed=0):
    cfg = r.cfg
    deps = [O.Deployment(d.group, rpm=d.rpm, tpm=d.tpm, weight=d.weight) for d in cfg.deployments]
    st = LatencySettings(strategy=cfg.strategy_id, enable_pre_call_checks=cfg.enable_pre_call_checks,
                         allowed_fails=cfg.allowed_fails, cooldown_ms=int(round(cfg.cooldown_time * 1000)),
                         latency_list_size=cfg.latency_list_size, latency_buffer_ppm=cfg.latency_buffer_ppm,
                         latency_ttl_ms=cfg.latency_ttl_ms)
    return LatencyOracleRouter(deps, len(cfg.groups), dict(cfg.fallbacks), st, seed=seed)


def test_gateway_routes_to_the_faster_replica_and_avoids_a_timed_out_one(capsys):
    from rr_b200 import APITimeoutError, Engine, EngineBackend, Router, SPECS, make_weights
    fast = Engine(make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda"), max_batch=8, ctx_max=256,
                  max_prefill_tokens=512)
    slow = Engine(make_weights(SPECS["llama-3-8b-2l"], seed=2, sigma=0.02, device="cuda"), max_batch=8, ctx_max=256,
                  max_prefill_tokens=512)
    for eng in (fast, slow):                                       # start-up costs stay out of the samples
        eng.wait(eng.submit(list(range(3, 40)), 32), timeout=60)
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny@fast", "gpu": 0}},
          {"model_name": "chat", "litellm_params": {"model": "b200/llama-3-8b-2l@slow", "gpu": 1}}]
    r = Router(model_list=ml, routing_strategy="latency-based-routing", allowed_fails=1000,
               routing_strategy_args={"lowest_latency_buffer": 0, "max_latency_list_size": 10, "ttl": 3600},
               backends={0: EngineBackend(fast), 1: EngineBackend(slow)}, seed=0)
    r.record_trace = 4096
    prompt = list(range(3, 40))
    try:
        first = [r.completion(model="chat", prompt_ids=prompt, max_tokens=32, timeout=60)._deployment for _ in range(2)]
        assert sorted(first) == [0, 1]                             # unmeasured deployments are tried first
        later = [r.completion(model="chat", prompt_ids=prompt, max_tokens=32, timeout=60)._deployment for _ in range(8)]
        assert later == [0] * 8
        lat = r.latency_snapshot()
        assert lat[0][1] == 9 and lat[1][1] == 1
        ratio = lat[1][0] / lat[0][0]
        with capsys.disabled():
            print(f"\n[latency routing] us per output token: tiny {lat[0][0]:.1f}, llama-3-8b-2l {lat[1][0]:.1f} "
                  f"(x{ratio:.2f})")
        assert ratio > 1.5          # H100 80GB HBM3, 400 W power limit: 80-84 vs 715-716 us / token, 8.5-9x
        # a timed-out request on the fast deployment: FAIL with the timeout flag -> penalty sample 1e9
        with pytest.raises(APITimeoutError):
            r.completion(model="chat", prompt_ids=list(range(3, 60)), max_tokens=190, timeout=0.002)
        deadline = time.time() + 10
        while time.time() < deadline and fast.stats()["active_rows"] + fast.stats()["queued"] > 0:
            time.sleep(0.01)
            fast.submit([5, 6, 7], 1)                              # keeps the worker stepping so that it sees the cancel
        snap = r.snapshot()                                        # quiesces: the FAIL has been through K1
        assert snap[0]["fail_count"] == 1 and snap[0]["inflight"] == 0
        lat = r.latency_snapshot()
        assert lat[0][1] == 10 and lat[0][0] > 1e8
        assert r.completion(model="chat", prompt_ids=prompt, max_tokens=32, timeout=60)._deployment == 1
        # the recorded trace replays through the oracle: every ADMIT decision and the final latency state
        trace = r.gateway_trace()
        assert any(e[0] == O.EV_FAIL and e[3] == 1 for e, _ in trace)
        assert all(e[3] > 0 for e, _ in trace if e[0] == O.EV_DONE)
        orc = _oracle_for(r)
        n_admit = 0
        for (typ, target, tokens, aux, now_ms), got in trace:
            want = orc.process([O.Event(typ, target, tokens, aux, now_ms)])[0].as_tuple()
            if typ == O.EV_ADMIT:
                assert got == want, (n_admit, got, want)
                n_admit += 1
        assert n_admit == 12
        assert r.latency_snapshot() == orc.latency_snapshot()
    finally:
        r.close()
        fast.close()
        slow.close()


# ---------------------------------------------------------------- native gateway, mock replicas (StubBackend)
def test_stub_replicas_post_latencies():
    from rr_b200 import APIError, Router, StubBackend
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny@a", "gpu": 0}},
          {"model_name": "chat", "litellm_params": {"model": "b200/tiny@b", "gpu": 1}},
          {"model_name": "spill", "litellm_params": {"model": "b200/tiny@c", "gpu": 2}}]
    r = Router(model_list=ml, routing_strategy="latency-based-routing", fallbacks=[{"chat": ["spill"]}],
               allowed_fails=1000, routing_strategy_args={"lowest_latency_buffer": 10, "max_latency_list_size": 32},
               backends={0: StubBackend(), 1: StubBackend(), 2: StubBackend(fail_every=2)}, seed=1)
    r.record_trace = 4096

    def events():
        return [e for e, _ in r.gateway_trace()]
    try:
        for _ in range(5):
            r.completion(model="chat", prompt_ids=[5, 6, 7], max_tokens=4)
        out = r.completion_batch("chat", [[5, 6, 7]] * 6, 4)
        assert all(not isinstance(o, Exception) for o in out)
        toks = [t for _, t, _, _ in r.completion_stream(model="chat", prompt_ids=[5, 6], max_tokens=3)]
        assert sum(len(t) for t in toks) == 3
        lat = r.latency_snapshot()
        assert lat[0][1] + lat[1][1] == 12 and lat[2] == (0.0, 0)
        assert all(m > 0.0 for m, n in lat[:2] if n)
        dones = [e for e in events() if e[0] == O.EV_DONE]
        assert len(dones) == 12 and all(e[3] >= 1 for e in dones)
        # a backend failure is not a timeout: FAIL without the flag, no sample
        r.completion(model="spill", prompt_ids=[5], max_tokens=2)
        n_before = len(events())
        with pytest.raises(APIError):
            r.completion(model="spill", prompt_ids=[5], max_tokens=2)
        fails = [e for e in events() if e[0] == O.EV_FAIL]
        assert len(fails) == 1 and fails[0][3] == 0
        assert r.latency_snapshot()[2][1] == 1
        # the failing request: ADMIT, FAIL, re-ADMIT one step down the chain, rejected (no fallback for `spill`)
        spill = r.gateway_trace()[n_before:]
        assert [(e[0], e[3]) for e, _ in spill] == [(O.EV_ADMIT, 0), (O.EV_FAIL, 0), (O.EV_ADMIT, 1)]
        assert spill[0][1][0] == 0 and spill[2][1][0] != 0
    finally:
        r.close()
