"""GPU: the native per-request path (csrc/rr_gateway.cu) -- concurrent Router.completion() callers coalesced into shared
K1 launches, admitted prompts handed to the engines without a Python hop, fallback walk / cancel / timeout inside the
library.  The admission trace the gateway recorded is replayed through the CPU oracle (oracle/router.py): decisions must
be bit-exact, which is the parity statement for the reference's concurrent dispatch loops
(reference src/demo_load_balancing.py:195-203, src/demo_fallback.py:212-220, src/demo_quota_isolation.py:135-139)."""
import threading
import time

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("rpm_window")]


def _oracle_for(r, seed=0):
    from oracle import router as O
    cfg = r.cfg
    deps = [O.Deployment(d.group, rpm=d.rpm, tpm=d.tpm, weight=d.weight) for d in cfg.deployments]
    return O.OracleRouter(deps, len(cfg.groups), dict(cfg.fallbacks),
                          O.Settings(strategy=cfg.strategy_id, enable_pre_call_checks=cfg.enable_pre_call_checks,
                                     allowed_fails=cfg.allowed_fails, cooldown_ms=int(round(cfg.cooldown_time * 1000))),
                          seed=seed)


def _replay(r, trace, seed=0):
    """Run the recorded events through the oracle; compare every decision."""
    from oracle import router as O
    orc = _oracle_for(r, seed)
    n_admit = 0
    for (typ, target, tokens, chain_start, now_ms), got in trace:
        want = orc.process([O.Event(typ, target, tokens, chain_start, now_ms)])[0].as_tuple()
        if typ == 0:
            assert got == want, (n_admit, got, want)
            n_admit += 1
    return n_admit


def _tiny_engine(**kw):
    from rr_b200 import Engine, SPECS, make_weights
    w = make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda")
    return Engine(w, max_batch=8, ctx_max=256, max_prefill_tokens=512, **kw)


def test_concurrent_callers_are_coalesced_and_decisions_replay_bit_exact():
    from rr_b200 import EngineBackend, RateLimitError, Router
    eng = _tiny_engine()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}, "rpm": 40, "tpm": 100000},
          {"model_name": "chat", "litellm_params": {"model": "b200/tiny@b", "gpu": 0}, "rpm": 15},
          {"model_name": "spill", "litellm_params": {"model": "b200/tiny-spill", "gpu": 0}, "rpm": 30}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", enable_pre_call_checks=True, fallbacks=[{"chat": ["spill"]}],
               backends={0: EngineBackend(eng)}, seed=0)
    r.record_trace = 4096
    N = 96
    out, lock = [None] * N, threading.Lock()
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, 1000, size=int(rng.randint(4, 40))).tolist() for _ in range(N)]

    def work(i):
        try:
            out[i] = r.completion(model="chat", prompt_ids=prompts[i], max_tokens=4, timeout=120)
        except RateLimitError as e:
            out[i] = e
    ths = [threading.Thread(target=work, args=(i,)) for i in range(N)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    ok = [o for o in out if not isinstance(o, Exception)]
    assert len(ok) == 85 and len(out) - len(ok) == 11            # rpm 40 + 15 + 30 admit 85 of 96
    assert all(len(o._token_ids) == 4 for o in ok)
    assert sum(o._fell_back for o in ok) == 30 and all(o.model == "tiny-spill" for o in ok if o._fell_back)
    snap = r.snapshot()                                            # quiesces: every DONE report has been through K1
    assert sum(s["inflight"] for s in snap) == 0 and sum(s["total_admitted"] for s in snap) == 85
    st = r.gateway_stats()
    assert st["submitted"] == N and st["admitted"] == 85 and st["rate_limited"] == 11 and st["completed"] == 85
    assert st["events"] == N + 85                                  # one ADMIT per request + one DONE per completion
    assert st["launches"] < st["events"]                           # concurrent admissions shared launches
    trace = r.gateway_trace()
    assert len(trace) == st["events"] and _replay(r, trace) == N
    # same prompt, same greedy tokens whichever deployment label served it
    by_prompt = {}
    for i, o in enumerate(out):
        if not isinstance(o, Exception):
            by_prompt.setdefault(tuple(prompts[i]), set()).add(tuple(o._token_ids))
    assert all(len(v) == 1 for v in by_prompt.values())
    r.close(); eng.close()


def _failures_walk_the_chain(bad, good):
    """BASELINE config #4 shape: primary replica `bad` fails about half its requests, fallback replica `good` is healthy.
    Checks the fallback walk inside the library and returns how many requests fell back."""
    from rr_b200 import APIError, RateLimitError, Router
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    now = [7000.0]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends={0: bad, 1: good}, seed=0, clock=lambda: now[0])
    r.record_trace = 4096
    outs = r.completion_batch("primary", [list(range(3, 20))] * 40, 3)
    assert all(not isinstance(o, Exception) for o in outs)
    n_fb = sum(o._fell_back for o in outs)
    assert 8 <= n_fb <= 32 and all((o.model == "tiny-backup") == o._fell_back for o in outs)
    assert len({tuple(o._token_ids) for o in outs}) == 1           # both replicas hold the same weights
    snap = r.snapshot()
    assert snap[0]["fail_count"] == n_fb and sum(s["inflight"] for s in snap) == 0
    st = r.gateway_stats()
    assert st["failed_over"] == n_fb and st["completed"] == 40 and st["failed"] == 0
    trace = r.gateway_trace()
    assert _replay(r, trace) == 40 + n_fb                          # every re-admission is an ADMIT with chain_start = 1
    assert sum(1 for e, _ in trace if e[0] == 0 and e[3] == 1) == n_fb
    # no fallback left: the error is a backend failure (500), not a 429
    r2 = Router(model_list=ml[:1], backends={0: bad}, seed=0, clock=lambda: now[0], allowed_fails=1000)
    res = r2.completion_batch("primary", [list(range(3, 20))] * 20, 2)
    errs = [o for o in res if isinstance(o, Exception)]
    assert errs and all(isinstance(e, APIError) and not isinstance(e, RateLimitError) and e.status_code == 500 for e in errs)
    assert sum(s["inflight"] for s in r2.snapshot()) == 0
    r2.close(); r.close()
    return n_fb


def test_backend_failures_walk_the_chain_inside_the_library():
    """Engine replicas: the primary has a seeded 50 % failure mask."""
    from rr_b200 import EngineBackend
    bad, good = _tiny_engine(fail_prob=0.5, fail_seed=42), _tiny_engine()
    try:
        _failures_walk_the_chain(EngineBackend(bad), EngineBackend(good))
    finally:
        bad.close(); good.close()


def test_mock_replica_failures_walk_the_chain_inside_the_library():
    """Mock replicas take the same native path: the primary fails every second request handed to it, exactly."""
    from rr_b200 import StubBackend
    assert _failures_walk_the_chain(StubBackend(fail_every=2), StubBackend()) == 20


def test_mock_replica_descriptors_are_checked_and_a_logprobs_struct_refused():
    """rr_gateway_create refuses a NULL engine without a valid rr_stub_desc and creates nothing; a gateway with a mock
    replica refuses logprobs at submit (no logits to fill the pairs from) and serves its fixed reply."""
    import ctypes as C
    from rr_b200 import Router, StubBackend, _lib
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}]
    r = Router(model_list=ml, backends={0: StubBackend()}, seed=0)
    try:
        engs, reps, gw = (C.c_void_p * 1)(), (C.c_int32 * 1)(0), C.c_void_p()
        assert _lib.lib.rr_gateway_create(r._h, engs, reps, 1, None, None, C.byref(gw)) == 4
        for bad in ((-1, 0, 100, 0), (8, -1, 100, 0), (8, 0, 0, 0)):
            stubs = (_lib.StubDesc * 1)(_lib.StubDesc(*bad))
            assert _lib.lib.rr_gateway_create(r._h, engs, reps, 1, stubs, None, C.byref(gw)) == 4
        assert not gw.value
        ids, t = (C.c_int32 * 3)(5, 6, 7), C.c_uint64()
        lp = _lib.GenParams(n_choices=1, top_logprobs=0, top_p=1.0)
        assert _lib.lib.rr_gateway_submit(r._gateway(), 0, ids, 3, 4, C.byref(lp), C.byref(t)) == 4
        assert _lib.lib.rr_gateway_submit(r._gateway(), 0, ids, 3, 4, None, C.byref(t)) == 0
        res, toks = _lib.GatewayResult(), (C.c_int32 * 4)()
        assert _lib.lib.rr_gateway_wait(r._gateway(), t.value, 30.0, C.byref(res), toks, 4, None, None, None, None) == 0
        assert list(toks) == [3, 4, 5, 6] and res.n_generated == 4 and res.deployment == 0
    finally:
        r.close()


def test_bad_requests_are_rejected_before_any_debit_and_timeouts_release_the_row():
    from rr_b200 import APITimeoutError, BadRequestError, EngineBackend, Router
    eng = _tiny_engine()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}, "rpm": 1000}]
    r = Router(model_list=ml, enable_pre_call_checks=True, backends={0: EngineBackend(eng)}, seed=0)
    with pytest.raises(BadRequestError):                           # 250 + 64 > ctx_max 256: HTTP 400, not an unhandled 500
        r.completion(model="chat", prompt_ids=list(range(3, 253)), max_tokens=64)
    with pytest.raises(BadRequestError):
        r.completion(model="chat", prompt_ids=[5, 99999], max_tokens=4)         # id outside the vocabulary
    with pytest.raises(BadRequestError):
        r.completion(model="nope", prompt_ids=[5], max_tokens=4)
    snap = r.snapshot()
    assert snap[0]["total_admitted"] == 0 and snap[0]["inflight"] == 0
    # a request that cannot finish inside its timeout: the caller gets 408, the decode row is given back, the deployment
    # gets a FAIL event (what litellm does with a timed-out call)
    with pytest.raises(APITimeoutError):
        r.completion(model="chat", prompt_ids=list(range(3, 60)), max_tokens=190, timeout=0.002)
    deadline = time.time() + 10
    while time.time() < deadline and eng.stats()["active_rows"] + eng.stats()["queued"] > 0:
        time.sleep(0.01)
        eng.submit([5, 6, 7], 1)                                   # keeps the worker stepping so that it sees the cancel
    snap = r.snapshot()
    assert snap[0]["inflight"] == 0 and snap[0]["fail_count"] == 1
    ok = r.completion(model="chat", prompt_ids=[5, 6, 7], max_tokens=3, timeout=60)
    assert len(ok._token_ids) == 3
    r.close(); eng.close()


def test_stream_close_releases_the_request():
    from rr_b200 import EngineBackend, Router
    eng = _tiny_engine()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}]
    r = Router(model_list=ml, routing_strategy="least-busy", backends={0: EngineBackend(eng)}, seed=0)
    full = [t for _, toks, _, _ in r.completion_stream(model="chat", prompt_ids=[9, 8, 7, 6], max_tokens=12) for t in toks]
    assert len(full) == 12
    assert full == r.completion(model="chat", prompt_ids=[9, 8, 7, 6], max_tokens=12)._token_ids
    gen = r.completion_stream(model="chat", prompt_ids=[9, 8, 7, 6], max_tokens=200)
    label, toks, done, _ = next(gen)
    assert label == "tiny" and toks and not done
    gen.close()                                                    # SSE client went away after the first chunk
    deadline = time.time() + 10
    while time.time() < deadline and sum(s["inflight"] for s in r.snapshot()) > 0:
        time.sleep(0.01)
    snap = r.snapshot()
    assert snap[0]["inflight"] == 0 and snap[0]["fail_count"] == 0  # a disconnect is not a backend failure
    assert r.gateway_stats()["in_flight"] == 0
    r.close(); eng.close()
