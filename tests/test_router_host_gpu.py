"""GPU: the reference-facing host interface (Router.completion / OpenAI facade / HTTP gateway / demo drivers) on top of the
device-resident router K1.  Scenarios and expected outcomes are the reference README's (README.md:167-171, 206-213,
262-264); the response `model` field and the 429 mapping follow the demos' call sites
(src/demo_load_balancing.py:116, src/demo_quota_isolation.py:80)."""
import os
import sys
import threading
import time

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("rpm_window")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "config", "config.yaml")


def _stub_router(clock=None, **kw):
    from rr_b200 import Router, StubBackend, load_config
    cfg = load_config(CFG)
    return Router(config=cfg, backends={0: StubBackend(), 1: StubBackend()}, seed=0, clock=clock, **kw)


def test_fallback_scenario_threads():
    from rr_b200 import OpenAI
    r = _stub_router()
    client = OpenAI(r)
    out, lock = [], threading.Lock()

    def work(i):
        resp = client.chat.completions.create(model="claude-sonnet-fallback-demo",
                                              messages=[{"role": "user", "content": f"q{i}"}], timeout=30)
        with lock:
            out.append(resp)
    ths = [threading.Thread(target=work, args=(i,)) for i in range(10)]
    for t in ths:
        t.start(); time.sleep(0.005)
    for t in ths:
        t.join()
    fallback = [o for o in out if "claude-3-5-sonnet" in o.model]
    assert len(out) == 10 and len(fallback) == 7 and all(o._fell_back for o in fallback)
    assert all(o.usage.completion_tokens == 8 and o.choices[0].message.role == "assistant" for o in out)
    assert not any(o.model.startswith("b200/") for o in out)          # provider prefix stripped
    r.close()


def test_load_balancing_and_quota_scenarios():
    from rr_b200 import RateLimitError
    r = _stub_router()
    models = [r.completion(model="claude-sonnet-loadbalance-demo", messages=[{"role": "user", "content": "x"}]).model
              for _ in range(10)]
    counts = sorted(models.count(m) for m in set(models))
    assert counts == [3, 3, 4] and models.count("llama-3-8b@claude-3-5-sonnet") == 4
    ok, limited = {}, {}
    for c in "abc":
        for _ in range(5):
            try:
                r.completion(model=f"consumer-{c}-model", messages=[{"role": "user", "content": "x"}], timeout=10)
                ok[c] = ok.get(c, 0) + 1
            except RateLimitError as e:
                assert e.status_code == 429
                limited[c] = limited.get(c, 0) + 1
    assert ok == {"a": 3, "b": 5, "c": 5} and limited == {"a": 2}
    snap = r.snapshot()
    assert sum(s["inflight"] for s in snap) == 0 and sum(s["total_admitted"] for s in snap) == 23
    r.close()


def test_unknown_model_and_minute_refill_with_injected_clock():
    from rr_b200 import BadRequestError, RateLimitError
    now = [1000.0]
    r = _stub_router(clock=lambda: now[0])
    with pytest.raises(BadRequestError):
        r.completion(model="no-such-group", messages=[])
    for _ in range(3):
        r.completion(model="consumer-a-model", messages=[{"role": "user", "content": "x"}])
    with pytest.raises(RateLimitError):
        r.completion(model="consumer-a-model", messages=[{"role": "user", "content": "x"}])
    now[0] = 1020.0                                    # next wall-clock minute (1020 // 60 = 17)
    assert r.completion(model="consumer-a-model", messages=[{"role": "user", "content": "x"}]).model
    r.close()


def test_backend_failure_walks_fallback_chain_and_cools_down():
    """BASELINE config #4 semantics: injected primary failures are retried on the fallback group; after
    allowed_fails (2) + 1 failures in a minute the primary cools down and is skipped without being tried."""
    from rr_b200 import Router, StubBackend, load_config
    cfg = load_config(CFG)
    bad, good = StubBackend(fail_every=1), StubBackend()
    now = [5000.0]
    r = Router(config=cfg, backends={0: bad, 1: good}, seed=0, clock=lambda: now[0])
    outs = [r.completion(model="claude-sonnet-fallback-demo", messages=[{"role": "user", "content": "x"}]) for _ in range(5)]
    assert all(o._fell_back and "claude-3-5-sonnet" in o.model for o in outs)
    snap = r.snapshot()
    # every admission of the primary is one hand-off to the failing replica
    assert snap[0]["total_admitted"] == 3               # 4th and 5th request never reached the cooling primary
    assert snap[0]["fail_count"] == 3 and snap[0]["cooldown_until_ms"] == int(now[0] * 1000) + 15000
    now[0] += 61.0                                    # past the cooldown AND into a fresh rpm window
    r.completion(model="claude-sonnet-fallback-demo", messages=[{"role": "user", "content": "x"}])
    assert r.snapshot()[0]["total_admitted"] == 4       # cooldown over: the primary is tried again
    r.close()


def test_engine_backed_completion_and_batch():
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    w = make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda")
    eng = Engine(w, max_batch=8, ctx_max=256, max_prefill_tokens=512)
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}, "rpm": 100, "tpm": 400}]
    r = Router(model_list=ml, routing_strategy="least-busy", enable_pre_call_checks=True, backends={0: EngineBackend(eng)})
    a = r.completion(model="chat", messages=[{"role": "user", "content": "What is machine learning?"}], max_tokens=12)
    b = r.completion(model="chat", messages=[{"role": "user", "content": "What is machine learning?"}], max_tokens=12)
    assert a._token_ids == b._token_ids and len(a._token_ids) == 12        # deterministic greedy decode
    assert a.usage.prompt_tokens == len("user: What is machine learning?") + 1
    outs = r.completion_batch("chat", [list(range(5, 40))] * 12, 4)      # tpm 400: 12 x 35 tokens do not fit
    n_ok = sum(not isinstance(o, Exception) for o in outs)
    assert 1 <= n_ok < 12 and all(len(o._token_ids) == 4 for o in outs if not isinstance(o, Exception))
    eng.close(); r.close()


@pytest.mark.skipif(__import__("torch").cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_one_process_two_gpu_replicas_round_robin():
    """The gateway layout of the reference (one server process, `start-gateway.sh:54`) with one replica per GPU:
    a burst over a two-deployment group lands on both engines and every request decodes the same tokens."""
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    engs = []
    for dev in (0, 1):
        w = make_weights(SPECS["tiny"], seed=2, sigma=0.05, device=f"cuda:{dev}")
        engs.append(Engine(w, device=dev, max_batch=8, ctx_max=256, max_prefill_tokens=512))
    ml = [{"model_name": "chat", "litellm_params": {"model": f"b200/tiny@gpu{d}", "gpu": d}} for d in (0, 1)]
    r = Router(model_list=ml, routing_strategy="round-robin", backends={d: EngineBackend(engs[d]) for d in (0, 1)})
    try:
        outs = r.completion_batch("chat", [list(range(7, 60))] * 10, 6)
        assert not any(isinstance(o, Exception) for o in outs)
        assert sorted(o.model for o in outs) == ["tiny@gpu0"] * 5 + ["tiny@gpu1"] * 5
        assert all(o._token_ids == outs[0]._token_ids and len(o._token_ids) == 6 for o in outs)
    finally:
        for e in engs:
            e.close()
        r.close()


def test_http_gateway_with_openai_sdk():
    import openai
    import uvicorn
    from rr_b200.server import create_app
    r = _stub_router()
    port = 18000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(r), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(100):
        if server.started:
            break
        time.sleep(0.05)
    try:
        client = openai.OpenAI(api_key="demo-key", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        got = [client.chat.completions.create(model="consumer-a-model", messages=[{"role": "user", "content": "hi"}], timeout=10)
               for _ in range(3)]
        assert all(g.model == "llama-3-8b@sonnet-3-7" and g.usage.completion_tokens == 8 for g in got)
        with pytest.raises(openai.RateLimitError):
            client.chat.completions.create(model="consumer-a-model", messages=[{"role": "user", "content": "hi"}], timeout=10)
        with pytest.raises(openai.BadRequestError):
            client.chat.completions.create(model="nope", messages=[{"role": "user", "content": "hi"}], timeout=10)
        v1 = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}/v1", max_retries=0)
        assert v1.chat.completions.create(model="consumer-b-model", messages=[{"role": "user", "content": "hi"}]).model
    finally:
        server.should_exit = True
        th.join(10)
        r.close()


def test_demo_drivers_in_process(capsys, monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "demos"))
    import demo_fallback
    import demo_load_balancing
    import demo_quota_isolation
    monkeypatch.setattr(sys, "argv", ["demo", "--stub"])
    assert demo_fallback.main() == {"primary": 3, "fallback": 7, "failed": 0}
    res = demo_load_balancing.main()
    assert res["ok"] == 10 and sorted(res["distribution"].values()) == [3, 3, 4]
    q = demo_quota_isolation.main()
    assert q == {"A": (3, 2), "B": (5, 0), "C": (5, 0)}


def test_streaming_over_http_with_real_replica():
    """SSE through the OpenAI SDK against an engine-backed router: chunks arrive, concatenate to the non-streamed
    completion, and admission errors still map to 429."""
    import openai
    import uvicorn
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    from rr_b200.server import create_app
    w = make_weights(SPECS["tiny"], seed=4, sigma=0.05, device="cuda")
    eng = Engine(w, max_batch=8, ctx_max=256, max_prefill_tokens=512)
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny@stream", "gpu": 0}, "rpm": 3}]
    r = Router(model_list=ml, enable_pre_call_checks=True, backends={0: EngineBackend(eng)}, default_max_tokens=24,
               clock=lambda: 1000.0)                     # frozen clock: the rpm window cannot roll over mid-test
    port = 19000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(r), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(100):
        if server.started:
            break
        time.sleep(0.05)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        msgs = [{"role": "user", "content": "stream me"}]
        full = client.chat.completions.create(model="chat", messages=msgs, timeout=30)
        parts, n_chunks = [], 0
        for ch in client.chat.completions.create(model="chat", messages=msgs, timeout=30, stream=True):
            n_chunks += 1
            assert ch.model == "tiny@stream"
            parts.append(ch.choices[0].delta.content or "")
        # >= 1 content chunk + the closing chunk (a tiny model may finish all 24 tokens before the first poll)
        assert n_chunks >= 2 and "".join(parts) == full.choices[0].message.content
        direct = list(r.completion_stream(model="chat", messages=msgs))
        assert direct[-1][2] is True and sum(len(t) for _, t, _, _ in direct) == 24
        with pytest.raises(openai.RateLimitError):
            client.chat.completions.create(model="chat", messages=msgs, timeout=30, stream=True)   # rpm 3 used up
    finally:
        server.should_exit = True
        th.join(10)
        eng.close(); r.close()
