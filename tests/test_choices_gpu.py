"""GPU: several choices per request (`n`), from the engine's fan-out (prompt prefilled once, its KV copied to the other
choices' slots) through the native gateway and the router to the OpenAI endpoint.

The contract is exact: choice i of a request is bit-identical, in tokens and in logprob pairs, to an n=1 request with
seed + i, because a sampled token depends only on the prompt, the weights and the parameters, never on the batch, the
slot or the prefix cache."""
import ctypes as C
import time

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

SAMPLED = dict(temperature=0.8, top_p=0.9, top_logprobs=5, frequency_penalty=0.5,
               logit_bias={7: 5.0, 11: -3.0, 100: 2.0})


def _engine(spec="tiny", B=8, ctx_max=512, **kw):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    w = make_weights(SPECS[spec], seed=5, sigma=0.05, device="cuda")
    return Engine(w, max_batch=B, ctx_max=ctx_max, max_prefill_tokens=1024, **kw)


def _prompt(n, seed=0):
    return np.random.RandomState(seed + n).randint(3, 1000, size=n).tolist()


def _alone(eng, prompt, max_new, seeds, **kw):
    """n=1 requests, one per seed, submitted together."""
    ts = [eng.submit(prompt, max_new, seed=s, **kw) for s in seeds]
    return [eng.wait(t) for t in ts]


@pytest.mark.parametrize("spec", ["tiny", "small", "tiny96"])
def test_each_choice_equals_the_single_request_with_its_seed(spec):
    B, max_new, seed = 8, 6, 2**64 - 2                             # seed + i wraps modulo 2^64
    eng = _engine(spec, B)
    try:
        for L in (1, 63, 64, 65, 300):
            p = _prompt(L)
            for n in (2, 3, B):
                eng.reset_stats()
                rec = eng.wait(eng.submit(p, max_new, seed=seed, n=n, **SAMPLED))
                st = eng.stats()
                assert rec.status == 0 and len(rec.choices) == n and all(len(c) == max_new for c in rec.choices)
                assert st["prefill_tokens"] == L and st["kv_copy_tokens"] == (n - 1) * L
                assert st["generated_tokens"] == n * max_new
                ref = _alone(eng, p, max_new, [(seed + i) % 2**64 for i in range(n)], **SAMPLED)
                for i in range(n):
                    assert rec.choices[i] == ref[i].tokens, (spec, L, n, i)
                    assert rec.choice_logprobs[i] == ref[i].logprobs, (spec, L, n, i)
                assert rec.tokens == rec.choices[0] and rec.logprobs == rec.choice_logprobs[0]
                assert len({tuple(c) for c in rec.choices}) > 1                      # the seeds differ
    finally:
        eng.close()


def test_greedy_choices_are_the_greedy_completion():
    eng = _engine()
    try:
        p = _prompt(70)
        want = eng.wait(eng.submit(p, 12, top_logprobs=3))
        rec = eng.wait(eng.submit(p, 12, n=4, top_logprobs=3))
        assert rec.choices == [want.tokens] * 4 and rec.choice_logprobs == [want.logprobs] * 4
    finally:
        eng.close()


def test_mixed_burst_counts_the_prompt_once():
    eng = _engine()
    try:
        a, x, b = _prompt(40), _prompt(50), _prompt(30)
        want_a, want_b = eng.wait(eng.submit(a, 8)), eng.wait(eng.submit(b, 8, seed=3, temperature=1.0))
        ref = _alone(eng, x, 8, [9, 10, 11], temperature=1.0)
        eng.reset_stats()
        ta, tx, tb = eng.submit(a, 8), eng.submit(x, 8, n=3, seed=9, temperature=1.0), eng.submit(b, 8, seed=3,
                                                                                                 temperature=1.0)
        ra, rx, rb = eng.wait(ta), eng.wait(tx), eng.wait(tb)
        st = eng.stats()
        assert ra.tokens == want_a.tokens and rb.tokens == want_b.tokens
        assert rx.choices == [r.tokens for r in ref]
        assert st["prefill_tokens"] == 40 + 50 + 30 and st["kv_copy_tokens"] == 2 * 50
        assert st["generated_tokens"] == 8 * 5
    finally:
        eng.close()


def test_rows_admission_order_cancel_and_peek_refusal():
    from rr_b200 import _lib
    B = 8
    eng = _engine(B=B, ctx_max=8192)
    try:
        with pytest.raises(_lib.RRError) as ei:
            eng.submit(_prompt(10), 4, n=B + 1)
        assert ei.value.rc == 4
        # n = B while a row is busy: waits for it, and the request behind it does not overtake it
        t1 = eng.submit(_prompt(20), 40)
        tx = eng.submit(_prompt(30), 4, n=B, temperature=1.0, seed=1)
        tq = eng.submit(_prompt(25), 4)
        r1, rx, rq = eng.wait(t1), eng.wait(tx), eng.wait(tq)
        assert r1.status == rx.status == rq.status == 0 and len(rx.choices) == B
        assert rx.t_first_token >= r1.t_done and rq.t_first_token > rx.t_first_token
        # peek refuses an n-choice ticket, which stays in flight
        tc = eng.submit(_prompt(30), 8000, n=4)                     # long enough to be cancelled mid-decode
        n, d = C.c_int32(), C.c_int32()
        assert _lib.lib.rr_engine_peek(eng._h, tc, 0, 0.01, None, 0, C.byref(n), C.byref(d), None, None, None) == 4
        eng.reset_stats()
        deadline = time.time() + 30
        while eng.stats()["active_rows"] != 4 and time.time() < deadline:
            time.sleep(0.005)
        assert eng.stats()["active_rows"] == 4
        assert _lib.lib.rr_engine_cancel(eng._h, tc) == 0
        while eng.stats()["active_rows"] != 0 and time.time() < deadline:
            time.sleep(0.005)
        st = eng.stats()
        assert st["active_rows"] == 0 and 0 < st["generated_tokens"] < 4 * 8000
        rb = eng.wait(eng.submit(_prompt(30), 4, n=B))
        assert rb.status == 0 and len(rb.choices) == B
    finally:
        eng.close()


def test_prefix_cache_with_choices():
    on, off = _engine(prefix_cache=True), _engine()
    try:
        p = _prompt(200)
        kw = dict(temperature=0.7, seed=21, top_logprobs=2)
        outs = []
        for eng in (on, off):
            x = eng.wait(eng.submit(p, 6, n=3, **kw))
            y = eng.wait(eng.submit(p, 6, **kw))
            outs.append((x, y))
        (xo, yo), (xf, yf) = outs
        assert xo.n_cached == 0 and yo.n_cached > 0 and yf.n_cached == 0
        assert xo.choices == xf.choices and xo.choice_logprobs == xf.choice_logprobs
        assert yo.tokens == yf.tokens == xo.choices[0] and yo.logprobs == yf.logprobs
        # an n-request on a cached prompt: the copy to the other choices includes the cached prefix
        z = on.wait(on.submit(p, 6, n=3, **kw))
        assert z.n_cached > 0 and z.choices == xf.choices
    finally:
        on.close(); off.close()


def _router(backends, **kw):
    from rr_b200 import Router
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends=backends, seed=0, clock=lambda: 7000.0, **kw)
    r.record_trace = 4096
    return r


def test_fallback_readmission_gives_the_same_choices_and_the_gateway_caps_n():
    from rr_b200 import BadRequestError, EngineBackend, _lib
    from test_gateway_gpu import _replay
    bad, good, ref = _engine(fail_prob=0.5, fail_seed=42), _engine(), _engine()
    r = _router({0: EngineBackend(bad), 1: EngineBackend(good)})
    try:
        n, max_new = 3, 5
        outs, fell = [], 0
        for k in range(12):
            p = _prompt(20 + k)
            o = r.completion(model="primary", prompt_ids=p, max_tokens=max_new, n=n, temperature=0.9, seed=100 + k,
                             logprobs=True, top_logprobs=2)
            want = ref.wait(ref.submit(p, max_new, n=n, temperature=0.9, seed=100 + k))
            assert o._choice_token_ids == want.choices and o._token_ids == want.choices[0]
            assert [c.index for c in o.choices] == [0, 1, 2] and all(c.logprobs for c in o.choices)
            assert o.usage.prompt_tokens == len(p) and o.usage.completion_tokens == n * max_new
            fell += o._fell_back
        assert 0 < fell < 12
        trace = r.gateway_trace()
        admits = [e for e, _ in trace if e[0] == 0]
        dones = [e for e, _ in trace if e[0] == 1]
        assert len(admits) == 12 + fell and len(dones) == 12 and all(e[2] == n * max_new for e in dones)
        assert _replay(r, trace) == 12 + fell
        with pytest.raises(BadRequestError) as ei:
            r.completion(model="primary", prompt_ids=[5, 6], max_tokens=2, n=9)
        assert "`n`" in str(ei.value)
        t = C.c_uint64()
        ids = (C.c_int32 * 2)(5, 6)
        p = _lib.GenParams(n_choices=9, top_logprobs=-1, top_p=1.0)
        assert _lib.lib.rr_gateway_submit(r._gateway(), 0, ids, 2, 2, C.byref(p), C.byref(t)) == 4
        with pytest.raises(BadRequestError):
            next(r.completion_stream(model="primary", prompt_ids=[5, 6], max_tokens=2, n=2))
    finally:
        r.close(); bad.close(); good.close(); ref.close()


def test_mock_replicas_reply_n_copies_and_fall_back():
    from rr_b200 import StubBackend
    r = _router({0: StubBackend(fail_every=2), 1: StubBackend()})
    try:
        outs = [r.completion(model="primary", prompt_ids=[5, 6, 7], max_tokens=4, n=5) for _ in range(4)]
        assert [o._fell_back for o in outs] == [False, True, False, True]
        for o in outs:
            assert o._choice_token_ids == [[3, 4, 5, 6]] * 5 and o.usage.completion_tokens == 20
        assert [e[2] for e, _ in r.gateway_trace() if e[0] == 1] == [20] * 4
    finally:
        r.close()


def test_endpoint_returns_n_choices():
    from starlette.testclient import TestClient
    from rr_b200 import EngineBackend, Router
    from rr_b200.server import create_app
    eng = _engine()
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, seed=0)
    try:
        c = TestClient(create_app(r))
        body = {"model": "chat", "messages": [{"role": "user", "content": "hello"}], "max_tokens": 5, "temperature": 1.0,
                "seed": 4, "n": 3}
        res = c.post("/v1/chat/completions", json=body)
        assert res.status_code == 200
        d = res.json()
        assert [ch["index"] for ch in d["choices"]] == [0, 1, 2]
        assert d["usage"]["completion_tokens"] == 15 and d["usage"]["total_tokens"] == d["usage"]["prompt_tokens"] + 15
        one = [c.post("/v1/chat/completions", json=dict(body, n=1, seed=4 + i)).json()["choices"][0]["message"]
               for i in range(3)]
        assert [ch["message"] for ch in d["choices"]] == one
        res = c.post("/v1/chat/completions", json=dict(body, n=9))
        assert res.status_code == 400 and "decode rows" in res.json()["error"]["message"]
        assert c.post("/v1/chat/completions", json=dict(body, stream=True)).status_code == 400
    finally:
        r.close(); eng.close()
