"""CPU: the logprobs surface without a device -- argument checks of the new C entry points (they return
RR_INVALID_ARGUMENT before touching the device), OpenAI's validation rules at the HTTP front (400), and the JSON / SSE
shapes through a fake router, parsed by the OpenAI SDK into its ChoiceLogprobs objects."""
import ctypes as C
import json

import pytest
from starlette.testclient import TestClient

from rr_b200.router import (BadRequestError, Choice, Message, ModelResponse, Usage, check_logprobs, detokenize,
                            logprobs_content)
from rr_b200.server import create_app

RR_INVALID_ARGUMENT = 4


def test_logprobs_entry_points_and_unified_calls_validate_before_touching_the_device():
    from rr_b200 import _lib
    L = _lib.lib
    dummy = C.c_void_p(16)                       # never dereferenced: every call below is rejected first
    ok = dict(logits=dummy, ld=128256, rows=64, vocab=128256, top_n=dummy, max_top=20, lp=dummy, ids=dummy)

    def op(**kw):
        a = dict(ok, **kw)
        return L.rr_op_logprobs(a["logits"], a["ld"], a["rows"], a["vocab"], a["top_n"], a["max_top"], a["lp"], a["ids"],
                                None)
    for bad in (dict(logits=None), dict(top_n=None), dict(lp=None), dict(ids=None), dict(rows=0), dict(rows=65536),
                dict(vocab=0), dict(vocab=128260), dict(ld=1003, vocab=1003), dict(max_top=0), dict(max_top=21),
                dict(ld=524292, vocab=524292)):
        assert op(**bad) == RR_INVALID_ARGUMENT, bad
    t = C.c_uint64(77)
    ids = (C.c_int32 * 4)(1, 2, 3, 4)
    p = _lib.GenParams(n_choices=1, top_logprobs=3, top_p=1.0)
    for params in (None, C.byref(p)):
        assert L.rr_engine_submit(None, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
        assert L.rr_gateway_submit(None, 0, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
    assert L.rr_engine_wait(None, 1, 0.0, None, None, 0, None, None, None, None) == RR_INVALID_ARGUMENT
    n, d = C.c_int32(-1), C.c_int32(-1)
    assert L.rr_engine_peek(None, 1, 0, 0.0, None, 0, C.byref(n), C.byref(d), None, None, None) == RR_INVALID_ARGUMENT
    assert L.rr_gateway_wait(None, 1, 0.0, None, None, 0, None, None, None, None) == RR_INVALID_ARGUMENT
    assert L.rr_gateway_peek(None, 1, 0, 0.0, None, 0, C.byref(n), C.byref(d), None, None, None) == RR_INVALID_ARGUMENT
    assert t.value == 77 and (n.value, d.value) == (-1, -1)


def test_validation_follows_openai_rules():
    assert check_logprobs(None, None) is None and check_logprobs(False, None) is None
    assert check_logprobs(True, None) == 0 and check_logprobs(True, 0) == 0 and check_logprobs(True, 20) == 20
    for lp, top in [(False, 3), (None, 3), (True, -1), (True, 21), (True, 2.5), (True, True), (True, "3"), (1, None),
                    ("true", None)]:
        with pytest.raises(BadRequestError):
            check_logprobs(lp, top)


def _content(toks, top):
    pairs = [[(t, -0.25 * (j + 1))] + [(t + 1 + i, -1.0 - i - j) for i in range(max(1, top) - 1)] for j, t in enumerate(toks)]
    return logprobs_content(toks, pairs, top)


class _Cfg:
    groups = ["g"]
    deployments = []


class _FakeRouter:
    """Records what reached it; replies with token ids [h, i] and their logprobs when asked for them."""
    cfg = _Cfg()
    TOKS = [3 + ord("h"), 3 + ord("i")]

    def __init__(self):
        self.calls = []

    def completion(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        top = check_logprobs(kw.get("logprobs", False), kw.get("top_logprobs"))
        lp = None if top is None else {"content": _content(self.TOKS, top), "refusal": None}
        return ModelResponse("chatcmpl-1", "tiny@x", [Choice(0, Message("assistant", detokenize(self.TOKS)), logprobs=lp)],
                             Usage(3, 2, 5))

    def completion_stream(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        top = check_logprobs(kw.get("logprobs", False), kw.get("top_logprobs"))
        for t in self.TOKS:
            yield ("tiny@x", [t], False, 0.01) if top is None else ("tiny@x", [t], False, 0.01, _content([t], top))
        yield ("tiny@x", [], True, 0.01) if top is None else ("tiny@x", [], True, 0.01, [])

    def snapshot(self):
        return []


BODY = {"model": "g", "messages": [{"role": "user", "content": "x"}]}


@pytest.mark.parametrize("stream", [False, True])
def test_server_rejects_invalid_logprobs_with_400(stream):
    r = _FakeRouter()
    c = TestClient(create_app(r))
    for extra in ({"top_logprobs": 3}, {"logprobs": False, "top_logprobs": 3}, {"logprobs": True, "top_logprobs": -1},
                  {"logprobs": True, "top_logprobs": 21}, {"logprobs": True, "top_logprobs": 2.5},
                  {"logprobs": True, "top_logprobs": True}, {"logprobs": "yes"}, {"logprobs": 1}):
        resp = c.post("/chat/completions", json=dict(BODY, stream=stream, **extra))
        assert resp.status_code == 400 and resp.json()["error"]["type"] == "invalid_request_error", extra
    assert r.calls == []                                     # rejected before the router saw anything


def test_json_shape_and_no_key_when_not_requested():
    r = _FakeRouter()
    c = TestClient(create_app(r))
    plain = c.post("/chat/completions", json=BODY).json()
    assert "logprobs" not in plain["choices"][0] and r.calls == [{}]
    assert c.post("/chat/completions", json=dict(BODY, logprobs=False)).json() == dict(plain, id=plain["id"],
                                                                                       created=plain["created"])
    got = c.post("/chat/completions", json=dict(BODY, logprobs=True, top_logprobs=3)).json()["choices"][0]["logprobs"]
    assert r.calls[-1] == {"logprobs": True, "top_logprobs": 3}
    assert got["refusal"] is None and len(got["content"]) == 2
    e = got["content"][0]
    assert e["token"] == "h" and e["bytes"] == [ord("h")] and e["logprob"] == -0.25
    assert len(e["top_logprobs"]) == 3 and e["top_logprobs"][0] == {"token": "h", "logprob": -0.25, "bytes": [ord("h")]}
    zero = c.post("/chat/completions", json=dict(BODY, logprobs=True)).json()["choices"][0]["logprobs"]
    assert all(x["top_logprobs"] == [] for x in zero["content"]) and r.calls[-1] == {"logprobs": True, "top_logprobs": None}


def test_token_fields_follow_the_byte_tokenizer():
    c = logprobs_content([1, 3 + 0xE2, 3 + ord("a")], [[(1, -3.0)], [(3 + 0xE2, -1.0)], [(3 + ord("a"), -0.5)]], 1)
    assert [(x["token"], x["bytes"]) for x in c] == [("", []), ("�", [0xE2]), ("a", [ord("a")])]
    assert [x["top_logprobs"][0]["logprob"] for x in c] == [-3.0, -1.0, -0.5]


def test_sse_chunks_carry_the_logprobs_of_their_delta():
    r = _FakeRouter()
    c = TestClient(create_app(r))
    for lp in (False, True):
        extra = {"logprobs": True, "top_logprobs": 2} if lp else {}
        text = c.post("/chat/completions", json=dict(BODY, stream=True, **extra)).text
        chunks = [json.loads(x[6:]) for x in text.splitlines() if x.startswith("data: ") and x != "data: [DONE]"]
        assert len(chunks) == 3
        if not lp:
            assert all("logprobs" not in ch["choices"][0] for ch in chunks)
            continue
        for ch, t in zip(chunks[:2], "hi"):
            content = ch["choices"][0]["logprobs"]["content"]
            assert [x["token"] for x in content] == [ch["choices"][0]["delta"]["content"]] == [t]
            assert len(content[0]["top_logprobs"]) == 2
        assert chunks[-1]["choices"][0]["logprobs"] is None


def test_openai_sdk_parses_both_shapes():
    from openai.types.chat import ChatCompletion, ChatCompletionChunk
    from openai.types.chat.chat_completion import ChoiceLogprobs
    r = _FakeRouter()
    c = TestClient(create_app(r))
    body = c.post("/chat/completions", json=dict(BODY, logprobs=True, top_logprobs=3)).json()
    cc = ChatCompletion.model_validate(body)
    lp = cc.choices[0].logprobs
    assert isinstance(lp, ChoiceLogprobs) and len(lp.content) == cc.usage.completion_tokens
    assert lp.content[1].token == "i" and lp.content[1].top_logprobs[0].logprob == lp.content[1].logprob
    assert ChatCompletion.model_validate(c.post("/chat/completions", json=BODY).json()).choices[0].logprobs is None
    text = c.post("/chat/completions", json=dict(BODY, stream=True, logprobs=True, top_logprobs=3)).text
    chunks = [ChatCompletionChunk.model_validate(json.loads(x[6:])) for x in text.splitlines()
              if x.startswith("data: ") and x != "data: [DONE]"]
    toks = [e.token for ch in chunks if ch.choices[0].logprobs for e in ch.choices[0].logprobs.content]
    assert toks == ["h", "i"] and chunks[-1].choices[0].logprobs is None
