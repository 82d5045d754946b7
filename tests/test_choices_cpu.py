"""CPU: the `n` request field (several choices per request) -- its validation, the HTTP front with a fake router, and the
shape of an n-choice response (indices, usage counted as OpenAI and litellm count it)."""
import types

import numpy as np
import pytest
from starlette.testclient import TestClient

from rr_b200.router import (BadRequestError, Choice, Message, ModelResponse, Router, Usage, check_n)
from rr_b200.server import create_app


def test_check_n_accepts_openai_range_only():
    assert check_n(None) == 1
    for n in (1, 2, 64, 128):
        assert check_n(n) == n
    for bad in (True, False, 2.0, 0, -1, 129, "3", [2]):
        with pytest.raises(BadRequestError):
            check_n(bad)


class _Cfg:
    groups = ["g"]
    deployments = []


class _Router:
    """Records the keyword arguments each completion call gets; replies with one choice per requested `n`."""
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def completion(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        n = kw.get("n") or 1
        ch = [Choice(i, Message("assistant", "ab"[i % 2])) for i in range(n)]
        return ModelResponse("chatcmpl-1", "m", ch, Usage(3, 2 * n, 3 + 2 * n))

    def completion_stream(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        yield "m", [3 + ord("h")], False, 0.01
        yield "m", [], True, 0.01


def test_http_forwards_n_only_when_present_and_rejects_bad_values():
    r = _Router()
    c = TestClient(create_app(r))
    body = {"model": "g", "messages": [{"role": "user", "content": "x"}]}
    assert c.post("/chat/completions", json=body).status_code == 200
    assert r.calls[-1] == {}                                       # absent: the router is called exactly as before
    res = c.post("/chat/completions", json=dict(body, n=3))
    assert res.status_code == 200 and r.calls[-1] == {"n": 3}
    assert [ch["index"] for ch in res.json()["choices"]] == [0, 1, 2]
    n_calls = len(r.calls)
    for bad in (0, 129, 2.5, True, "2"):
        res = c.post("/chat/completions", json=dict(body, n=bad))
        assert res.status_code == 400 and "`n`" in res.json()["error"]["message"], bad
    res = c.post("/chat/completions", json=dict(body, n=2, stream=True))
    assert res.status_code == 400 and "stream" in res.json()["error"]["message"]
    assert len(r.calls) == n_calls                                 # refused before the router is called
    res = c.post("/chat/completions", json=dict(body, n=1, stream=True))
    assert res.status_code == 200 and r.calls[-1] == {"n": 1}


def test_n_choice_response_counts_the_prompt_once():
    """Router._gw_response, the shaping of every gateway result, over a fake result of 3 choices of 4 tokens."""
    from rr_b200.config import build_config
    cfg = build_config([{"model_name": "g", "litellm_params": {"model": "b200/tiny", "gpu": 0, "prefix_cache": True}}], {})
    fake = types.SimpleNamespace(cfg=cfg)
    fake._usage = lambda *a: Router._usage(fake, *a)
    res = types.SimpleNamespace(deployment=0, served_group=0, chain_pos=0, n_generated=4, n_cached=64,
                                t_first_token_s=1.0, t_submit_s=0.5)
    toks = np.array([[3 + ord(ch) for ch in w] + [0] for w in ("abcd", "efgh", "ijkl")], dtype=np.int32)
    out = Router._gw_response(fake, res, toks, 100, 0.0, logprobs=[{"content": [i]} for i in range(3)])
    d = out.model_dump()
    assert [c["index"] for c in d["choices"]] == [0, 1, 2]
    assert [c["message"]["content"] for c in d["choices"]] == ["abcd", "efgh", "ijkl"]
    assert [c["logprobs"] for c in d["choices"]] == [{"content": [i]} for i in range(3)]
    assert all(c["finish_reason"] == "length" for c in d["choices"])
    assert d["usage"] == {"prompt_tokens": 100, "completion_tokens": 12, "total_tokens": 112,
                          "prompt_tokens_details": {"cached_tokens": 64}}
    assert out._token_ids == toks[0, :4].tolist() and out._choice_token_ids == toks[:, :4].tolist()
    one = Router._gw_response(fake, res, toks[1], 100, 0.0)                   # one choice: the n=1 shape
    assert len(one.choices) == 1 and one._token_ids == toks[1, :4].tolist() and one.usage.completion_tokens == 4
