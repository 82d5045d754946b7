"""CPU: /v1/completions (Router.text_completion, server.py) -- request validation, response formatting from synthetic
engine pairs, and the prompt-logprob entry points' argument checks, which run before anything touches the device."""
import ctypes as C
import math

import numpy as np
import pytest
from starlette.testclient import TestClient

from rr_b200 import _lib
from rr_b200.router import (BadRequestError, Router, _lib as router_lib, check_text_completion, completion_logprobs,
                            detokenize, text_offsets, top_logprobs_dict)
from rr_b200.server import create_app


def _b(s: str):
    """Token ids of the bytes of s (no BOS)."""
    return [3 + b for b in s.encode("utf-8")]


# ---------------------------------------------------------------- validation
@pytest.mark.parametrize("kw, field", [
    (dict(prompt=""), None), (dict(prompt=[]), "prompt"), (dict(prompt=[[]]), "prompt"), (dict(prompt=[1, "a"]), "prompt"),
    (dict(prompt=[[1], 2]), "prompt"), (dict(prompt=[True]), "prompt"), (dict(prompt=None), "prompt"),
    (dict(prompt="x", max_tokens=0), "max_tokens"), (dict(prompt="x", max_tokens=-1), "max_tokens"),
    (dict(prompt="x", echo=True, stream=True), "echo"), (dict(prompt="x", best_of=2), "best_of"),
    (dict(prompt="x", best_of=True), "best_of"), (dict(prompt="x", suffix="s"), "suffix"),
    (dict(prompt="x", logprobs=6), "logprobs"), (dict(prompt="x", logprobs=-1), "logprobs"),
    (dict(prompt="x", logprobs=True), "logprobs"), (dict(prompt="x", logprobs=1.0), "logprobs"),
    (dict(prompt="x", echo="yes"), "echo"),
])
def test_each_refusal_names_its_field(kw, field):
    if field is None:                   # an empty string is a prompt: BOS alone
        assert check_text_completion(**kw) == ([""], None)
        return
    with pytest.raises(BadRequestError) as e:
        check_text_completion(**kw)
    assert f"`{field}`" in e.value.message


def test_the_four_prompt_forms_and_accepted_values():
    assert check_text_completion("ab") == (["ab"], None)
    assert check_text_completion(["a", "b"], logprobs=5) == (["a", "b"], 5)
    assert check_text_completion([1, 2, 3], echo=True, logprobs=0) == ([[1, 2, 3]], 0)
    assert check_text_completion([[1, 2], [3]], max_tokens=1, best_of=1) == ([[1, 2], [3]], None)
    assert check_text_completion("x", stream=True)[0] == ["x"]


# ---------------------------------------------------------------- formatting
def test_text_offset_on_multibyte_and_invalid_utf8():
    toks = [1] + _b("aé€b")            # é = c3 a9, € = e2 82 ac
    text, offs = text_offsets(toks)
    assert text == "aé€b"
    assert offs == [0, 0, 1, 1, 2, 2, 2, 3]
    # an invalid sequence: e2 41 -> U+FFFD, 'A'; a lone continuation byte 80 -> U+FFFD; a truncated tail e2 82
    toks = [1, 3 + 0xE2, 3 + 0x41, 3 + 0x80, 3 + ord("z"), 3 + 0xE2, 3 + 0x82]
    text, offs = text_offsets(toks)
    assert text == b"\xe2A\x80z\xe2\x82".decode("utf-8", errors="replace") == "�A�z�"
    assert offs == [0, 0, 1, 2, 3, 4, 4]


def test_top_logprobs_dict_keeps_the_largest_of_colliding_strings():
    a = 3 + ord("a")
    # ids a and a + 256 (and a + 512) are all the byte "a"
    d = top_logprobs_dict(a + 512, -3.0, [(a, -1.5), (a + 256, -0.5), (3 + ord("b"), -2.0)])
    assert d == {"a": -0.5, "b": -2.0}
    assert top_logprobs_dict(a, -0.25, []) == {"a": -0.25}
    assert top_logprobs_dict(a, -1.0, [(3 + ord("c"), -math.inf)]) == {"a": -1.0}


def test_bos_entry_is_null():
    toks = [1] + _b("hi")
    lp = completion_logprobs(toks, [None, -1.0, -2.0], [None, [(3 + ord("x"), -0.5)], [(3 + ord("i"), -2.0)]])
    assert lp["tokens"] == ["", "h", "i"]
    assert lp["token_logprobs"] == [None, -1.0, -2.0]
    assert lp["top_logprobs"] == [None, {"x": -0.5, "h": -1.0}, {"i": -2.0}]
    assert lp["text_offset"] == [0, 0, 1]


# ---------------------------------------------------------------- Router.text_completion on a fake gateway
class _Dep:
    response_model = "tiny@fake"
    prefix_cache = False


class _Cfg:
    groups = ["g"]
    deployments = [_Dep()]
    routing_strategy = "simple-shuffle"

    def group_index(self, m):
        return 0 if m == "g" else -1


class _Res:
    deployment = 0
    n_cached = 0


def _fake_router(scores):
    """A Router whose gateway calls are replaced: prompt i scores to scores(i, prompt) = (targets, [(ids, lps)] per
    position), and every choice c of it generates [3 + ord("A") + c] with pairs [(tok, -0.1 * (c + 1)), (other, -2)]."""
    r = Router.__new__(Router)
    r.cfg, r.backends, r.default_max_tokens, r._gw = _Cfg(), {}, 4, None
    r._custom_clock = False
    sub = []
    r._gateway = lambda: "gw"

    def submit(gw, g, p, max_new, model, gen, prompt_top=None):
        sub.append((list(p), max_new, prompt_top, gen.params.n_choices, gen.top))
        return len(sub) - 1
    r._gw_submit = submit

    def collect(gw, model, p, ticket, max_new, timeout, gen, score):
        n = gen.params.n_choices
        toks = np.array([[3 + ord("A") + c] + [0] * (max_new - 1) for c in range(n)], dtype=np.int32)
        pairs = None
        if gen.top is not None:
            w = gen.width
            lp, ids = np.zeros((n, max_new, w), np.float32), np.zeros((n, max_new, w), np.int32)
            for c in range(n):
                ids[c, 0, :2] = [3 + ord("A") + c, 3 + ord("B")][:w] if w >= 2 else [3 + ord("A") + c]
                lp[c, 0, :2] = [-0.1 * (c + 1), -2.0][:w] if w >= 2 else [-0.1 * (c + 1)]
            pairs = [(lp[c], ids[c]) for c in range(n)]
        plp = None
        if score is not None:
            tgt, alts = scores(ticket, p)
            plp = ([None] + list(tgt), [None] + [a[:score] for a in alts])
        return "tiny@fake", plp, (_Res(), toks, pairs, [1] * n, [0] * n)
    r._collect_prompt = collect
    return r, sub


def _scores(i, p):
    """Prompt position t: the target's logprob -(t + i) / 10 and the pairs [(target, that), (3, -5.0)]."""
    tgt = [-(t + i) / 10 for t in range(1, len(p))]
    return tgt, [[(p[t], tgt[t - 1]), (3, -5.0)] for t in range(1, len(p))]


def test_prompt_major_choice_indices_usage_and_echo_text():
    r, sub = _fake_router(_scores)
    prompts = [[1] + _b("ab"), [1] + _b("xyz"), [1] + _b("q")]
    resp = r.text_completion("g", prompts, max_tokens=1, echo=True, n=2)
    assert [c.index for c in resp.choices] == list(range(6))
    assert [c.text for c in resp.choices] == ["abA", "abB", "xyzA", "xyzB", "qA", "qB"]
    assert all(c.logprobs is None for c in resp.choices)
    assert [s[2] for s in sub] == [None] * 3 and [s[3] for s in sub] == [2] * 3       # no scoring without logprobs
    u = resp.usage
    assert (u.prompt_tokens, u.completion_tokens, u.total_tokens) == (3 + 4 + 2, 6, 15)
    d = resp.model_dump()
    assert d["object"] == "text_completion" and d["id"].startswith("cmpl-") and d["model"] == "tiny@fake"
    assert set(d["choices"][0]) == {"index", "text", "logprobs", "finish_reason"}


def test_lm_eval_parse_of_echo_logprobs():
    """lm-evaluation-harness's loglikelihood request (max_tokens 1, logprobs 1, echo, temperature 0) and its parse:
    sum(token_logprobs[ctxlen:-1]) and is_greedy from the best key of each top_logprobs entry."""
    r, sub = _fake_router(_scores)
    ctx, cont = [1] + _b("ab"), _b("cd")
    resp = r.text_completion("g", [ctx + cont], max_tokens=1, echo=True, logprobs=1, temperature=0)
    assert sub[0][2] == 1
    lp = resp.choices[0].logprobs
    toks = ctx + cont
    assert lp["tokens"] == [""] + list("abcd") + ["A"]
    assert lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None
    assert lp["text_offset"] == [0, 0, 1, 2, 3, 4]
    ctxlen = len(ctx)
    got = sum(lp["token_logprobs"][ctxlen:-1])
    assert got == pytest.approx(sum(-t / 10 for t in range(ctxlen, len(toks))), abs=1e-6)
    is_greedy = all(max(top, key=top.get) == tok for tok, top in zip(lp["tokens"][ctxlen:-1], lp["top_logprobs"][ctxlen:-1]))
    assert is_greedy
    # the generated token: its own logprob and its one alternative
    assert lp["token_logprobs"][-1] == pytest.approx(-0.1) and lp["top_logprobs"][-1] == {"A": pytest.approx(-0.1)}


def test_logprobs_without_echo_cover_the_completion_only():
    r, sub = _fake_router(_scores)
    resp = r.text_completion("g", "ignored-by-fake" and [[1, 5, 6]], logprobs=2)
    assert sub[0][2] is None and sub[0][4] == 2
    lp = resp.choices[0].logprobs
    assert lp["tokens"] == ["A"] and lp["top_logprobs"] == [{"A": pytest.approx(-0.1), "B": -2.0}]


def test_token_ids_out_of_range_are_refused():
    r, _ = _fake_router(_scores)
    with pytest.raises(BadRequestError, match="`prompt`"):
        r.text_completion("g", [[1, 128256]])


# ---------------------------------------------------------------- HTTP
def test_http_completions_echo_without_logprobs_and_refusals():
    r, _ = _fake_router(_scores)
    c = TestClient(create_app(r))
    for path in ("/completions", "/v1/completions"):
        got = c.post(path, json={"model": "g", "prompt": [[1] + _b("hi"), [1, 3 + ord("k")]], "echo": True,
                                 "max_tokens": 1})
        assert got.status_code == 200, got.text
        j = got.json()
        assert j["object"] == "text_completion" and [ch["text"] for ch in j["choices"]] == ["hiA", "kA"]
        assert [ch["logprobs"] for ch in j["choices"]] == [None, None]
    for body, field in [({"prompt": "x", "echo": True, "stream": True}, "echo"), ({"prompt": "x", "best_of": 3}, "best_of"),
                        ({"prompt": "x", "suffix": "y"}, "suffix"), ({"prompt": "x", "max_tokens": 0}, "max_tokens"),
                        ({"prompt": [], "echo": True}, "prompt"), ({"prompt": "x", "logprobs": 9}, "logprobs")]:
        got = c.post("/v1/completions", json=dict(body, model="g"))
        assert got.status_code == 400 and f"`{field}`" in got.json()["error"]["message"], (body, got.text)
    assert c.post("/v1/completions", json={"model": "g"}).status_code == 400


def test_openai_sdk_parses_the_response():
    """The SDK builds responses without validation (its types say List[float], the API sends null for the first
    token), as openai._models.construct_type does."""
    pytest.importorskip("openai")
    from openai._models import construct_type
    from openai.types import Completion
    r, _ = _fake_router(_scores)
    d = r.text_completion("g", [[1] + _b("ab")], max_tokens=1, echo=True, logprobs=1).model_dump()
    comp = construct_type(type_=Completion, value=d)
    assert comp.choices[0].logprobs.token_logprobs[0] is None
    assert comp.choices[0].logprobs.text_offset == [0, 0, 1, 2]


# ---------------------------------------------------------------- C ABI
def test_entry_points_reject_bad_arguments_before_touching_the_device():
    L = _lib.lib
    t = C.c_uint64(77)
    ids = (C.c_int32 * 3)(1, 2, 3)
    assert L.rr_engine_submit_scored(None, ids, 3, 1, None, 0, C.byref(t)) == 4 and t.value == 77
    assert L.rr_engine_prompt_logprobs(None, 1, 0.0, None, None, None) == 4
    assert L.rr_gateway_submit_scored(None, 0, ids, 3, 1, None, 0, C.byref(t)) == 4 and t.value == 77
    assert L.rr_gateway_prompt_logprobs(None, 1, 0.0, None, None, None) == 4
    # rr_op_prefill_gemm: the fp32 mode is a consumer mode; null pointers are refused first, modes 1 and 4 stay refused
    for mode in (1, 4, 6, 7):
        assert L.rr_op_prefill_gemm(None, 128, 64, 4096, None, 128256, 4096, None, 128256, mode, None, 32, 4096, 1e-5,
                                    None, None, None, 0, None) == 4
    assert router_lib is _lib
    assert all(n in _lib.PROTOTYPES for n in ("rr_engine_submit_scored", "rr_engine_prompt_logprobs",
                                              "rr_gateway_submit_scored", "rr_gateway_prompt_logprobs"))
