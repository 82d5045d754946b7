"""CPU: the `stop` request field -- its validation, the oracle of the byte-matching contract on hand-written cases, the
HTTP front with a recording router, and the ctypes side of the calls it added."""
import ctypes as C
import gc
import json

import numpy as np
import pytest
from starlette.testclient import TestClient

from rr_b200.router import (BadRequestError, Choice, Message, ModelResponse, StreamItem, Usage, check_stop, gen_args)
from rr_b200.server import create_app
from stop_oracle import stop_cut, stop_scan, visible


def T(s):
    """Token ids of a text, as the byte tokenizer gives them."""
    return [3 + b for b in (s.encode() if isinstance(s, str) else s)]


def test_check_stop_accepts_openai_shapes_only():
    assert check_stop(None) == [] and check_stop([]) == []
    assert check_stop("\n\n") == [b"\n\n"]
    assert check_stop(["a", "bc", "é", "x" * 64]) == [b"a", b"bc", "é".encode(), b"x" * 64]
    for bad, word in ((3, "string"), ([b"a"], "string"), (["a", 1], "string"), ({"a": 1}, "string"), ("", "empty"),
                      (["a", ""], "empty"), (["a"] * 5, "4"), ("x" * 65, "64"), ("é" * 33, "64")):
        with pytest.raises(BadRequestError) as ei:
            check_stop(bad)
        assert ei.value.status_code == 400 and word in ei.value.message, bad


def test_gen_args_fills_the_stop_fields_and_keeps_the_rest_plain():
    plain = gen_args().params
    for p in (plain, gen_args(stop=[]).params):
        assert p.n_stop == 0 and not p.stop_bytes and not p.stop_off
    g = gen_args(stop=[b"ab", b"c"]).params
    same = ("n_choices", "top_logprobs", "temperature", "top_p", "seed", "frequency_penalty", "presence_penalty", "n_bias",
            "response_format")
    assert [getattr(g, f) for f in same] == [getattr(plain, f) for f in same] and not g.bias_ids
    assert g.n_stop == 2 and bytes(g.stop_bytes[:3]) == b"abc" and g.stop_off[:3] == [0, 2, 3]


def test_gen_args_struct_keeps_its_arrays_alive():
    g = gen_args(stop=[b"ab", b"c"], bias_ids=[5, 9], bias_vals=[1.5, -2.0]).params
    gc.collect()
    junk = [np.full(64, -1, dtype=np.int32) for _ in range(256)]      # takes the memory of any array freed above
    assert g.bias_ids[:2] == [5, 9] and g.bias_vals[:2] == [1.5, -2.0] and len(junk) == 256
    assert bytes(g.stop_bytes[:3]) == b"abc" and g.stop_off[:3] == [0, 2, 3]


def test_oracle_cuts_at_the_first_match_and_keeps_what_precedes_it():
    assert stop_cut(T("hello world"), [b"o w"]) == (4, True)
    assert stop_cut(T("hello"), [b"xyz"]) == (5, False)
    assert stop_cut(T("hello"), []) == (5, False)
    assert stop_cut(T("hello"), [b"h"]) == (0, True)                     # the first token: nothing is returned
    assert stop_cut(T("hello"), [b"o"]) == (4, True)                     # the last token
    assert stop_cut(T("ab"), [b"abc"]) == (2, False)                     # a stop longer than the reply
    # the generation ends at the first point where a sequence is complete, whichever sequence that is
    assert stop_cut(T("xabcd"), [b"abcd", b"bc"]) == (2, True)


def test_oracle_overlapping_sequences_take_the_earliest_start():
    # "aa" completes first, at the second a
    assert stop_cut(T("xaaa"), [b"aa", b"aaa"]) == (1, True)
    # both end at the same token: the longer one starts earlier and decides the cut
    assert stop_scan(T("xbab"), [b"ab", b"bab"])[-1] == (1, 0)
    assert stop_scan(T("xbab"), [b"ab"])[-1] == (2, 0)
    # a self-overlapping sequence: the partial match falls back to its own border instead of breaking
    scan = stop_scan(T("abaabab"), [b"abab"])
    assert [c for c, _ in scan] == [-1] * 6 + [3]
    assert [h for _, h in scan[:6]] == [1, 2, 3, 1, 2, 3]


def test_oracle_byteless_tokens_and_aliased_ids():
    # ids 0..2 add no byte: they cannot complete a match, sit inside one without breaking it, and are kept before one
    toks = [0] + T("a") + [1] + T("b") + [2]
    assert stop_scan(toks, [b"ab"]) == [(-1, 0), (-1, 1), (-1, 2), (1, 0), (-1, 0)]
    assert stop_cut(toks, [b"ab"]) == (1, True)                          # the byteless token before the match is kept
    assert stop_cut([1, 2] + T("b"), [b"b"]) == (2, True)
    # ids >= 259 alias a byte: 3 + 256 + b is byte b
    assert stop_cut([3 + 256 + ord("a"), 3 + 512 + ord("b")], [b"ab"]) == (0, True)
    # a byteless newest token is held with a pending partial match
    assert stop_scan(T("xa") + [0, 0], [b"ab"])[-1] == (-1, 3)


def test_oracle_hold_is_released_when_a_partial_match_breaks():
    toks = T("x\n\ny\nz")
    assert visible(toks, [b"\n\n\n"]) == [1, 1, 1, 4, 4, 6]
    assert [h for _, h in stop_scan(toks, [b"\n\n\n"])] == [0, 1, 2, 0, 1, 0]
    shown = 0
    for v in visible(T("abaabab"), [b"abab"])[:-1]:                       # what is shown (before the hit at the last
        assert v >= shown                                                 # token) is never taken back
        shown = v
    assert shown <= stop_cut(T("abaabab"), [b"abab"])[0]


class _Cfg:
    groups = ["g"]
    deployments = []


class _Router:
    """Records the keyword arguments each call gets; its replies end by a stop sequence."""
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def completion(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        check_stop(kw.get("stop"))
        reason = "stop" if kw.get("stop") else "length"
        return ModelResponse("chatcmpl-1", "m", [Choice(0, Message("assistant", "ab"), reason)], Usage(3, 2, 5))

    def completion_stream(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        yield "m", T("h"), False, 0.01
        last = StreamItem(("m", [], True, 0.01))
        last.finish_reason = "stop" if kw.get("stop") else "length"
        yield last


def _chunks(res):
    return [json.loads(line[6:]) for line in res.text.splitlines() if line.startswith("data: {")]


def test_http_forwards_stop_only_when_present_and_reports_the_finish_reason():
    r = _Router()
    c = TestClient(create_app(r))
    body = {"model": "g", "messages": [{"role": "user", "content": "x"}]}
    res = c.post("/chat/completions", json=body)
    assert res.status_code == 200 and r.calls[-1] == {}                 # absent: the router is called exactly as before
    assert res.json()["choices"][0]["finish_reason"] == "length"
    assert c.post("/chat/completions", json=dict(body, stop=None)).status_code == 200 and r.calls[-1] == {}
    res = c.post("/chat/completions", json=dict(body, stop="\n\n"))
    assert res.status_code == 200 and r.calls[-1] == {"stop": "\n\n"}
    assert res.json()["choices"][0]["finish_reason"] == "stop"
    res = c.post("/chat/completions", json=dict(body, stop=["a", "b"]))
    assert res.status_code == 200 and r.calls[-1] == {"stop": ["a", "b"]}
    n_calls = len(r.calls)
    for bad, word in ((3, "string"), ([1], "string"), ("", "empty"), (["a"] * 5, "4"), ("x" * 65, "64")):
        for extra in ({}, {"stream": True}):
            res = c.post("/chat/completions", json=dict(body, stop=bad, **extra))
            assert res.status_code == 400 and word in res.json()["error"]["message"], bad
    assert len(r.calls) == n_calls                                      # refused before the router is called
    res = c.post("/chat/completions", json=dict(body, stop="h", stream=True))
    assert res.status_code == 200 and r.calls[-1] == {"stop": "h"}
    ch = _chunks(res)
    assert ch[-1]["choices"][0]["finish_reason"] == "stop" and ch[-1]["choices"][0]["delta"] == {}
    assert ch[0]["choices"][0]["finish_reason"] is None and ch[0]["choices"][0]["delta"]["content"] == "h"
    res = c.post("/chat/completions", json=dict(body, stream=True))
    assert _chunks(res)[-1]["choices"][0]["finish_reason"] == "length" and r.calls[-1] == {}


def test_submit_takes_the_stops_in_the_param_struct_and_wait_returns_each_choice():
    from rr_b200 import _lib
    P = _lib.PROTOTYPES
    i32p = C.POINTER(C.c_int32)
    # the sequences go in through the parameter struct; every choice's token count and finish reason come back from wait
    for name in ("rr_engine_submit", "rr_gateway_submit"):
        assert P[name][0] is C.c_int and P[name][1][-2:] == [C.POINTER(_lib.GenParams), C.POINTER(C.c_uint64)]
    for name in ("rr_engine_wait", "rr_gateway_wait"):
        assert P[name][0] is C.c_int and P[name][1][-4:] == [C.POINTER(C.c_float), i32p, i32p, i32p]
    assert len(P["rr_op_stop_match"][1]) == 13
    assert C.sizeof(_lib.Completion) == 48 and C.sizeof(_lib.GatewayResult) == 80
    # the raw arguments are checked before anything is queued: no engine is needed to be refused
    t = C.c_uint64(77)
    p = _lib.GenParams(n_choices=1, top_logprobs=-1, top_p=1.0, n_stop=1)
    assert _lib.lib.rr_engine_submit(None, None, 0, 0, C.byref(p), C.byref(t)) == 4
    assert _lib.lib.rr_gateway_submit(None, 0, None, 0, 0, C.byref(p), C.byref(t)) == 4 and t.value == 77
    assert _lib.lib.rr_op_stop_match(None, 8, None, None, None, None, None, None, None, None, None, 1, None) == 4
