"""CPU: JSON mode (`response_format: {"type": "json_object"}`) -- the Python oracle of the byte grammar pinned to Python's
`json` module, the request-field validation, the HTTP front with a recording router, and the ctypes side of the calls."""
import ctypes as C
import json
import random

import pytest
from starlette.testclient import TestClient

import json_oracle as J
from rr_b200.router import (BadRequestError, Choice, Message, ModelResponse, StreamItem, Usage, check_response_format,
                            gen_args, logprobs_content)
from rr_b200.server import create_app


def _reject(name):
    raise ValueError(name)


def loads_dict(data: bytes):
    """json.loads on the strict UTF-8 decode, NaN / Infinity refused: the dict, or None when Python rejects the text."""
    try:
        v = json.loads(data.decode("utf-8"), parse_constant=_reject)
    except (ValueError, UnicodeDecodeError):
        return None
    return v if isinstance(v, dict) else None


_docs = J.random_docs


def _walk(data: bytes):
    """The states before each byte of data and after the last, asserting every byte is accepted."""
    states = [J.initial()]
    for c in data:
        states.append(J.advance(states[-1], c))
    return states


def test_json_dumps_output_is_accepted_byte_by_byte_and_done_exactly_at_the_end():
    for data in _docs(60, 1):
        states = _walk(data)
        assert J.done(states[-1]), data
        assert not any(J.done(s) for s in states[:-1]), data
        for s in states:
            assert J.allowed(s), s                                   # never an empty allowed set
        # trailing whitespace is still a JSON text; anything else after the object is not
        assert J.accepts(data + b" \n", states[0])[1] == len(data) + 2
        assert J.allowed(states[-1]) == set(J.WS)


def test_every_accepted_prefix_completes_to_a_dict():
    for data in _docs(8, 2):
        states = _walk(data)
        for i, s in enumerate(states):
            text = data[:i] + J.completion(s)
            assert loads_dict(text) is not None, text


def test_mutations_are_rejected_exactly_where_python_rejects_them():
    rng = random.Random(3)
    docs = _docs(40, 4)
    agree = rejected = 0
    for _ in range(1500):
        d = bytearray(rng.choice(docs))
        op, i = rng.randint(0, 2), rng.randrange(len(d))
        b = rng.choice([rng.randrange(256), rng.choice(b'{}[]":,\\0123456789.eE+-tfnu \t\n\r')])
        if op == 0:
            d[i] = b
        elif op == 1:
            d.insert(i, b)
        else:
            del d[i]
        data = bytes(d)
        s, k = J.accepts(data)
        ours = k == len(data) and J.done(s)
        assert ours == (loads_dict(data) is not None), data
        agree += 1
        if k < len(data):
            rejected += 1
            assert loads_dict(data[:k] + J.completion(s)) is not None     # everything before the rejected byte is valid
            assert data[k] not in J.allowed(s)
    assert agree == 1500 and rejected > 300


@pytest.mark.parametrize("text", [
    b'{"a":NaN}', b'{"a":Infinity}', b'{"a":-Infinity}', b'{"a":nan}', b'[1]', b'"x"', b'1', b'null', b'\xef\xbb\xbf{}',
    b'{"a":01}', b'{"a":1.}', b'{"a":.5}', b'{"a":1e}', b'{"a":1e+}', b'{"a":+1}', b'{"a":-}', b'{"a":--1}',
    b'{"a":tru}', b'{"a":True}', b'{a:1}', b'{1:1}', b'{"a":1,}', b'{"a" 1}', b'{"a":[1,]}', b'{"a":[1 2]}',
    b'{"a":"\x00"}', b'{"a":"\x1f"}', b'{"a":"\n"}', b'{"\\x":1}', b'{"\\U0041":1}', b'{"\\u12G4":1}', b'{"\\u12":1}',
    b'{"a":"\xc0\x80"}', b'{"a":"\xc1\xbf"}', b'{"a":"\xe0\x80\x80"}', b'{"a":"\xe0\x9f\xbf"}', b'{"a":"\xf0\x80\x80\x80"}',
    b'{"a":"\xf0\x8f\xbf\xbf"}', b'{"a":"\xed\xa0\x80"}', b'{"a":"\xed\xbf\xbf"}', b'{"a":"\xf4\x90\x80\x80"}',
    b'{"a":"\xf5\x80\x80\x80"}', b'{"a":"\xff"}', b'{"a":"\x80"}', b'{"a":"\xc3"}', b'{"a":"\xe2\x82"}',
    b'{"a":"\xc3\xc3"}', b'{} {}', b'{}x', b'{"a":1}}',
])
def test_edge_cases_python_rejects_are_rejected(text):
    s, k = J.accepts(text)
    assert not (k == len(text) and J.done(s))
    assert loads_dict(text) is None


@pytest.mark.parametrize("text", [
    b'{}', b' \t\r\n{ } ', b'{"":""}', b'{"a":0,"b":-0,"c":1.5e-3,"d":1E+10,"e":0.0,"f":-12.5E3}', b'{"a":[]}',
    b'{"a":[{}, [], "", 0, true, false, null]}', b'{"a":"\\" \\\\ \\/ \\b \\f \\n \\r \\t \\u00e9 \\uD83D\\uDE00"}',
    b'{"a":"\x7f\xc2\x80\xdf\xbf\xe0\xa0\x80\xed\x9f\xbf\xee\x80\x80\xef\xbf\xbf\xf0\x90\x80\x80\xf4\x8f\xbf\xbf"}',
    b'{"a":{"a":{"a":{}}}, "a":1}',
])
def test_edge_cases_python_accepts_are_accepted(text):
    s, k = J.accepts(text)
    assert k == len(text) and J.done(s)
    assert loads_dict(text) is not None


def test_depth_cap():
    # 63 more containers inside the top-level object, objects and arrays alternating: 64 open
    text = b'{"a":' + b"".join(b"[" if d % 2 else b'{"": ' for d in range(2, J.MAX_DEPTH + 1))
    s, k = J.accepts(text)
    assert k == len(text) and len(s.stack) == J.MAX_DEPTH
    a = J.allowed(s)
    assert ord("[") not in a and ord("{") not in a and ord('"') in a and ord("0") in a
    s1, _ = J.accepts(text[:-1] if text.endswith(b"[") else text[:-5])
    assert ord("[") in J.allowed(s1) or ord("{") in J.allowed(s1)             # one level less: containers open
    assert loads_dict(text + J.completion(s)) is not None


def test_whitespace_cap():
    for lead in (b"", b'{', b'{"a"', b'{"a":', b'{"a":1', b'{"a":[', b'{"a":[1'):
        s, k = J.accepts(lead + b" " * J.MAX_WS)
        assert k == len(lead) + J.MAX_WS
        a = J.allowed(s)
        assert not (a & J.WS) and a                       # whitespace masked, something else still allowed
        s, k = J.accepts(lead + b"\t" * (J.MAX_WS - 1) + b"\n")
        assert J.allowed(s) & J.WS == set()
    # a run ends at any other byte: two runs of 64 separated by a token are fine
    text = b"{" + b" " * 64 + b'"a"' + b"\n" * 64 + b":" + b"\r" * 64 + b"1" + b" " * 64 + b"}"
    assert J.accepts(text) == (J.accepts(text)[0], len(text)) and J.done(J.accepts(text)[0])
    assert loads_dict(text) is not None


def test_random_walks_never_reach_an_empty_allowed_set():
    rng = random.Random(5)
    seen = 0
    for walk in range(60):
        s = J.initial()
        bias = [None, b"[", b" ", b"\\", b"\xf0", b"e"][walk % 6]
        for _ in range(400):
            a = J.allowed(s)
            assert a, s
            seen += 1
            if J.done(s):
                break
            pick = [c for c in (bias or b"") if c in a]
            c = pick[0] if pick and rng.random() < 0.7 else rng.choice(sorted(a))
            s = J.advance(s, c)
    assert seen > 5000


def test_mask_columns_follow_the_byte_tokenizer():
    s = J.advance(J.initial(), ord("{"))
    m = J.mask_columns(s, 600)
    assert m[0] and m[1] and m[2]
    for c in range(3, 600):
        assert m[c] == (J.token_byte(c) not in {ord('"'), ord("}"), 0x20, 0x09, 0x0A, 0x0D})


def test_check_response_format():
    assert check_response_format(None) is False
    assert check_response_format({"type": "text"}) is False
    assert check_response_format({"type": "json_object"}) is True
    with pytest.raises(BadRequestError) as ei:
        check_response_format({"type": "json_schema", "json_schema": {"name": "x", "schema": {}}})
    assert ei.value.status_code == 400 and "not supported" in ei.value.message and "json_object" in ei.value.message
    for bad in ("json_object", {"type": "xml"}, {}, {"type": None}, ["json_object"], 1, True):
        with pytest.raises(BadRequestError) as ei:
            check_response_format(bad)
        assert ei.value.status_code == 400 and "response_format" in ei.value.message, bad


def test_gen_args_json_object_fills_response_format():
    g, plain = gen_args(json_object=True).params, gen_args().params
    assert g.response_format == 1 and plain.response_format == 0
    for p in (g, plain):              # otherwise a plain request: greedy, one choice, nothing else asked for
        assert (p.n_choices, p.top_logprobs, p.temperature, p.top_p, p.seed, p.frequency_penalty, p.presence_penalty,
                p.n_bias, p.n_stop) == (1, -1, 0.0, 1.0, 0, 0.0, 0.0, 0, 0)
        assert not (p.bias_ids or p.bias_vals or p.stop_bytes or p.stop_off)
    st = gen_args(stop=[b"ab"], json_object=True).params
    assert st.n_stop == 1 and st.response_format == 1


def test_top_logprobs_drop_minus_infinity():
    inf = float("-inf")
    c = logprobs_content([3 + ord("{")], [[(3 + ord("{"), 0.0), (3 + ord(" "), inf), (1, inf)]], 3)
    assert c[0]["logprob"] == 0.0 and [e["logprob"] for e in c[0]["top_logprobs"]] == [0.0]
    json.dumps(c, allow_nan=False)
    c = logprobs_content([10], [[(10, -0.5), (11, -1.0)]], 2)               # finite entries are all kept
    assert [e["logprob"] for e in c[0]["top_logprobs"]] == [-0.5, -1.0]


class _Cfg:
    groups = ["g"]
    deployments = []


class _Router:
    """Records the keyword arguments each call gets; a JSON-mode reply is an object that ended with `stop`."""
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def completion(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        js = check_response_format(kw.get("response_format"))
        return ModelResponse("chatcmpl-1", "m", [Choice(0, Message("assistant", "{}" if js else "ab"),
                                                        "stop" if js else "length")], Usage(3, 2, 5))

    def completion_stream(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        js = check_response_format(kw.get("response_format"))
        yield "m", [3 + ord("{")], False, 0.01
        yield "m", [3 + ord("}")], False, 0.01
        last = StreamItem(("m", [], True, 0.01))
        last.finish_reason = "stop" if js else "length"
        yield last


def _chunks(res):
    return [json.loads(line[6:]) for line in res.text.splitlines() if line.startswith("data: {")]


def test_http_forwards_response_format_only_when_present_and_not_text():
    r = _Router()
    c = TestClient(create_app(r))
    body = {"model": "g", "messages": [{"role": "user", "content": "x"}]}
    js = {"type": "json_object"}
    for extra in ({}, {"response_format": None}, {"response_format": {"type": "text"}}):
        res = c.post("/chat/completions", json=dict(body, **extra))
        assert res.status_code == 200 and r.calls[-1] == {}, extra        # the router is called exactly as before
    res = c.post("/chat/completions", json=dict(body, response_format=js))
    assert res.status_code == 200 and r.calls[-1] == {"response_format": js}
    assert json.loads(res.json()["choices"][0]["message"]["content"]) == {}
    assert res.json()["choices"][0]["finish_reason"] == "stop"
    n_calls = len(r.calls)
    for bad, word in (({"type": "json_schema", "json_schema": {}}, "not supported"), ({"type": "xml"}, "response_format"),
                      ("json_object", "response_format")):
        for extra in ({}, {"stream": True}):
            res = c.post("/chat/completions", json=dict(body, response_format=bad, **extra))
            assert res.status_code == 400 and word in res.json()["error"]["message"], bad
    assert len(r.calls) == n_calls                                          # refused before the router is called
    res = c.post("/chat/completions", json=dict(body, response_format=js, stream=True))
    assert res.status_code == 200 and r.calls[-1] == {"response_format": js}
    ch = _chunks(res)
    assert "".join(x["choices"][0]["delta"].get("content", "") for x in ch) == "{}"
    assert ch[-1]["choices"][0]["finish_reason"] == "stop"
    res = c.post("/chat/completions", json=dict(body, response_format={"type": "text"}, stream=True))
    assert _chunks(res)[-1]["choices"][0]["finish_reason"] == "length" and r.calls[-1] == {}


def test_submit_takes_the_format_in_the_param_struct():
    from rr_b200 import _lib
    P = _lib.PROTOTYPES
    # the format goes in through the parameter struct (its layout: tests/test_abi.py)
    for name in ("rr_engine_submit", "rr_gateway_submit"):
        assert P[name][0] is C.c_int and C.POINTER(_lib.GenParams) in P[name][1]
    assert len(P["rr_op_json_mask"][1]) == 8 and len(P["rr_op_json_advance"][1]) == 9
    # the raw arguments are checked before anything is queued or launched: no engine or GPU is needed to be refused
    t = C.c_uint64(77)
    p = _lib.GenParams(n_choices=1, top_logprobs=-1, top_p=1.0, response_format=1)
    assert _lib.lib.rr_engine_submit(None, None, 0, 0, C.byref(p), C.byref(t)) == 4
    assert _lib.lib.rr_gateway_submit(None, 0, None, 0, 0, C.byref(p), C.byref(t)) == 4 and t.value == 77
    assert _lib.lib.rr_op_json_mask(None, 8, 1, 8, None, None, None, None) == 4
    assert _lib.lib.rr_op_json_advance(0, None, None, None, None, None, None, None, None) == 4
