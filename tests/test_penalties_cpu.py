"""CPU: the penalties / logit-bias surface without a device -- the float32 oracle against hand-computed answers, OpenAI's
validation rules for frequency_penalty / presence_penalty / logit_bias (BadRequestError, HTTP 400), forwarding at the
front only when the fields are present, and the argument checks of the new C entry points (RR_INVALID_ARGUMENT before
touching the device)."""
import ctypes as C

import numpy as np
import pytest
from starlette.testclient import TestClient

import penalty_oracle as O
from rr_b200.router import BadRequestError, check_penalties
from rr_b200.server import create_app

RR_INVALID_ARGUMENT = 4


# ---------------------------------------------------------------- oracle
def test_oracle_known_answers():
    x = np.array([1.0, 2.0, 3.0, -4.0, 0.5, 7.0], dtype=np.float32)
    # token 1 generated 3 times, token 2 once, token 5 never; bias on 2 and 5
    y = O.apply_row(x, [1, 2, 1, 1], frequency_penalty=0.5, presence_penalty=1.0, bias={2: -1.5, 5: 100})
    assert y.tolist() == [1.0, 2.0 - (3 * 0.5 + 1.0), (3.0 - 1.5) - (0.5 + 1.0), -4.0, 0.5, 107.0]
    # negative penalties reward repeats
    y = O.apply_row(x, [3, 3], frequency_penalty=-2.0, presence_penalty=-0.25)
    assert y[3] == np.float32(-4.0 + 4.0 + 0.25) and np.array_equal(np.delete(y, 3), np.delete(x, 3))
    # nothing to apply: bitwise the same row, -0.0 included
    z = np.array([-0.0, np.inf, -np.inf, 1e-45], dtype=np.float32)
    assert O.apply_row(z, [0, 1, 2], 0.0, 0.0, {}).tobytes() == z.tobytes()
    # history ids outside the vocabulary are ignored
    assert O.apply_row(x, [-1, 6, 99], 1.0, 1.0).tobytes() == x.tobytes()


def test_oracle_rounds_every_operation_in_float32():
    # (x + b) - (c * af + ap) with float32 rounding after each op differs from the exact / float64 result here
    x = np.array([16777216.0, 0.1], dtype=np.float32)
    y = O.apply_row(x, [0] * 3 + [1] * 7, frequency_penalty=0.1, presence_penalty=0.3, bias={0: 1.0})
    f32 = np.float32
    assert y[0] == f32(f32(f32(16777216.0) + f32(1.0)) - f32(f32(f32(3) * f32(0.1)) + f32(0.3)))
    assert y[1] == f32(f32(0.1) - f32(f32(f32(7) * f32(0.1)) + f32(0.3)))


# ---------------------------------------------------------------- validation
def test_validation_accepts_openai_ranges():
    assert check_penalties() is None
    assert check_penalties(0, 0.0, {}) is None
    assert check_penalties(0.5) == (0.5, 0.0, [], [])
    assert check_penalties(None, -2) == (0.0, -2.0, [], [])
    assert check_penalties(2, 2, {"7": 100, "0": -100, "+12": 0.5}, vocab=13) == (2.0, 2.0, [7, 0, 12], [100.0, -100.0, 0.5])
    assert check_penalties(logit_bias={5: 1}) == (0.0, 0.0, [5], [1.0])
    big = {str(i): 1 for i in range(300)}
    assert len(check_penalties(logit_bias=big, vocab=300)[2]) == 300


@pytest.mark.parametrize("kw", [
    dict(frequency_penalty=2.01), dict(frequency_penalty=-2.5), dict(presence_penalty=3), dict(presence_penalty=-2.0001),
    dict(frequency_penalty=True), dict(presence_penalty=False), dict(frequency_penalty="1"),
    dict(frequency_penalty=float("nan")), dict(presence_penalty=float("inf")),
    dict(logit_bias=[1, 2]), dict(logit_bias="x"), dict(logit_bias={"a": 1}), dict(logit_bias={"1.5": 1}),
    dict(logit_bias={"": 1}), dict(logit_bias={" 7": 1}), dict(logit_bias={True: 1}),
    dict(logit_bias={"7": 1, "07": 2}), dict(logit_bias={"7": 1, 7: 2}),
    dict(logit_bias={"-1": 1}), dict(logit_bias={"1000": 1}, vocab=1000), dict(logit_bias={str(2**40): 1}, vocab=128256),
    dict(logit_bias={"1": 100.5}), dict(logit_bias={"1": -101}), dict(logit_bias={"1": "5"}), dict(logit_bias={"1": True}),
    dict(logit_bias={"1": None}), dict(logit_bias={"1": float("nan")}),
    dict(logit_bias={str(i): 1 for i in range(301)}),
])
def test_validation_rejects_with_bad_request(kw):
    with pytest.raises(BadRequestError) as ei:
        check_penalties(**kw)
    assert ei.value.status_code == 400


# ---------------------------------------------------------------- HTTP front
class _Cfg:
    groups = ["g"]
    deployments = []


class _FakeRouter:
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def completion(self, model, messages, timeout=None, max_tokens=None, **kw):
        from rr_b200.router import Choice, Message, ModelResponse, Usage
        self.calls.append(kw)
        return ModelResponse("chatcmpl-1", "tiny@x", [Choice(0, Message("assistant", "hi"))], Usage(3, 2, 5))

    def completion_stream(self, model, messages, timeout=None, max_tokens=None, **kw):
        self.calls.append(kw)
        yield "tiny@x", [3 + ord("h")], False, 0.01
        yield "tiny@x", [], True, 0.01


BODY = {"model": "g", "messages": [{"role": "user", "content": "x"}]}


@pytest.mark.parametrize("stream", [False, True])
def test_http_forwards_the_fields_only_when_present(stream):
    fake = _FakeRouter()
    client = TestClient(create_app(fake))
    base = dict(BODY, stream=stream)
    for extra, want in [({}, {}), ({"frequency_penalty": None, "presence_penalty": None, "logit_bias": None}, {}),
                        ({"frequency_penalty": 0.5}, {"frequency_penalty": 0.5}),
                        ({"presence_penalty": -1, "logit_bias": {"72": 100}},
                         {"presence_penalty": -1, "logit_bias": {"72": 100}}),
                        ({"logit_bias": {}}, {"logit_bias": {}}),
                        ({"temperature": 0.7, "frequency_penalty": 1}, {"temperature": 0.7, "frequency_penalty": 1})]:
        r = client.post("/v1/chat/completions", json=dict(base, **extra))
        assert r.status_code == 200, r.text
        assert fake.calls[-1] == want


@pytest.mark.parametrize("stream", [False, True])
@pytest.mark.parametrize("extra", [{"frequency_penalty": 2.5}, {"presence_penalty": -3}, {"frequency_penalty": "x"},
                                   {"presence_penalty": True}, {"logit_bias": [1]}, {"logit_bias": {"x": 1}},
                                   {"logit_bias": {"7": 1, "07": 1}}, {"logit_bias": {"-3": 1}},
                                   {"logit_bias": {"7": 101}}, {"logit_bias": {"7": "1"}},
                                   {"logit_bias": {str(i): 1 for i in range(301)}}])
def test_http_rejects_invalid_values_with_400(stream, extra):
    fake = _FakeRouter()
    r = TestClient(create_app(fake)).post("/v1/chat/completions", json=dict(BODY, stream=stream, **extra))
    assert r.status_code == 400 and r.json()["error"]["type"] == "invalid_request_error"
    assert fake.calls == []


# ---------------------------------------------------------------- C entry points
def test_penalty_entry_points_and_unified_submit_validate_before_touching_the_device():
    from rr_b200 import _lib
    L = _lib.lib
    dummy = C.c_void_p(16)                       # never dereferenced: every call below is rejected first
    ok = dict(logits=dummy, ld=128256, rows=64, vocab=128256, hist=dummy, hist_ld=4096, hist_len=dummy, fp=dummy,
              pp=dummy, ids=dummy, vals=dummy, bias_ld=300, nb=dummy)

    def op(**kw):
        a = dict(ok, **kw)
        return L.rr_op_logit_penalties(a["logits"], a["ld"], a["rows"], a["vocab"], a["hist"], a["hist_ld"],
                                       a["hist_len"], a["fp"], a["pp"], a["ids"], a["vals"], a["bias_ld"], a["nb"], None)
    for bad in (dict(logits=None), dict(hist=None), dict(hist_len=None), dict(fp=None), dict(pp=None), dict(ids=None),
                dict(vals=None), dict(nb=None), dict(rows=0), dict(rows=-1), dict(rows=65536), dict(vocab=0),
                dict(vocab=128260), dict(ld=1003, vocab=1003), dict(ld=524292, vocab=524292), dict(hist_ld=-1),
                dict(bias_ld=-1), dict(bias_ld=301)):
        assert op(**bad) == RR_INVALID_ARGUMENT, bad
    t = C.c_uint64(77)
    ids = (C.c_int32 * 4)(1, 2, 3, 4)
    b_ids, b_vals = (C.c_int32 * 1)(5), (C.c_float * 1)(1.0)
    p = _lib.GenParams(n_choices=1, top_logprobs=-1, top_p=1.0, frequency_penalty=0.5, n_bias=1, bias_ids=b_ids,
                       bias_vals=b_vals)
    for params in (None, C.byref(p)):
        assert L.rr_engine_submit(None, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
        assert L.rr_gateway_submit(None, 0, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
    assert t.value == 77
