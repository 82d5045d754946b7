"""CPU: the sampling surface without a device -- the fp64 oracle (Philox4x32-10 against its published answers, the nucleus,
the Gumbel-max draw against softmax), OpenAI's validation rules for temperature / top_p / seed, HTTP 400s and forwarding at
the front, and the argument checks of the new C entry points (RR_INVALID_ARGUMENT before touching
the device)."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats
from starlette.testclient import TestClient

import sampling_oracle as O
from rr_b200.router import BadRequestError, check_sampling
from rr_b200.server import create_app

RR_INVALID_ARGUMENT = 4


# ---------------------------------------------------------------- oracle
@pytest.mark.parametrize("ctr,key,want", [
    # Random123 known-answer vectors for philox4x32_10
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = O.philox4x32_10(*ctr, *key)
    assert tuple(int(w) for w in got) == want


def test_uniforms_are_exact_and_inside_the_open_interval():
    u = O.uniforms(12345, 7, 100000)
    assert u.min() > 0 and u.max() < 1
    assert np.all(u.astype(np.float32).astype(np.float64) == u)          # exact in fp32, as the kernel computes it
    assert np.all((u * 2**24) % 2 == 1)
    assert stats.kstest(u, "uniform").pvalue > 1e-3
    # the counter is (token id, position): another position or seed gives other words
    assert not np.array_equal(O.random_words(12345, 7, 64), O.random_words(12345, 8, 64))
    assert not np.array_equal(O.random_words(12345, 7, 64), O.random_words(12346, 7, 64))
    assert np.array_equal(O.random_words(-1, 3, 16), O.random_words(2**64 - 1, 3, 16))


def test_nucleus_is_the_smallest_value_prefix_with_enough_mass():
    rng = np.random.default_rng(0)
    x = rng.normal(0, 1, 500).astype(np.float32)
    x[10:14] = x[3]                                                       # ties
    for T in (0.05, 0.7, 2.0):
        for p in (1e-6, 0.3, 0.9, 0.999):
            tau = O.threshold(x, T, p)
            w = np.exp((x.astype(np.float64) - x.max()) / T)
            share = w[x >= tau].sum() / w.sum()
            above = w[x > tau].sum() / w.sum()
            assert share >= np.float32(p) and above < np.float32(p)
    assert O.threshold(x, 1.0, 1.0) == -np.inf


def test_gumbel_max_draws_follow_the_renormalised_nucleus():
    x = np.array([2.0, 1.5, 1.5, 0.3, -1.0, 0.0, 1.0, -3.0], dtype=np.float32)
    T, p, n = 0.8, 0.85, 6000
    toks = np.array([O.sample(x, T, p, seed=99, position=j).token for j in range(n)])
    tau = O.threshold(x, T, p)
    inside = x >= tau
    assert set(toks.tolist()) <= set(np.flatnonzero(inside).tolist())
    w = np.where(inside, np.exp((x.astype(np.float64) - x.max()) / T), 0.0)
    want = w / w.sum() * n
    got = np.bincount(toks, minlength=len(x))
    assert stats.chisquare(got[inside], want[inside]).pvalue > 1e-3


# ---------------------------------------------------------------- validation
def test_validation_follows_openai_rules():
    assert check_sampling() is None and check_sampling(0) is None and check_sampling(0.0, 0.5, 3) is None
    assert check_sampling(0.7) == (0.7, 1.0, None)
    assert check_sampling(2, 0, -1) == (2.0, 0.0, 2**64 - 1)
    assert check_sampling(1.0, 1, 2**64 - 1) == (1.0, 1.0, 2**64 - 1)
    assert check_sampling(1.0, None, -2**63) == (1.0, 1.0, 2**63)
    for kw in [dict(temperature=-0.1), dict(temperature=2.01), dict(temperature=True), dict(temperature="1"),
               dict(temperature=float("nan")), dict(temperature=float("inf")), dict(top_p=-0.01), dict(top_p=1.5),
               dict(top_p=False), dict(top_p="0.9"), dict(top_p=float("nan")), dict(seed=1.0), dict(seed=True),
               dict(seed="7"), dict(seed=2**64), dict(seed=-2**63 - 1), dict(temperature=1.0, seed=2**70)]:
        with pytest.raises(BadRequestError):
            check_sampling(**kw)


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
    for extra, want in [({}, {}), ({"temperature": None, "top_p": None, "seed": None}, {}),
                        ({"temperature": 0.7}, {"temperature": 0.7}),
                        ({"temperature": 1, "top_p": 0.9, "seed": 42}, {"temperature": 1, "top_p": 0.9, "seed": 42}),
                        ({"seed": -5}, {"seed": -5})]:
        r = client.post("/v1/chat/completions", json=dict(base, **extra))
        assert r.status_code == 200, r.text
        assert fake.calls[-1] == want


@pytest.mark.parametrize("stream", [False, True])
@pytest.mark.parametrize("extra", [{"temperature": 2.5}, {"temperature": -1}, {"temperature": "hot"}, {"temperature": True},
                                   {"top_p": 1.01}, {"top_p": -0.5}, {"seed": 0.5}, {"seed": "1"}, {"seed": 2**64},
                                   {"seed": False}])
def test_http_rejects_invalid_values_with_400(stream, extra):
    fake = _FakeRouter()
    r = TestClient(create_app(fake)).post("/v1/chat/completions", json=dict(BODY, stream=stream, **extra))
    assert r.status_code == 400 and r.json()["error"]["type"] == "invalid_request_error"
    assert fake.calls == []


# ---------------------------------------------------------------- C entry points
def test_sampling_entry_points_and_unified_submit_validate_before_touching_the_device():
    from rr_b200 import _lib
    L = _lib.lib
    dummy = C.c_void_p(16)                       # never dereferenced: every call below is rejected first
    ok = dict(logits=dummy, ld=128256, rows=64, vocab=128256, temp=dummy, top_p=dummy, seed=dummy, pos=dummy, out=dummy)

    def op(**kw):
        a = dict(ok, **kw)
        return L.rr_op_sample(a["logits"], a["ld"], a["rows"], a["vocab"], a["temp"], a["top_p"], a["seed"], a["pos"],
                              a["out"], None)
    for bad in (dict(logits=None), dict(temp=None), dict(top_p=None), dict(seed=None), dict(pos=None), dict(out=None),
                dict(rows=0), dict(rows=-3), dict(rows=65536), dict(vocab=0), dict(vocab=128260), dict(ld=1003, vocab=1003),
                dict(ld=524292, vocab=524292)):
        assert op(**bad) == RR_INVALID_ARGUMENT, bad
    t = C.c_uint64(77)
    ids = (C.c_int32 * 4)(1, 2, 3, 4)
    p = _lib.GenParams(n_choices=1, top_logprobs=-1, temperature=0.7, top_p=0.9, seed=1)
    for params in (None, C.byref(p)):
        assert L.rr_engine_submit(None, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
        assert L.rr_gateway_submit(None, 0, ids, 4, 8, params, C.byref(t)) == RR_INVALID_ARGUMENT
    assert t.value == 77
