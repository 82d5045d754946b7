"""CPU: /v1/embeddings (Router.embedding, server.py) -- request validation, the base64 encoding, the response shape through
a fake router, and the refusals of the new C entry points before they touch the device.  The pooling kernel, the engine's
embedding rows and the gateway path are checked in test_embeddings_gpu.py."""
import base64
import ctypes as C

import numpy as np
import pytest
from starlette.testclient import TestClient

from rr_b200 import _lib
from rr_b200.router import (APIError, BadRequestError, EmbeddingResponse, RateLimitError, check_embedding,
                            encode_embedding)
from rr_b200.server import create_app

_P = C.c_void_p(16)              # a 16-byte aligned stand-in pointer: a refused call never dereferences it
_ODD = C.c_void_p(24)            # 8-byte but not 16-byte aligned


# ---------------------------------------------------------------- validation
@pytest.mark.parametrize("inp", ["", [], [""], ["a", ""], [[]], [[1], []], [1, "a"], ["a", 1], [True], [[1, True]],
                                 [1.5], None, 7, {"a": 1}, [["a"]], [[1], 2]])
def test_bad_input_forms_are_refused(inp):
    with pytest.raises(BadRequestError, match="`input`"):
        check_embedding(inp)


def test_the_four_input_forms():
    assert check_embedding("hi") == (["hi"], "float")
    assert check_embedding(["a", "bc"]) == (["a", "bc"], "float")
    assert check_embedding([1, 2, 3]) == ([[1, 2, 3]], "float")
    assert check_embedding([[1], [2, 3]]) == ([[1], [2, 3]], "float")
    assert check_embedding("x", "base64", 4096) == (["x"], "base64")
    assert len(check_embedding(["a"] * 2048)[0]) == 2048


def test_limits_and_fields():
    with pytest.raises(BadRequestError, match="2048"):
        check_embedding(["a"] * 2049)
    with pytest.raises(BadRequestError, match="2048"):
        check_embedding([[1]] * 2049)
    for fmt in ("FLOAT", "binary", "", 1):
        with pytest.raises(BadRequestError, match="`encoding_format`"):
            check_embedding("x", fmt)
    for dims in (0, -1, 1.0, "8", True):
        with pytest.raises(BadRequestError, match="`dimensions`"):
            check_embedding("x", None, dims)


def test_base64_round_trips_to_the_same_fp32_bits():
    g = np.random.default_rng(0)
    v = np.concatenate([g.standard_normal(509).astype(np.float32) * 1e-3, np.float32([0.0, -0.0, 1.0, -1.0]),
                        np.float32([1e-45, 3.4e38, np.nextafter(np.float32(1), np.float32(2))])])
    s = encode_embedding(v, "base64")
    back = np.frombuffer(base64.b64decode(s), dtype="<f4")
    assert back.tobytes() == v.astype("<f4").tobytes()
    f = encode_embedding(v, "float")
    assert np.array(f, dtype=np.float32).tobytes() == v.tobytes()


# ---------------------------------------------------------------- HTTP
class _Cfg:
    groups = ["g", "limited"]
    deployments = []


class _FakeRouter:
    """Router.embedding's contract on synthetic vectors: [i, i + 0.5, -0.25] per input."""
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def embedding(self, model, input, encoding_format=None, dimensions=None, timeout=None, user=None):
        self.calls.append(dict(model=model, input=input, encoding_format=encoding_format, dimensions=dimensions))
        inputs, fmt = check_embedding(input, encoding_format, dimensions)
        if model == "limited":
            raise RateLimitError("No deployments available")
        if model == "boom":
            raise APIError("the embedding holds a non-finite value")
        if model not in self.cfg.groups:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        if dimensions is not None and dimensions != 3:
            raise BadRequestError("`dimensions` must be the model's hidden size [3]")
        vecs = [np.float32([i, i + 0.5, -0.25]) for i in range(len(inputs))]
        n = sum(len(p) if isinstance(p, list) else len(p.encode()) + 1 for p in inputs)
        return EmbeddingResponse("tiny", [encode_embedding(v, fmt) for v in vecs], n)


def test_http_embeddings_routes_and_status_codes():
    r = _FakeRouter()
    c = TestClient(create_app(r))
    for path in ("/embeddings", "/v1/embeddings"):
        got = c.post(path, json={"model": "g", "input": ["ab", "c"]})
        assert got.status_code == 200, got.text
        j = got.json()
        assert j["object"] == "list" and j["model"] == "tiny"
        assert [d["index"] for d in j["data"]] == [0, 1] and all(d["object"] == "embedding" for d in j["data"])
        assert j["data"][1]["embedding"] == [1.0, 1.5, -0.25]
        assert j["usage"] == {"prompt_tokens": 5, "total_tokens": 5}
    got = c.post("/v1/embeddings", json={"model": "g", "input": [[1, 2, 3]], "encoding_format": "base64"})
    assert got.status_code == 200
    v = np.frombuffer(base64.b64decode(got.json()["data"][0]["embedding"]), dtype="<f4")
    assert v.tolist() == [0.0, 0.5, -0.25]
    assert c.post("/v1/embeddings", json={"model": "limited", "input": "x"}).status_code == 429
    assert c.post("/v1/embeddings", json={"model": "nope", "input": "x"}).status_code == 400
    assert c.post("/v1/embeddings", json={"model": "boom", "input": "x"}).status_code == 500
    assert c.post("/v1/embeddings", json={"model": "g", "input": "x", "dimensions": 4}).status_code == 400
    assert c.post("/v1/embeddings", json={"model": "g", "input": "x", "dimensions": 3}).status_code == 200
    n_calls = len(r.calls)
    # refused before the router is called, naming the field
    for body, field in [({"input": ""}, "input"), ({"input": []}, "input"), ({"input": [[]]}, "input"),
                        ({"input": ["a"] * 2049}, "input"), ({"input": [1, "a"]}, "input"),
                        ({"input": "x", "encoding_format": "int8"}, "encoding_format"),
                        ({"input": "x", "dimensions": 0}, "dimensions")]:
        got = c.post("/v1/embeddings", json=dict(body, model="g"))
        assert got.status_code == 400 and f"`{field}`" in got.json()["error"]["message"], (body, got.text)
    assert c.post("/v1/embeddings", json={"model": "g"}).status_code == 400
    assert c.post("/v1/embeddings", json={"input": "x"}).status_code == 400
    assert c.post("/v1/embeddings", content=b"{not json").status_code == 400
    assert len(r.calls) == n_calls


def test_openai_sdk_parses_the_response():
    pytest.importorskip("openai")
    from openai._models import construct_type
    from openai.types import CreateEmbeddingResponse
    d = _FakeRouter().embedding("g", ["a", "b"]).model_dump()
    resp = construct_type(type_=CreateEmbeddingResponse, value=d)
    assert resp.data[1].embedding == [1.0, 1.5, -0.25] and resp.usage.prompt_tokens == 4


# ---------------------------------------------------------------- C ABI
POOL_GOOD = (_P, 4096, None, 64, 4096, _P, 4096)
POOL_ARGS = ("xn", "ld", "rows", "n", "hidden", "out", "out_ld")
POOL_BAD = {
    "null-xn": dict(xn=None),
    "null-out": dict(out=None),
    "n-0": dict(n=0),
    "n-negative": dict(n=-1),
    "n-65536": dict(n=65536),
    "hidden-0": dict(hidden=0),
    "hidden-negative": dict(hidden=-8),
    "hidden-4": dict(hidden=4),
    "hidden-not-multiple-of-8": dict(hidden=4092, ld=4096, out_ld=4096),
    "hidden-above-16384": dict(hidden=16392, ld=16392, out_ld=16392),
    "ld-below-hidden": dict(ld=4088),
    "ld-not-multiple-of-8": dict(ld=4100),
    "out_ld-below-hidden": dict(out_ld=4095),
    "xn-8-byte-aligned": dict(xn=_ODD),
}


@pytest.mark.parametrize("case", list(POOL_BAD))
def test_embed_pool_refuses_before_touching_the_device(case):
    a = dict(zip(POOL_ARGS, POOL_GOOD))
    a.update(POOL_BAD[case])
    assert _lib.lib.rr_op_embed_pool(*(a[k] for k in POOL_ARGS), None) == 4


def test_engine_and_gateway_entry_points_refuse_before_touching_the_device():
    L = _lib.lib
    t = C.c_uint64(77)
    ids = (C.c_int32 * 3)(1, 2, 3)
    out = (C.c_float * 8)()
    dim = C.c_int32(-5)
    assert L.rr_engine_submit_embed(None, ids, 3, C.byref(t)) == 4 and t.value == 77
    assert L.rr_engine_embedding(None, 1, 0.0, out, 8, C.byref(dim)) == 4 and dim.value == -5
    assert L.rr_gateway_submit_embed(None, 0, ids, 3, C.byref(t)) == 4 and t.value == 77
    assert L.rr_gateway_embedding(None, 1, 0.0, out, 8, C.byref(dim)) == 4 and dim.value == -5
    assert all(n in _lib.PROTOTYPES for n in ("rr_op_embed_pool", "rr_engine_submit_embed", "rr_engine_embedding",
                                              "rr_gateway_submit_embed", "rr_gateway_embedding"))
