"""CPU: prompt prefix caching -- the config key, the OpenAI usage shape, argument checks of the two kernel entry points
(rejected before any device is touched) and the C structs."""
import ctypes as C
import types

import pytest


def _cfg(params_a, params_b=None):
    from rr_b200.config import build_config
    ml = [{"model_name": "chat", "litellm_params": dict({"model": "b200/tiny", "gpu": 0}, **params_a)}]
    if params_b is not None:
        ml.append({"model_name": "other", "litellm_params": dict({"model": "b200/tiny", "gpu": 0}, **params_b)})
    return build_config(ml)


def test_config_key_parsed_and_checked(tmp_path):
    from rr_b200.config import load_config
    assert _cfg({"prefix_cache": True}).deployments[0].prefix_cache is True
    assert _cfg({"prefix_cache": False}).deployments[0].prefix_cache is False
    assert _cfg({}).deployments[0].prefix_cache is False
    for bad in ("yes", 1, None, 0.0):
        with pytest.raises(ValueError, match="prefix_cache"):
            _cfg({"prefix_cache": bad})
    # deployments on one GPU share one engine
    with pytest.raises(ValueError, match="prefix_cache"):
        _cfg({"prefix_cache": True}, {})
    assert [d.prefix_cache for d in _cfg({"prefix_cache": True}, {"prefix_cache": True}).deployments] == [True, True]
    p = tmp_path / "c.yaml"
    p.write_text("model_list:\n"
                 "  - model_name: chat\n    litellm_params: {model: b200/tiny, gpu: 0, prefix_cache: true}\n"
                 "  - model_name: plain\n    litellm_params: {model: b200/tiny, gpu: 1}\n")
    cfg = load_config(str(p))
    assert [(d.gpu, d.prefix_cache) for d in cfg.deployments] == [(0, True), (1, False)]
    p.write_text("model_list:\n"
                 "  - model_name: chat\n    litellm_params: {model: b200/tiny, gpu: 0, prefix_cache: true}\n"
                 "  - model_name: plain\n    litellm_params: {model: b200/tiny, gpu: 0}\n")
    with pytest.raises(ValueError, match="disagree"):
        load_config(str(p))


def test_usage_carries_cached_tokens_only_for_caching_deployments():
    from rr_b200.router import Choice, Message, ModelResponse, Router
    cfg = _cfg({"prefix_cache": True})
    cfg.deployments.append(_cfg({}).deployments[0])
    cfg.deployments[1].index = 1
    fake = types.SimpleNamespace(cfg=cfg)
    on, off = Router._usage(fake, 0, 130, 7, 101), Router._usage(fake, 1, 130, 7, 0)
    assert on.prompt_tokens == 130 and on.total_tokens == 137          # the whole prompt still counts
    d_on = ModelResponse("chatcmpl-1", "tiny", [Choice(0, Message("assistant", "hi"))], on).model_dump()
    d_off = ModelResponse("chatcmpl-2", "tiny", [Choice(0, Message("assistant", "hi"))], off).model_dump()
    assert d_on["usage"] == {"prompt_tokens": 130, "completion_tokens": 7, "total_tokens": 137,
                             "prompt_tokens_details": {"cached_tokens": 101}}
    assert d_off["usage"] == {"prompt_tokens": 130, "completion_tokens": 7, "total_tokens": 137}
    from openai.types.chat import ChatCompletion
    assert ChatCompletion.model_validate(d_on).usage.prompt_tokens_details.cached_tokens == 101
    assert ChatCompletion.model_validate(d_off).usage.prompt_tokens_details is None


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def test_kv_copy_prefix_rejects_bad_arguments_without_a_device():
    from rr_b200 import _lib
    f = _lib.lib.rr_op_kv_copy_prefix
    k, v = C.c_void_p(256), C.c_void_p(512)                  # never dereferenced: every call below is rejected first
    L, S, KV, ctx = 2, 8, 2, 128

    def call(src, dst, n, cnt=None, kc=k, vc=v):
        return f(kc, vc, L, S, KV, ctx, _i32(*src), _i32(*dst), _i32(*n), len(src) if cnt is None else cnt, None)
    assert call([0], [1], [4], kc=None) == 4 and call([0], [1], [4], vc=None) == 4
    assert f(k, v, L, S, KV, ctx, None, _i32(1), _i32(4), 1, None) == 4
    assert call([0], [1], [4], cnt=0) == 4
    assert call([0] * 257, list(range(1, 258)), [4] * 257) == 4                      # n_copies above 256
    assert call([-1], [1], [4]) == 4 and call([0], [S], [4]) == 4 and call([S], [1], [4]) == 4
    assert call([0], [1], [0]) == 4 and call([0], [1], [ctx + 1]) == 4
    assert call([0, 2], [1, 1], [4, 4]) == 4                                         # duplicate destination
    assert call([0, 1], [1, 2], [4, 4]) == 4                                         # slot 1 is a source and a destination
    assert call([3], [3], [4]) == 4
    assert f(k, v, 0, S, KV, ctx, _i32(0), _i32(1), _i32(4), 1, None) == 4


def test_prefill_attn_cached_rejects_bad_arguments_without_a_device():
    from rr_b200 import _lib
    f = _lib.lib.rr_op_prefill_attn_cached
    p = [C.c_void_p(256 * (i + 1)) for i in range(7)]

    def call(ptrs=p, n_seqs=2, max_len=64, H=8, KV=2, ctx=256):
        return f(*ptrs, n_seqs, max_len, H, KV, ctx, 0.088, None)
    for i in range(7):
        assert call(ptrs=p[:i] + [None] + p[i + 1:]) == 4, i                         # seq_pos0 is required too
    assert call(n_seqs=0) == 4 and call(max_len=0) == 4
    assert call(KV=0) == 4 and call(H=6, KV=4) == 4
    assert call(ctx=0) == 4 and call(ctx=100) == 4


def test_abi_of_the_new_fields():
    from rr_b200 import _lib
    assert not _lib.MISSING
    assert C.sizeof(_lib.Completion) == 48 and _lib.Completion.n_cached.offset == 20
    assert C.sizeof(_lib.EngineOpts) == 48 and _lib.EngineOpts.prefix_cache.offset == 44
    assert C.sizeof(_lib.GatewayResult) == 80 and _lib.GatewayResult.n_cached.offset == 72
    assert [n for n, _ in _lib.EngineStats._fields_][-3:] == ["prefix_hits", "prefix_cached_tokens", "kv_copy_tokens"]
    hdr = open(_lib._PKG.parent / "include" / "rr_b200.h").read()
    assert "rr_op_prefill_attn_cached(" in hdr and "rr_op_kv_copy_prefix(" in hdr
