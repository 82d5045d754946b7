"""CPU checks of the paged KV cache: the option's place in rr_engine_opts, the refusals of rr_engine_create and of the four
`_paged` kernel entry points (all made before any CUDA call, so they run without a GPU), and the config keys
`litellm_params.context_window` / `kv_cache_tokens`."""
import ctypes as C

import pytest


def test_engine_opts_layout():
    from rr_b200 import _lib
    O = _lib.EngineOpts
    assert C.sizeof(O) == 48
    assert O.kv_cache_tokens.offset == 28 and O.prefix_cache.offset == 44


@pytest.mark.parametrize("kv", [-64, 1, 63, 512 + 32, 512 - 64, 4 * 512 + 64])
def test_engine_create_refuses_bad_pool(kv):
    """max_batch 4, ctx_max 512: the pool must be a multiple of 64 in [512, 2048]; anything else is refused before any CUDA
    call."""
    from rr_b200 import _lib
    desc = _lib.ModelDesc(256, 256, 512, 2, 4, 2, 64, 10000.0, 1e-5)
    w = _lib.ModelWeights()
    opts = _lib.EngineOpts(0, 4, 512, 256, 0, 0, 0.0, kv, (C.c_int32 * 3)(), 0)
    h = C.c_void_p()
    assert _lib.lib.rr_engine_create(C.byref(desc), C.byref(w), C.byref(opts), C.byref(h)) == 4
    assert h.value is None


_T = (C.c_int32 * 4)()           # a host array stands in for the table: a refused call never reads it
_F = C.c_void_p(16)              # never dereferenced either


def _calls(table, pps, n_pages, ctx):
    from rr_b200 import _lib
    L = _lib.lib
    out = C.c_int32(-1)
    src, dst, n_tok = (C.c_int32 * 1)(0), (C.c_int32 * 1)(1), (C.c_int32 * 1)(64)   # a list the counterpart accepts
    return {
        "decode": lambda: L.rr_op_decode_attn_qkv_paged(_F, 1, 0, 1536, _F, _F, _F, _F, _F, 1, 8, 2, 128, ctx, 1, 5e5,
                                                         C.byref(out), table, pps, n_pages, None),
        "prefill_qkv": lambda: L.rr_op_prefill_qkv_paged(_F, _F, 128, 64, 256, _F, 8, 2, 128, ctx, 5e5, 1e-5, _F, _F, _F,
                                                         _F, _F, C.byref(out), table, pps, n_pages, None),
        "prefill_attn": lambda: L.rr_op_prefill_attn_cached_paged(_F, _F, _F, _F, _F, _F, _F, 1, 1, 8, 2, ctx, 0.1, table,
                                                                   pps, n_pages, None),
        "kv_copy": lambda: L.rr_op_kv_copy_prefix_paged(_F, _F, 1, 2, 2, ctx, src, dst, n_tok, 1, table, pps, n_pages, None),
    }, out


@pytest.mark.parametrize("op", ["decode", "prefill_qkv", "prefill_attn", "kv_copy"])
@pytest.mark.parametrize("table,pps,n_pages,ctx", [(None, 2, 4, 128), (_T, 0, 4, 0), (_T, -1, 4, -64), (_T, 2, 0, 128),
                                                   (_T, 2, -3, 128), (_T, 2, 4, 192), (_T, 2, 4, 64)])
def test_paged_entry_points_refuse_bad_tables(op, table, pps, n_pages, ctx):
    calls, out = _calls(table, pps, n_pages, ctx)
    assert calls[op]() == 4 and out.value == -1


def test_paged_entry_points_then_apply_the_counterpart_checks():
    """A good table leaves the counterpart's refusals in place: a null q / qkv / cache pointer."""
    from rr_b200 import _lib
    L = _lib.lib
    ks = C.c_int32(-1)
    assert L.rr_op_decode_attn_qkv_paged(None, 1, 0, 1536, None, None, None, None, None, 1, 8, 2, 128, 128, 1, 5e5,
                                         C.byref(ks), _T, 2, 4, None) == 4 and ks.value == -1
    n = (C.c_int32 * 1)(1)
    assert L.rr_op_kv_copy_prefix_paged(None, None, 1, 1, 2, 128, n, n, n, 1, _T, 2, 4, None) == 4


# ---------------------------------------------------------------------------------------------------------------- config
def _cfg(*lps):
    from rr_b200.config import build_config
    return build_config([{"model_name": "m", "litellm_params": dict(model="b200/tiny", **lp)} for lp in lps])


def test_config_defaults():
    d = _cfg({}).deployments[0]
    assert d.context_window == 1024 and d.kv_cache_tokens is None


def test_config_values():
    d = _cfg({"context_window": 8192, "kv_cache_tokens": 262144}).deployments[0]
    assert d.context_window == 8192 and d.kv_cache_tokens == 262144


@pytest.mark.parametrize("lp", [{"context_window": 100}, {"context_window": 0}, {"context_window": "8192"},
                                {"context_window": True}, {"context_window": 8192.0},
                                {"kv_cache_tokens": 1000}, {"kv_cache_tokens": 512}, {"kv_cache_tokens": False},
                                {"context_window": 2048, "kv_cache_tokens": 1024}])
def test_config_errors(lp):
    with pytest.raises(ValueError):
        _cfg(lp)


@pytest.mark.parametrize("a,b", [({"context_window": 2048}, {}), ({"kv_cache_tokens": 4096}, {}),
                                 ({"kv_cache_tokens": 4096}, {"kv_cache_tokens": 8192})])
def test_config_deployments_on_one_gpu_must_agree(a, b):
    with pytest.raises(ValueError, match="disagree"):
        _cfg(dict(gpu=0, **a), dict(gpu=0, **b))
    _cfg(dict(gpu=0, **a), dict(gpu=1, **b))                    # separate GPUs: separate engines


def test_long_context_example_config():
    from pathlib import Path
    from rr_b200.config import load_config
    cfg = load_config(str(Path(__file__).resolve().parents[1] / "config" / "long-context.yaml"))
    d = cfg.deployments[0]
    assert d.context_window == 8192 and d.kv_cache_tokens == 262144


@pytest.mark.parametrize("cw,kv,max_batch,ctx_max", [(8192, 8192 * 4 + 64, 4, None), (1024, 2048, 4, 4096)])
def test_build_backends_refuses_a_pool_outside_its_range(cw, kv, max_batch, ctx_max):
    """A pool larger than max_batch x the context window, or smaller than the context window the engine serves, is
    refused, not resized."""
    from rr_b200.server import build_backends
    cfg = _cfg({"context_window": cw, "kv_cache_tokens": kv})
    with pytest.raises(ValueError, match="kv_cache_tokens"):
        build_backends(cfg, stub=False, max_batch=max_batch, ctx_max=ctx_max)
