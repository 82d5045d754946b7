"""CPU: the host side of long prompts -- the 65536-token example config, and the Router's HTTP 400s without the former
prefill-chunk limit (a prompt longer than max_prefill_tokens is prefilled in pieces)."""
from pathlib import Path
from types import SimpleNamespace

import pytest


def test_long_prompts_example_config():
    from rr_b200.config import load_config
    cfg = load_config(str(Path(__file__).resolve().parents[1] / "config" / "long-prompts.yaml"))
    d = cfg.deployments[0]
    assert d.context_window == 65536 and d.kv_cache_tokens == 262144


def _router_with(ctx_max, max_batch, kv, max_prefill_tokens=8192):
    from rr_b200.router import EngineBackend, Router
    eng = SimpleNamespace(spec=SimpleNamespace(vocab=256), ctx_max=ctx_max, max_batch=max_batch, kv_cache_tokens=kv,
                          max_prefill_tokens=max_prefill_tokens)
    fake = SimpleNamespace(backends={0: EngineBackend(eng)})
    fake._limits = lambda: Router._limits(fake)
    return fake


def test_limits_no_longer_name_the_prefill_chunk():
    from rr_b200.router import Router
    fake = _router_with(65536, 64, 262144)
    assert Router._limits(fake) == (65536, 64, 262144)
    msg = Router._invalid(fake, 40000, 8).message
    assert "prefill chunk" not in msg and "vocabulary" in msg


@pytest.mark.parametrize("n_prompt,max_new,n,want", [(65000, 1000, 1, "context window"), (40000, 8, 65, "decode rows"),
                                                     (40000, 8, 7, "KV cache")])
def test_the_other_400s_keep_their_messages(n_prompt, max_new, n, want):
    from rr_b200.router import Router
    msg = Router._invalid(_router_with(65536, 64, 262144), n_prompt, max_new, n).message
    assert want in msg and "prefill chunk" not in msg
