"""CPU: sliding-window attention without a GPU -- the oracle's window against the real transformers
MistralForCausalLM (tests/golden/sliding_window_golden.pt), the KV ring's size bound by exhaustive simulation, the spec
and ABI plumbing, and the Router's KV 400 under the ring rule."""
import ctypes as C
import os
from types import SimpleNamespace

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "sliding_window_golden.pt")


def golden_case():
    from rr_b200.models import SPECS, make_weights
    g = torch.load(GOLDEN)
    spec = SPECS[g["spec"]]
    assert spec.sliding_window == g["sliding_window"] == 100
    w = make_weights(spec, seed=g["seed"], sigma=g["sigma"], device="cpu", norm_jitter=g["norm_jitter"])
    chk = float(sum(t.float().abs().sum() for t in w.tensors()))
    assert abs(chk - g["weight_checksum"]) < 1e-3 * g["weight_checksum"], "seeded weights drifted from fixture"
    return spec, w, g


def test_oracle_window_matches_hf_mistral():
    """The windowed oracle (tests/window_oracle.py) against HF MistralForCausalLM(sliding_window=100), at the tolerance of
    test_restatement_matches_hf_mistral_and_phi3.  The unwindowed restatement matches only rows below the window."""
    import dataclasses
    from oracle import llama_ref
    from window_oracle import forward_logits
    spec, w, g = golden_case()
    w0 = dataclasses.replace(w, spec=dataclasses.replace(spec, sliding_window=0))
    below = past = 0
    for p, lg, tk in zip(g["prompts"], g["logits"], g["tokens"]):
        toks = list(p)
        for j in range(len(tk)):
            mine = forward_logits(w, toks)[-1]
            assert torch.allclose(mine, lg[j], atol=2e-4, rtol=1e-4), (len(p), j, (mine - lg[j]).abs().max())
            assert int(mine.argmax()) == tk[j]
            full = llama_ref.forward_logits(w0, toks)[-1]
            if len(toks) <= spec.sliding_window:          # the last row's position < W: the window changes nothing
                assert torch.equal(full, mine)
                below += 1
            else:
                assert (full - lg[j]).abs().max() > 1e-2, (len(toks), "the window made no difference")
                past += 1
            toks.append(tk[j])
    assert below >= 4 and past >= 9


@pytest.mark.parametrize("T,W", [(2500, 100), (2500, 1500), (3000, 1024)])
def test_oracle_window_blocks_equal_one_masked_softmax(T, W):
    """The oracle's blocked window attention equals one masked T x T softmax."""
    import math
    from window_oracle import window_attn
    g = torch.Generator().manual_seed(T + W)
    q, k, v = (torch.randn(T, 2, 32, generator=g, dtype=torch.float64) for _ in range(3))
    i = torch.arange(T)
    vis = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - W)
    sc = torch.einsum("thd,shd->hts", q, k) / math.sqrt(32)
    want = torch.einsum("hts,shd->thd", torch.softmax(sc.masked_fill(~vis[None], float("-inf")), -1), v)
    assert torch.allclose(window_attn(q, k, v, W), want, atol=1e-12, rtol=1e-12)


def _live_pages(pos0, n, W):
    """Logical pages a prefill piece (or, n = 1, a decode step) at positions pos0 .. pos0 + n - 1 reads or writes."""
    return range(max(0, pos0 - W + 1) // 64, (pos0 + n - 1) // 64 + 1)


def _ring_ok(R, W, tmax):
    """Every piece alignment and length, and every decode position: the live pages are distinct mod R."""
    for pos0 in range(0, 4 * 64 + W + tmax):
        for n in range(1, tmax + 1):
            pages = _live_pages(pos0, n, W)
            if len({p % R for p in pages}) != len(pages):
                return False
    return True


@pytest.mark.parametrize("W", [1, 2, 63, 64, 65, 100, 128, 130])
@pytest.mark.parametrize("tmax", [16, 17, 64, 66, 100, 129])
def test_ring_bound_is_exact(W, tmax):
    """R = ceil((W + Tmax - 2) / 64) + 1 pages hold every piece and decode step without a write landing on a page still
    read (pages mapped p -> p mod R); R - 1 pages fail for some alignment."""
    from rr_b200.models import ring_pages
    R = ring_pages(W, tmax)
    assert R == -(-(W + tmax - 2) // 64) + 1
    assert _ring_ok(R, W, tmax)
    assert not _ring_ok(R - 1, W, tmax)


def test_ring_pages_mirror():
    from rr_b200.models import ring_pages
    assert ring_pages(0, 8192) == 0
    assert ring_pages(4096, 8192) == 193                 # 1.51 GiB of Mistral-7B KV at 128 KiB per token
    assert ring_pages(4096, 0) == 193                    # max_prefill_tokens 0: the 8192-token default
    assert ring_pages(100, 512) == 11 and ring_pages(100, 1) == ring_pages(100, 16) == 3


def test_specs_and_abi():
    """The window belongs to the model; rr_model_weights carries it where `reserved` was, so no offset moves."""
    from rr_b200 import _lib
    from rr_b200.models import SPECS
    assert SPECS["mistral-7b"].sliding_window == SPECS["mistral-7b-2l"].sliding_window == 4096
    assert SPECS["tiny-sw"].sliding_window == 100
    for name in ("llama-3-8b", "phi-3-mini", "tiny", "small", "llama-3-8b-2l", "phi-3-mini-2l", "tiny96", "small96"):
        assert SPECS[name].sliding_window == 0, name
    t = SPECS["tiny-sw"]
    assert (t.vocab, t.hidden, t.inter, t.n_layers, t.n_heads, t.n_kv_heads, t.head_dim) == \
        (1024, 512, 1024, 2, 4, 2, 128)
    M = _lib.ModelWeights
    assert [f[0] for f in M._fields_][9:11] == ["flags", "sliding_window"]
    assert M.flags.offset == 72 and M.sliding_window.offset == 76 and M.wqkv_scale.offset == 80
    assert C.sizeof(M) == 112 and M.sliding_window.size == 4


def _router(*engines):
    from rr_b200.router import EngineBackend, Router
    fake = SimpleNamespace(backends={i: EngineBackend(SimpleNamespace(
        spec=SimpleNamespace(vocab=256, sliding_window=w), ctx_max=ctx, max_batch=8, kv_cache_tokens=kv,
        max_prefill_tokens=tmax)) for i, (w, ctx, kv, tmax) in enumerate(engines)})
    fake._limits = lambda: Router._limits(fake)
    return fake


@pytest.mark.parametrize("n_prompt,max_new,n,ok", [
    (2000, 100, 1, True),          # 33 pages linearly > 16, ring 11 <= 16
    (600, 100, 1, True),           # 11 pages: linear, fits
    (2000, 100, 2, False),         # 2 x 11 > 16
    (700, 100, 2, False),          # 2 x 11 (13 linearly, ring 11) > 16
    (300, 100, 2, True),           # 2 x 7 linear pages
])
def test_router_kv_400_follows_the_ring(n_prompt, max_new, n, ok):
    """A windowed replica (W = 100, Tmax 512: a ring of 11 pages) of 16 pages: a choice reserves min(ceil(reach / 64),
    11) pages, so the 400 names the KV cache exactly when the engine would refuse."""
    from rr_b200.router import Router
    msg = Router._invalid(_router((100, 4096, 1024, 512)), n_prompt, max_new, n).message
    assert ("KV cache" in msg) == (not ok), msg


def test_router_kv_400_names_any_engine_that_could_never_fit():
    """Each engine counts its own pages: a windowed pool serves what a same-sized unwindowed pool refuses, and a fleet
    refuses what one of its engines could never hold."""
    from rr_b200.router import Router
    assert "KV cache" not in Router._invalid(_router((100, 4096, 1024, 512)), 2000, 100).message
    assert "KV cache (1024 tokens)" in Router._invalid(_router((0, 4096, 1024, 512)), 2000, 100).message
    assert "KV cache (1024 tokens)" in Router._invalid(_router((100, 4096, 65536, 512), (0, 4096, 1024, 512)),
                                                       2000, 100).message


_T = (C.c_int32 * 4)()           # a host array stands in for the table: a refused call never reads it
_F = C.c_void_p(16)              # never dereferenced either


def _window_calls(window, table=_T, pps=2, n_pages=4, ctx=128):
    from rr_b200 import _lib
    L = _lib.lib
    out = C.c_int32(-1)
    return {
        "decode": lambda: L.rr_op_decode_attn_qkv_window(_F, 1, 0, 1536, _F, _F, _F, _F, _F, 1, 8, 2, 128, ctx, 1, 5e5,
                                                         C.byref(out), table, pps, n_pages, window, None),
        "prefill": lambda: L.rr_op_prefill_attn_window(_F, _F, _F, _F, _F, _F, _F, 1, 1, 8, 2, ctx, 0.1, table, pps,
                                                       n_pages, window, None),
    }, out


@pytest.mark.parametrize("op", ["decode", "prefill"])
@pytest.mark.parametrize("window", [-1, -4096, -(2**31)])
def test_window_entry_points_refuse_a_negative_window(op, window):
    calls, out = _window_calls(window)
    assert calls[op]() == 4 and out.value == -1


@pytest.mark.parametrize("op", ["decode", "prefill"])
@pytest.mark.parametrize("table,pps,n_pages,ctx", [(None, 2, 4, 128), (_T, 0, 4, 0), (_T, 2, 0, 128), (_T, 2, 4, 192)])
def test_window_entry_points_refuse_bad_tables(op, table, pps, n_pages, ctx):
    calls, out = _window_calls(100, table, pps, n_pages, ctx)
    assert calls[op]() == 4 and out.value == -1


def test_engine_create_refuses_a_negative_window():
    """Refused before any CUDA call, like a bad pool."""
    from rr_b200 import _lib
    desc = _lib.ModelDesc(256, 256, 512, 2, 4, 2, 64, 10000.0, 1e-5)
    w = _lib.ModelWeights()
    w.sliding_window = -1
    opts = _lib.EngineOpts(0, 4, 512, 256, 0, 0, 0.0, 0, (C.c_int32 * 3)(), 0)
    h = C.c_void_p()
    assert _lib.lib.rr_engine_create(C.byref(desc), C.byref(w), C.byref(opts), C.byref(h)) == 4
    assert h.value is None


def test_sliding_window_example_config():
    """config/sliding-window.yaml: Mistral-7B (W = 4096) at a 32768-token context window; its header's ring arithmetic."""
    from pathlib import Path
    from rr_b200.config import load_config
    from rr_b200.models import resolve_spec, ring_pages
    cfg = load_config(str(Path(__file__).resolve().parents[1] / "config" / "sliding-window.yaml"))
    d = cfg.deployments[0]
    assert d.context_window == 32768 and d.kv_cache_tokens == 262144
    spec = resolve_spec(d.model)
    R = ring_pages(spec.sliding_window, 8192)
    assert spec.sliding_window == 4096 and R == 193
    assert (d.kv_cache_tokens // 64) // R == 21 and (d.kv_cache_tokens // 64) // (32768 // 64) == 8
    assert abs(R * 64 * spec.kv_bytes_per_token / 2**30 - 1.51) < 0.005
