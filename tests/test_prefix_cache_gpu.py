"""GPU: prompt prefix caching, from the kernels (prefill attention over a cached prefix, the KV prefix copy) through the
engine's index to the OpenAI endpoint.

A cache hit is checked bit for bit: the KV at position p depends only on tokens 0..p, every prefill kernel computes a row
independently of the chunk it is in and of its place in a tile, and in attention a fully masked key tile leaves the
online-softmax state unchanged.  So with caching on, tokens and top-20 logprobs equal those of an engine without it."""
import ctypes as C
import math
import os
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


def _lib():
    from rr_b200 import _lib
    return _lib


def P(t):
    return C.c_void_p(t.data_ptr())


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ kernel: attention
CASES = [(0, 1), (1, 1), (63, 1), (64, 64), (65, 127), (127, 129), (128, 128), (300, 212), (448, 64), (511, 1), (0, 512)]


def _attn_call(fn, q, kc, vc, out, lens, slots, H, KV, ctx, scale, pos0=None):
    L = _lib()
    start = torch.tensor([0] + np.cumsum(lens).tolist(), device=DEV, dtype=torch.int32)
    sl = torch.tensor(slots, device=DEV, dtype=torch.int32)
    if pos0 is None:
        rc = L.lib.rr_op_prefill_attn(P(q), P(kc), P(vc), P(out), P(start), P(sl), len(lens), max(lens), H, KV, ctx,
                                      scale, None)
    else:
        p0 = torch.tensor(pos0, device=DEV, dtype=torch.int32)
        rc = L.lib.rr_op_prefill_attn_cached(P(q), P(kc), P(vc), P(out), P(start), P(sl), P(p0), len(lens), max(lens),
                                             H, KV, ctx, scale, None)
    L.check(rc, fn)
    torch.cuda.synchronize()
    return start.tolist()


@pytest.mark.parametrize("hd", [128, 96])
@pytest.mark.parametrize("H,KV", [(32, 8), (8, 8), (4, 1), (16, 2)])
def test_prefill_attention_over_cached_prefix(H, KV, hd):
    g = torch.Generator(device=DEV).manual_seed(H * 7 + KV + hd)
    ctx, n = 576, len(CASES)
    slots = list(range(n))
    pad = torch.zeros(128, device=DEV)
    pad[:hd] = 1

    def rnd(*shape):
        return (torch.randn(*shape, 128, device=DEV, generator=g) * pad).bfloat16()
    kc, vc = rnd(n + 1, KV, ctx), rnd(n + 1, KV, ctx)
    full = [p0 + ln for p0, ln in CASES]
    qf = [rnd(m, H) for m in full]                                # whole sequences; the suffix is the last `len` rows
    qs = torch.cat([qf[i][p0:].reshape(ln, H * 128) for i, (p0, ln) in enumerate(CASES)])
    scale = 1 / math.sqrt(hd)
    out = torch.zeros(qs.shape, device=DEV, dtype=torch.bfloat16)
    lens, pos0 = [ln for _, ln in CASES], [p0 for p0, _ in CASES]
    st = _attn_call("cached", qs, kc, vc, out, lens, slots, H, KV, ctx, scale, pos0)

    # cold run over the whole sequences, same cache
    qfull = torch.cat([x.reshape(-1, H * 128) for x in qf])
    cold = torch.zeros(qfull.shape, device=DEV, dtype=torch.bfloat16)
    stf = _attn_call("cold", qfull, kc, vc, cold, full, slots, H, KV, ctx, scale)
    G = H // KV
    for i, (p0, ln) in enumerate(CASES):
        got = out[st[i]:st[i] + ln]
        assert torch.equal(_bits(got), _bits(cold[stf[i] + p0:stf[i + 1]])), (i, p0, ln)
        # fp64 reference
        qq = qf[i][p0:].double().transpose(0, 1)                                  # [H, ln, 128]
        k = kc[i, :, :p0 + ln].double().repeat_interleave(G, 0)
        v = vc[i, :, :p0 + ln].double().repeat_interleave(G, 0)
        sc = (qq @ k.transpose(1, 2)) * scale
        keep = torch.arange(p0 + ln, device=DEV)[None, :] <= (p0 + torch.arange(ln, device=DEV))[:, None]
        ref = (torch.softmax(sc.masked_fill(~keep, float("-inf")), -1) @ v).transpose(0, 1)
        gv = got.view(ln, H, 128).double()
        assert torch.allclose(gv[..., :hd], ref[..., :hd], atol=3e-2, rtol=3e-2), (i, (gv - ref).abs().max().item())
        assert (gv[..., hd:] == 0).all()

    # seq_pos0 all zero: the bits of rr_op_prefill_attn
    zero = torch.zeros(qfull.shape, device=DEV, dtype=torch.bfloat16)
    _attn_call("zero", qfull, kc, vc, zero, full, slots, H, KV, ctx, scale, [0] * n)
    assert torch.equal(_bits(zero), _bits(cold))

    # different finite garbage beyond each sequence's last position changes no bit
    for i, m in enumerate(full):
        kc[i, :, m:] = rnd(KV, ctx - m) * 40
        vc[i, :, m:] = rnd(KV, ctx - m) * 40
    again = torch.zeros(qs.shape, device=DEV, dtype=torch.bfloat16)
    _attn_call("garbage", qs, kc, vc, again, lens, slots, H, KV, ctx, scale, pos0)
    assert torch.equal(_bits(again), _bits(out))


# ------------------------------------------------------------------------------------------------ kernel: copy
def test_kv_copy_prefix():
    L = _lib()
    layers, S, KV, ctx = 3, 12, 2, 320
    g = torch.Generator(device=DEV).manual_seed(9)
    kc = torch.randn(layers, S, KV, ctx, 128, device=DEV, generator=g).bfloat16()
    vc = torch.randn(layers, S, KV, ctx, 128, device=DEV, generator=g).bfloat16()
    for copies in ([(0, 5, 1), (1, 6, 63), (2, 7, 64), (0, 8, 65), (3, 9, ctx)], [(9, 0, 200)]):
        k0, v0 = kc.clone(), vc.clone()
        src, dst, n = zip(*copies)
        arr = lambda x: (C.c_int32 * len(x))(*x)                                    # noqa: E731
        L.check(L.lib.rr_op_kv_copy_prefix(P(kc), P(vc), layers, S, KV, ctx, arr(src), arr(dst), arr(n), len(copies),
                                           None), "copy")
        torch.cuda.synchronize()
        want_k, want_v = k0.clone(), v0.clone()
        for s, d, m in copies:
            want_k[:, d, :, :m] = k0[:, s, :, :m]
            want_v[:, d, :, :m] = v0[:, s, :, :m]
        assert torch.equal(_bits(kc), _bits(want_k)) and torch.equal(_bits(vc), _bits(want_v))


# ------------------------------------------------------------------------------------------------ engine
N_NEW = 8


class Pair:
    """The same weights behind a caching engine and a plain one."""

    def __init__(self, spec_name):
        from rr_b200 import SPECS, make_weights
        from rr_b200.engine import Engine
        self.spec = SPECS[spec_name]
        w = make_weights(self.spec, seed=11, sigma=0.05, device="cuda")
        kw = dict(max_batch=64, ctx_max=1024, max_prefill_tokens=8192, use_cuda_graph=True)
        self.on = Engine(w, prefix_cache=True, **kw)
        self.off = Engine(w, **kw)
        self.rng = np.random.RandomState(len(spec_name))
        self.refs = {}

    def close(self):
        self.on.close()
        self.off.close()

    def toks(self, n):
        return self.rng.randint(3, self.spec.vocab, size=n).tolist()

    def other(self, t):
        return t + 1 if t + 1 < self.spec.vocab else 3

    def ref(self, prompts, n_new=N_NEW):
        todo = [p for p in prompts if (tuple(p), n_new) not in self.refs]
        tk = [self.off.submit(p, n_new, top_logprobs=20) for p in todo]
        for p, t in zip(todo, tk):
            r = self.off.wait(t)
            assert r.status == 0 and r.n_cached == 0
            self.refs[(tuple(p), n_new)] = (r.tokens, r.logprobs)
        return [self.refs[(tuple(p), n_new)] for p in prompts]

    def check(self, recs, prompts, n_new=N_NEW):
        for r, want in zip(recs, self.ref(prompts, n_new)):
            assert r.status == 0
            assert r.tokens == want[0]
            got = [[(i, np.float32(v).view(np.int32)) for i, v in row] for row in r.logprobs]
            exp = [[(i, np.float32(v).view(np.int32)) for i, v in row] for row in want[1]]
            assert got == exp

    def run(self, prompts, n_new=N_NEW):
        """Sequentially on the caching engine: -> records (checked against the plain engine)."""
        recs = [self.on.wait(self.on.submit(p, n_new, top_logprobs=20)) for p in prompts]
        self.check(recs, prompts, n_new)
        return recs

    def delta(self, fn):
        self.on.reset_stats()
        out = fn()
        s = self.on.stats()
        return out, (s["prefill_tokens"], s["prefix_hits"], s["prefix_cached_tokens"], s["kv_copy_tokens"])


@pytest.fixture(scope="module", params=["tiny", "tiny96", "llama-3-8b-2l"])
def pair(request):
    p = Pair(request.param)
    yield p
    s = p.off.stats()
    p.close()
    assert s["prefix_hits"] == s["prefix_cached_tokens"] == s["kv_copy_tokens"] == 0


def test_hit_on_a_freed_slot(pair):
    a = pair.toks(200)
    b = a[:150] + [pair.other(a[150])] + pair.toks(49)
    (ra,), d = pair.delta(lambda: pair.run([a]))
    assert ra.n_cached == 0 and d == (200, 0, 0, 0)
    (rb,), d = pair.delta(lambda: pair.run([b]))
    assert rb.n_cached == 150 and d == (50, 1, 150, 0)


def test_hit_on_a_busy_slot_copies(pair):
    c = pair.toks(300)
    e = c + pair.toks(20)
    long_new = 200

    def go():
        tc = pair.on.submit(c, long_new, top_logprobs=20)
        pair.on.peek(tc, 0, timeout=60)                                   # prefilled, decoding
        re = pair.on.wait(pair.on.submit(e, N_NEW, top_logprobs=20))
        rc = pair.on.wait(tc)
        return rc, re
    (rc, re), d = pair.delta(go)
    pair.check([rc], [c], long_new)                                       # the running request is unchanged
    pair.check([re], [e])
    assert rc.n_cached == 0 and re.n_cached == 300 and d == (300 + 20, 1, 300, 300)


def test_identical_prompt(pair):
    p = pair.toks(130)
    _, d = pair.delta(lambda: pair.run([p, p]))
    assert d == (130 + 1, 1, 129, 0)


def test_lcp_63_misses_64_hits(pair):
    f = pair.toks(100)
    alt = [pair.other(t) for t in f]
    g63 = f[:63] + alt[63:]
    g64 = f[:64] + alt[64:]
    recs, d = pair.delta(lambda: pair.run([f, g63, g64]))
    # g63 shares 63 tokens with f: a miss.  g64 shares 64 with f (and 63 with g63): a hit on f's freed slot
    assert [r.n_cached for r in recs] == [0, 0, 64] and d == (100 + 100 + 36, 1, 64, 0)


def test_conversation_caches_the_previous_prompt_only(pair):
    h1 = pair.toks(100)
    (r1,) = pair.run([h1])
    h2 = h1 + r1.tokens + pair.toks(30)
    (r2,), d = pair.delta(lambda: pair.run([h2]))
    assert r2.n_cached == len(h1) and d == (len(h2) - len(h1), 1, len(h1), 0)


def test_lru_eviction(pair):
    B = pair.on.max_batch
    xs = [pair.toks(70) for _ in range(B + 1)]
    pair.run(xs)                                                  # every slot now holds one of them; xs[0] was evicted
    (r1, r0), d = pair.delta(lambda: pair.run([xs[1] + pair.toks(5), xs[0] + pair.toks(5)]))
    assert (r1.n_cached, r0.n_cached) == (70, 0) and d == (5 + 75, 1, 70, 0)


def test_low_level_call_clears_the_index(pair):
    p = pair.toks(120)
    pair.run([p])
    pair.on.prefill([pair.toks(10)], [0])
    pair.on.decode_step([0], [5], [10])                            # (also leaves the row inactive again)
    (r,), d = pair.delta(lambda: pair.run([p]))
    assert r.n_cached == 0 and d == (120, 0, 0, 0)
    pair.on.decode_step([0], [5], [0])
    (r,), d = pair.delta(lambda: pair.run([p]))
    assert r.n_cached == 0 and d == (120, 0, 0, 0)
    (r,), d = pair.delta(lambda: pair.run([p]))
    assert r.n_cached == 119 and d == (1, 1, 119, 0)


def test_burst_with_a_shared_prefix(pair):
    """64 requests, a 448-token shared prefix and 64 distinct tokens each.  Requests of one chunk never share, so the first
    chunk (at most 8192 / 512 = 16 requests) is cold and the later ones copy the prefix from its busy slots: at least 48
    hits, 8192 + 48 x 64 = 11264 prefill tokens when the first chunk is full.  Every request stays busy far longer than
    the submissions take (96 tokens), so every hit is on a busy slot: a copy."""
    shared = pair.toks(448)
    prompts = [shared + [3 + i] + pair.toks(63) for i in range(64)]          # suffixes differ at their first token
    n_new = 96

    def go():
        tk = [pair.on.submit(p, n_new, top_logprobs=20) for p in prompts]
        return [pair.on.wait(t) for t in tk]
    recs, d = pair.delta(go)
    pair.check(recs, prompts, n_new)
    cached = [r.n_cached for r in recs]
    hits = sum(c > 0 for c in cached)
    assert set(cached) <= {0, 448} and cached[0] == 0 and hits >= 48
    assert d == (64 * 512 - 448 * hits, hits, 448 * hits, 448 * hits)


# ------------------------------------------------------------------------------------------------ HTTP
def _server(router):
    import uvicorn
    from rr_b200.server import create_app
    port = 22000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(router), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(200):
        if server.started:
            break
        time.sleep(0.05)
    return server, th, port


def test_http_conversation_reports_cached_tokens():
    import openai
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    w = make_weights(SPECS["tiny"], seed=4, sigma=0.05, device="cuda")
    on = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=2048, prefix_cache=True)
    off = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=2048)
    ml = [{"model_name": "cached", "litellm_params": {"model": "b200/tiny", "gpu": 0, "prefix_cache": True}},
          {"model_name": "plain", "litellm_params": {"model": "b200/tiny-plain", "gpu": 1}}]
    r = Router(model_list=ml, backends={0: EngineBackend(on), 1: EngineBackend(off)}, default_max_tokens=16, seed=0)
    server, th, port = _server(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        msgs = [{"role": "system", "content": "You are a terse assistant. Answer in one short sentence, no lists."}]
        prev = None
        for turn in ("hello there", "and then?", "thanks"):
            msgs.append({"role": "user", "content": turn})
            a = client.chat.completions.create(model="cached", messages=msgs, timeout=60)
            b = client.chat.completions.create(model="plain", messages=msgs, timeout=60)
            assert a.choices[0].message.content == b.choices[0].message.content
            assert a.usage.prompt_tokens == b.usage.prompt_tokens
            assert b.usage.prompt_tokens_details is None
            assert a.usage.prompt_tokens_details.cached_tokens == (0 if prev is None else prev)
            prev = a.usage.prompt_tokens
            msgs.append({"role": "assistant", "content": a.choices[0].message.content})
    finally:
        server.should_exit = True
        th.join(10)
        r.close(); on.close(); off.close()
