"""GPU: long prompts, prefilled in pieces over several chunks between decode steps.

Every prefill kernel computes a row independently of the chunk it is in, and prefill attention takes each sequence's
first position (seq_pos0).  So a prompt cut into pieces gives the KV, logits and tokens of the same prompt in one chunk,
bit for bit: an engine whose max_prefill_tokens holds the whole prompt is the oracle of one that does not.

Kernel level: prefill attention for an 8192-row query piece deep in a 65536-token context over a scattered page pool,
against the matching rows of one cold whole-sequence call and the exact answer of selection operands.  Engine level: piece invariance (greedy,
sampled, n choices with bias / penalties / stop / JSON), long contexts at size, interleaving with decode, the exact cost
of a chunk without tail rows, cancel / failure / prefix caching mid-prompt, FIFO on a small pool.  Gateway: a
65536-token context window through Router.completion, streaming and fallback."""
import ctypes as C
import math
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


def _weights(name, seed=11):
    from rr_b200 import SPECS, make_weights
    return SPECS[name], make_weights(SPECS[name], seed=seed, sigma=0.05, device="cuda")


def _toks(spec, n, seed):
    return np.random.RandomState(seed).randint(3, spec.vocab, size=n).tolist()


def _res(r):
    """tokens, finish reasons and logprob pairs (values as their bits) of a completion record"""
    assert r.status == 0, r.status
    lp = None if r.choice_logprobs is None else [[[(i, np.float32(v).view(np.int32)) for i, v in row] for row in c]
                                                 for c in r.choice_logprobs]
    return r.choices, r.finish_reasons, lp


def _run(eng, reqs, timeout=600):
    tk = [eng.submit(p, m, **kw) for p, m, kw in reqs]
    return [_res(eng.wait(t, timeout=timeout)) for t in tk]


def _idle(eng):
    for _ in range(500):
        st = eng.stats()
        if st["active_rows"] == 0 and st["queued"] == 0:
            break
        time.sleep(0.01)
    return eng.kv_usage()


def _wait_chunks(eng, n, limit=30.0):
    t0 = time.time()
    while eng.stats()["prefill_chunks"] < n:
        assert time.time() - t0 < limit
        time.sleep(0.0005)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("H,KV", [(32, 8), (16, 2)])
def test_prefill_attention_pieces_deep_in_a_65536_context(H, KV):
    """Query pieces of 8192 rows at pos0 = 8192, 24576 and 57344 (up to 1024 key tiles per query tile) over pages
    scattered through the pool, on the selection operands of test_long_context_attn_gpu.py: the rows of one cold call over
    the whole sequences, bit for bit, and every row the exact mean of V over the keys its heads select."""
    from test_long_context_attn_gpu import check_prefill_rows, prefill_queries, prefill_sequence
    L = _lib()
    PAGE, ctx, piece = 64, 65536, 8192
    pos0 = [8192, 24576, 57344]
    full = [p + piece for p in pos0]
    n = len(pos0)
    pps = ctx // PAGE
    G = H // KV
    g = torch.Generator().manual_seed(H + KV)
    n_pages = sum(m // PAGE for m in full) + 16
    perm = torch.randperm(n_pages, generator=g)
    table = torch.zeros(n, pps, dtype=torch.int32)
    k = 0
    for s, m in enumerate(full):
        table[s, :m // PAGE] = perm[k:k + m // PAGE]
        table[s, m // PAGE:] = perm[-1]
        k += m // PAGE
    dtable = table.to(DEV)
    gd = torch.Generator(device=DEV).manual_seed(H * 3 + KV)
    kp = torch.full((n_pages, KV, PAGE, 128), 7.0, device=DEV, dtype=torch.bfloat16)
    vp = kp.clone()
    seqs, qf = [], []
    for s, m in enumerate(full):
        res, K, V = prefill_sequence(H, KV, m, g, gd)
        pages = table[s, :m // PAGE].long().to(DEV)
        kp[pages] = K.view(KV, m // PAGE, PAGE, 128).transpose(0, 1)
        vp[pages] = V.view(KV, m // PAGE, PAGE, 128).transpose(0, 1)
        qf.append(prefill_queries(res, torch.arange(m, device=DEV), H, G))
        seqs.append((res, V))
        del K
    scale = 1 / math.sqrt(128)

    def call(q, lens, p0):
        start = torch.tensor([0] + np.cumsum(lens).tolist(), device=DEV, dtype=torch.int32)
        sl = torch.arange(n, device=DEV, dtype=torch.int32)
        dp0 = torch.tensor(p0, device=DEV, dtype=torch.int32)
        out = torch.zeros_like(q)
        L.check(L.lib.rr_op_prefill_attn_cached_paged(P(q), P(kp), P(vp), P(out), P(start), P(sl), P(dp0), n, max(lens),
                                                      H, KV, ctx, scale, P(dtable), pps, n_pages, None), "attn")
        torch.cuda.synchronize()
        return out, start.tolist()

    out, st = call(torch.cat([q[p:] for q, p in zip(qf, pos0)]), [piece] * n, pos0)
    cold, stf = call(torch.cat(qf), full, [0] * n)
    for i, p in enumerate(pos0):
        got = out[st[i]:st[i] + piece]
        assert torch.equal(_bits(got), _bits(cold[stf[i] + p:stf[i + 1]])), i
        res, V = seqs[i]
        check_prefill_rows(got, res, V, torch.arange(p, p + piece, device=DEV), H, G)


# ------------------------------------------------------------------------------------------------ piece invariance
def _mixed(spec, T):
    """greedy and seeded sampled requests, with top-20 logprobs, at every prompt length around the chunk size"""
    out = []
    for i, n in enumerate([T + 1, 2 * T - 1, 2 * T, 2 * T + 1, 5 * T + 37]):
        p = _toks(spec, n, 100 + n)
        out += [(p, 12, dict(top_logprobs=20)), (p, 12, dict(top_logprobs=20, temperature=0.9, top_p=0.9, seed=40 + i))]
    return out


def _combined(spec, T, seed, n):
    bias = {3 + ord("{"): 4.0, 3 + ord('"'): 2.0, 7: -5.0}
    return (_toks(spec, 2 * T + 9, 77), 16,
            dict(n=n, temperature=1.0, seed=seed, logit_bias=bias, frequency_penalty=0.5, presence_penalty=0.3,
                 stop=[b"\x22\x3a", b"}"], response_format={"type": "json_object"}, top_logprobs=3))


@pytest.mark.parametrize("name", ["tiny", "tiny96", "llama-3-8b-2l"])
def test_pieces_give_the_bits_of_one_chunk(name):
    from rr_b200.engine import Engine
    spec, w = _weights(name)
    kw = dict(max_batch=16, ctx_max=4096, use_cuda_graph=True)
    ref = Engine(w, max_prefill_tokens=4096, **kw)
    try:
        want = {T: _run(ref, _mixed(spec, T)) for T in (512, 500)}
        singles = {T: [_run(ref, [_combined(spec, T, 9 + i, 1)])[0] for i in range(3)] for T in (512, 500)}
    finally:
        ref.close()
    for T in (512, 500):
        eng = Engine(w, max_prefill_tokens=T, **kw)
        try:
            reqs = _mixed(spec, T)
            assert _run(eng, reqs) == want[T]
            st = eng.stats()
            assert st["prefill_tokens"] == sum(len(p) for p, _, _ in reqs)          # every prompt token once
            assert st["prefill_chunks"] >= -(-st["prefill_tokens"] // T)
            toks, fin, lp = _run(eng, [_combined(spec, T, 9, 3)])[0]
            for i, (t1, f1, l1) in enumerate(singles[T]):
                assert toks[i] == t1[0] and fin[i] == f1[0] and lp[i] == l1[0], i
            assert _idle(eng) == (16 * 4096 // 64,) * 2
        finally:
            eng.close()


# ------------------------------------------------------------------------------------------------ long contexts at size
def _one_vs_pieces(w, spec, ctx, n_prompt, piece, max_batch=2):
    from rr_b200.engine import Engine
    p = _toks(spec, n_prompt, n_prompt)
    out = []
    for T in (ctx, piece):
        eng = Engine(w, max_batch=max_batch, ctx_max=ctx, max_prefill_tokens=T, kv_cache_tokens=ctx,
                     use_cuda_graph=True)
        try:
            out.append(_run(eng, [(p, 4, dict(top_logprobs=20))]))
            st = eng.stats()
            assert st["prefill_chunks"] == -(-n_prompt // T) and st["prefill_tokens"] == n_prompt
        finally:
            eng.close()
        torch.cuda.empty_cache()
    assert out[0] == out[1]


def test_64000_token_prompt_in_8_pieces_llama_2l():
    spec, w = _weights("llama-3-8b-2l")
    _one_vs_pieces(w, spec, 65536, 64000, 8192)


def test_32000_token_prompt_in_4_pieces_full_llama():
    spec, w = _weights("llama-3-8b")
    _one_vs_pieces(w, spec, 32768, 32000, 8192)


def test_32000_token_prompt_matches_the_oracle():
    from oracle import llama_ref
    from rr_b200.engine import Engine
    spec, w = _weights("tiny", seed=13)
    eng = Engine(w, max_batch=2, ctx_max=32768, max_prefill_tokens=8192, kv_cache_tokens=32768, use_cuda_graph=True)
    try:
        p = _toks(spec, 32000, 8)
        r = eng.wait(eng.submit(p, 2))
        assert r.status == 0 and eng.stats()["prefill_chunks"] == 4
    finally:
        eng.close()
    seq = list(p)
    with torch.no_grad():
        for t in r.tokens[:2]:
            assert t == int(llama_ref.forward_logits(w, seq)[-1].argmax())        # fp32 on the GPU
            seq.append(t)
            torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ interleaving, costs
def test_decode_runs_between_pieces():
    """R short requests that each want k tokens share the first chunk of a k-piece prompt: one decode step follows each
    non-final piece, so every short request is done before the long one's first token."""
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    T, R, k, short = 512, 4, 6, 20
    eng = Engine(w, max_batch=8, ctx_max=4096, max_prefill_tokens=T, use_cuda_graph=True)
    try:
        eng.wait(eng.submit(_toks(spec, short, 1), 2))                              # warm-up: the decode graph
        long_p = _toks(spec, (T - R * short) + (k - 1) * T, 2)
        tk = [eng.submit(_toks(spec, short, 10 + i), k) for i in range(R)]
        tl = eng.submit(long_p, 3)
        rs = [eng.wait(t) for t in tk]
        rl = eng.wait(tl)
        assert rl.status == 0 and all(r.status == 0 and len(r.tokens) == k for r in rs)
        assert all(r.t_done <= rl.t_first_token for r in rs), ([r.t_done for r in rs], rl.t_first_token)
        # without a long prompt: one chunk and k - 1 decode steps, F + (k - 1) P launches
        eng.reset_stats()
        eng.wait(eng.submit(_toks(spec, short, 3), 1))
        F = eng.stats()["kernel_launches"]
        eng.reset_stats()
        eng.wait(eng.submit(_toks(spec, short, 3), 2))
        Pst = eng.stats()["kernel_launches"] - F
        eng.reset_stats()
        eng.wait(eng.submit(_toks(spec, short, 3), k))
        st = eng.stats()
        assert st["decode_steps"] == k - 1 and st["prefill_chunks"] == 1
        assert st["kernel_launches"] == F + (k - 1) * Pst
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["tiny", "tiny96"])
def test_a_chunk_without_tail_rows_costs_exactly(name):
    """A three-piece prompt with max_tokens 1 (no decode step): the two non-final chunks launch embed + norm + L x (QKV,
    rope_kv unless fused) + (L - 1) x (attention, O, gate/up, down, silu_mul unless fused) each, copy nothing back, and
    upload the chunk's ids / positions / slots / sequence arrays, with the pos0 column only for a continuation."""
    from rr_b200.engine import Engine
    spec, w = _weights(name)
    T = 256
    eng = Engine(w, max_batch=32, ctx_max=1024, max_prefill_tokens=T, use_cuda_graph=True)
    try:
        fuse_rope, fuse_silu = spec.head_dim == 128, hasattr(eng, "_wgu_il")
        Lr = spec.n_layers
        NF = 2 + Lr * (1 + (0 if fuse_rope else 1)) + (Lr - 1) * (4 + (0 if fuse_silu else 1))
        short, long_p = _toks(spec, 100, 1), _toks(spec, 2 * T + 100, 2)
        eng.wait(eng.submit(long_p, 1))                  # the slot's pages and table row are in place from here on
        eng.wait(eng.submit(short, 1))
        eng.reset_stats()
        eng.wait(eng.submit(short, 1))
        one = eng.stats()
        eng.reset_stats()
        eng.wait(eng.submit(long_p, 1))
        st = eng.stats()
        assert st["prefill_chunks"] == 3 and st["decode_steps"] == 0 and st["prefill_tokens"] == 2 * T + 100
        assert st["kernel_launches"] == one["kernel_launches"] + 2 * NF
        assert st["d2h_bytes"] == one["d2h_bytes"] == 4
        # ids | pos | slot (3 per token) + seq_start (2) + seq_slot + last per chunk, pos0 for the two continuations
        assert one["h2d_bytes"] == 4 * (3 * 100 + 4)
        assert st["h2d_bytes"] == 4 * (3 * (2 * T + 100) + 3 * 4 + 2)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ lifecycle
def test_cancel_and_failure_mid_prompt_return_rows_and_pages():
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    kw = dict(max_batch=4, ctx_max=32768, max_prefill_tokens=128, kv_cache_tokens=32768, use_cuda_graph=True)
    eng = Engine(w, **kw)
    fresh = Engine(w, **kw)
    try:
        t = eng.submit(_toks(spec, 30000, 5), 8)
        _wait_chunks(eng, 3)
        assert _lib().lib.rr_engine_cancel(eng._h, t) == 0
        assert _idle(eng) == (512, 512)
        assert eng.stats()["generated_tokens"] == 0                  # cancelled before its last piece
        p = _toks(spec, 1000, 6)
        assert _run(eng, [(p, 8, dict(top_logprobs=5))]) == _run(fresh, [(p, 8, dict(top_logprobs=5))])
    finally:
        eng.close()
        fresh.close()
    failing = Engine(w, fail_prob=0.5, fail_seed=3, **kw)
    try:
        recs = [failing.wait(failing.submit(_toks(spec, 3000 + i, i), 4)) for i in range(6)]
        assert {r.status for r in recs} >= {0}
        assert _idle(failing) == (512, 512)
    finally:
        failing.close()


def test_prefix_cache_with_long_prompts():
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    kw = dict(max_batch=8, ctx_max=16384, max_prefill_tokens=512, use_cuda_graph=True)
    plain, cached = Engine(w, **kw), Engine(w, prefix_cache=True, **kw)
    try:
        def both(p, n=8):
            want = plain.wait(plain.submit(p, n, top_logprobs=2))
            got = cached.wait(cached.submit(p, n, top_logprobs=2), timeout=300)
            assert got.status == 0 and got.tokens == want.tokens and got.logprobs == want.logprobs
            return got
        turn1 = _toks(spec, 3000, 1)
        r1 = both(turn1)
        assert r1.n_cached == 0
        # turn 2 of the conversation: the whole first prompt is cached, and the uncached rest still takes pieces
        turn2 = turn1 + r1.tokens + _toks(spec, 1500, 2)
        assert both(turn2).n_cached == 3000
        # a shorter prompt sharing a long prefix of turn 2 hits it too
        assert both(turn2[:3200] + _toks(spec, 700, 3)).n_cached == 3200
        assert cached.stats()["prefix_hits"] == 2
        # a low-level call mid-prompt clears the index: the prompt starts again and its tokens do not change
        long_p = _toks(spec, 12000, 4)
        want = plain.wait(plain.submit(long_p, 8, top_logprobs=2))
        cached.reset_stats()
        t = cached.submit(long_p, 8, top_logprobs=2)
        _wait_chunks(cached, 3)
        cached.prefill([_toks(spec, 10, 5)], [7])
        got = cached.wait(t, timeout=300)
        assert got.status == 0 and got.tokens == want.tokens and got.logprobs == want.logprobs
        assert cached.stats()["prefill_tokens"] > 12000                             # some pieces ran twice
    finally:
        plain.close()
        cached.close()


def test_small_pool_keeps_fifo_behind_a_long_prompt():
    """The pool holds one long request: the short ones submitted behind it wait for its pages and start in order."""
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    eng = Engine(w, max_batch=8, ctx_max=8192, max_prefill_tokens=512, kv_cache_tokens=8192, use_cuda_graph=True)
    try:
        tl = eng.submit(_toks(spec, 8000, 1), 190)                       # 128 pages: the whole pool
        ts = [eng.submit(_toks(spec, 50 + i, 2 + i), 4) for i in range(5)]
        rl = eng.wait(tl)
        rs = [eng.wait(t) for t in ts]
        assert rl.status == 0 and all(r.status == 0 for r in rs)
        assert all(r.t_first_token >= rl.t_done for r in rs)
        assert all(a.t_first_token <= b.t_first_token for a, b in zip(rs, rs[1:]))
        assert _idle(eng) == (128, 128)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ gateway
def _long_router():
    from rr_b200.config import build_config
    from rr_b200.router import Router
    from rr_b200.server import build_backends
    cfg = build_config([{"model_name": "m", "litellm_params": {"model": "b200/tiny", "context_window": 65536,
                                                               "kv_cache_tokens": 262144}}])
    backends = build_backends(cfg, stub=False, max_batch=8)
    return Router(config=cfg, backends=backends, seed=0), backends


def test_router_serves_a_40000_byte_message():
    from rr_b200.router import BadRequestError, messages_to_text, tokenize
    router, backends = _long_router()
    eng = backends[0].engine
    try:
        msgs = [{"role": "user", "content": "".join(chr(97 + (i * 7) % 26) for i in range(40000))}]
        ids = tokenize(messages_to_text(msgs), eng.spec.vocab).tolist()
        assert len(ids) > 40000
        want = eng.wait(eng.submit(ids, 8))
        r = router.completion(model="m", messages=msgs, max_tokens=8)
        assert r._token_ids == want.tokens and r.usage.prompt_tokens == len(ids)
        # streaming: the first chunk comes after the last of the prompt's pieces
        eng.reset_stats()
        got = []
        for item in router.completion_stream(model="m", messages=msgs, max_tokens=8):
            if not got:
                assert eng.stats()["prefill_chunks"] >= -(-len(ids) // 8192)
            got += item[1]
        assert got == want.tokens
        with pytest.raises(BadRequestError, match="context window"):
            router.completion(model="m", messages=[{"role": "user", "content": "x" * 65536}], max_tokens=8)
    finally:
        router.close()
        for b in backends.values():
            b.engine.close()


def test_fallback_replays_a_long_prompt_and_the_trace_replays():
    from rr_b200 import EngineBackend, Router
    from rr_b200.engine import Engine
    from test_gateway_gpu import _replay
    spec, w = _weights("tiny", seed=0)
    kw = dict(max_batch=4, ctx_max=65536, max_prefill_tokens=8192, kv_cache_tokens=65536 * 2)
    bad, good, ref = Engine(w, fail_prob=0.5, fail_seed=42, **kw), Engine(w, **kw), Engine(w, **kw)
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny", "gpu": 1}}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends={0: EngineBackend(bad), 1: EngineBackend(good)}, seed=0,
               clock=lambda: 7000.0)
    r.record_trace = 4096
    try:
        fell = 0
        for k in range(12):
            p = _toks(spec, 9000 + 997 * k, k)
            want = ref.wait(ref.submit(p, 6))
            o = r.completion(model="primary", prompt_ids=p, max_tokens=6)
            assert o._token_ids == want.tokens
            fell += o._fell_back
        assert 0 < fell < 12
        assert _replay(r, r.gateway_trace()) == 12 + fell
    finally:
        r.close(); bad.close(); good.close(); ref.close()
