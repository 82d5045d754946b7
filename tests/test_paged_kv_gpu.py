"""The paged KV cache on the GPU.

Kernel level: every `_paged` entry point against its slot-contiguous counterpart, over a pool larger than needed whose
pages a random permutation hands out and whose unused bytes hold a finite sentinel.  Outputs and kv_splits match bit for
bit, the pool gathered through the table equals the contiguous cache at every written position, and every other byte still
holds the sentinel.

Engine level: placement invariance (the same requests on a fresh engine, on one whose pool fits about three of them, and
after traffic that scatters the free list give the same bits), pool pressure (FIFO, the submit refusal, pages coming back
after cancel, failure and early stops), prefix caching on a small pool, long contexts against the reference model, and the
Router's 400."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu]
DEV = "cuda"
PAGE = 64
SENT = 7.0


def _lib():
    from rr_b200 import _lib
    return _lib


def P(t):
    return C.c_void_p(t.data_ptr())


def _bits(t):
    return t.contiguous().view(torch.int16)


class Pool:
    """A paged pool for `n_slots` slots of ctx positions, pages_needed[s] pages each, plus `extra` unused pages, handed out
    by a random permutation; table entries past a slot's pages name unused pages (never read)."""

    def __init__(self, layers, kv, ctx, pages_needed, extra, g):
        self.pps = ctx // PAGE
        self.n_pages = sum(pages_needed) + extra
        perm = torch.randperm(self.n_pages, generator=g).tolist()
        self.table = torch.empty(len(pages_needed), self.pps, dtype=torch.int32)
        it = iter(perm)
        for s, n in enumerate(pages_needed):
            for j in range(self.pps):
                self.table[s, j] = next(it) if j < n else perm[-1 - (j % max(extra, 1))]
        self.dtable = self.table.to(DEV)
        shape = (layers, self.n_pages, kv, PAGE, 128)
        self.k = torch.full(shape, SENT, device=DEV, dtype=torch.bfloat16)
        self.v = torch.full(shape, SENT, device=DEV, dtype=torch.bfloat16)

    def scatter(self, dst, src, slot, n):
        """positions [0, n) of contiguous src [layers][kv][ctx][128] -> slot's pages of dst"""
        for j in range((n + PAGE - 1) // PAGE):
            m = min(PAGE, n - j * PAGE)
            dst[:, int(self.table[slot, j]), :, :m] = src[:, :, j * PAGE:j * PAGE + m]

    def expect(self, kc, vc, written):
        """the pool that holds exactly contiguous kc / vc [layers][slot][kv][ctx][128] at written[slot] positions"""
        ek, ev = torch.full_like(self.k, SENT), torch.full_like(self.v, SENT)
        for s, n in written.items():
            self.scatter(ek, kc[:, s], s, n)
            self.scatter(ev, vc[:, s], s, n)
        return ek, ev

    def check(self, kc, vc, written):
        ek, ev = self.expect(kc, vc, written)
        assert torch.equal(_bits(self.k), _bits(ek)) and torch.equal(_bits(self.v), _bits(ev))


# ------------------------------------------------------------------------------------------------ decode attention
POSITIONS = [0, 63, 64, 65, 8191, 200, 4095, 1000]


@pytest.mark.parametrize("hd", [128, 96])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("rows", [1, 5, 64, 128])
def test_decode_attn_paged_matches_contiguous(G, hd, rows):
    L = _lib()
    KV, ctx, n_splits = 2, 8192, 3
    H = G * KV
    g = torch.Generator().manual_seed(G * 1000 + hd + rows)
    pos = [POSITIONS[(r + rows) % len(POSITIONS)] for r in range(rows)]          # by slot
    # at head_dim 96 row r decodes slot (7 r + 3) % rows: the kernel then reads the table row of another slot than its own
    perm = [(7 * r + 3) % rows if hd == 96 else r for r in range(rows)]
    pad = torch.zeros(128, device=DEV)
    pad[:hd] = 1
    gd = torch.Generator(device=DEV).manual_seed(G * 1000 + hd + rows)
    kc = (torch.randn(1, rows, KV, ctx, 128, device=DEV, generator=gd) * pad).bfloat16()
    vc = (torch.randn(1, rows, KV, ctx, 128, device=DEV, generator=gd) * pad).bfloat16()
    ld = (H + 2 * KV) * hd
    qkv = torch.randn(n_splits, rows, ld, generator=g).to(DEV)
    slot = torch.tensor(perm, device=DEV, dtype=torch.int32)
    dpos = torch.tensor([pos[perm[r]] for r in range(rows)], device=DEV, dtype=torch.int32)
    pool = Pool(1, KV, ctx, [p // PAGE + 1 for p in pos], 5, g)
    for s, p in enumerate(pos):            # position p too: its padding columns beyond head_dim are not written
        pool.scatter(pool.k, kc[:, s], s, p + 1)
        pool.scatter(pool.v, vc[:, s], s, p + 1)
    out_c = torch.zeros(rows, H * hd, device=DEV, dtype=torch.bfloat16)
    out_p = torch.zeros_like(out_c)
    ks_c, ks_p = C.c_int32(), C.c_int32()
    L.check(L.lib.rr_op_decode_attn_qkv(P(qkv), n_splits, qkv.stride(0), ld, P(kc), P(vc), P(out_c), P(slot), P(dpos),
                                        rows, H, KV, hd, ctx, rows, 5e5, C.byref(ks_c), None), "contiguous")
    L.check(L.lib.rr_op_decode_attn_qkv_paged(P(qkv), n_splits, qkv.stride(0), ld, P(pool.k), P(pool.v), P(out_p),
                                              P(slot), P(dpos), rows, H, KV, hd, ctx, rows, 5e5, C.byref(ks_p),
                                              P(pool.dtable), pool.pps, pool.n_pages, None), "paged")
    torch.cuda.synchronize()
    assert ks_c.value == ks_p.value
    assert torch.equal(_bits(out_c), _bits(out_p))
    pool.check(kc, vc, {s: p + 1 for s, p in enumerate(pos)})


def test_decode_attn_paged_more_rows_than_slots():
    """rows = 4 over a table of 2 slots, rows 2 and 3 inactive (slot -1): the kernel reads only the table rows of the slots
    it decodes, and matches the contiguous counterpart bit for bit."""
    L = _lib()
    KV, G, hd, ctx, rows, n_slots = 2, 4, 128, 1024, 4, 2
    H = G * KV
    g = torch.Generator().manual_seed(17)
    pos = [700, 65]
    kc = torch.randn(1, n_slots, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    vc = torch.randn(1, n_slots, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    ld = (H + 2 * KV) * hd
    qkv = torch.randn(2, rows, ld, generator=g).to(DEV)
    slot = torch.tensor([1, 0, -1, -1], device=DEV, dtype=torch.int32)
    dpos = torch.tensor([pos[1], pos[0], 0, 0], device=DEV, dtype=torch.int32)
    pool = Pool(1, KV, ctx, [p // PAGE + 1 for p in pos], 3, g)
    assert pool.dtable.shape == (n_slots, ctx // PAGE)
    for s, p in enumerate(pos):
        pool.scatter(pool.k, kc[:, s], s, p + 1)
        pool.scatter(pool.v, vc[:, s], s, p + 1)
    out_c = torch.zeros(rows, H * hd, device=DEV, dtype=torch.bfloat16)
    out_p = torch.zeros_like(out_c)
    ks_c, ks_p = C.c_int32(), C.c_int32()
    L.check(L.lib.rr_op_decode_attn_qkv(P(qkv), 2, qkv.stride(0), ld, P(kc), P(vc), P(out_c), P(slot), P(dpos), rows, H,
                                        KV, hd, ctx, n_slots, 5e5, C.byref(ks_c), None), "contiguous")
    L.check(L.lib.rr_op_decode_attn_qkv_paged(P(qkv), 2, qkv.stride(0), ld, P(pool.k), P(pool.v), P(out_p), P(slot),
                                              P(dpos), rows, H, KV, hd, ctx, n_slots, 5e5, C.byref(ks_p), P(pool.dtable),
                                              pool.pps, pool.n_pages, None), "paged")
    torch.cuda.synchronize()
    assert ks_c.value == ks_p.value
    assert torch.equal(_bits(out_c), _bits(out_p))
    assert (out_p[2:] == 0).all()
    pool.check(kc, vc, {s: p + 1 for s, p in enumerate(pos)})


# ------------------------------------------------------------------------------------------------ prefill QKV
@pytest.mark.parametrize("hd", [128, 96])
def test_prefill_qkv_paged_matches_contiguous(hd):
    L = _lib()
    KV, H, hidden, ctx = 2, 8, 256, 8192
    g = torch.Generator().manual_seed(hd)
    # tokens of 3 slots at the page edges and at the end of the context
    toks = [(0, p) for p in (0, 1, 62, 63, 64, 65, 127, 128)] + [(1, p) for p in range(8100, 8192)] + [(2, 5), (2, 4000)]
    T = len(toks)
    plan = ((T + 127) // 128) * 128
    xhat = (torch.randn(plan, hidden, generator=g) * 0.5).to(DEV).bfloat16()
    rowss = (torch.rand(plan, hidden // 128, generator=g) * 50 + 10).to(DEV)
    wqkv = (torch.randn((H + 2 * KV) * hd, hidden, generator=g) * 0.05).to(DEV).bfloat16()
    slot = torch.tensor([s for s, _ in toks], device=DEV, dtype=torch.int32)
    pos = torch.tensor([p for _, p in toks], device=DEV, dtype=torch.int32)
    kc = torch.full((1, 3, KV, ctx, 128), SENT, device=DEV, dtype=torch.bfloat16)
    vc = kc.clone()
    need = [max(p for s, p in toks if s == q) // PAGE + 1 for q in range(3)]
    pool = Pool(1, KV, ctx, need, 4, g)
    qc = torch.zeros(T, H * 128, device=DEV, dtype=torch.bfloat16)
    qp = torch.zeros_like(qc)
    fc, fp = C.c_int32(), C.c_int32()
    L.check(L.lib.rr_op_prefill_qkv(P(xhat), P(rowss), plan, T, hidden, P(wqkv), H, KV, hd, ctx, 5e5, 1e-5, P(slot), P(pos),
                                    P(qc), P(kc), P(vc), C.byref(fc), None), "contiguous")
    L.check(L.lib.rr_op_prefill_qkv_paged(P(xhat), P(rowss), plan, T, hidden, P(wqkv), H, KV, hd, ctx, 5e5, 1e-5, P(slot),
                                          P(pos), P(qp), P(pool.k), P(pool.v), C.byref(fp), P(pool.dtable), pool.pps,
                                          pool.n_pages, None), "paged")
    torch.cuda.synchronize()
    assert fc.value == fp.value == (1 if hd == 128 else 0)
    assert torch.equal(_bits(qc), _bits(qp))
    # written positions only: gather them through the table
    for s, p in toks:
        pg = int(pool.table[s, p // PAGE])
        assert torch.equal(_bits(pool.k[0, pg, :, p % PAGE]), _bits(kc[0, s, :, p]))
        assert torch.equal(_bits(pool.v[0, pg, :, p % PAGE]), _bits(vc[0, s, :, p]))
    # and nothing else: put the sentinel back where tokens wrote, the whole pool is the sentinel again
    for s, p in toks:
        pg = int(pool.table[s, p // PAGE])
        pool.k[0, pg, :, p % PAGE] = SENT
        pool.v[0, pg, :, p % PAGE] = SENT
    assert (pool.k == SENT).all() and (pool.v == SENT).all()


# ------------------------------------------------------------------------------------------------ prefill attention
@pytest.mark.parametrize("H,KV", [(8, 8), (4, 1), (16, 2), (32, 8)])
def test_prefill_attn_cached_paged_matches_contiguous(H, KV):
    L = _lib()
    ctx = 1024
    cases = [(0, 1), (0, 200), (64, 1), (64, 130), (100, 27), (100, 300), (0, 64), (64, 64)]
    n = len(cases)
    g = torch.Generator().manual_seed(H + KV)
    kc = torch.randn(1, n, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    vc = torch.randn(1, n, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    lens, pos0 = [ln for _, ln in cases], [p for p, _ in cases]
    q = torch.randn(sum(lens), H * 128, generator=g).to(DEV).bfloat16()
    pool = Pool(1, KV, ctx, [(p + ln + PAGE - 1) // PAGE for p, ln in cases], 6, g)
    for s, (p, ln) in enumerate(cases):
        pool.scatter(pool.k, kc[:, s], s, p + ln)
        pool.scatter(pool.v, vc[:, s], s, p + ln)
    k_before, v_before = pool.k.clone(), pool.v.clone()
    start = torch.tensor([0] + np.cumsum(lens).tolist(), device=DEV, dtype=torch.int32)
    sl = torch.arange(n, device=DEV, dtype=torch.int32)
    p0 = torch.tensor(pos0, device=DEV, dtype=torch.int32)
    oc, op = torch.zeros_like(q), torch.zeros_like(q)
    scale = 1 / math.sqrt(128)
    L.check(L.lib.rr_op_prefill_attn_cached(P(q), P(kc), P(vc), P(oc), P(start), P(sl), P(p0), n, max(lens), H, KV, ctx,
                                            scale, None), "contiguous")
    L.check(L.lib.rr_op_prefill_attn_cached_paged(P(q), P(pool.k), P(pool.v), P(op), P(start), P(sl), P(p0), n, max(lens),
                                                  H, KV, ctx, scale, P(pool.dtable), pool.pps, pool.n_pages, None), "paged")
    torch.cuda.synchronize()
    assert torch.equal(_bits(oc), _bits(op))
    assert torch.equal(_bits(pool.k), _bits(k_before)) and torch.equal(_bits(pool.v), _bits(v_before))


# ------------------------------------------------------------------------------------------------ prefix copy
def test_kv_copy_prefix_paged_matches_contiguous():
    L = _lib()
    layers, S, KV, ctx = 3, 10, 2, 512
    g = torch.Generator().manual_seed(5)
    kc = torch.randn(layers, S, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    vc = torch.randn(layers, S, KV, ctx, 128, generator=g).to(DEV).bfloat16()
    copies = [(0, 5, 1), (1, 6, 63), (2, 7, 64), (0, 8, 65), (3, 9, ctx)]
    src_n = {s: ctx for s in range(5)}
    pool = Pool(layers, KV, ctx, [ctx // PAGE] * S, 7, g)
    for s in range(5):
        pool.scatter(pool.k, kc[:, s], s, ctx)
        pool.scatter(pool.v, vc[:, s], s, ctx)
    src, dst, nn = zip(*copies)
    arr = lambda x: (C.c_int32 * len(x))(*x)                                        # noqa: E731
    L.check(L.lib.rr_op_kv_copy_prefix(P(kc), P(vc), layers, S, KV, ctx, arr(src), arr(dst), arr(nn), len(copies), None),
            "contiguous")
    L.check(L.lib.rr_op_kv_copy_prefix_paged(P(pool.k), P(pool.v), layers, S, KV, ctx, arr(src), arr(dst), arr(nn),
                                             len(copies), P(pool.dtable), pool.pps, pool.n_pages, None), "paged")
    torch.cuda.synchronize()
    written = dict(src_n)
    written.update({d: m for _, d, m in copies})
    pool.check(kc, vc, written)


# ------------------------------------------------------------------------------------------------ engine
def _weights(name, seed=11):
    from rr_b200 import SPECS, make_weights
    return SPECS[name], make_weights(SPECS[name], seed=seed, sigma=0.05, device="cuda")


def _mix(spec, rng):
    """(prompt, max_new, kwargs) of greedy, seeded sampling, logprobs, stop, n = 3 and JSON-mode requests"""
    def toks(n):
        return rng.randint(3, spec.vocab, size=n).tolist()
    out = []
    for i in range(4):
        out += [(toks(40 + 37 * i), 30, {}),
                (toks(100 + 11 * i), 24, dict(temperature=0.9, top_p=0.9, seed=7 + i)),
                (toks(70), 20, dict(top_logprobs=3)),
                (toks(90 + i), 40, dict(stop=[b"\x10", b"\x20\x21"])),
                (toks(60), 16, dict(n=3, temperature=1.0, seed=3 + i, top_logprobs=1)),
                (toks(50 + i), 30, dict(response_format={"type": "json_object"}))]
    return out


def _run(eng, reqs):
    tk = [eng.submit(p, m, **kw) for p, m, kw in reqs]
    res = []
    for t in tk:
        r = eng.wait(t)
        assert r.status == 0
        lp = None if r.choice_logprobs is None else [[[(i, np.float32(v).view(np.int32)) for i, v in row] for row in c]
                                                     for c in r.choice_logprobs]
        res.append((r.choices, r.finish_reasons, lp))
    return res


def _idle_pages(eng):
    import time
    for _ in range(200):
        if eng.stats()["active_rows"] == 0 and eng.stats()["queued"] == 0:
            break
        time.sleep(0.01)
    return eng.kv_usage()


@pytest.mark.parametrize("name", ["tiny", "llama-3-8b-2l"])
def test_placement_invariance(name):
    from rr_b200.engine import Engine
    spec, w = _weights(name)
    reqs = _mix(spec, np.random.RandomState(1))
    kw = dict(max_batch=16, ctx_max=512, max_prefill_tokens=2048, use_cuda_graph=True)
    fresh = Engine(w, **kw)
    try:
        ref = _run(fresh, reqs)
        assert fresh.kv_usage() == (16 * 512 // 64, 16 * 512 // 64)
    finally:
        fresh.close()
    # 27 pages: about nine of the mix's reservations (2 to 3 pages a request, 6 for n = 3) against 16 rows, so requests
    # wait for pages, not only for rows
    small = Engine(w, kv_cache_tokens=27 * 64, **kw)
    try:
        assert small.kv_usage() == (27, 27)
        assert _run(small, reqs) == ref                               # waits and page reuse
        warm = _mix(spec, np.random.RandomState(2))[::-1]
        _run(small, warm)                                             # scatters the free list
        assert _run(small, reqs) == ref
        assert _idle_pages(small) == (27, 27)
    finally:
        small.close()


def test_pool_pressure_fifo_refusal_and_page_return():
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    rng = np.random.RandomState(3)
    eng = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=2048, kv_cache_tokens=1024, use_cuda_graph=True,
                 fail_prob=0.0)
    try:
        big = rng.randint(3, spec.vocab, size=600).tolist()
        small = rng.randint(3, spec.vocab, size=20).tolist()
        # submit refuses what the pool can never hold, with nothing queued
        with pytest.raises(Exception):
            eng.submit(small, 120, n=8)                               # 8 x 3 pages
        with pytest.raises(Exception):
            eng.submit(small, 1000, n=2)
        assert eng.stats()["queued"] == 0 and eng.kv_usage() == (16, 16)
        # FIFO: a 10-page request runs, the big 16-page one waits at the head, the small ones behind it do not overtake
        t0 = eng.submit(rng.randint(3, spec.vocab, size=600).tolist(), 40)
        t1 = eng.submit(big, 400)
        ts = [eng.submit(small, 5) for _ in range(3)]
        r0, r1 = eng.wait(t0), eng.wait(t1)
        rs = [eng.wait(t) for t in ts]
        assert r0.status == r1.status == 0 and all(r.status == 0 for r in rs)
        assert r1.t_first_token >= r0.t_done
        assert all(r.t_first_token >= r1.t_first_token for r in rs)
        assert _idle_pages(eng) == (16, 16)
        # cancel returns the pages
        t = eng.submit(big, 400)
        eng.peek(t, 0, timeout=60)
        assert _lib().lib.rr_engine_cancel(eng._h, t) == 0
        assert _idle_pages(eng) == (16, 16)
        # an early stop returns them too
        ref = eng.wait(eng.submit(small, 100))
        tok = next(t for t in ref.tokens[5:] if t >= 3)
        cut = eng.wait(eng.submit(small, 100, stop=[bytes([(tok - 3) % 256])]))
        assert cut.finish_reasons == ["stop"]
        assert _idle_pages(eng) == (16, 16)
    finally:
        eng.close()
    failing = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=2048, kv_cache_tokens=1024, use_cuda_graph=True,
                     fail_prob=0.5, fail_seed=1)
    try:
        recs = [failing.wait(failing.submit(small, 20)) for _ in range(8)]
        assert {r.status for r in recs} >= {0}
        assert _idle_pages(failing) == (16, 16)
    finally:
        failing.close()


def test_prefix_cache_on_a_small_pool():
    """12 pages, ctx_max 512.  Hits give the bits of a plain engine and report n_cached; under pressure the least recently
    used retained prefix goes first, and a request that needs the whole pool still runs (no page leaks)."""
    from rr_b200.engine import Engine
    spec, w = _weights("tiny")
    rng = np.random.RandomState(4)
    kw = dict(max_batch=8, ctx_max=512, max_prefill_tokens=2048, use_cuda_graph=True)
    plain = Engine(w, **kw)
    cached = Engine(w, prefix_cache=True, kv_cache_tokens=12 * 64, **kw)

    def toks(n):
        return rng.randint(3, spec.vocab, size=n).tolist()
    try:
        def both(p, n=8):
            want = plain.wait(plain.submit(p, n, top_logprobs=2))
            got = cached.wait(cached.submit(p, n, top_logprobs=2), timeout=120)
            assert got.status == 0 and got.tokens == want.tokens and got.logprobs == want.logprobs
            return got.n_cached
        a, b = toks(300), toks(300)
        assert both(a) == 0
        assert both(a[:200] + b[:50]) == 200            # hit on a's slot, which kept its 5 pages; it now keeps 4
        assert both(b) == 0                             # a second slot keeps 5 pages: 9 of 12 held
        assert both(toks(400)) == 0                     # 7 pages: the older prefix (a's slot) is reclaimed, b's stays
        assert both(b[:100] + a[:10]) == 100
        assert both(a[:200] + b[:10]) == 0
        # every choice of this request needs 4 pages: all 12, so every page must come back
        t = cached.submit(toks(200), 50, n=3)
        assert cached.wait(t, timeout=120).status == 0
        assert cached.stats()["prefix_hits"] == 2
    finally:
        plain.close()
        cached.close()


def test_long_context_matches_oracle():
    from oracle import llama_ref
    from rr_b200.engine import Engine
    spec, w = _weights("tiny", seed=13)
    eng = Engine(w, max_batch=8, ctx_max=8192, max_prefill_tokens=8192, kv_cache_tokens=2 * 8192, use_cuda_graph=True)
    try:
        g = torch.Generator().manual_seed(8)
        prompts = [torch.randint(3, spec.vocab, (n,), generator=g).tolist() for n in (8000, 7900)]
        tk = [eng.submit(p, 6) for p in prompts]
        recs = [eng.wait(t) for t in tk]
        w_cpu = w.to("cpu")
        for p, r in zip(prompts, recs):
            assert r.status == 0
            seq = list(p)
            for t in r.tokens[:2]:
                want = int(llama_ref.forward_logits(w_cpu, seq)[-1].argmax())
                assert t == want
                seq.append(t)
        assert _idle_pages(eng) == (256, 256)
    finally:
        eng.close()


def test_router_long_message_and_pool_400():
    from rr_b200.config import build_config
    from rr_b200.router import Router, BadRequestError
    from rr_b200.server import build_backends
    cfg = build_config([{"model_name": "m", "litellm_params": {"model": "b200/tiny", "context_window": 8192,
                                                               "kv_cache_tokens": 8192 + 1024}}])
    backends = build_backends(cfg, stub=False, max_batch=4)
    router = Router(config=cfg, backends=backends, seed=0)
    try:
        assert backends[0].engine.kv_usage() == (144, 144)
        msg = "x" * 6000
        r = router.completion(model="m", messages=[{"role": "user", "content": msg}], max_tokens=8)
        assert r.usage.prompt_tokens > 6000 and len(r.choices) == 1
        with pytest.raises(BadRequestError, match="exceed the KV cache"):
            router.completion(model="m", messages=[{"role": "user", "content": msg}], max_tokens=8, n=2)
    finally:
        router.close()
        for b in backends.values():
            b.engine.close()
