"""GPU: seeded temperature / top-p sampling from the kernel (rr_op_sample) through the engine, the native gateway and the
HTTP front, against the fp64 oracle of the contract (tests/sampling_oracle.py).

When the GPU's token must equal the oracle's.  The kernel computes in fp32 what the oracle computes in fp64; a draw is
compared only when both of these hold (u = 2^-24):
  * Nucleus.  The kernel's weight of token j is trunc(expf(fl(fl(x_j - m) / T)) 2^40) / 2^40.  x_j - m and the division
    each round once (relative u of the argument a = (x_j - m) / T), expf is within 2 ulp, so a weight is off by at most
    (2 |a| + 4) u relative, plus 2^-40 absolute from the fixed point.  Weights with |a| > 40 are below 5e-18 of the row
    max and never matter; so every share F(v) / Z of the nucleus masses is off by at most
    2 (80 + 4) u + vocab 2^-40 < 2e-5 = MASS_SLACK (Z >= 1 since the max's weight is 1; the integer sums are exact).  The
    kernel's tau therefore lies between the oracle's taus for masses moved by -MASS_SLACK and +MASS_SLACK.  The draw is
    clear of the nucleus boundary when the best token over the larger of those nuclei also lies in the smaller one.
  * Scores.  s = fl(fl(x / T) + fl(-logf(-logf(u)))).  logf is within 1 ulp, so L = -log u is off by <= 2u relative and
    G = -log L by <= 2u + 2u |G|; x / T rounds once (u |x / T|) and the sum once (u |s|).  So one score is within
    2^-22 (1 + |G| + |x / T| + |s|) of the fp64 score, and the best two are ordered the same when their gap exceeds the
    sum of their two bounds (Draw.score_bound).
A draw that misses either condition is ambiguous: counted and reported, never compared.  The generator itself is pinned
exactly: on an all-zero row with top_p = 1 every score is G_i, and the oracle predicts the token from integers alone.
"""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest
import torch
from scipy import stats

import sampling_oracle as O

pytestmark = [pytest.mark.gpu]

MASS_SLACK = 2e-5


def _lib():
    from rr_b200 import _lib
    return _lib.lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _run_op(logits, ld, vocab, temp, top_p, seed, pos):
    """rr_op_sample on device logits [rows][ld]; rows with temp <= 0 keep -7."""
    rows = len(temp)
    d_t = torch.tensor(temp, dtype=torch.float32, device="cuda")
    d_p = torch.tensor(top_p, dtype=torch.float32, device="cuda")
    d_s = torch.tensor(np.asarray([s % 2**64 for s in seed], dtype=np.uint64).view(np.int64), device="cuda")
    d_pos = torch.tensor(pos, dtype=torch.int32, device="cuda")
    out = torch.full((rows,), -7, dtype=torch.int32, device="cuda")
    rc = _lib().rr_op_sample(_ptr(logits), ld, rows, vocab, _ptr(d_t), _ptr(d_p), _ptr(d_s), _ptr(d_pos), _ptr(out), None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _compare(x_rows, T, P, S, Q, got):
    """-> number of ambiguous draws; asserts every clear draw equals the oracle's."""
    amb = 0
    for r in range(len(T)):
        if T[r] <= 0:
            assert got[r] == -7, r
            continue
        d = O.sample(x_rows[r], T[r], P[r], S[r], Q[r], mass_slack=MASS_SLACK)
        assert d.scores[got[r]] > -np.inf, (r, "token outside the nucleus")
        if not d.stable_nucleus or d.score_gap <= d.score_bound:
            amb += 1
            continue
        assert got[r] == d.token, (r, got[r], d.token, T[r], P[r])
    return amb


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("vocab,ld", [(128256, 128256), (32064, 32064), (32000, 32000), (1003, 1004)])
def test_kernel_against_oracle(vocab, ld):
    g = torch.Generator().manual_seed(vocab)
    rows = 24
    x = torch.randn(rows, ld, generator=g) * 2.0
    T, P, S, Q = [], [], [], []
    for r in range(rows):
        kind = r % 8
        t, p = [(1.0, 0.9), (0.7, 0.5), (2.0, 0.95), (0.05, 0.9), (1.0, 1.0), (1.3, 1e-6), (0.0, 0.9), (0.9, 0.8)][kind]
        if kind == 0:
            x[r] = torch.randn(ld, generator=g) * 0.02             # flat: the 0.9 nucleus holds most of the row
        elif kind == 1:
            x[r, int(torch.randint(0, vocab, (1,), generator=g))] = 40.0   # one dominant token
        elif kind == 7:                                            # ties straddling tau
            # at T = 0.9 the 12.0 group holds about 30 % of the mass and 12.0 + 11.0 about 97 % (the N(0, 0.5) bulk under
            # 2 % even at 128 k tokens): the 0.8 crossing falls inside the 35 tied 11.0 tokens at every vocabulary
            x[r] = torch.randn(ld, generator=g) * 0.5
            top = torch.randperm(vocab, generator=g)[:40]
            x[r, top[:5]] = 12.0
            x[r, top[5:40]] = 11.0
        T.append(t); P.append(p); S.append(int(torch.randint(-2**62, 2**62, (1,), generator=g)) * 3); Q.append(r * 37 + 5)
    x[:, vocab:] = float("nan")                                    # padding columns are never read
    for r in range(7, rows, 8):
        assert O.threshold(x[r, :vocab].numpy(), T[r], P[r]) == 11.0
    d_x = x.cuda()
    got = _run_op(d_x, ld, vocab, T, P, S, Q)
    amb = _compare(x[:, :vocab].numpy(), T, P, S, Q, got)
    print(f"vocab {vocab}: {amb} ambiguous of {sum(t > 0 for t in T)} draws")
    assert amb <= 3
    assert np.array_equal(got, _run_op(d_x, ld, vocab, T, P, S, Q))   # deterministic


def test_identical_rows_draw_identical_tokens():
    """Many CTAs of one launch resident together, each searching tau over the same flat row with the same parameters:
    every row must find the same nucleus and draw the same token, the oracle's when the draw is clear."""
    vocab, rows = 32064, 4096
    g = torch.Generator().manual_seed(5)
    row = torch.randn(vocab, generator=g) * 0.02
    x = row.cuda().expand(rows, vocab).contiguous()
    for T, p in ((1.0, 0.9), (0.7, 0.5)):
        got = _run_op(x, vocab, vocab, [T] * rows, [p] * rows, [77] * rows, [300] * rows)
        assert (got == got[0]).all(), np.unique(got)
        d = O.sample(row.numpy(), T, p, 77, 300, mass_slack=MASS_SLACK)
        assert d.scores[got[0]] > -np.inf
        if d.stable_nucleus and d.score_gap > d.score_bound:
            assert got[0] == d.token


def test_generator_pinned_exactly():
    n, rows = 1000, 4096
    x = torch.zeros(rows, n, device="cuda")
    rng = np.random.RandomState(1)
    seeds = [int(s) for s in rng.randint(0, 2**63, size=rows, dtype=np.int64)]
    seeds[:4] = [0, 1, 2**64 - 1, 2**63]
    pos = rng.randint(0, 1 << 20, size=rows).tolist()
    got = _run_op(x, n, n, [1.0] * rows, [1.0] * rows, seeds, pos)
    for r in range(rows):
        bits = O.random_words(seeds[r], pos[r], n) >> np.uint64(9)
        assert got[r] == int(np.argmax(bits)), r                   # argmax: the lowest id of the largest u


@pytest.mark.parametrize("T,p", [(1.0, 1.0), (0.6, 0.7), (1.7, 0.93), (1.0, 0.35)])
def test_distribution_of_draws(T, p):
    n, per_call, calls = 1000, 50000, 2
    g = torch.Generator().manual_seed(11)
    row = (torch.randn(n, generator=g) * 1.5).numpy().astype(np.float32)
    vals, frac = O.mass_profile(row, T)
    k = np.searchsorted(frac, np.float32(p))
    assert p >= 1 or min(frac[k] - np.float32(p), np.float32(p) - (frac[k - 1] if k else 0)) > 5 * MASS_SLACK   # clear of tau
    tau = O.threshold(row, T, p)
    inside = row >= tau
    w = np.where(inside, np.exp((row.astype(np.float64) - row.max()) / T), 0.0)
    want = w / w.sum()
    x = torch.from_numpy(row).cuda().expand(per_call, n).contiguous()
    counts = np.zeros(n, dtype=np.int64)
    for c in range(calls):
        pos = list(range(c * per_call, (c + 1) * per_call))
        got = _run_op(x, n, n, [T] * per_call, [p] * per_call, [1234 + c] * per_call, pos)
        assert np.array_equal(got, _run_op(x, n, n, [T] * per_call, [p] * per_call, [1234 + c] * per_call, pos))
        counts += np.bincount(got, minlength=n)
    N = counts.sum()
    assert counts[~inside].sum() == 0                              # never outside the nucleus
    exp = want[inside] * N
    obs = counts[inside]
    big = exp >= 5                                                 # pool the thin bins
    e2 = np.append(exp[big], exp[~big].sum()) if (~big).any() else exp[big]
    o2 = np.append(obs[big], obs[~big].sum()) if (~big).any() else obs[big]
    pv = stats.chisquare(o2, e2).pvalue
    print(f"T={T} top_p={p}: nucleus {inside.sum()} tokens, chi-square p = {pv:.3g}")
    assert pv > 1e-4


# ------------------------------------------------------------------------------------------------ engine
def _prompts(n, vocab, seed, lo=3, hi=60):
    rng = np.random.RandomState(seed)
    return [rng.randint(3, vocab, size=int(rng.randint(lo, hi))).tolist() for _ in range(n)]


def _lse(x):
    x = x.astype(np.float64)
    m = x.max()
    return m + np.log(np.exp(x - m).sum())


@pytest.mark.parametrize("spec_name,rows,N", [("tiny", 24, 6), ("llama-3-8b-2l", 32, 3)])
def test_engine_sampled_tokens_match_oracle_on_teacher_forced_logits(spec_name, rows, N):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS[spec_name]
    w = make_weights(spec, seed=5, sigma=0.05, device="cuda")
    eng = Engine(w, max_batch=rows, ctx_max=256, max_prefill_tokens=4096, use_cuda_graph=True)
    try:
        prompts = _prompts(rows, spec.vocab, rows)
        params = [([0.5, 1.0, 1.6, 0.8][i % 4], [1.0, 0.9, 0.5, 0.97][(i // 4) % 4], 1000 + 7919 * i) for i in range(rows)]
        tops = [[None, 0, 3][i % 3] for i in range(rows)]
        tk = [eng.submit(p, N, top_logprobs=k, temperature=t, top_p=q, seed=s)
              for p, k, (t, q, s) in zip(prompts, tops, params)]
        recs = [eng.wait(t) for t in tk]
        # teacher forcing on the engine's own token path
        slots = list(range(rows))
        _, lg = eng.prefill(prompts, slots, want_logits=True)
        steps = [lg]
        for j in range(1, N):
            _, lg = eng.decode_step(slots, [r.tokens[j - 1] for r in recs], [len(p) + j - 1 for p in prompts],
                                    want_logits=True)
            steps.append(lg)
        amb = 0
        for j in range(N):
            x = steps[j]
            amb += _compare(x, [p[0] for p in params], [p[1] for p in params], [p[2] for p in params],
                            [len(p) + j for p in prompts], np.array([r.tokens[j] for r in recs]))
            sel = [i for i in range(rows) if tops[i] is not None]
            top_n = torch.tensor([tops[i] for i in sel], dtype=torch.int32, device="cuda")
            lp = torch.full((len(sel), 20), float("nan"), device="cuda")
            ids = torch.full((len(sel), 20), -7, dtype=torch.int32, device="cuda")
            assert _lib().rr_op_logprobs(_ptr(torch.from_numpy(x[sel]).cuda()), spec.vocab, len(sel), spec.vocab,
                                         _ptr(top_n), 20, _ptr(lp), _ptr(ids), None) == 0
            lp, ids = lp.cpu().numpy(), ids.cpu().numpy()
            for a, i in enumerate(sel):
                k = max(1, tops[i])
                pairs = recs[i].logprobs[j]
                assert len(pairs) == k + 1
                # top_logprobs: what the same logits give under greedy, bit for bit
                assert [q[0] for q in pairs[:k]] == ids[a, :k].tolist()
                assert np.array_equal(np.array([q[1] for q in pairs[:k]], dtype=np.float32), lp[a, :k])
                # the token's own pair: x_tok - lse within the logprobs bound (a few 1e-6 here; 1e-4 is loose)
                tok, own = pairs[k]
                assert tok == recs[i].tokens[j]
                assert abs(own - (x[i, tok] - _lse(x[i]))) <= 1e-4 + 1e-6 * abs(own)
        print(f"{spec_name}: {amb} ambiguous of {rows * N} draws")
        assert amb <= max(2, rows * N // 20)
    finally:
        eng.close()


def test_seeded_request_is_reproducible_everywhere():
    from rr_b200 import EngineBackend, Router, SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS["tiny"]

    def tiny(**kw):
        return Engine(make_weights(spec, seed=9, sigma=0.05, device="cuda"), max_batch=64, ctx_max=512,
                      max_prefill_tokens=4096, **kw)
    eng = tiny()
    prompt = _prompts(1, spec.vocab, 77, 90, 100)[0]
    kw = dict(temperature=1.3, top_p=0.95, seed=2**63 + 12345)
    N = 24
    try:
        alone = eng.wait(eng.submit(prompt, N, **kw)).tokens
        assert eng.wait(eng.submit(prompt, N, **kw)).tokens == alone
        other = eng.wait(eng.submit(prompt, N, **dict(kw, seed=5))).tokens
        assert other != alone                                          # another seed draws other tokens
        greedy = eng.wait(eng.submit(prompt, N)).tokens
        assert eng.wait(eng.submit(prompt, N, temperature=0, top_p=0.5, seed=3)).tokens == greedy
        # inside a 63-request burst of mixed greedy / sampled requests, submitted last: another slot
        burst = [eng.submit(p, N, **({} if i % 2 else dict(temperature=0.9, seed=i)))
                 for i, p in enumerate(_prompts(62, spec.vocab, 5))]
        t = eng.submit(prompt, N, **kw)
        assert eng.wait(t).tokens == alone
        for b in burst:
            eng.wait(b)
        # streamed
        t, seen = eng.submit(prompt, N, **kw), []
        while True:
            toks, done, _ = eng.peek(t, len(seen), timeout=5)
            seen = toks
            if done:
                break
        assert eng.wait(t).tokens == alone and seen == alone
    finally:
        eng.close()
    # prefix cache: the prompt's first 80 tokens come from a slot another request left behind
    pc = tiny(prefix_cache=True)
    try:
        pc.wait(pc.submit(prompt[:85] + [7, 8, 9], 2))
        rec = pc.wait(pc.submit(prompt, N, **kw))
        assert rec.n_cached >= 64 and rec.tokens == alone
    finally:
        pc.close()
    # gateway, with fallback re-admission to a second replica of the same weights
    bad, good = tiny(fail_prob=0.5, fail_seed=42), tiny()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, fallbacks=[{"chat": ["backup"]}], allowed_fails=1000,
               backends={0: EngineBackend(bad), 1: EngineBackend(good)}, seed=0)
    try:
        fell = 0
        for _ in range(10):
            resp = r.completion("chat", prompt_ids=prompt, max_tokens=N, **kw)
            assert resp._token_ids == alone
            fell += resp._fell_back
            streamed = [t for item in r.completion_stream("chat", prompt_ids=prompt, max_tokens=N, **kw) for t in item[1]]
            assert streamed == alone
        assert fell > 0
    finally:
        r.close(); bad.close(); good.close()


def test_launches_and_copies_of_plain_logprobs_and_sampled_runs():
    """Whole runs, read while idle (see test_logprobs_gpu.py).  A sampled request adds three launches to its prefill chunk
    and to each of its max_new - 1 decode steps; with logprobs also the token's own logprob (4 bytes per sequence in
    prefill, 4 B per step).  Runs without sampled rows cost exactly what they cost before."""
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS["tiny"]
    w = make_weights(spec, seed=3, sigma=0.05, device="cuda")
    B, N = 16, 40
    eng = Engine(w, max_batch=B, ctx_max=1024, max_prefill_tokens=512, use_cuda_graph=True)
    keys = ("kernel_launches", "decode_steps", "prefill_chunks", "d2h_bytes", "h2d_bytes")
    prompt = list(range(5, 40))
    try:
        def run(**kw):
            eng.reset_stats()
            out = eng.wait(eng.submit(prompt, N, **kw)).tokens
            st = eng.stats()
            return out, {k: st[k] for k in keys}
        run()
        _, s1 = run()                                                   # plain graph captured by now
        eng.reset_stats()
        eng.wait(eng.submit(prompt, 1))
        F = eng.stats()["kernel_launches"]                             # one prefill chunk
        P = (s1["kernel_launches"] - F) // (N - 1)
        H = s1["h2d_bytes"]
        assert s1 == {"kernel_launches": F + (N - 1) * P, "decode_steps": N - 1, "prefill_chunks": 1,
                      "d2h_bytes": 4 + (N - 1) * 4 * B, "h2d_bytes": H}
        samp = dict(temperature=1.0, top_p=0.9, seed=1)
        run(**samp); run(top_logprobs=2, **samp); run(top_logprobs=2)   # capture every graph
        _, s = run(**samp)
        assert s == {"kernel_launches": F + 3 + (N - 1) * (P + 3), "decode_steps": N - 1, "prefill_chunks": 1,
                     "d2h_bytes": 4 + (N - 1) * 4 * B, "h2d_bytes": H + 16 * B + 20}
        _, s = run(top_logprobs=2)
        assert s == {"kernel_launches": F + 2 + (N - 1) * (P + 2), "decode_steps": N - 1, "prefill_chunks": 1,
                     "d2h_bytes": 4 + 20 * 8 + (N - 1) * (4 * B + 20 * 8 * B), "h2d_bytes": H + 4 * B + 4}
        _, s = run(top_logprobs=2, **samp)
        assert s == {"kernel_launches": F + 5 + (N - 1) * (P + 5), "decode_steps": N - 1, "prefill_chunks": 1,
                     "d2h_bytes": 4 + 20 * 8 + 4 + (N - 1) * (4 * B + 20 * 8 * B + 4 * B),
                     "h2d_bytes": H + 16 * B + 20 + 4 * B + 4}
        _, s = run()
        assert s == s1                                                  # plain again: today's totals
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ routers / HTTP
def test_stub_router_validates_and_keeps_its_fixed_reply():
    from rr_b200.router import BadRequestError, Router, StubBackend
    model_list = [{"model_name": "g", "litellm_params": {"model": "b200/tiny", "gpu": 0}, "rpm": 1000}]
    r = Router(model_list=model_list, backends={0: StubBackend()}, seed=0)
    try:
        msgs = [{"role": "user", "content": "hi"}]
        plain = r.completion("g", messages=msgs, max_tokens=5)
        samp = r.completion("g", messages=msgs, max_tokens=5, temperature=0.9, top_p=0.5, seed=3)
        assert samp._token_ids == plain._token_ids and samp.choices[0].message.content == plain.choices[0].message.content
        streamed = [t for item in r.completion_stream("g", messages=msgs, max_tokens=5, temperature=1.2, seed=4)
                    for t in item[1]]
        assert streamed == plain._token_ids
        with pytest.raises(BadRequestError):
            r.completion("g", messages=msgs, temperature=3.0)
        with pytest.raises(BadRequestError):
            next(r.completion_stream("g", messages=msgs, top_p=2))
        with pytest.raises(BadRequestError):                  # a mock replica has no logits to serve logprobs from
            r.completion("g", messages=msgs, logprobs=True)
    finally:
        r.close()


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


def test_http_sampling_with_the_openai_sdk():
    import openai
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    eng = Engine(make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda"), max_batch=8, ctx_max=256,
                 max_prefill_tokens=512)
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, default_max_tokens=16, seed=0)
    server, th, port = _server(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        msgs = [{"role": "user", "content": "tell me something"}]
        kw = dict(temperature=1.5, top_p=0.98, seed=31337)
        a = client.chat.completions.create(model="chat", messages=msgs, timeout=60, **kw)
        b = client.chat.completions.create(model="chat", messages=msgs, timeout=60, **kw)
        assert a.choices[0].message.content == b.choices[0].message.content
        s = "".join(ch.choices[0].delta.content or "" for ch in
                    client.chat.completions.create(model="chat", messages=msgs, timeout=60, stream=True, **kw))
        assert s == a.choices[0].message.content
        c = client.chat.completions.create(model="chat", messages=msgs, timeout=60, **dict(kw, seed=1))
        greedy = client.chat.completions.create(model="chat", messages=msgs, timeout=60)
        assert c.choices[0].message.content != a.choices[0].message.content
        assert greedy.choices[0].message.content != a.choices[0].message.content
        lp = client.chat.completions.create(model="chat", messages=msgs, timeout=60, logprobs=True, top_logprobs=2, **kw)
        assert lp.choices[0].message.content == a.choices[0].message.content
        assert all(len(c.top_logprobs) == 2 and c.logprob <= 0 for c in lp.choices[0].logprobs.content)
        for bad in (dict(temperature=2.5), dict(top_p=-1), dict(seed=0.5)):
            with pytest.raises(openai.BadRequestError):
                client.chat.completions.create(model="chat", messages=msgs, timeout=60, **bad)
            with pytest.raises(openai.BadRequestError):
                list(client.chat.completions.create(model="chat", messages=msgs, timeout=60, stream=True, **bad))
    finally:
        server.should_exit = True
        th.join(10)
        r.close(); eng.close()
