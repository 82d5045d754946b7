"""GPU: frequency / presence penalties and logit bias from the kernel (rr_op_logit_penalties) through the engine, the native
gateway and the HTTP front, against the float32 oracle of the contract (tests/penalty_oracle.py).

Every operation of the contract is one float32 round-to-nearest op, so the kernel must match the oracle bit for bit, and
every token the engine picks must be exactly what argmax, rr_op_sample or rr_op_logprobs give on the processed logits of
teacher-forced steps."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest
import torch

import penalty_oracle as O

pytestmark = [pytest.mark.gpu]


def _lib():
    from rr_b200 import _lib
    return _lib.lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).cuda()


def _run_op(x, vocab, hists, fp, pp, biases, hist_ld=None, bias_ld=300):
    """rr_op_logit_penalties on a copy of x [rows][ld] (float32, host) -> the processed copy (host)."""
    rows, ld = x.shape
    hist_ld = hist_ld or max(1, max(len(h) for h in hists))
    H = np.zeros((rows, hist_ld), dtype=np.int32)
    for r, h in enumerate(hists):
        H[r, :len(h)] = h
    ids = np.zeros((rows, bias_ld), dtype=np.int32)
    vals = np.zeros((rows, bias_ld), dtype=np.float32)
    for r, b in enumerate(biases):
        ids[r, :len(b)] = list(b.keys())
        vals[r, :len(b)] = list(b.values())
    d_x = _dev(x, np.float32)
    d_h, d_hl = _dev(H, np.int32), _dev([len(h) for h in hists], np.int32)
    d_fp, d_pp = _dev(fp, np.float32), _dev(pp, np.float32)
    d_ids, d_vals, d_nb = _dev(ids, np.int32), _dev(vals, np.float32), _dev([len(b) for b in biases], np.int32)
    rc = _lib().rr_op_logit_penalties(_ptr(d_x), ld, rows, vocab, _ptr(d_h), hist_ld, _ptr(d_hl), _ptr(d_fp), _ptr(d_pp),
                                      _ptr(d_ids), _ptr(d_vals), bias_ld, _ptr(d_nb), None)
    assert rc == 0
    torch.cuda.synchronize()
    return d_x.cpu().numpy()


def _oracle(x, vocab, hists, fp, pp, biases):
    want = x.copy()
    want[:, :vocab] = O.apply(x[:, :vocab], hists, fp, pp, biases)
    return want


def _cases(vocab, rng):
    """(histories, frequency penalties, presence penalties, bias maps): every shape the contract names, one row each."""
    f32 = lambda v: float(np.float32(v))                                # noqa: E731
    dup = rng.randint(0, vocab, 50)
    rows = [
        (rng.randint(0, vocab, 300).tolist(), 0.0, 0.0, {}),            # unprocessed: bitwise unchanged
        ([], 1.5, 0.5, {}),                                             # nothing generated yet: unchanged
        ([int(rng.randint(vocab))], 0.7, 0.3, {}),                      # one token
        ([int(rng.randint(vocab))] * 4096, 2.0, 2.0, {}),               # one token repeated 4096 times
        (dup[rng.randint(0, 50, 3000)].tolist(), f32(rng.uniform(-2, 2)), f32(rng.uniform(-2, 2)), {}),
        (rng.randint(0, vocab, 20000).tolist(), f32(rng.uniform(-2, 2)), f32(rng.uniform(-2, 2)), {}),   # no cap
        ([], 0.0, 0.0, {int(rng.randint(vocab)): 100.0}),               # bias only, first token
        (dup[rng.randint(0, 50, 500)].tolist(), -2.0, -1.25, {int(dup[0]): -100.0}),
        (dup[rng.randint(0, 50, 800)].tolist(), f32(rng.uniform(-2, 2)), f32(rng.uniform(-2, 2)), None),
        (rng.randint(0, vocab, 1000).tolist(), 0.0, f32(rng.uniform(-2, 2)), None),
        (rng.randint(0, vocab, 100).tolist(), 0.0, 0.0, None),          # bias only, with a history
        ([-1, vocab, vocab + 5, 3 % vocab, 3 % vocab], 1.0, 1.0, {}),   # history ids outside the vocabulary: ignored
    ]
    out = []
    for h, a, b, bias in rows:
        if bias is None:                                                # 300 entries overlapping the history
            ids = list(dict.fromkeys(list(dup) + h[:200] + rng.randint(0, vocab, 400).tolist()))[:300]
            vals = [float(np.float32(v)) for v in rng.choice([-100.0, 100.0, -0.5, 3.25, 77.7], size=len(ids))]
            bias = dict(zip(ids, vals))
        out.append((h, a, b, bias))
    return [list(c) for c in zip(*out)]


@pytest.mark.parametrize("vocab", [1024, 32000, 32064, 128256])
def test_kernel_matches_oracle_bit_for_bit(vocab):
    rng = np.random.RandomState(vocab)
    hists, fp, pp, biases = _cases(vocab, rng)
    rows, ld = len(hists), vocab + 12                                   # padded rows: columns >= vocab stay as they are
    x = (rng.standard_normal((rows, ld)) * 4).astype(np.float32)
    x[:, vocab:] = np.float32(-12345.5)
    x[0, 5] = np.float32(-0.0)
    got = _run_op(x, vocab, hists, fp, pp, biases)
    want = _oracle(x, vocab, hists, fp, pp, biases)
    assert got.tobytes() == want.tobytes()
    assert got[0].tobytes() == x[0].tobytes() and got[1].tobytes() == x[1].tobytes()
    changed = (got != x).any(axis=0)
    touched = {t for r in range(rows) for t in hists[r] if 0 <= t < vocab} | {j for b in biases for j in b}
    assert set(np.flatnonzero(changed).tolist()) <= touched
    # a second call on other rows (reversed, other penalties) gives the oracle's answer too
    hists2, biases2 = hists[::-1], biases[::-1]
    fp2 = [float(np.float32(v)) for v in rng.uniform(-2, 2, rows)]
    pp2 = [float(np.float32(v)) for v in rng.uniform(-2, 2, rows)]
    x2 = (rng.standard_normal((rows, ld)) * 4).astype(np.float32)
    got2 = _run_op(x2, vocab, hists2, fp2, pp2, biases2)
    assert got2.tobytes() == _oracle(x2, vocab, hists2, fp2, pp2, biases2).tobytes()


def test_kernel_full_batch_at_llama3_vocabulary():
    """64 rows x 128256, every row processed with a 4096-token history and 300 bias entries, as a full decode batch."""
    vocab, rows = 128256, 64
    rng = np.random.RandomState(64)
    hists = [rng.randint(0, vocab // (1 + r % 8), 4096).tolist() for r in range(rows)]
    fp = [float(np.float32(v)) for v in rng.uniform(-2, 2, rows)]
    pp = [float(np.float32(v)) for v in rng.uniform(-2, 2, rows)]
    biases = [dict(zip(rng.choice(vocab // 4, 300, replace=False).tolist(),
                       rng.uniform(-100, 100, 300).astype(np.float32).tolist())) for _ in range(rows)]
    x = (rng.standard_normal((rows, vocab)) * 4).astype(np.float32)
    assert _run_op(x, vocab, hists, fp, pp, biases).tobytes() == _oracle(x, vocab, hists, fp, pp, biases).tobytes()


# ------------------------------------------------------------------------------------------------ engine
def _prompts(n, vocab, seed, lo=3, hi=60):
    rng = np.random.RandomState(seed)
    return [rng.randint(3, vocab, size=int(rng.randint(lo, hi))).tolist() for _ in range(n)]


def _lse(x):
    x = x.astype(np.float64)
    m = x.max()
    return m + np.log(np.exp(x - m).sum())


def _sample_op(x, T, P, S, pos):
    rows = x.shape[0]
    out = torch.full((rows,), -7, dtype=torch.int32, device="cuda")
    d_s = torch.tensor(np.asarray([s % 2**64 for s in S], dtype=np.uint64).view(np.int64), device="cuda")
    assert _lib().rr_op_sample(_ptr(_dev(x, np.float32)), x.shape[1], rows, x.shape[1], _ptr(_dev(T, np.float32)),
                               _ptr(_dev(P, np.float32)), _ptr(d_s), _ptr(_dev(pos, np.int32)), _ptr(out), None) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _logprobs_op(x, tops):
    rows, vocab = x.shape
    lp = torch.full((rows, 20), float("nan"), device="cuda")
    ids = torch.full((rows, 20), -7, dtype=torch.int32, device="cuda")
    assert _lib().rr_op_logprobs(_ptr(_dev(x, np.float32)), vocab, rows, vocab, _ptr(_dev(tops, np.int32)), 20, _ptr(lp),
                                 _ptr(ids), None) == 0
    return lp.cpu().numpy(), ids.cpu().numpy()


def _params(i, vocab, rng):
    """Penalties and bias of request i: a mix of penalties only, bias only and both, negative values included."""
    fp = [0.0, 1.5, -0.5, 2.0, 0.75][i % 5]
    pp = [0.0, 0.5, 2.0, -1.0][i % 4]
    bias = {} if i % 3 == 0 else dict(zip(rng.choice(vocab, 1 + 7 * (i % 2), replace=False).tolist(),
                                          rng.choice([-100.0, 100.0, 4.5, -3.0], 1 + 7 * (i % 2)).tolist()))
    if fp == 0 and pp == 0 and not bias:
        fp = 1.0
    return fp, pp, bias


@pytest.mark.parametrize("spec_name,rows,N", [("tiny", 24, 10), ("llama-3-8b-2l", 32, 4)])
def test_engine_processed_tokens_match_oracle_on_teacher_forced_logits(spec_name, rows, N):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS[spec_name]
    w = make_weights(spec, seed=5, sigma=0.05, device="cuda")
    eng = Engine(w, max_batch=rows, ctx_max=256, max_prefill_tokens=4096, use_cuda_graph=True)
    rng = np.random.RandomState(11)
    try:
        prompts = _prompts(rows, spec.vocab, rows)
        pen = [_params(i, spec.vocab, rng) for i in range(rows)]
        temps = [[0.0, 0.8, 1.3][(i // 3) % 3] for i in range(rows)]
        seeds = [4000 + 31 * i for i in range(rows)]
        tops = [[None, 2, 0, None][i % 4] for i in range(rows)]
        tk = [eng.submit(p, N, top_logprobs=k, temperature=t, top_p=0.95, seed=s, frequency_penalty=a,
                         presence_penalty=b, logit_bias=c)
              for p, k, t, s, (a, b, c) in zip(prompts, tops, temps, seeds, pen)]
        recs = [eng.wait(t) for t in tk]
        slots = list(range(rows))
        _, lg = eng.prefill(prompts, slots, want_logits=True)
        steps = [lg]
        for j in range(1, N):
            _, lg = eng.decode_step(slots, [r.tokens[j - 1] for r in recs], [len(p) + j - 1 for p in prompts],
                                    want_logits=True)
            steps.append(lg)
        for j in range(N):
            x = O.apply(steps[j], [r.tokens[:j] for r in recs], [p[0] for p in pen], [p[1] for p in pen],
                        [p[2] for p in pen])
            tok = np.array([r.tokens[j] for r in recs])
            greedy = [i for i in range(rows) if temps[i] == 0]
            assert tok[greedy].tolist() == x[greedy].argmax(axis=1).tolist()
            samp = [i for i in range(rows) if temps[i] > 0]
            drawn = _sample_op(x[samp], [temps[i] for i in samp], [0.95] * len(samp), [seeds[i] for i in samp],
                               [len(prompts[i]) + j for i in samp])
            assert tok[samp].tolist() == drawn.tolist()
            sel = [i for i in range(rows) if tops[i] is not None]
            lp, ids = _logprobs_op(x[sel], [tops[i] for i in sel])
            for a, i in enumerate(sel):
                k = max(1, tops[i])
                pairs = recs[i].logprobs[j]
                assert len(pairs) == k + (1 if temps[i] > 0 else 0)
                assert [q[0] for q in pairs[:k]] == ids[a, :k].tolist()
                assert np.array_equal(np.array([q[1] for q in pairs[:k]], dtype=np.float32), lp[a, :k])
                if temps[i] > 0:
                    t, own = pairs[k]
                    assert t == tok[i] and abs(own - (x[i, t] - _lse(x[i]))) <= 1e-4 + 1e-6 * abs(own)
        # the processing changed something: not every row generated what the plain logits pick
        plain0 = steps[0].argmax(axis=1)
        assert any(recs[i].tokens[0] != plain0[i] for i in range(rows) if temps[i] == 0 and pen[i][2])
    finally:
        eng.close()


def _tiny(**kw):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    return Engine(make_weights(SPECS["tiny"], seed=9, sigma=0.05, device="cuda"), max_batch=kw.pop("max_batch", 64),
                  ctx_max=512, max_prefill_tokens=4096, **kw)


def test_no_leaks_between_requests_and_no_effect_on_plain_or_zero_param_rows():
    from rr_b200 import SPECS
    vocab = SPECS["tiny"].vocab
    prompt = _prompts(1, vocab, 3, 20, 30)[0]
    kw = dict(frequency_penalty=1.25, presence_penalty=0.5, logit_bias={7: 5.0, 300: -100.0})
    N = 40
    fresh = _tiny()
    try:
        want = fresh.wait(fresh.submit(prompt, N, **kw)).tokens
    finally:
        fresh.close()
    eng = _tiny()
    try:
        plain = eng.wait(eng.submit(prompt, N)).tokens
        assert plain != want
        # a long penalized request leaves slot 0 (history, counts, bias), then the same request takes that slot
        eng.wait(eng.submit(prompt[::-1], 200, frequency_penalty=-2.0, presence_penalty=2.0,
                            logit_bias={i: 50.0 for i in range(200)}))
        assert eng.wait(eng.submit(prompt, N, **kw)).tokens == want
        # zero penalties and no bias are plain, through Engine.submit and through the C entry point
        assert eng.wait(eng.submit(prompt, N, frequency_penalty=0, presence_penalty=0.0, logit_bias={})).tokens == plain
        ids = np.asarray(prompt, dtype=np.int32)
        t = C.c_uint64()
        from rr_b200._lib import GenParams
        zero = GenParams(n_choices=1, top_logprobs=-1, top_p=1.0)
        for p in (None, C.byref(zero)):
            assert _lib().rr_engine_submit(eng._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), N, p,
                                           C.byref(t)) == 0
            assert eng.wait(t.value).tokens == plain
        # a 64-request burst: plain rows bit-identical with and without processed rows beside them
        burst = _prompts(64, vocab, 17, 5, 40)
        base = [eng.submit(p, N) for p in burst]
        base = [eng.wait(t).tokens for t in base]
        mixed = [eng.submit(p, N, **(dict(kw, frequency_penalty=0.25 * (i % 8)) if i % 2 else {}))
                 for i, p in enumerate(burst)]
        mixed = [eng.wait(t).tokens for t in mixed]
        assert [mixed[i] for i in range(0, 64, 2)] == [base[i] for i in range(0, 64, 2)]
        assert any(mixed[i] != base[i] for i in range(1, 64, 2))
    finally:
        eng.close()


def test_seeded_penalized_request_is_reproducible_everywhere():
    from rr_b200 import EngineBackend, Router, SPECS
    vocab = SPECS["tiny"].vocab
    eng = _tiny()
    prompt = _prompts(1, vocab, 77, 90, 100)[0]
    kw = dict(temperature=1.1, top_p=0.95, seed=2**63 + 99, frequency_penalty=0.8, presence_penalty=-0.4,
              logit_bias={5: 3.0, 600: -100.0, 11: 2.5})
    N = 24
    try:
        alone = eng.wait(eng.submit(prompt, N, **kw)).tokens
        assert eng.wait(eng.submit(prompt, N, **kw)).tokens == alone
        assert eng.wait(eng.submit(prompt, N, **dict(kw, frequency_penalty=-2.0))).tokens != alone
        burst = [eng.submit(p, N, **({} if i % 2 else dict(kw, seed=i))) for i, p in enumerate(_prompts(62, vocab, 5))]
        t = eng.submit(prompt, N, **kw)                                  # another slot, inside a burst
        assert eng.wait(t).tokens == alone
        for b in burst:
            eng.wait(b)
        t, seen = eng.submit(prompt, N, **kw), []
        while True:
            toks, done, _ = eng.peek(t, len(seen), timeout=5)
            seen = toks
            if done:
                break
        assert eng.wait(t).tokens == alone and seen == alone
    finally:
        eng.close()
    pc = _tiny(prefix_cache=True)
    try:
        pc.wait(pc.submit(prompt[:85] + [7, 8, 9], 2, frequency_penalty=2.0))
        rec = pc.wait(pc.submit(prompt, N, **kw))
        assert rec.n_cached >= 64 and rec.tokens == alone
    finally:
        pc.close()
    bad, good = _tiny(fail_prob=0.5, fail_seed=42), _tiny()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, fallbacks=[{"chat": ["backup"]}], allowed_fails=1000,
               backends={0: EngineBackend(bad), 1: EngineBackend(good)}, seed=0)
    try:
        rkw = dict(kw, logit_bias={str(k): v for k, v in kw["logit_bias"].items()})
        fell = 0
        for _ in range(10):
            resp = r.completion("chat", prompt_ids=prompt, max_tokens=N, **rkw)
            assert resp._token_ids == alone
            fell += resp._fell_back
            streamed = [t for item in r.completion_stream("chat", prompt_ids=prompt, max_tokens=N, **rkw) for t in item[1]]
            assert streamed == alone
        assert fell > 0
    finally:
        r.close(); bad.close(); good.close()


def test_launches_and_copies_of_plain_and_processed_runs():
    """Whole runs, read while idle.  A processed request adds one launch to each of its max_new - 1 decode steps and one to
    its prefill chunk when it has a logit bias.  Its H2D bytes beyond a plain run's are exactly the parameter uploads: the
    decode rows' block (16 + 8 * 300 bytes per row) once when it joins, and the prefill chunk's block (16 + 8 * n_bias
    bytes per sequence) when it has a bias.  Plain runs cost exactly what they cost before."""
    B, N = 16, 40
    eng = _tiny(max_batch=B, use_cuda_graph=True)
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
        F = eng.stats()["kernel_launches"]
        P = (s1["kernel_launches"] - F) // (N - 1)
        pen = dict(frequency_penalty=0.5, presence_penalty=0.25)
        bias = dict(logit_bias={3: 1.0, 9: -2.0, 40: 0.5})
        samp = dict(temperature=1.0, top_p=0.9, seed=1)
        for kw in (pen, bias, dict(pen, **samp), dict(pen, top_logprobs=2)):
            run(**kw)                                                   # capture every graph
        dec = B * (16 + 8 * 300)
        _, s = run(**pen)
        assert s == dict(s1, kernel_launches=F + (N - 1) * (P + 1), h2d_bytes=s1["h2d_bytes"] + dec)
        _, s = run(**pen, **bias)
        assert s == dict(s1, kernel_launches=F + 1 + (N - 1) * (P + 1), h2d_bytes=s1["h2d_bytes"] + dec + 16 + 8 * 3)
        _, s = run(**bias)
        assert s == dict(s1, kernel_launches=F + 1 + (N - 1) * (P + 1), h2d_bytes=s1["h2d_bytes"] + dec + 16 + 8 * 3)
        _, s = run(**pen, **samp)
        assert s["kernel_launches"] == F + 3 + (N - 1) * (P + 4)
        _, s = run()
        assert s == s1                                                  # plain again: today's totals
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ routers / HTTP
def test_stub_router_validates_and_keeps_its_fixed_reply():
    from rr_b200.router import BadRequestError, Router, StubBackend
    model_list = [{"model_name": "g", "litellm_params": {"model": "b200/tiny", "gpu": 0}, "rpm": 1000}]
    r = Router(model_list=model_list, backends={0: StubBackend(vocab=1000)}, seed=0)
    try:
        msgs = [{"role": "user", "content": "hi"}]
        plain = r.completion("g", messages=msgs, max_tokens=5)
        pen = r.completion("g", messages=msgs, max_tokens=5, frequency_penalty=1, presence_penalty=-1,
                           logit_bias={"72": 100})
        assert pen._token_ids == plain._token_ids and pen.choices[0].message.content == plain.choices[0].message.content
        streamed = [t for item in r.completion_stream("g", messages=msgs, max_tokens=5, logit_bias={"5": -100})
                    for t in item[1]]
        assert streamed == plain._token_ids
        for bad in (dict(frequency_penalty=3), dict(presence_penalty="1"), dict(logit_bias={"x": 1}),
                    dict(logit_bias={"7": 1, "07": 1}), dict(logit_bias={"1000": 1}), dict(logit_bias={"1": 101})):
            with pytest.raises(BadRequestError):
                r.completion("g", messages=msgs, **bad)
            with pytest.raises(BadRequestError):
                next(r.completion_stream("g", messages=msgs, **bad))
    finally:
        r.close()


def _server(router):
    import uvicorn
    from rr_b200.server import create_app
    port = 23000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(router), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(200):
        if server.started:
            break
        time.sleep(0.05)
    return server, th, port


def _greedy_by_oracle(eng, prompt, n, fp, pp, bias):
    """Greedy decoding driven by the oracle through the engine's low-level calls: each token is the argmax of the
    oracle-processed logits of the tokens chosen so far."""
    _, lg = eng.prefill([prompt], [0], want_logits=True)
    toks = []
    for j in range(n):
        toks.append(int(O.apply_row(lg[0], toks, fp, pp, bias).argmax()))
        if j + 1 < n:
            _, lg = eng.decode_step([0], [toks[-1]], [len(prompt) + j], want_logits=True)
    return toks


def test_http_penalties_with_the_openai_sdk():
    import openai
    from rr_b200 import EngineBackend, Router
    from rr_b200.router import detokenize, messages_to_text, tokenize
    eng = _tiny(max_batch=8)
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, default_max_tokens=16, seed=0)
    server, th, port = _server(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        msgs = [{"role": "user", "content": "tell me something"}]
        e = client.chat.completions.create(model="chat", messages=msgs, timeout=60, logit_bias={"72": 100})
        assert e.choices[0].message.content == "E" * 16
        s = "".join(ch.choices[0].delta.content or "" for ch in client.chat.completions.create(
            model="chat", messages=msgs, timeout=60, stream=True, logit_bias={"72": 100}, temperature=1.0, seed=3))
        assert s == "E" * 16
        plain = client.chat.completions.create(model="chat", messages=msgs, timeout=60).choices[0].message.content
        # negative penalties reward what was generated: the plain reply, which repeats nothing, turns into repeats
        kw = dict(frequency_penalty=-2.0, presence_penalty=-1.5)
        got = client.chat.completions.create(model="chat", messages=msgs, timeout=60, **kw).choices[0].message.content
        prompt = tokenize(messages_to_text(msgs), 1024).tolist()
        assert got == detokenize(_greedy_by_oracle(eng, prompt, 16, -2.0, -1.5, {}))
        assert got != plain
        for bad in (dict(frequency_penalty=2.5), dict(presence_penalty=-3), dict(logit_bias={"abc": 1}),
                    dict(logit_bias={"72": 101}), dict(logit_bias={"1024": 1})):
            with pytest.raises(openai.BadRequestError):
                client.chat.completions.create(model="chat", messages=msgs, timeout=60, **bad)
            with pytest.raises(openai.BadRequestError):
                list(client.chat.completions.create(model="chat", messages=msgs, timeout=60, stream=True, **bad))
    finally:
        server.should_exit = True
        th.join(10)
        r.close(); eng.close()
