"""GPU: JSON mode (`response_format: {"type": "json_object"}`), from rr_op_json_mask / rr_op_json_advance through the
engine's logits tail, early row release, the native gateway and the router to the OpenAI endpoint.

The contract is exact.  The mask only writes -inf to the columns tests/json_oracle.py disallows, so every token is the
argmax / the sampler's draw over the oracle-masked logits of the row's own prefix, and the reply is always a prefix of a
JSON object."""
import ctypes as C
import dataclasses
import json
import threading
import time

import numpy as np
import pytest

import json_oracle as J
import sampling_oracle as S

pytestmark = [pytest.mark.gpu]

JS = {"type": "json_object"}


def _lib():
    from rr_b200 import _lib as L
    return L.lib


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _allowed_mask(state):
    a = np.zeros(256, dtype=bool)
    a[list(J.allowed(state))] = True
    return a


def _masked_cols(state, vocab):
    c = np.arange(vocab)
    return (c < 3) | ~_allowed_mask(state)[(c - 3) % 256]


def _loads(data: bytes):
    v = json.loads(data.decode("utf-8"), parse_constant=lambda n: (_ for _ in ()).throw(ValueError(n)))
    assert isinstance(v, dict)
    return v


def _text(tokens):
    return bytes((t - 3) % 256 for t in tokens if t >= 3)


def _valid_prefix(tokens):
    assert all(t >= 3 for t in tokens), tokens
    s, k = J.accepts(_text(tokens))
    assert k == len(tokens), (_text(tokens), k)
    return s


# ---------------------------------------------------------------- 1. kernels against the oracle
ADVERSARIAL = [
    b'{"a":' + b"[" * 63 + b"1" + b"]" * 63 + b"}",                  # depth 64
    b"{" + b" " * 64 + b'"k"' + b"\t" * 64 + b":" + b"\n" * 64 + b"0" + b"\r" * 64 + b"}",   # whitespace runs at the cap
    b'{"\xf0\x9f\x98\x80\xf4\x8f\xbf\xbf":"\xe0\xa0\x80\xed\x9f\xbf"}',  # 4-byte characters pending
    b'{"\\u00e9\\uD83D\\uDE00":"\\"\\\\\\/\\b\\f\\n\\r\\t"}',          # \u escapes
    b'{"a":-0.5e+10,"b":[true,false,null,0,1E-2]}',
]


def _run_kernels(docs, vocab, ld, fmt, active, seed):
    """Feed doc[r]'s bytes to row r through rr_op_json_mask / rr_op_json_advance, one token per step, checking every
    step against the oracle.  Rows with fmt 0 or inactive, and rows whose document has ended, must not be touched.
    -> the final state bytes."""
    import torch
    rows = len(docs)
    rng = np.random.RandomState(seed)
    d_fmt = torch.tensor(fmt, dtype=torch.int32, device="cuda")
    d_act = torch.tensor(active, dtype=torch.int32, device="cuda")
    state = torch.zeros((rows, 16), dtype=torch.uint8, device="cuda")
    done = torch.full((rows,), -5, dtype=torch.int32, device="cuda")
    ost = [J.initial() for _ in range(rows)]
    live = [fmt[r] != 0 and active[r] >= 0 for r in range(rows)]
    steps = max(len(d) for d in docs)
    for j in range(steps):
        x = torch.from_numpy(rng.standard_normal((rows, ld)).astype(np.float32)).cuda()
        x0 = x.clone()
        step_fmt = d_fmt.clone()
        for r in range(rows):
            if j >= len(docs[r]):
                step_fmt[r] = 0                               # ended: from now on a format-0 row
        assert _lib().rr_op_json_mask(_ptr(x), ld, rows, vocab, _ptr(step_fmt), _ptr(d_act),
                                      _ptr(state) if j else None, None) == 0
        got, ref = x.cpu().numpy(), x0.cpu().numpy()
        for r in range(rows):
            if live[r] and j < len(docs[r]):
                m = _masked_cols(ost[r], vocab)
                assert (np.isneginf(got[r, :vocab]) == m).all(), (r, j, docs[r][:j])
                keep = np.concatenate([~m, np.ones(ld - vocab, dtype=bool)])
                assert (got[r][keep].view(np.uint32) == ref[r][keep].view(np.uint32)).all()
            else:
                assert (got[r].view(np.uint32) == ref[r].view(np.uint32)).all()
        # the token: the document's byte under an id of its byte class, ids >= 259 included
        tok = []
        for r in range(rows):
            b = docs[r][j] if j < len(docs[r]) else 32
            k = int(rng.randint(0, (vocab - 3 - b - 1) // 256 + 1))
            tok.append(3 + b + 256 * k)
        d_tok = torch.tensor(tok, dtype=torch.int32, device="cuda")
        done.fill_(-5)
        before = state.clone()
        assert _lib().rr_op_json_advance(rows, _ptr(step_fmt), _ptr(d_act), _ptr(d_tok), _ptr(state) if j else None,
                                         _ptr(state), None, _ptr(done), None) == 0
        dn = done.cpu().numpy()
        for r in range(rows):
            if live[r] and j < len(docs[r]):
                ost[r] = J.advance(ost[r], docs[r][j])
                assert dn[r] == int(J.done(ost[r])), (r, j)
            else:
                assert dn[r] == -5 and (state[r] == before[r]).all()
    return state.cpu().numpy()


@pytest.mark.parametrize("rows,vocab,ld", [(1, 1024, 1024), (7, 1003, 1004), (64, 32000, 32000), (3, 32064, 32064),
                                           (4, 128256, 128256), (5, 2 * 8192 + 100, 2 * 8192 + 100), (256, 1024, 1028)])
def test_kernels_equal_the_oracle(rows, vocab, ld):
    docs = (ADVERSARIAL + J.random_docs(rows, rows))[:rows]
    if vocab > 100000 or rows >= 64:
        docs = [d[:40] for d in docs]                           # prefixes: the states the documents open with
    fmt = [0 if r % 7 == 6 else 1 for r in range(rows)]
    active = [-1 if r % 5 == 4 else r for r in range(rows)]
    if rows == 1:
        fmt, active = [1], [0]
    a = _run_kernels(docs, vocab, ld, fmt, active, seed=rows)
    b = _run_kernels(docs, vocab, ld, fmt, active, seed=rows)
    assert (a == b).all()                                        # two runs agree bit for bit


def test_prefill_slot_indirection():
    import torch
    rows = 3
    fmt = torch.ones(rows, dtype=torch.int32, device="cuda")
    tok = torch.tensor([3 + ord("{"), 3 + ord(" "), 3 + ord("x")], dtype=torch.int32, device="cuda")
    slot = torch.tensor([5, 0, 2], dtype=torch.int32, device="cuda")
    out = torch.full((8, 16), 0xAB, dtype=torch.uint8, device="cuda")
    done = torch.zeros(rows, dtype=torch.int32, device="cuda")
    assert _lib().rr_op_json_advance(rows, _ptr(fmt), None, _ptr(tok), None, _ptr(out), _ptr(slot), _ptr(done), None) == 0
    o = out.cpu().numpy()
    untouched = [1, 3, 4, 6, 7]
    assert (o[untouched] == 0xAB).all()
    assert (o[2] == 0).all()                                      # 'x' is not allowed: the initial state is written
    assert not (o[0] == 0).all() and not (o[5] == 0).all()        # a whitespace run of 1; the open object
    assert done.tolist() == [0, 0, 0]
    assert _lib().rr_op_json_mask(None, 8, 1, 8, None, None, None, None) == 4
    x = torch.zeros((1, 8), device="cuda")
    assert _lib().rr_op_json_mask(_ptr(x), 6, 1, 8, _ptr(fmt), None, None, None) == 4      # ld % 4, vocab > ld


# ---------------------------------------------------------------- 2. tail kernels on masked rows
def _masked_logits(states, vocab, seed):
    rng = np.random.RandomState(seed)
    x = rng.standard_normal((len(states), vocab)).astype(np.float32) * 3
    for r, s in enumerate(states):
        x[r, _masked_cols(s, vocab)] = -np.inf
    return x


# states: after '{' (6 bytes), inside a string (most bytes), after 't' (only 'r': whole chunks masked), after '-'
_STATES = [b"{", b'{"', b'{"a":t', b'{"a":-', b"", b'{"a":"\xf0']


def _states():
    return [J.accepts(p)[0] for p in _STATES]


@pytest.mark.parametrize("vocab", [1024, 8192 + 100, 32064])
def test_logprobs_on_masked_rows(vocab):
    import torch
    st = _states()
    x = _masked_logits(st, vocab, vocab)
    rows = len(st)
    tops = torch.full((rows,), 20, dtype=torch.int32, device="cuda")
    lp = torch.full((rows, 20), float("nan"), device="cuda")
    ids = torch.full((rows, 20), -7, dtype=torch.int32, device="cuda")
    xd = torch.from_numpy(x).cuda()
    assert _lib().rr_op_logprobs(_ptr(xd), vocab, rows, vocab, _ptr(tops), 20, _ptr(lp), _ptr(ids), None) == 0
    lp, ids = lp.cpu().numpy(), ids.cpu().numpy()
    for r in range(rows):
        ok = np.isfinite(x[r])
        x64 = x[r][ok].astype(np.float64)
        lse = x64.max() + np.log(np.exp(x64 - x64.max()).sum())
        n = int(ok.sum())
        for j in range(20):
            if j < n:
                i = ids[r, j]
                assert ok[i] and abs(lp[r, j] - (x[r, i] - lse)) <= 1e-4 + 1e-5 * abs(lp[r, j]), (r, j)
            else:
                assert np.isneginf(lp[r, j]) and not ok[ids[r, j]]
        order = np.argsort(-x[r][ok], kind="stable")
        assert ids[r, : min(n, 20)].tolist() == np.flatnonzero(ok)[order][: min(n, 20)].tolist()
    # after 't' only 'r' is allowed: with vocab % 8192 in 1..255 the last chunk is all -inf and the lse stays finite
    assert np.isfinite(lp[2, 0])


@pytest.mark.parametrize("top_p", [1.0, 0.9])
def test_sampler_never_draws_a_masked_token(top_p):
    import torch
    vocab = 32064
    st = _states() * 6
    x = _masked_logits(st, vocab, 7)
    rows = len(st)
    T = np.full(rows, 1.3, dtype=np.float32)
    seeds = np.arange(rows, dtype=np.uint64) * 977 + 5
    pos = np.arange(rows, dtype=np.int32) + 40
    out = torch.full((rows,), -7, dtype=torch.int32, device="cuda")
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a.astype(dt))).cuda()
    assert _lib().rr_op_sample(_ptr(dev(x, np.float32)), vocab, rows, vocab, _ptr(dev(T, np.float32)),
                               _ptr(dev(np.full(rows, top_p), np.float32)), _ptr(dev(seeds.view(np.int64), np.int64)),
                               _ptr(dev(pos, np.int32)), _ptr(out), None) == 0
    got = out.cpu().numpy()
    for r in range(rows):
        assert np.isfinite(x[r, got[r]]), r
        d = S.sample(x[r], float(T[r]), top_p, int(seeds[r]), int(pos[r]), mass_slack=1e-6)
        if d.stable_nucleus and d.score_gap > d.score_bound:
            assert got[r] == d.token, r


# ---------------------------------------------------------------- 3. engine tokens against the oracle
def _engine(spec="tiny", B=8, ctx_max=512, **kw):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    sp = SPECS[spec] if isinstance(spec, str) else spec
    w = make_weights(sp, seed=5, sigma=0.05, device="cuda")
    return Engine(w, max_batch=B, ctx_max=ctx_max, max_prefill_tokens=4096, **kw)


def _prompt(n, seed=0):
    return np.random.RandomState(seed + n).randint(3, 1000, size=n).tolist()


@pytest.mark.parametrize("spec,B,N", [("tiny", 64, 24), ("llama-3-8b-2l", 64, 8)])
def test_engine_tokens_are_the_oracle_on_masked_teacher_forced_logits(spec, B, N):
    eng = _engine(spec, B, use_cuda_graph=True)
    try:
        prompts = [_prompt(10 + i) for i in range(B)]
        temps = [0.0 if i % 2 == 0 else 1.1 for i in range(B)]
        seeds = [300 + 7 * i for i in range(B)]
        tops = [3 if i % 4 == 1 else None for i in range(B)]
        ts = [eng.submit(p, N, temperature=t, top_p=1.0 if i % 3 else 0.9, seed=s, top_logprobs=k, response_format=JS)
              for i, (p, t, s, k) in enumerate(zip(prompts, temps, seeds, tops))]
        recs = [eng.wait(t) for t in ts]
        for rec in recs:
            s = _valid_prefix(rec.tokens)
            assert rec.finish_reasons == (["stop"] if J.done(s) else ["length"])
            assert J.done(s) or len(rec.tokens) == N
            if J.done(s):
                _loads(_text(rec.tokens))
        # teacher forcing: each row's logits of its own prefix, masked by the oracle, pick the same token
        slots = list(range(B))
        _, lg = eng.prefill(prompts, slots, want_logits=True)
        states = [J.initial() for _ in range(B)]
        for j in range(N):
            if j:
                live = [i for i in range(B) if len(recs[i].tokens) > j]
                if not live:
                    break
                _, lg = eng.decode_step(slots, [recs[i].tokens[j - 1] if len(recs[i].tokens) >= j else 3 for i in slots],
                                        [len(prompts[i]) + j - 1 for i in slots], want_logits=True)
            for i in range(B):
                if len(recs[i].tokens) <= j:
                    continue
                x = lg[i].copy()
                x[_masked_cols(states[i], len(x))] = -np.inf
                tok = recs[i].tokens[j]
                if temps[i] == 0:
                    assert tok == int(np.argmax(x)), (i, j)
                else:
                    d = S.sample(x, temps[i], 1.0 if i % 3 else 0.9, seeds[i], len(prompts[i]) + j, mass_slack=1e-6)
                    if d.stable_nucleus and d.score_gap > d.score_bound:
                        assert tok == d.token, (i, j)
                    assert np.isfinite(x[tok])
                if tops[i] is not None:
                    pairs = recs[i].logprobs[j]
                    for t, v in pairs[:3]:
                        assert (v == -np.inf) == (not np.isfinite(x[t]))
                states[i] = J.advance(states[i], (tok - 3) % 256)
    finally:
        eng.close()


def test_logit_bias_steers_and_cannot_override_the_grammar():
    eng = _engine()
    try:
        p = _prompt(20)
        b = lambda ch: 3 + ord(ch)
        rec = eng.wait(eng.submit(p, 32, logit_bias={b("{"): 100, b("}"): 100}, response_format=JS))
        assert _text(rec.tokens) == b"{}" and rec.finish_reasons == ["stop"]
        bias = {b('"'): 100, b(":"): 95, b("{"): 90, b("}"): 80}
        rec = eng.wait(eng.submit(p, 32, logit_bias=bias, response_format=JS))
        assert _text(rec.tokens) == b'{"":""}' and rec.finish_reasons == ["stop"] and _loads(_text(rec.tokens)) == {"": ""}
        # +100 on tokens no state ever allows (0..2, the bytes C0, C1, F5..FF) changes nothing
        never = {t: 100.0 for t in [0, 1, 2] + [3 + c for c in (0xC0, 0xC1, 0xF5, 0xFF)]}
        for kw in ({}, dict(temperature=1.0, seed=4)):
            a = eng.wait(eng.submit(p, 24, response_format=JS, **kw))
            c = eng.wait(eng.submit(p, 24, response_format=JS, logit_bias=never, **kw))
            assert a.tokens == c.tokens
    finally:
        eng.close()


# ---------------------------------------------------------------- 4. neighbours, reuse, choices, combinations
def test_plain_neighbours_are_untouched_and_slots_are_reused_cleanly():
    B, N = 64, 16
    eng, fresh = _engine(B=B, use_cuda_graph=True), _engine(B=B, use_cuda_graph=True)
    try:
        prompts = [_prompt(20 + i) for i in range(B)]
        plain = [eng.wait(t).tokens for t in [eng.submit(p, N) for p in prompts]]
        mixed = [eng.submit(p, N, response_format=JS if i % 2 else None) for i, p in enumerate(prompts)]
        recs = [eng.wait(t) for t in mixed]
        for i in range(0, B, 2):
            assert recs[i].tokens == plain[i], i
        for i in range(1, B, 2):
            _valid_prefix(recs[i].tokens)
        # JSON requests in the slots JSON requests just left equal a fresh engine's
        again = [eng.wait(t).tokens for t in [eng.submit(_prompt(33 + i, 1), N, response_format=JS) for i in range(B)]]
        want = [fresh.wait(t).tokens for t in [fresh.submit(_prompt(33 + i, 1), N, response_format=JS) for i in range(B)]]
        assert again == want
    finally:
        eng.close(); fresh.close()


def test_a_closed_object_gives_its_row_back_at_once():
    eng = _engine(B=2)
    try:
        p1, p2, p3, N = _prompt(30), _prompt(31), _prompt(32), 40
        bias = {3 + ord("{"): 100, 3 + ord("}"): 100}
        eng.reset_stats()
        t1 = eng.submit(p1, N, logit_bias=bias, response_format=JS)
        t2, t3 = eng.submit(p2, N), eng.submit(p3, N)
        r1, r2, r3 = eng.wait(t1), eng.wait(t2), eng.wait(t3)
        assert _text(r1.tokens) == b"{}" and r1.finish_reasons == ["stop"] and len(r2.tokens) == len(r3.tokens) == N
        assert r1.t_done < r3.t_first_token < r2.t_done
        assert eng.stats()["decode_steps"] == 1 + (N - 1)
    finally:
        eng.close()


def test_choices_end_on_their_own_and_equal_single_requests():
    eng = _engine(B=4)
    try:
        p, N, n = _prompt(50), 40, 3
        kw = dict(temperature=1.0, top_p=0.95, top_logprobs=2, response_format=JS,
                  logit_bias={3 + ord("}"): 4.5, 3 + ord('"'): 4.0, 3 + ord("{"): 8.0})
        singles = [eng.wait(eng.submit(p, N, seed=70 + i, **kw)) for i in range(n)]
        rec = eng.wait(eng.submit(p, N, seed=70, n=n, **kw))
        for i in range(n):
            assert rec.choices[i] == singles[i].tokens and rec.choice_logprobs[i] == singles[i].logprobs
            assert rec.finish_reasons[i] == singles[i].finish_reasons[0]
            _valid_prefix(rec.choices[i])
        assert "stop" in rec.finish_reasons
    finally:
        eng.close()


def test_combinations_with_stop_penalties_logprobs_and_the_prefix_cache():
    eng = _engine(B=8, prefix_cache=True)
    try:
        p, N = _prompt(150), 30
        full = dict(temperature=0.8, top_p=0.9, seed=3, top_logprobs=4, frequency_penalty=0.4, presence_penalty=0.2,
                    logit_bias={3 + ord("}"): 3.0, 3 + ord("a"): 2.0})
        ref = eng.wait(eng.submit(p, N, response_format=JS, **full))
        s = _valid_prefix(ref.tokens)
        # a prefix-cache hit gives the same reply
        hit = eng.wait(eng.submit(p, N, response_format=JS, **full))
        assert hit.tokens == ref.tokens and hit.logprobs == ref.logprobs and hit.n_cached > 0
        # stop cuts the JSON reply where the stop oracle says; a cut on the token that closes the object wins
        from stop_oracle import stop_cut
        text = _text(ref.tokens)
        stop = [text[len(text) // 2: len(text) // 2 + 2]] if len(text) > 4 else [text[-1:]]
        rec = eng.wait(eng.submit(p, N, response_format=JS, stop=stop, **full))
        keep, stopped = stop_cut(ref.tokens, stop)
        assert stopped and rec.tokens == ref.tokens[:keep] and rec.finish_reasons == ["stop"]
        if J.done(s):
            rec = eng.wait(eng.submit(p, N, response_format=JS, stop=[text[-1:]], **full))
            keep, _ = stop_cut(ref.tokens, [text[-1:]])
            assert rec.tokens == ref.tokens[:keep] and len(rec.tokens) < len(ref.tokens)
    finally:
        eng.close()


# ---------------------------------------------------------------- 5. exact counts
def test_counts_of_a_step_with_json_rows():
    """A JSON request adds two launches to its prefill chunk and to each decode step, 4 bytes per row read back with the
    tokens, and the uploads of its parameter block: 4 bytes for the chunk's row and 4 x max_batch for the decode rows
    when it joins.  A plain run afterwards costs exactly what it did before."""
    B, N = 16, 40
    eng = _engine(B=B)
    keys = ("kernel_launches", "decode_steps", "prefill_chunks", "d2h_bytes", "h2d_bytes")
    prompt = list(range(5, 40))
    # a string that never ends: no token of the reply closes the object before N
    bias = {3 + ord("{"): 50, 3 + ord('"'): 50, 3 + ord("a"): 100}     # '{' also lies inside strings: below 'a'
    try:
        def run(**kw):
            eng.reset_stats()
            rec = eng.wait(eng.submit(prompt, N, logit_bias=bias, **kw))
            st = eng.stats()
            return rec, {k: st[k] for k in keys}
        run()
        plain, s1 = run()
        eng.reset_stats()
        eng.wait(eng.submit(prompt, 1, logit_bias=bias))
        F = eng.stats()["kernel_launches"]
        P = (s1["kernel_launches"] - F) // (N - 1)
        run(response_format=JS)                                          # allocates, captures the graph of mode 20
        rec, s = run(response_format=JS)
        assert _text(rec.tokens) == b'{"' + b"a" * (N - 2) and rec.finish_reasons == ["length"]
        assert s == dict(s1, kernel_launches=F + 2 + (N - 1) * (P + 2), h2d_bytes=s1["h2d_bytes"] + 4 + 4 * B,
                         d2h_bytes=s1["d2h_bytes"] + 4 + (N - 1) * 4 * B)
        _, s = run()
        assert s == s1
    finally:
        eng.close()


# ---------------------------------------------------------------- 6. serving paths
def _serve(r):
    import socket
    import uvicorn
    from rr_b200.server import create_app
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    srv = uvicorn.Server(uvicorn.Config(create_app(r), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=srv.run, daemon=True)
    th.start()
    deadline = time.time() + 30
    while not srv.started and time.time() < deadline:
        time.sleep(0.05)
    return srv, th, port


def test_streaming_router_and_http_with_the_openai_sdk():
    openai = pytest.importorskip("openai")
    import httpx
    from rr_b200 import EngineBackend, Router
    eng = _engine(ctx_max=1024)
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, seed=0)
    bias = {str(3 + ord(c)): v for c, v in (("{", 90), ('"', 100), (":", 95), ("}", 80), ("a", 85))}
    try:
        p = _prompt(30)
        full = r.completion(model="chat", prompt_ids=p, max_tokens=40, response_format=JS, logit_bias=bias)
        assert full.choices[0].finish_reason == "stop"
        _loads(full.choices[0].message.content.encode())
        items = list(r.completion_stream(model="chat", prompt_ids=p, max_tokens=40, response_format=JS, logit_bias=bias))
        assert sum((it[1] for it in items[:-1]), []) == full._token_ids and items[-1].finish_reason == "stop"
        srv, th, port = _serve(r)
        try:
            client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}/v1", max_retries=0)
            msgs = [{"role": "user", "content": "reply in JSON"}]
            kw = dict(model="chat", messages=msgs, max_tokens=40, response_format={"type": "json_object"})
            res = client.chat.completions.create(logit_bias=bias, **kw)
            assert res.choices[0].finish_reason == "stop"
            obj = _loads(res.choices[0].message.content.encode())
            chunks = list(client.chat.completions.create(logit_bias=bias, stream=True, **kw))
            assert "".join(c.choices[0].delta.content or "" for c in chunks) == res.choices[0].message.content
            assert chunks[-1].choices[0].finish_reason == "stop" and isinstance(obj, dict)
            # top_logprobs: a masked alternative has logprob -inf and is left out; the body is strict JSON
            raw = httpx.post(f"http://127.0.0.1:{port}/v1/chat/completions", timeout=60,
                             json=dict(kw, logprobs=True, top_logprobs=20, logit_bias=bias))
            assert raw.status_code == 200
            body = json.loads(raw.text, parse_constant=lambda n: (_ for _ in ()).throw(ValueError(n)))
            content = body["choices"][0]["logprobs"]["content"]
            s = J.initial()
            for c in content:                                             # min(20, allowed ids) entries, all finite
                assert len(c["top_logprobs"]) == min(20, int((~_masked_cols(s, 1024)).sum()))
                assert all(e["logprob"] > -1e30 for e in c["top_logprobs"])
                s = J.advance(s, c["bytes"][0])
            for bad in ({"type": "json_schema", "json_schema": {"name": "x", "schema": {}}}, {"type": "yaml"}):
                with pytest.raises(openai.BadRequestError):
                    client.chat.completions.create(model="chat", messages=msgs, max_tokens=4, response_format=bad)
            plain = client.chat.completions.create(model="chat", messages=msgs, max_tokens=8,
                                                   response_format={"type": "text"})
            ref = client.chat.completions.create(model="chat", messages=msgs, max_tokens=8)
            assert plain.choices[0].message.content == ref.choices[0].message.content
        finally:
            srv.should_exit = True
            th.join(timeout=10)
    finally:
        r.close(); eng.close()


def _router(backends, **kw):
    from rr_b200 import Router
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends=backends, seed=0, clock=lambda: 7000.0, **kw)
    r.record_trace = 4096
    return r


def test_fallback_readmission_gives_the_same_reply_and_the_trace_replays():
    from rr_b200 import EngineBackend
    from test_gateway_gpu import _replay
    bad, good, ref = _engine(fail_prob=0.5, fail_seed=42), _engine(), _engine()
    r = _router({0: EngineBackend(bad), 1: EngineBackend(good)})
    try:
        N, fell = 24, 0
        bias = {3 + ord("}"): 5.0, 3 + ord("{"): 6.0}
        for k in range(12):
            p = _prompt(20 + k)
            want = ref.wait(ref.submit(p, N, temperature=0.9, seed=100 + k, logit_bias=bias, response_format=JS))
            o = r.completion(model="primary", prompt_ids=p, max_tokens=N, temperature=0.9, seed=100 + k,
                             logit_bias={str(t): v for t, v in bias.items()}, response_format=JS, logprobs=True)
            assert o._token_ids == want.tokens and o.choices[0].finish_reason == want.finish_reasons[0]
            json.dumps(o.choices[0].logprobs, allow_nan=False)
            fell += o._fell_back
        assert 0 < fell < 12
        assert _replay(r, r.gateway_trace()) == 12 + fell
    finally:
        r.close(); bad.close(); good.close(); ref.close()


def test_refusals_mock_replicas_and_small_vocabularies_via_gen_params():
    from rr_b200 import BadRequestError, EngineBackend, SPECS, StubBackend, _lib as L
    r = _router({0: StubBackend(), 1: StubBackend()})
    try:
        with pytest.raises(BadRequestError) as ei:
            r.completion(model="primary", prompt_ids=[5, 6, 7], max_tokens=4, response_format=JS)
        assert ei.value.status_code == 400 and "response_format" in ei.value.message
        t, ids = C.c_uint64(), (C.c_int32 * 2)(5, 6)
        p = L.GenParams(n_choices=1, top_logprobs=-1, top_p=1.0, response_format=1)
        assert L.lib.rr_gateway_submit(r._gateway(), 0, ids, 2, 2, C.byref(p), C.byref(t)) == 4
        assert len(r.completion(model="primary", prompt_ids=[5, 6, 7], max_tokens=4,
                                response_format={"type": "text"})._token_ids) == 4
    finally:
        r.close()
    small = _engine(dataclasses.replace(SPECS["tiny"], vocab=256))
    try:
        with pytest.raises(L.RRError) as ei:
            small.submit([5, 6, 7], 4, response_format=JS)
        assert ei.value.rc == 4
        assert len(small.wait(small.submit([5, 6, 7], 4)).tokens) == 4
    finally:
        small.close()
    eng = _engine()
    try:
        with pytest.raises(BadRequestError):
            eng.submit([5, 6], 4, response_format={"type": "json_schema"})
    finally:
        eng.close()
