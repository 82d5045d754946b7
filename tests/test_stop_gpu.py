"""GPU: stop sequences, from rr_op_stop_match through the engine's early row release, the native gateway and the router
to the OpenAI endpoint.

The contract is exact.  Stop sequences change no logit and no draw, so the reply with `stop` is the reply without it cut
where tests/stop_oracle.py says; the kernel's (cut, hold) equal the oracle's for any history."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from stop_oracle import stop_cut, stop_state

pytestmark = [pytest.mark.gpu]


# ---------------------------------------------------------------- 1. the kernel against the oracle
def _stop_block(stops_per_row):
    rows = len(stops_per_row)
    n = np.array([len(s) for s in stops_per_row], dtype=np.int32)
    ln = np.zeros((rows, 4), dtype=np.uint8)
    by = np.zeros((rows, 4, 64), dtype=np.uint8)
    for r, stops in enumerate(stops_per_row):
        for i, s in enumerate(stops):
            ln[r, i] = len(s)
            by[r, i, : len(s)] = np.frombuffer(s, dtype=np.uint8)
    return n, ln, by


def _match(histories, stops_per_row, active=None, ld=None, gen0=None):
    """rr_op_stop_match over rows whose generated tokens are histories[r] (the last one is the token just picked).
    -> (cut, hold, history buffer before, after), outputs poisoned with -99 and free history cells with -7."""
    import torch
    from rr_b200 import _lib
    rows = len(histories)
    ld = ld or max(len(h) for h in histories) + 3
    hist = np.full((rows, ld), -7, dtype=np.int32)
    for r, h in enumerate(histories):
        hist[r, : len(h) - 1] = h[:-1]
    gen0 = np.arange(rows, dtype=np.int32) * 7 + 5 if gen0 is None else np.asarray(gen0, dtype=np.int32)
    pos = gen0 + np.array([len(h) - 1 for h in histories], dtype=np.int32)
    tok = np.array([h[-1] for h in histories], dtype=np.int32)
    n, ln, by = _stop_block(stops_per_row)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (hist, tok, pos, n, gen0, ln, by)]
    act = None if active is None else torch.tensor(active, dtype=torch.int32).cuda()
    cut, hold = torch.full((rows,), -99, dtype=torch.int32).cuda(), torch.full((rows,), -99, dtype=torch.int32).cuda()
    d_hist, d_tok, d_pos, d_n, d_g0, d_ln, d_by = dev
    rc = _lib.lib.rr_op_stop_match(d_hist.data_ptr(), ld, d_tok.data_ptr(), d_pos.data_ptr(),
                                   act.data_ptr() if act is not None else None, d_n.data_ptr(), d_g0.data_ptr(),
                                   d_ln.data_ptr(), d_by.data_ptr(), cut.data_ptr(), hold.data_ptr(), rows, None)
    assert rc == 0
    torch.cuda.synchronize()
    return cut.cpu().numpy(), hold.cpu().numpy(), hist, d_hist.cpu().numpy()


def _random_case(rng, length, alphabet):
    """A history over a few letters (hits and partial matches are frequent), byteless ids and ids that alias the letters."""
    letters = [3 + b for b in alphabet]
    pool = letters * 3 + [0, 1, 2] + [t + 256 * int(rng.randint(1, 4)) for t in letters]
    h = [int(pool[i]) for i in rng.randint(0, len(pool), size=length)]
    stops = []
    for _ in range(int(rng.randint(0, 5))):
        k = int(rng.choice([1, 2, 3, 5, 17, 63, 64]))
        if rng.rand() < 0.6 and length >= 2:                     # taken from the text itself, so it does occur
            text = bytes((t - 3) % 256 for t in h if t >= 3)
            a = int(rng.randint(0, max(1, len(text))))
            s = text[max(0, a - k): a] or bytes([alphabet[0]])
        else:
            s = bytes(int(alphabet[i]) for i in rng.randint(0, len(alphabet), size=k))
        stops.append(s)
    return h, stops


@pytest.mark.parametrize("rows", [1, 3, 64, 256])
def test_kernel_equals_the_oracle(rows):
    rng = np.random.RandomState(rows)
    lengths = [1, 2, 3, 31, 32, 33, 64, 65, 100, 700, 3000]
    cases = [_random_case(rng, lengths[r % len(lengths)] if r < 2 * len(lengths) else int(rng.randint(1, 200)),
                          b"abc" if r % 2 else b"abcd") for r in range(rows)]
    cases[0] = ([5] + [0] * 100 + [3 + 97], [b"\x02a", b"a" * 64])        # a run of byteless tokens inside a match
    if rows > 2:
        cases[1] = ([3 + 97] * 70, [b"a" * 64, b"a" * 63])               # 64-byte hit
        cases[2] = ([3 + 97] * 5, [b"a" * 64])                           # sequence longer than the history: hold only
    active = [-1 if r % 5 == 4 else r for r in range(rows)]
    hs, ss = [c[0] for c in cases], [c[1] for c in cases]
    cut, hold, before, after = _match(hs, ss, active)
    cut2, hold2, _, after2 = _match(hs, ss, active)
    assert (cut == cut2).all() and (hold == hold2).all() and (after == after2).all()
    hit = part = 0
    for r in range(rows):
        touched = active[r] >= 0 and len(ss[r]) > 0
        want = stop_state(hs[r], ss[r]) if touched else (-99, -99)
        assert (cut[r], hold[r]) == want, (r, hs[r][-80:], ss[r])
        if touched:
            before[r, len(hs[r]) - 1] = hs[r][-1]                    # the new cell is written, and no other
            hit += want[0] >= 0
            part += want[1] > 0
    assert (before == after).all()
    if rows >= 64:
        assert hit >= 4 and part >= 4                                    # the cases do exercise both outcomes


def test_kernel_index_outside_the_history_is_no_hit_and_no_store():
    cut, hold, before, after = _match([[3 + 97, 3 + 98]], [[b"ab"]], ld=4, gen0=[9])
    assert (cut[0], hold[0]) == (0, 0)
    import torch
    from rr_b200 import _lib
    z = torch.zeros(8, dtype=torch.int32).cuda()
    one = torch.ones(8, dtype=torch.int32).cuda()
    by = torch.zeros(256, dtype=torch.uint8).cuda()
    out = torch.full((2,), -99, dtype=torch.int32).cuda()
    pos = torch.tensor([4], dtype=torch.int32).cuda()                    # index 4 of a 4-token history
    assert _lib.lib.rr_op_stop_match(z.data_ptr(), 4, z.data_ptr(), pos.data_ptr(), None, one.data_ptr(), z.data_ptr(),
                                     by.data_ptr(), by.data_ptr(), out.data_ptr(), out[1:].data_ptr(), 1, None) == 0
    torch.cuda.synchronize()
    assert out.tolist() == [-1, 0] and z.tolist() == [0] * 8


# ---------------------------------------------------------------- engines
def _engine(spec="tiny", B=8, ctx_max=512, **kw):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    w = make_weights(SPECS[spec], seed=5, sigma=0.05, device="cuda")
    return Engine(w, max_batch=B, ctx_max=ctx_max, max_prefill_tokens=1024, **kw)


def _prompt(n, seed=0):
    return np.random.RandomState(seed + n).randint(3, 1000, size=n).tolist()


def _text(tokens):
    return bytes((t - 3) % 256 for t in tokens if t >= 3)


def _stops_from(reply):
    """Stop sets taken from the reply's own bytes: at the first token, the second, mid-reply, the last, never."""
    n = len(reply)
    one = lambda i: _text(reply[i: i + 1])
    sets = [[one(0)], [one(1)], [_text(reply[n // 2: n // 2 + 3])], [one(n - 1)], [b"\x00\x01\x02\x03never"],
            [_text(reply[n // 2 + 1: n // 2 + 3]), _text(reply[n // 2: n // 2 + 3]), b"\xff" * 64, one(n - 2)]]
    return [[s for s in st if s] for st in sets]


SAMPLED = dict(temperature=0.9, top_p=0.95, seed=11)


@pytest.mark.parametrize("spec,B", [("tiny", 8), ("llama-3-8b-2l", 64)])
@pytest.mark.parametrize("kw", [{}, SAMPLED], ids=["greedy", "sampled"])
def test_reply_with_stop_is_the_oracle_cut_of_the_reply_without(spec, B, kw):
    eng = _engine(spec, B)
    try:
        p, N = _prompt(40), 24
        ref = eng.wait(eng.submit(p, N, top_logprobs=3, **kw))
        assert len(ref.tokens) == N and ref.finish_reasons == ["length"]
        stop_sets = _stops_from(ref.tokens)
        ts = [eng.submit(p, N, top_logprobs=3, stop=st, **kw) for st in stop_sets]       # side by side in one batch
        reasons = []
        for st, t in zip(stop_sets, ts):
            rec = eng.wait(t)
            keep, stopped = stop_cut(ref.tokens, st)
            assert rec.status == 0 and rec.tokens == ref.tokens[:keep], (st, keep)
            assert rec.finish_reasons == ["stop" if stopped else "length"]
            assert rec.logprobs == ref.logprobs[:keep]                                   # bit for bit
            reasons.append((keep, stopped))
        assert reasons[0] == (0, True) and reasons[4] == (N, False) and reasons[3][1]
    finally:
        eng.close()


def test_neighbours_of_stopping_requests_are_untouched():
    B, N = 64, 16
    eng, fresh = _engine(B=B), _engine(B=B)
    try:
        prompts = [_prompt(20 + i) for i in range(B)]
        plain = [eng.wait(t).tokens for t in [eng.submit(p, N) for p in prompts]]
        stops = [[_text(plain[i][5 + i % 7: 7 + i % 7])] if i % 2 else None for i in range(B)]
        recs = [eng.wait(t) for t in [eng.submit(p, N, stop=s) for p, s in zip(prompts, stops)]]
        for i, rec in enumerate(recs):
            keep, stopped = stop_cut(plain[i], stops[i] or [])
            assert rec.tokens == plain[i][:keep] and (stopped or not i % 2), i
        assert sum(r.finish_reasons == ["stop"] for r in recs) >= B // 2 - 2
        # rows that stopped requests just left serve the next requests as a fresh engine does
        again = [eng.wait(t).tokens for t in [eng.submit(_prompt(33 + i, 1), N) for i in range(B)]]
        want = [fresh.wait(t).tokens for t in [fresh.submit(_prompt(33 + i, 1), N) for i in range(B)]]
        assert again == want
    finally:
        eng.close(); fresh.close()


def test_a_stopped_choice_gives_its_row_back_at_once():
    eng = _engine(B=2)
    try:
        p1, p2, p3, N = _prompt(30), _prompt(31), _prompt(32), 40
        ref = eng.wait(eng.submit(p1, N)).tokens
        stop = [_text(ref[4:6])]
        keep, stopped = stop_cut(ref, stop)
        assert stopped and keep <= 4
        eng.reset_stats()
        t1, t2, t3 = eng.submit(p1, N, stop=stop), eng.submit(p2, N), eng.submit(p3, N)
        r1, r2, r3 = eng.wait(t1), eng.wait(t2), eng.wait(t3)
        st = eng.stats()
        assert r1.tokens == ref[:keep] and r1.finish_reasons == ["stop"] and len(r2.tokens) == len(r3.tokens) == N
        assert r1.t_done < r3.t_first_token < r2.t_done                  # the third runs in the row the first gave back
        # 1 and 2 decode together until 1 stops at token keep + len(stop) (steps: one less, the first token is prefill's);
        # 3 is prefilled at once and needs N - 1 steps: the schedule, not max_tokens, decides the step count
        n1 = next(i for i in range(1, N + 1) if stop_cut(ref[:i], stop)[1])
        assert st["decode_steps"] == (n1 - 1) + (N - 1) and st["generated_tokens"] == n1 + 2 * N
    finally:
        eng.close()


def _produced(tokens, stop):
    """Tokens the engine generates for a reply that would be `tokens`: up to the one that completes a stop sequence."""
    return next((i for i in range(1, len(tokens) + 1) if stop_cut(tokens[:i], stop)[1]), len(tokens))


def test_choices_end_on_their_own():
    eng = _engine(B=3)
    try:
        p, N, n = _prompt(50), 30, 3
        kw = dict(temperature=1.0, top_p=0.9, top_logprobs=2)
        free = [eng.wait(eng.submit(p, N, seed=70 + i, **kw)) for i in range(n)]
        stop = [_text(free[0].tokens[3:5]), _text(free[1].tokens[14:16])]
        singles = [eng.wait(eng.submit(p, N, seed=70 + i, stop=stop, **kw)) for i in range(n)]
        cuts = [stop_cut(f.tokens, stop) for f in free]
        assert cuts[0][1] and cuts[1][1] and len({c for c, _ in cuts}) >= 2
        eng.reset_stats()
        t = eng.submit(p, N, seed=70, n=n, stop=stop, **kw)
        late = eng.submit(_prompt(20), 4)                                 # needs a row: gets one a choice gave back
        rec, rl = eng.wait(t), eng.wait(late)
        for i in range(n):
            assert rec.choices[i] == singles[i].tokens == free[i].tokens[:cuts[i][0]], i
            assert rec.choice_logprobs[i] == singles[i].logprobs
            assert rec.finish_reasons[i] == singles[i].finish_reasons[0] == ("stop" if cuts[i][1] else "length")
        assert len({len(c) for c in rec.choices}) >= 2
        assert rl.status == 0 and len(rl.tokens) == 4
        made = [_produced(f.tokens, stop) for f in free]
        assert eng.stats()["generated_tokens"] == sum(made) + 4
        assert max(made) - min(made) > 8 and rl.t_done < rec.t_done       # served in a freed row while the longest ran
        c = eng.wait(eng.submit(p, N, seed=70, n=n, stop=stop, **kw))
        assert c.choices == rec.choices
    finally:
        eng.close()


def test_counts_of_a_step_with_stop_rows():
    """Whole runs, read while idle.  A request with stop sequences adds one launch to its prefill chunk and to each decode
    step, 8 bytes per row read back with the tokens, and the uploads of its parameter block: 268 bytes for the chunk's
    one row and 268 x max_batch for the decode rows when it joins.  Plain runs cost exactly what they cost before."""
    B, N = 16, 40
    eng = _engine(B=B)
    keys = ("kernel_launches", "decode_steps", "prefill_chunks", "d2h_bytes", "h2d_bytes")
    prompt = list(range(5, 40))
    never = [b"\x00\x01never", b"\xfe" * 64]
    try:
        def run(**kw):
            eng.reset_stats()
            rec = eng.wait(eng.submit(prompt, N, **kw))
            st = eng.stats()
            return rec, {k: st[k] for k in keys}
        run()
        plain, s1 = run()
        eng.reset_stats()
        eng.wait(eng.submit(prompt, 1))
        F = eng.stats()["kernel_launches"]
        P = (s1["kernel_launches"] - F) // (N - 1)
        run(stop=never)                                                  # captures the graph of mode 8
        rec, s = run(stop=never)
        assert rec.tokens == plain.tokens
        assert s == dict(s1, kernel_launches=F + 1 + (N - 1) * (P + 1), h2d_bytes=s1["h2d_bytes"] + 268 + 268 * B,
                         d2h_bytes=s1["d2h_bytes"] + 8 + (N - 1) * 8 * B)
        _, s = run()
        assert s == s1                                                   # plain again: today's totals
        # every tail kernel at once (mode 15): still the oracle cut of the same request without stop
        full = dict(temperature=0.8, top_p=0.9, seed=3, top_logprobs=4, frequency_penalty=0.4, presence_penalty=0.2,
                    logit_bias={7: 4.0, 11: -3.0})
        ref = eng.wait(eng.submit(prompt, N, **full))
        stop = [_text(ref.tokens[20:23]), b"\xfd" * 9]
        keep, stopped = stop_cut(ref.tokens, stop)
        rec = eng.wait(eng.submit(prompt, N, stop=stop, **full))
        assert stopped and rec.tokens == ref.tokens[:keep] and rec.logprobs == ref.logprobs[:keep]
        # the raw arguments are checked before anything is queued
        from rr_b200 import _lib
        for bad in ([b""], [b"a"] * 5, [b"x" * 65]):
            with pytest.raises(_lib.RRError) as ei:
                eng.submit(prompt, 4, stop=bad)
            assert ei.value.rc == 4
    finally:
        eng.close()


def test_peek_never_shows_a_token_it_would_take_back():
    eng = _engine(B=2, ctx_max=2048)
    try:
        p, N = _prompt(25), 60
        ref = eng.wait(eng.submit(p, N)).tokens
        for stop in ([_text(ref[30:34])], [_text(ref[N - 2:]) + b"\x00zz"]):       # a hit; a partial match pending at the end
            keep, stopped = stop_cut(ref, stop)
            t = eng.submit(p, N, stop=stop)
            seen, done = [], False
            while not done:
                toks, done, _ = eng.peek(t, len(seen), timeout=1.0)
                assert toks[: len(seen)] == seen and toks == ref[: len(toks)]
                if not done:
                    assert len(toks) <= keep
                seen = toks
            rec = eng.wait(t)
            assert seen == rec.tokens == ref[:keep] and rec.finish_reasons == ["stop" if stopped else "length"]
    finally:
        eng.close()


# ---------------------------------------------------------------- router, gateway, HTTP
def _ascii_stop(reply, lo):
    """A one-character stop string that occurs in the reply at or after token lo (and maybe before)."""
    i = next(i for i in range(lo, len(reply)) if reply[i] >= 3 and (reply[i] - 3) % 256 < 128)
    return chr((reply[i] - 3) % 256)


def test_streaming_shows_only_what_stays():
    from rr_b200 import EngineBackend, Router, detokenize
    eng = _engine(ctx_max=1024)
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, seed=0)
    try:
        p, N = _prompt(30), 80
        ref = r.completion(model="chat", prompt_ids=p, max_tokens=N)._token_ids
        s = _ascii_stop(ref, 40)
        for stop, want_reason in ((s, "stop"), (["\x01never", s + "\x02\x03"], "length")):
            keep, stopped = stop_cut(ref, [x.encode() for x in ([stop] if isinstance(stop, str) else stop)])
            full = r.completion(model="chat", prompt_ids=p, max_tokens=N, stop=stop)
            assert full._token_ids == ref[:keep] and full.choices[0].finish_reason == want_reason
            assert full.usage.completion_tokens == keep
            items = list(r.completion_stream(model="chat", prompt_ids=p, max_tokens=N, stop=stop))
            got = []
            for it in items[:-1]:
                got += it[1]
                assert got == ref[: len(got)] and len(got) <= keep       # nothing shown is ever taken back
            assert got == full._token_ids and items[-1][2] and items[-1].finish_reason == want_reason
            if want_reason == "stop":
                assert s not in detokenize(got)
    finally:
        r.close(); eng.close()


def test_stop_over_http_with_the_openai_sdk():
    openai = pytest.importorskip("openai")
    import uvicorn
    from rr_b200 import EngineBackend, Router
    from rr_b200.server import create_app
    eng = _engine(ctx_max=1024)
    r = Router(model_list=[{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}}],
               backends={0: EngineBackend(eng)}, seed=0)
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    srv = uvicorn.Server(uvicorn.Config(create_app(r), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=srv.run, daemon=True)
    th.start()
    try:
        deadline = time.time() + 30
        while not srv.started and time.time() < deadline:
            time.sleep(0.05)
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}/v1", max_retries=0)
        msgs = [{"role": "user", "content": "tell me about stop sequences"}]
        # a bias that keeps the reply printable ASCII, so its text does not depend on where the chunks split it
        kw = dict(model="chat", messages=msgs, max_tokens=60, logit_bias={str(3 + b): 100 for b in range(32, 127)},
                  frequency_penalty=1.5)
        free = client.chat.completions.create(**kw)
        text = free.choices[0].message.content
        assert free.choices[0].finish_reason == "length" and len(text) == 60
        s = text[30:32]
        keep = text.index(s)
        res = client.chat.completions.create(stop=s, **kw)
        assert res.choices[0].finish_reason == "stop" and res.usage.completion_tokens == keep
        assert res.choices[0].message.content == text[:keep]
        chunks = list(client.chat.completions.create(stop=["\x01never", s], stream=True, **kw))
        shown = ""
        for c in chunks:
            shown += c.choices[0].delta.content or ""
            assert text[:keep].startswith(shown)
        assert shown == text[:keep] and chunks[-1].choices[0].finish_reason == "stop"
        pending = text[58:] + "\x01"                                       # a partial match is pending when the reply ends
        chunks = list(client.chat.completions.create(stop=pending, stream=True, **kw))
        assert "".join(c.choices[0].delta.content or "" for c in chunks) == text
        assert chunks[-1].choices[0].finish_reason == "length" and chunks[-1].choices[0].delta.content is None
        with pytest.raises(openai.BadRequestError):
            client.chat.completions.create(stop=["a"] * 5, **kw)
    finally:
        srv.should_exit = True
        th.join(timeout=10)
        r.close(); eng.close()


def _router(backends, **kw):
    from rr_b200 import Router
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends=backends, seed=0, clock=lambda: 7000.0, **kw)
    r.record_trace = 4096
    return r


def test_fallback_readmission_gives_the_same_cut_reply_and_the_trace_replays():
    from rr_b200 import EngineBackend
    from test_gateway_gpu import _replay
    bad, good, ref = _engine(fail_prob=0.5, fail_seed=42), _engine(), _engine()
    r = _router({0: EngineBackend(bad), 1: EngineBackend(good)})
    try:
        N, fell, kept = 24, 0, []
        for k in range(12):
            p = _prompt(20 + k)
            free = ref.wait(ref.submit(p, N, temperature=0.9, seed=100 + k)).tokens
            s = _ascii_stop(free, 6)
            keep, stopped = stop_cut(free, [s.encode()])
            o = r.completion(model="primary", prompt_ids=p, max_tokens=N, temperature=0.9, seed=100 + k, stop=s,
                             logprobs=True)
            assert stopped and o._token_ids == free[:keep] and o.choices[0].finish_reason == "stop"
            assert o.usage.completion_tokens == keep == len(o.choices[0].logprobs["content"])
            fell += o._fell_back
            kept.append(keep)
        assert 0 < fell < 12
        trace = r.gateway_trace()
        admits = [e for e, _ in trace if e[0] == 0]
        dones = [e for e, _ in trace if e[0] == 1]
        fails = [e for e, _ in trace if e[0] == 2]
        assert len(admits) == 12 + fell and len(fails) == fell
        assert [e[2] for e in dones] == kept                             # one DONE each, with the tokens returned
        assert _replay(r, trace) == 12 + fell
    finally:
        r.close(); bad.close(); good.close(); ref.close()


def test_mock_replicas_refuse_a_stop_struct_and_the_prefix_cache_does_not_change_the_cut():
    from rr_b200 import BadRequestError, EngineBackend, StubBackend, _lib
    r = _router({0: StubBackend(), 1: StubBackend()})
    try:
        with pytest.raises(BadRequestError) as ei:
            r.completion(model="primary", prompt_ids=[5, 6, 7], max_tokens=4, stop="a")
        assert ei.value.status_code == 400 and "`stop`" in ei.value.message
        t, ids, off = C.c_uint64(), (C.c_int32 * 2)(5, 6), (C.c_int32 * 2)(0, 1)
        by = (C.c_uint8 * 1)(97)
        p = _lib.GenParams(n_choices=1, top_logprobs=-1, top_p=1.0, n_stop=1, stop_bytes=by, stop_off=off)
        assert _lib.lib.rr_gateway_submit(r._gateway(), 0, ids, 2, 2, C.byref(p), C.byref(t)) == 4
        assert len(r.completion(model="primary", prompt_ids=[5, 6, 7], max_tokens=4)._token_ids) == 4
    finally:
        r.close()
    on = _engine(prefix_cache=True)
    r = _router({0: EngineBackend(on), 1: EngineBackend(on)})
    try:
        p, N = _prompt(200), 30
        free = r.completion(model="primary", prompt_ids=p, max_tokens=N)._token_ids
        s = _ascii_stop(free, 10)
        keep, _ = stop_cut(free, [s.encode()])
        outs = [r.completion(model="primary", prompt_ids=p, max_tokens=N, stop=s, n=n) for n in (1, 2)]
        for o in outs:
            assert all(t == free[:keep] for t in o._choice_token_ids) and o.usage.prompt_tokens_details is None
            assert all(c.finish_reason == "stop" for c in o.choices)
        assert outs[1].usage.completion_tokens == 2 * keep
        assert on.stats()["prefix_hits"] >= 2                            # cold once, then hits: the same cut reply
    finally:
        r.close(); on.close()
