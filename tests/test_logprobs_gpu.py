"""GPU: per-token logprobs / top_logprobs from the kernel (rr_op_logprobs) through the engine, the native gateway and the
HTTP front.

Error bound of the kernel (logprob = x - lse against fp64 log_softmax of the same fp32 logits), u = 2^-24:
  * s = sum exp(x - m) is built from fp32 additions: 32 sequential terms per thread (8192-column chunk / 256 threads),
    a 10-level shuffle tree over the block, then the chunks in order (n_chunks additions).  A term goes through at most
    D = 32 + 10 + n_chunks roundings of the running sum, each a relative error <= u of a sum of positive terms.
  * expf is within 2 ulp (<= 4u relative) for each term and for each chunk's rescale factor exp(m_c - m); the rescale
    multiply rounds once (u).
  * x - m_c and m_c - m are rounded (relative <= u of their value); a term's exponent error is then <= |x - m| u, so
    summed over terms weighted by their share p = softmax(x) of s it is <= 2 A u with A = sum p |x - m| (fp64).
  => |ds / s| <= (D + 9) u + 2 A u.  lse = m + logf(s): logf is within 1 ulp (<= 2u |log s|), the addition rounds
  (u |lse|), and x - lse rounds once more (u |lp|):
      |lp - lp64| <= 1.05 ((D + 9) u + 2 A u + 2u |log s| + u |lse| + u |lp|)
  (the factor 1.05 covers second-order terms).  This is a few 1e-6 at a 128 k vocabulary.
"""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu]

U = 2.0 ** -24
CHUNK = 8192


def _lib():
    from rr_b200 import _lib
    return _lib.lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _run_op(logits, ld, vocab, top_n, max_top=20):
    rows = top_n.numel()
    lp = torch.full((rows, max_top), float("nan"), device="cuda")
    ids = torch.full((rows, max_top), -7, dtype=torch.int32, device="cuda")
    rc = _lib().rr_op_logprobs(_ptr(logits), ld, rows, vocab, _ptr(top_n), max_top, _ptr(lp), _ptr(ids), None)
    assert rc == 0
    torch.cuda.synchronize()
    return lp.cpu().numpy(), ids.cpu().numpy()


def _reference(x):
    """(ids in the stable (-logit, id) order, fp64 log_softmax, tolerance per element) of one fp32 row."""
    x64 = x.astype(np.float64)
    order = np.lexsort((np.arange(x.size), -x64))
    m = x64.max()
    e = np.exp(x64 - m)
    s = e.sum()
    lse = m + np.log(s)
    A = float((e / s * (m - x64)).sum())
    D = 32 + 10 + (x.size + CHUNK - 1) // CHUNK
    lp = x64 - lse
    tol = 1.05 * ((D + 9) * U + 2 * A * U + 2 * U * abs(np.log(s)) + U * abs(lse) + U * np.abs(lp))
    return order, lp, tol


def _check_rows(x, top_n, lp, ids, max_top=20):
    for r in range(x.shape[0]):
        tn = int(top_n[r])
        if tn < 0:
            assert np.isnan(lp[r]).all() and (ids[r] == -7).all(), r
            continue
        k = min(max(1, tn), max_top)
        order, ref, tol = _reference(x[r])
        assert (ids[r, :k] == order[:k]).all(), (r, ids[r, :k], order[:k])
        err = np.abs(lp[r, :k].astype(np.float64) - ref[order[:k]])
        assert (err <= tol[order[:k]]).all(), (r, err.max(), tol[order[:k]].min())
        assert np.isfinite(lp[r, :k]).all()
        assert np.isnan(lp[r, k:]).all() and (ids[r, k:] == -7).all(), r


@pytest.mark.parametrize("vocab,ld", [(128256, 128256), (32064, 32064), (32000, 32000), (1003, 1004)])
@pytest.mark.parametrize("rows", [1, 37, 128])
def test_kernel_against_fp64(vocab, ld, rows):
    g = torch.Generator().manual_seed(vocab + rows)
    x = torch.randn(rows, ld, generator=g) * 3.0
    # planted ties: several equal maxima; a run of equal values straddling position k = 5 / 20; a row far above the rest
    for r in range(rows):
        kind = r % 4
        if kind == 1:
            x[r, torch.randperm(vocab, generator=g)[:4]] = 60.0
        elif kind == 2:
            top = torch.randperm(vocab, generator=g)[:30]
            x[r, top[:3]] = 45.0
            x[r, top[3:30]] = 40.0                      # positions 3..29 tie: k = 5 and k = 20 cut through them
        elif kind == 3 and r % 8 == 3:
            x[r, int(torch.randint(0, vocab, (1,), generator=g))] = float(x[r, :vocab].max()) + 80.0
    x[:, vocab:] = float("nan")                           # padding columns are never read
    choices = torch.tensor([-1, 0, 1, 5, 20], dtype=torch.int32)
    top_n = choices[torch.randint(0, 5, (rows,), generator=g)]
    if rows == 1:
        top_n[0] = 20
    d_x, d_top = x.cuda(), top_n.cuda()
    lp, ids = _run_op(d_x, ld, vocab, d_top)
    xs = x[:, :vocab].numpy()
    _check_rows(xs, top_n.numpy(), lp, ids)
    # entry 0 is the greedy token
    tok = torch.zeros(rows, dtype=torch.int32, device="cuda")
    assert _lib().rr_op_argmax(_ptr(d_x), ld, rows, vocab, _ptr(tok), None, None, None, None) == 0
    tok = tok.cpu().numpy()
    on = top_n.numpy() >= 0
    assert (ids[on, 0] == tok[on]).all()
    # deterministic: a second call gives the same bits
    lp2, ids2 = _run_op(d_x, ld, vocab, d_top)
    assert np.array_equal(lp.view(np.int32), lp2.view(np.int32)) and np.array_equal(ids, ids2)


def test_kernel_max_top_below_20_and_far_maximum():
    x = torch.full((3, 4096), -5.0)
    x[0, 17] = 75.0                                       # 80 above the rest: logprob 0, the others -80 - log(1 + ...)
    x[1] = torch.linspace(-1, 1, 4096)
    x[2] = 0.0                                            # all equal: ids 0.. in order
    top_n = torch.tensor([20, 3, 7], dtype=torch.int32)
    lp, ids = _run_op(x.cuda(), 4096, 4096, top_n.cuda(), max_top=6)
    assert ids[0, 0] == 17 and list(ids[0, 1:6]) == [0, 1, 2, 3, 4] and np.isfinite(lp[[0, 2]]).all()
    assert list(ids[2]) == [0, 1, 2, 3, 4, 5]
    _check_rows(x.numpy(), top_n.numpy(), lp, ids, max_top=6)


# ------------------------------------------------------------------------------------------------ engine
def _prompts(n, vocab, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(3, vocab, size=int(rng.randint(3, 60))).tolist() for _ in range(n)]


@pytest.mark.parametrize("spec_name,rows", [("tiny", 24), ("llama-3-8b-2l", 64)])
def test_engine_logprobs_match_teacher_forced_logits(spec_name, rows):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS[spec_name]
    w = make_weights(spec, seed=5, sigma=0.05, device="cuda")
    eng = Engine(w, max_batch=rows, ctx_max=256, max_prefill_tokens=4096, use_cuda_graph=True)
    try:
        N = 6
        prompts = _prompts(rows, spec.vocab, rows)
        tops = [[0, 1, 5, 20, 3][(i // 2) % 5] if i % 2 else None for i in range(rows)]
        plain = [eng.wait(t).tokens for t in [eng.submit(p, N) for p in prompts]]
        tk = [eng.submit(p, N, top_logprobs=k) for p, k in zip(prompts, tops)]
        recs = [eng.wait(t) for t in tk]
        assert [r.tokens for r in recs] == plain                       # logprobs never change the tokens
        for r, k in zip(recs, tops):
            assert (r.logprobs is None) == (k is None)
            if k is not None:
                assert len(r.logprobs) == N and all(len(p) == max(1, k) for p in r.logprobs)
        # teacher forcing on the same token path: prefill logits for token 0, decode_step logits for tokens 1..N-1
        slots = list(range(rows))
        first, lg = eng.prefill(prompts, slots, want_logits=True)
        assert first.tolist() == [t[0] for t in plain]
        steps = [lg]
        for j in range(1, N):
            nxt, lg = eng.decode_step(slots, [t[j - 1] for t in plain], [len(p) + j - 1 for p in prompts], want_logits=True)
            assert nxt.tolist() == [t[j] for t in plain]
            steps.append(lg)
        for j in range(N):
            lg = steps[j]
            sel = [i for i in range(rows) if tops[i] is not None]
            top_n = torch.tensor([tops[i] for i in sel], dtype=torch.int32)
            d = torch.from_numpy(lg[sel]).cuda()
            lp, ids = _run_op(d, spec.vocab, spec.vocab, top_n.cuda())
            for a, i in enumerate(sel):
                k = max(1, tops[i])
                got = recs[i].logprobs[j]
                # the serving loop's logits are bit-identical to the teacher-forced ones: the same kernel gives the same bits
                assert [g[0] for g in got] == ids[a, :k].tolist(), (i, j)
                assert np.array_equal(np.array([g[1] for g in got], dtype=np.float32).view(np.int32),
                                      lp[a, :k].view(np.int32)), (i, j)
                assert got[0][0] == plain[i][j]
            _check_rows(lg[sel], top_n.numpy(), lp, ids)
    finally:
        eng.close()


def test_graph_switching_keeps_plain_steps_unchanged():
    """Launch and copy counts of whole runs, read while the engine is idle (a read during a run waits for the worker's GPU
    lock and can land hundreds of steps late, so counts are never sampled mid-run).  A request with logprobs is active
    in exactly max_new - 1 decode steps, and each such step replays the logprobs graph (two more launches, the pairs' D2H);
    every other step must cost exactly what a plain step costs."""
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS["tiny"]
    w = make_weights(spec, seed=3, sigma=0.05, device="cuda")
    B = 16
    eng = Engine(w, max_batch=B, ctx_max=1024, max_prefill_tokens=512, use_cuda_graph=True)
    keys = ("kernel_launches", "decode_steps", "prefill_chunks", "d2h_bytes")
    try:
        long_prompt = list(range(5, 40))

        def run(fn):
            eng.reset_stats()
            out = fn()
            st = eng.stats()
            return out, {k: st[k] for k in keys}

        # plain costs: a prefill chunk (F launches) and a decode step (P launches)
        _, s = run(lambda: eng.wait(eng.submit(long_prompt, 1)))
        F = s["kernel_launches"]
        assert s["decode_steps"] == 0 and s["prefill_chunks"] == 1
        solo, s = run(lambda: eng.wait(eng.submit(long_prompt, 600)).tokens)
        assert s["decode_steps"] == 599
        P = (s["kernel_launches"] - F) // 599
        assert s["kernel_launches"] == F + 599 * P and s["d2h_bytes"] == 4 + 599 * 4 * B

        # a long plain request; short logprobs requests come and go next to it, one at a time
        def mixed():
            t = eng.submit(long_prompt, 600)
            eng.peek(t, 0, timeout=30)                                  # prefilled in a chunk of its own
            recs = []
            for i in range(6):
                x = eng.submit(_prompts(1, spec.vocab, 100 + i)[0], 8, top_logprobs=[0, 3, 20][i % 3])
                recs.append(eng.wait(x))
            return eng.wait(t).tokens, recs
        (toks, recs), s = run(mixed)
        assert toks == solo and all(len(r.logprobs) == 8 for r in recs)
        assert s["prefill_chunks"] == 7
        lp_steps = 6 * 7                                                # each short request: 7 decode steps
        assert s["kernel_launches"] == 7 * F + 6 * 2 + s["decode_steps"] * P + lp_steps * 2
        assert s["d2h_bytes"] == 4 + 6 * (4 + 20 * 8) + s["decode_steps"] * 4 * B + lp_steps * 20 * 8 * B
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ gateway / HTTP
def _server(router):
    import uvicorn
    from rr_b200.server import create_app
    port = 21000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(router), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(200):
        if server.started:
            break
        time.sleep(0.05)
    return server, th, port


def _pairs_of(content):
    return [(c.token, c.logprob, [(t.token, t.logprob) for t in c.top_logprobs]) for c in content]


def test_gateway_and_http_logprobs_with_fallback():
    import openai
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights

    def tiny(**kw):
        w = make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda")
        return Engine(w, max_batch=8, ctx_max=256, max_prefill_tokens=512, **kw)
    bad, good = tiny(fail_prob=0.5, fail_seed=42), tiny()
    ml = [{"model_name": "chat", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny-backup", "gpu": 1}}]
    r = Router(model_list=ml, fallbacks=[{"chat": ["backup"]}], allowed_fails=1000, backends={0: EngineBackend(bad),
               1: EngineBackend(good)}, default_max_tokens=12, seed=0)
    server, th, port = _server(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        fell_back, ref = 0, None
        for i in range(12):
            msgs = [{"role": "user", "content": "score me"}]
            full = client.chat.completions.create(model="chat", messages=msgs, logprobs=True, top_logprobs=3, timeout=60)
            content = full.choices[0].logprobs.content
            assert len(content) == full.usage.completion_tokens == 12
            assert all(c.logprob == c.top_logprobs[0].logprob and len(c.top_logprobs) == 3 for c in content)
            fell_back += full.model == "tiny-backup"
            got = _pairs_of(content)
            assert ref is None or got == ref                  # same weights on both replicas: same tokens and logprobs
            ref = got
            streamed = []
            for ch in client.chat.completions.create(model="chat", messages=msgs, logprobs=True, top_logprobs=3,
                                                     timeout=60, stream=True):
                if ch.choices[0].logprobs is not None:
                    streamed += _pairs_of(ch.choices[0].logprobs.content)
            assert streamed == ref
        assert fell_back > 0                                  # some requests failed over and still carried full lists
        plain = client.chat.completions.create(model="chat", messages=[{"role": "user", "content": "score me"}], timeout=60)
        assert plain.choices[0].logprobs is None
    finally:
        server.should_exit = True
        th.join(10)
        r.close(); bad.close(); good.close()
