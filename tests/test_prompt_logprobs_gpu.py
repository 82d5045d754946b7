"""GPU: prompt logprobs (`echo` + `logprobs` on /v1/completions) from the prefill GEMM's fp32 epilogue
(rr_op_prefill_gemm mode RR_OUT_ROWMAJOR_F32) through the engine's scoring chunks, the native gateway and the HTTP front.

Bound of the kernel test.  out[t][n] = fl(fl(sum_k a_tk w_nk) * r_t), r_t = rsqrtf(fl(sum_p ss_tp) / hidden + eps), with
bf16 operands (exact products in fp32) and an fp32 accumulation of K products in whatever order the tensor cores take.
Any order of K - 1 fp32 additions errs by at most gamma_{K-1} sum_k |a_tk w_nk| <= 1.01 (K - 1) u S (u = 2^-24); the
tensor cores' adder aligns the addends of one k-group of 16 to the largest and truncates, which at worst doubles the
per-addition error, so the sum is within 2.02 K u S.  r_t carries rsqrtf's 2 ulp and the fp32 sum of n_part partials
(n_part u), relative; the final product rounds once (u).  So |out - ref| <= 2.02 K u S r + (n_part + 4) u |ref|, with ref
the fp64 product of the same bf16 values and the fp64 factor of the same fp32 partial sums.

Tolerance of the engine against the reference model.  The engine keeps activations in bf16 between its GEMMs while
oracle/llama_ref runs fp32 throughout; smoke() holds its logits within 0.02 std(logits) in rms.  A logprob is a logit
minus logsumexp, and logsumexp moves by at most the largest logit error, so |dlp| <= 2 max |dlogit|.  Taking the largest
error at 6x the rms gives TOL = 0.25 std(reference logits of the row); top-1 ids must agree where the reference's margin
between its two best tokens exceeds 2 TOL."""
import ctypes as C
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu]

U = 2.0 ** -24


def _lib():
    from rr_b200 import _lib
    return _lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ---------------------------------------------------------------- kernel
@pytest.mark.parametrize("vocab, K, plan_rows, T", [(128256, 4096, 384, 300), (32000, 512, 256, 129),
                                                     (32064, 1024, 128, 77), (32000, 256, 64, 64)])
def test_fp32_epilogue_against_fp64(vocab, K, plan_rows, T):
    g = torch.Generator(device="cuda").manual_seed(vocab + T)
    A = (torch.randn(plan_rows, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    W = (torch.randn(vocab, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    n_part = (K + 127) // 128
    rowss = torch.rand(plan_rows, n_part, device="cuda", generator=g) * 2.0 + 0.1
    ldo = vocab + 6                                       # columns >= vocab stay untouched
    out = torch.full((plan_rows + 3, ldo), float("nan"), device="cuda")
    L = _lib()
    rc = L.lib.rr_op_prefill_gemm(_ptr(A), plan_rows, T, K, _ptr(W), vocab, K, _ptr(out), ldo, 6, _ptr(rowss), n_part,
                                  K, 1e-5, None, None, None, 0, None)
    L.check(rc, "rr_op_prefill_gemm")
    torch.cuda.synchronize()
    a64, w64 = A[:T].double(), W.double()
    ss = rowss[:T].float().sum(1).double()                # the kernel sums the fp32 partials in order
    r = 1.0 / torch.sqrt(ss / K + 1e-5)
    ref = (a64 @ w64.T) * r[:, None]
    S = (a64.abs() @ w64.abs().T) * r[:, None]
    bound = 2.02 * K * U * S + (n_part + 4) * U * ref.abs()
    got = out[:T, :vocab].double()
    assert torch.isfinite(got).all()
    assert ((got - ref).abs() <= bound).all(), float(((got - ref).abs() - bound).max())
    assert torch.isnan(out[T:]).all() and torch.isnan(out[:T, vocab:]).all()
    # no deferred norm (n_part 0): the plain product
    out2 = torch.full((plan_rows, vocab), float("nan"), device="cuda")
    L.check(L.lib.rr_op_prefill_gemm(_ptr(A), plan_rows, T, K, _ptr(W), vocab, K, _ptr(out2), vocab, 6, None, 0, 0, 0.0,
                                     None, None, None, 0, None), "rr_op_prefill_gemm")
    torch.cuda.synchronize()
    ref2 = a64 @ w64.T
    assert ((out2[:T].double() - ref2).abs() <= 2.02 * K * U * (a64.abs() @ w64.abs().T) + 4 * U * ref2.abs()).all()
    # an odd ldo cannot hold 8-byte pairs
    assert L.lib.rr_op_prefill_gemm(_ptr(A), plan_rows, T, K, _ptr(W), vocab, K, _ptr(out2), vocab - 1, 6, None, 0, 0,
                                    0.0, None, None, None, 0, None) == 4


# ---------------------------------------------------------------- engine helpers
def _engine(spec_name, seed=3, sigma=0.05, weights=None, **kw):
    from rr_b200 import Engine, SPECS, make_weights
    w = weights if weights is not None else make_weights(SPECS[spec_name], seed=seed, sigma=sigma, device="cuda",
                                                         norm_jitter=0.1)
    kw = dict(dict(max_batch=8, ctx_max=1024, max_prefill_tokens=512), **kw)
    return Engine(w, **kw), w


def _score(e, prompt, k=5, max_new=1, **kw):
    t = e.submit(prompt, max_new, prompt_logprobs=k, **kw)
    tgt, lp, ids = e.prompt_logprobs(t, timeout=120)
    rec = e.wait(t, timeout=120)
    assert rec.status == 0
    return tgt, lp, ids, rec


def _prompt(vocab, n, seed):
    g = torch.Generator().manual_seed(seed)
    return [1] + torch.randint(3, vocab, (n - 1,), generator=g).tolist()


def _reference(w, prompt):
    if getattr(w.spec, "sliding_window", 0):
        import window_oracle
        logits = window_oracle.forward_logits(w, prompt)
    else:
        from oracle import llama_ref
        logits = llama_ref.forward_logits(w, prompt)
    return logits.double().cpu()


@pytest.mark.parametrize("spec_name, n", [("tiny", 300), ("small", 200), ("tiny96", 250), ("tiny-sw", 330)])
def test_engine_prompt_logprobs_against_the_reference_model(spec_name, n):
    e, w = _engine(spec_name, max_prefill_tokens=128)          # several pieces, and past the window of tiny-sw
    try:
        prompt = _prompt(w.spec.vocab, n, 11)
        tgt, lp, ids, rec = _score(e, prompt, k=5)
        assert rec.n_cached == 0 and len(tgt) == n - 1
        ref = _reference(w, prompt)[:-1]                      # row t - 1 predicts prompt[t]
        ref_lp = torch.log_softmax(ref, -1)
        tol = 0.25 * ref.std(-1)
        want = ref_lp[torch.arange(n - 1), torch.tensor(prompt[1:])]
        err = (torch.from_numpy(tgt).double() - want).abs()
        assert (err <= tol).all(), (float(err.max()), float(tol.min()))
        top2 = ref.topk(2, -1)
        sure = (top2.values[:, 0] - top2.values[:, 1]) > 2 * tol
        assert sure.sum() > 0
        assert (torch.from_numpy(ids[:, 0]).long()[sure] == top2.indices[sure, 0]).all()
        # pairs: ordered by logprob descending, the best ones within the tolerance of the reference's values
        assert (np.diff(lp, axis=1) <= 0).all()
        got_best = torch.from_numpy(lp[:, 0]).double()
        assert ((got_best - ref_lp.max(-1).values).abs() <= tol).all()
    finally:
        e.close()


def test_bit_identical_across_chunks_pieces_slots_choices_and_prefix_cache():
    from rr_b200 import SPECS, make_weights
    w = make_weights(SPECS["tiny"], seed=5, sigma=0.05, device="cuda", norm_jitter=0.1)
    prompt = _prompt(1024, 400, 21)
    others = [_prompt(1024, m, 30 + m) for m in (37, 90)]
    e, _ = _engine("tiny", weights=w, max_prefill_tokens=1024)
    try:
        base = _score(e, prompt, k=3, max_new=6, top_logprobs=2)
        # with other prompts in the same chunk (submitted first, so the scored one lands at another row offset / slot)
        ts = [e.submit(p, 4) for p in others]
        again = _score(e, prompt, k=3, max_new=6, top_logprobs=2)
        for t in ts:
            e.wait(t, timeout=60)
        # n = 3: scored once, every choice the same tokens
        multi = _score(e, prompt, k=3, max_new=6, top_logprobs=2, n=3)
        # no scoring: the same generated tokens and logprobs
        t = e.submit(prompt, 6, top_logprobs=2)
        plain = e.wait(t, timeout=60)
    finally:
        e.close()
    runs = [again, multi]
    for mp, pc in ((64, False), (150, False), (1024, True)):
        e, _ = _engine("tiny", weights=w, max_prefill_tokens=mp, prefix_cache=pc)
        try:
            if pc:                                            # a retained prefix would be a hit for a plain request
                e.wait(e.submit(prompt[:300] + [5] * 10, 2), timeout=60)
            runs.append(_score(e, prompt, k=3, max_new=6, top_logprobs=2))
        finally:
            e.close()
    for r in runs:
        for a, b in zip(base[:3], r[:3]):
            assert np.array_equal(a, b)
        assert r[3].tokens == base[3].tokens and r[3].logprobs == base[3].logprobs and r[3].n_cached == 0
    assert all(c == base[3].tokens for c in multi[3].choices)
    assert plain.tokens == base[3].tokens and plain.logprobs == base[3].logprobs


def test_fp8_scores_equal_bf16_on_dequantized_weights():
    from rr_b200 import Engine, SPECS, make_weights
    from rr_b200.models import quantize_fp8
    w = make_weights(SPECS["small"], seed=8, sigma=0.05, device="cuda", norm_jitter=0.1)
    q = quantize_fp8(w)
    prompt = _prompt(SPECS["small"].vocab, 300, 4)
    out = []
    for weights in (q, q.dequantize()):
        e = Engine(weights, max_batch=8, ctx_max=1024, max_prefill_tokens=128)
        try:
            out.append(_score(e, prompt, k=4, max_new=4, top_logprobs=1))
        finally:
            e.close()
    for a, b in zip(out[0][:3], out[1][:3]):
        assert np.array_equal(a, b)
    assert out[0][3].tokens == out[1][3].tokens


def test_teacher_forcing_matches_the_decode_path():
    """Greedy reply with logprobs on sharpened weights, then prompt + reply scored.  Each reply token's scored logprob is
    the decode path's within TOL, and it is among the scored best five.  It is the scored top-1 wherever the decode step's
    own margin between its two best tokens exceeds 2 TOL: the two paths round differently (the decode step normalises
    before its split-K GEMMs and runs lm_head in decode orientation, the scoring chunk applies the deferred norm after
    its prefill GEMMs), so two tokens closer than that may swap places."""
    e, w = _engine("tiny", sigma=0.08)
    try:
        prompt = _prompt(1024, 60, 9)
        t = e.submit(prompt, 24, top_logprobs=2)
        rec = e.wait(t, timeout=60)
        reply = rec.tokens
        tgt, lp, ids, _ = _score(e, prompt + reply, k=5)
        n = len(prompt)
        ref = _reference(w, prompt + reply)[n - 1: -1]
        tol = 0.25 * ref.std(-1)
        checked = 0
        for j, tok in enumerate(reply):
            (t0, l0), (_, l1) = rec.logprobs[j][:2]
            assert t0 == tok
            assert abs(float(tgt[n - 1 + j]) - l0) <= float(tol[j]), j
            assert tok in ids[n - 1 + j].tolist(), j
            if l0 - l1 > 2 * float(tol[j]):
                assert ids[n - 1 + j, 0] == tok, j
                checked += 1
        assert checked >= 1, "no reply token had a clear margin: sharpen the weights"
    finally:
        e.close()


def test_cancel_and_fallback():
    from rr_b200 import Engine, EngineBackend, Router, SPECS, make_weights
    w = make_weights(SPECS["tiny"], seed=2, sigma=0.05, device="cuda")
    e = Engine(w, max_batch=8, ctx_max=4096, max_prefill_tokens=256)
    try:
        total, free0 = e.kv_usage()
        for delay in (0.0, 0.002, 0.02):                     # queued, in a scoring chunk, in the middle of the pieces
            t = e.submit(_prompt(1024, 3000, 1), 4, prompt_logprobs=2)
            time.sleep(delay)
            _lib().check(_lib().lib.rr_engine_cancel(e._h, t), "cancel")
            deadline = time.time() + 30
            while e.kv_usage()[1] != free0 and time.time() < deadline:
                time.sleep(0.01)
            assert e.kv_usage() == (total, free0)
        ref = _score(e, _prompt(1024, 200, 3), k=2)
    finally:
        e.close()
    bad = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=512, fail_prob=1.0, fail_seed=1)
    good = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=512)
    ml = [{"model_name": "a", "litellm_params": {"model": "b200/tiny", "gpu": 0}},
          {"model_name": "b", "litellm_params": {"model": "b200/tiny-b", "gpu": 1}}]
    r = Router(model_list=ml, fallbacks=[{"a": ["b"]}], allowed_fails=1000,
               backends={0: EngineBackend(bad), 1: EngineBackend(good)}, seed=0)
    try:
        resp = r.text_completion("a", [_prompt(1024, 200, 3)], max_tokens=1, echo=True, logprobs=2)
        assert resp.model == "tiny-b"
        lp = resp.choices[0].logprobs
        assert lp["token_logprobs"][0] is None
        assert np.array_equal(np.array(lp["token_logprobs"][1:200], np.float32), ref[0])
    finally:
        r.close(); bad.close(); good.close()


def test_engine_that_never_scores_allocates_nothing_new():
    from rr_b200 import SPECS
    e, w = _engine("tiny", ctx_max=512)
    try:
        torch.cuda.synchronize()
        before = torch.cuda.mem_get_info()[0]
        e.wait(e.submit(_prompt(1024, 100, 1), 4, top_logprobs=3), timeout=60)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == before
        _score(e, _prompt(1024, 100, 1), k=1)
        torch.cuda.synchronize()
        # the scoring buffers, allocated by the first scoring request only
        assert before - torch.cuda.mem_get_info()[0] >= min(1024, 512) * SPECS["tiny"].vocab * 4
    finally:
        e.close()


def test_full_model_long_prompt_in_pieces_equals_one_chunk():
    from rr_b200 import Engine, SPECS, make_weights
    w = make_weights(SPECS["llama-3-8b"], seed=0, device="cuda")
    prompt = _prompt(SPECS["llama-3-8b"].vocab, 12000, 7)
    out = []
    for mp in (12032, 4096):
        e = Engine(w, max_batch=2, ctx_max=12288, max_prefill_tokens=mp, kv_cache_tokens=12288)
        try:
            out.append(_score(e, prompt, k=5))
        finally:
            e.close()
            torch.cuda.empty_cache()
    for a, b in zip(out[0][:3], out[1][:3]):
        assert np.array_equal(a, b)
    assert np.isfinite(out[0][0]).all() and out[0][3].tokens == out[1][3].tokens


def _serve(r):
    import socket
    import uvicorn
    from rr_b200.server import create_app
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    srv = uvicorn.Server(uvicorn.Config(create_app(r), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=srv.run, daemon=True)
    th.start()
    while not srv.started:
        time.sleep(0.05)
    return srv, th, port


def test_http_openai_sdk_lm_eval_request():
    openai = pytest.importorskip("openai")
    from rr_b200 import EngineBackend, Router
    e, w = _engine("tiny", sigma=0.05)
    prompts = [_prompt(1024, m, 40 + m) for m in (20, 75, 130)]
    want = [_score(e, p, k=1) for p in prompts]
    ml = [{"model_name": "m", "litellm_params": {"model": "b200/tiny", "gpu": 0}}]
    r = Router(model_list=ml, backends={0: EngineBackend(e)}, seed=0)
    srv, th, port = _serve(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}/v1", max_retries=0)
        resp = client.completions.create(model="m", prompt=prompts, echo=True, logprobs=1, max_tokens=1, temperature=0,
                                         timeout=60)
        assert resp.object == "text_completion" and len(resp.choices) == 3
        for i, (p, (tgt, lp, ids, rec)) in enumerate(zip(prompts, want)):
            c = resp.choices[i]
            assert c.index == i
            got = c.logprobs.token_logprobs
            assert got[0] is None and len(got) == len(p) + 1
            assert np.array_equal(np.array(got[1:len(p)], np.float32), tgt)
            chat = r.completion("m", prompt_ids=p, max_tokens=1)
            assert chat._token_ids == rec.tokens
        assert resp.usage.prompt_tokens == sum(len(p) for p in prompts)
    finally:
        srv.should_exit = True
        th.join(10)
        r.close(); e.close()
