"""GPU: parity at BASELINE.json's full size (Llama-3-8B shape, 32 layers, vocab 128256, 512-token prompts) against the
fp32 generated-token oracle on the same seeded bf16 weights.

Stated tolerance for the 32-layer model (north_star: "within a stated fp16 logit tolerance"): per position, with
d = logit_engine - logit_oracle and s = std of the oracle's logits over the vocabulary,
    rms(d) <= 0.08 * s   and   max|d| <= 0.40 * s,
and the engine's greedy token equals the oracle's wherever the oracle's top-2 margin exceeds 0.8 * s.
bf16 rounding noise grows ~sqrt(layers) from the 2-layer bound.
(HF's own bf16 execution deviates from its fp32 execution by more than this: DESIGN.md §parity.)"""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL_RMS, TOL_MAX = 0.08, 0.40


def _check(got, ref, what):
    ref = ref.float().cpu(); got = torch.as_tensor(got).float().cpu()
    s = ref.std().item(); d = got - ref
    rms, mx = d.pow(2).mean().sqrt().item() / s, d.abs().max().item() / s
    assert torch.isfinite(got).all() and rms <= TOL_RMS and mx <= TOL_MAX, (what, rms, mx)
    top2 = ref.topk(2).values
    margin_ok = (top2[0] - top2[1]).item() > 2 * TOL_MAX * s
    agree = int(got.argmax()) == int(ref.argmax())
    if margin_ok:
        assert agree, what
    return rms, mx, agree


def test_llama3_8b_shape_prefill_and_decode_logits():
    from oracle import llama_ref
    from rr_b200.engine import Engine
    from rr_b200.models import SPECS, make_weights
    spec = SPECS["llama-3-8b"]
    w = make_weights(spec, seed=0, sigma=0.02, device="cuda")
    eng = Engine(w, max_batch=64, ctx_max=640, max_prefill_tokens=2048, use_cuda_graph=False)
    try:
        lens = [512, 512, 37]
        prompts = []
        for r, n in enumerate(lens):
            g = torch.Generator().manual_seed(1234 + r)           # the bench's prompt generator
            prompts.append(torch.randint(0, spec.vocab, (n,), generator=g).tolist())
        slots = [0, 63, 17]
        first, logits = eng.prefill(prompts, slots, want_logits=True)
        worst = [0.0, 0.0]
        n_agree = 0
        refs = [llama_ref.forward_logits(w, p)[-1] for p in prompts]
        for i in range(3):
            rms, mx, ag = _check(logits[i], refs[i], f"prefill len={lens[i]}")
            worst = [max(worst[0], rms), max(worst[1], mx)]; n_agree += ag
        # two teacher-forced decode steps on the ORACLE's tokens
        toks = [list(p) for p in prompts]
        cur = [int(r.argmax()) for r in refs]
        for j in range(2):
            pos = [len(t) for t in toks]
            for t, c in zip(toks, cur):
                t.append(c)
            nxt, lg = eng.decode_step(slots, cur, pos, want_logits=True)
            refs = [llama_ref.forward_logits(w, t)[-1] for t in toks]
            for i in range(3):
                rms, mx, ag = _check(lg[i], refs[i], f"decode step {j} seq {i}")
                worst = [max(worst[0], rms), max(worst[1], mx)]; n_agree += ag
            cur = [int(r.argmax()) for r in refs]
        print(f"\n[llama-3-8b, 32 layers] worst rms/std = {worst[0]:.4f}, worst max/std = {worst[1]:.4f}, "
              f"greedy token agreement {n_agree}/9")
    finally:
        eng.close()
