"""Generate tests/golden/sliding_window_golden.pt with the REAL transformers MistralForCausalLM (fp32, CPU, eager
attention) with sliding_window = 100, on seeded bf16-rounded weights of the tiny-sw spec (the tiny shape with a 100-token
window).  Position q attends to positions q - 99 .. q (transformers.masking_utils.sliding_window_overlay), so prompts of
1, 99, 100, 101, 300 and 700 tokens cover rows below, at and far past the window; 3 greedy steps each.
Run in the build container:  python tests/golden/make_sliding_window_golden.py
Pins tests/window_oracle.py, the windowed restatement the GPU engine is checked against."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from rr_b200.models import SPECS, make_weights  # noqa: E402

SPEC = "tiny-sw"
SEED, SIGMA, JITTER, STEPS = 11, 0.05, 0.1, 3
LENGTHS = (1, 99, 100, 101, 300, 700)


def build_mistral(w):
    from transformers import MistralConfig, MistralForCausalLM
    s = w.spec
    cfg = MistralConfig(vocab_size=s.vocab, hidden_size=s.hidden, intermediate_size=s.inter, num_hidden_layers=s.n_layers,
                        num_attention_heads=s.n_heads, num_key_value_heads=s.n_kv_heads, head_dim=s.head_dim,
                        rope_theta=s.rope_theta, rms_norm_eps=s.rms_eps, max_position_embeddings=4096,
                        sliding_window=s.sliding_window, tie_word_embeddings=False, attn_implementation="eager")
    m = MistralForCausalLM(cfg).float()
    H, KV, D = s.n_heads, s.n_kv_heads, s.head_dim
    sd = {"model.embed_tokens.weight": w.embed, "lm_head.weight": w.lm_head, "model.norm.weight": w.final_norm}
    for l in range(s.n_layers):
        p = f"model.layers.{l}."
        sd[p + "self_attn.q_proj.weight"] = w.wqkv[l][: H * D]
        sd[p + "self_attn.k_proj.weight"] = w.wqkv[l][H * D:(H + KV) * D]
        sd[p + "self_attn.v_proj.weight"] = w.wqkv[l][(H + KV) * D:]
        sd[p + "self_attn.o_proj.weight"] = w.wo[l]
        sd[p + "mlp.gate_proj.weight"] = w.wgu[l][: s.inter]
        sd[p + "mlp.up_proj.weight"] = w.wgu[l][s.inter:]
        sd[p + "mlp.down_proj.weight"] = w.wdown[l]
        sd[p + "input_layernorm.weight"] = w.norm_attn[l]
        sd[p + "post_attention_layernorm.weight"] = w.norm_mlp[l]
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if "rotary" not in k] and not unexpected, (missing, unexpected)
    assert m.config.sliding_window == s.sliding_window
    return m.eval()


def main():
    import transformers
    spec = SPECS[SPEC]
    w = make_weights(spec, seed=SEED, sigma=SIGMA, device="cpu", norm_jitter=JITTER)
    hf = build_mistral(w)
    g = torch.Generator().manual_seed(2468)
    prompts = [torch.randint(0, spec.vocab, (n,), generator=g).tolist() for n in LENGTHS]
    logits, tokens = [], []
    with torch.no_grad():
        for p in prompts:
            toks, lg, tk = list(p), [], []
            for _ in range(STEPS):
                lo = hf(torch.tensor([toks])).logits[0, -1].float()
                t = int(lo.argmax())
                lg.append(lo); tk.append(t); toks.append(t)
            logits.append(torch.stack(lg)); tokens.append(tk)
    out = {"spec": SPEC, "seed": SEED, "sigma": SIGMA, "norm_jitter": JITTER, "torch": str(torch.__version__),
           "transformers": transformers.__version__, "sliding_window": spec.sliding_window, "prompts": prompts,
           "logits": logits, "tokens": tokens,
           "weight_checksum": float(sum(t.float().abs().sum() for t in w.tensors()))}
    torch.save(out, os.path.join(os.path.dirname(__file__), "sliding_window_golden.pt"))
    print("ok", [len(p) for p in prompts])


if __name__ == "__main__":
    main()
