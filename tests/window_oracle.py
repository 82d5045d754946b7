"""Sliding-window restatement of oracle/llama_ref.forward_logits, for the tests: the same fp32 forward pass, with the
spec's window W > 0 applied, so position q attends to positions max(0, q - W + 1) .. q.  Pinned against the real
transformers MistralForCausalLM(sliding_window=100) by tests/golden/sliding_window_golden.pt
(tests/golden/make_sliding_window_golden.py, tests/test_sliding_window_cpu.py).

Attention runs in blocks of at most 1024 query rows, each against the keys its rows may see, so a long prompt never holds
a T x T score tensor (a 12000-token prompt at 32 heads would need about 18 GB).  A sequence no longer than W, or a spec
without a window, is llama_ref.forward_logits itself."""
from __future__ import annotations

import math
from typing import Sequence

import torch

from oracle import llama_ref
from oracle.llama_ref import _rms, _rope

BLOCK = 1024


def window_attn(q, k, v, W):
    """Sliding-window attention of q, k, v [T, H, D] (k, v already repeated per query head) -> [T, H, D]."""
    T, _, D = q.shape
    out = torch.empty_like(q)
    for t0 in range(0, T, BLOCK):
        t1 = min(T, t0 + BLOCK)
        k0 = max(0, t0 - W + 1)
        qp = torch.arange(t0, t1, device=q.device)[:, None]
        kp = torch.arange(k0, t1, device=q.device)[None, :]
        vis = (kp <= qp) & (kp > qp - W)
        sc = torch.einsum("thd,shd->hts", q[t0:t1], k[k0:t1]) / math.sqrt(D)
        sc = sc.masked_fill(~vis[None], float("-inf"))
        out[t0:t1] = torch.einsum("hts,shd->thd", torch.softmax(sc, -1), v[k0:t1])
    return out


@torch.no_grad()
def forward_logits(w, tokens: Sequence[int], dtype=torch.float32) -> torch.Tensor:
    """Forward of one sequence under the spec's sliding window -> logits [T, vocab] (fp32 math on the given weights)."""
    s = w.spec
    W = getattr(s, "sliding_window", 0)
    T = len(tokens)
    if not 0 < W < T:               # every key a row may see lies inside the window
        return llama_ref.forward_logits(w, tokens, dtype)
    dev = w.embed.device
    ids = torch.as_tensor(list(tokens), device=dev, dtype=torch.long)
    pos = torch.arange(T, device=dev)
    x = w.embed[ids].to(dtype)
    H, KV, D = s.n_heads, s.n_kv_heads, s.head_dim
    for l in range(s.n_layers):
        h = _rms(x, w.norm_attn[l].to(dtype), s.rms_eps)
        qkv = h @ w.wqkv[l].to(dtype).t()
        q = _rope(qkv[:, : H * D].view(T, H, D), pos, s.rope_theta)
        k = _rope(qkv[:, H * D:(H + KV) * D].view(T, KV, D), pos, s.rope_theta)
        v = qkv[:, (H + KV) * D:].view(T, KV, D)
        a = window_attn(q, k.repeat_interleave(H // KV, 1), v.repeat_interleave(H // KV, 1), W).reshape(T, H * D)
        x = x + a @ w.wo[l].to(dtype).t()
        h = _rms(x, w.norm_mlp[l].to(dtype), s.rms_eps)
        gu = h @ w.wgu[l].to(dtype).t()
        act = torch.nn.functional.silu(gu[:, : s.inter]) * gu[:, s.inter:]
        x = x + act @ w.wdown[l].to(dtype).t()
    x = _rms(x, w.final_norm.to(dtype), s.rms_eps)
    return x @ w.lm_head.to(dtype).t()
