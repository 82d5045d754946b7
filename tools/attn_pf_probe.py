"""Standalone prefill-attention probe: correctness vs an fp32 torch reference and CUDA-event timing at the
bench chunk shape (16 prompts x 512 tokens, 32 query heads, 8 kv heads) and a ragged batch, on the wgmma kernel
(prefill_attn_tc_kernel)."""
import math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rr_b200 import _lib

def P(t): return t.data_ptr()
DEV = "cuda"
H, KV, ctx_max = 32, 8, 640
lens_sets = {"bench 16x512": [512] * 16, "ragged": [1, 17, 64, 65, 200, 512, 333, 128, 129, 640]}
for name, lens in lens_sets.items():
    n = len(lens); slots = n
    g = torch.Generator(device=DEV).manual_seed(1)
    T = sum(lens)
    start = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device=DEV, dtype=torch.int32)
    seq_slot = torch.randperm(n, device=DEV, generator=g).int()
    q = torch.randn(T, H * 128, device=DEV, generator=g).bfloat16()
    kc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    vc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    out = torch.zeros(T, H * 128, device=DEV, dtype=torch.bfloat16)
    scale = 1 / math.sqrt(128)
    def run():
        _lib.check(_lib.lib.rr_op_prefill_attn(P(q), P(kc), P(vc), P(out), P(start), P(seq_slot), n, max(lens), H, KV,
                                               ctx_max, scale, None))
    run(); torch.cuda.synchronize()
    G = H // KV
    worst = 0.0
    for s, L in enumerate(lens):
        a0 = int(start[s]); sl = int(seq_slot[s])
        qs = q[a0:a0 + L].float().view(L, H, 128).transpose(0, 1)
        k = kc[sl, :, :L].float().repeat_interleave(G, 0)
        v = vc[sl, :, :L].float().repeat_interleave(G, 0)
        sc = (qs @ k.transpose(1, 2)) * scale
        sc = sc.masked_fill(~torch.ones(L, L, device=DEV, dtype=torch.bool).tril(), float("-inf"))
        ref = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(L, H * 128)
        worst = max(worst, (out[a0:a0 + L].float() - ref).abs().max().item())
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(3): run()
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(20): run()
    ev[1].record(); torch.cuda.synchronize()
    us = ev[0].elapsed_time(ev[1]) / 20 * 1e3
    flops = sum(4 * 128 * H * (L * (L + 1) / 2) for L in lens)
    print(f"{name:14s} max|err| {worst:.4f}  {us:8.1f} us/call (incl. host map setup)  {flops / us / 1e6:7.1f} TFLOP/s causal")
