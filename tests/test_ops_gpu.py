"""Parity of the elementwise / attention kernels (through the C-ABI) against plain torch fp32
references of the same ops.  Tolerances: outputs are bf16 (rel 2^-8) of fp32 math; stated per test."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def L():
    from rr_b200 import _lib
    return _lib


def P(t):
    return t.data_ptr() if t is not None else None


def test_embed_and_rmsnorm_splitk_reduce():
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(0)
    rows, hidden, vocab = 37, 4096, 1000
    table = torch.randn(vocab, hidden, device=DEV, generator=g).bfloat16()
    ids = torch.randint(0, vocab, (rows,), device=DEV, generator=g, dtype=torch.int32)
    active = torch.ones(rows, device=DEV, dtype=torch.int32); active[5] = -1
    x = torch.zeros(rows, hidden, device=DEV)
    lib.check(lib.lib.rr_op_embed(P(ids), P(table), P(x), rows, hidden, P(active), None))
    ref = table[ids.long()].float(); ref[5] = 0
    assert torch.equal(x, ref)

    w = (1 + 0.1 * torch.randn(hidden, device=DEV, generator=g)).bfloat16()
    xn = torch.empty(rows, hidden, device=DEV, dtype=torch.bfloat16)
    # fp32 split-K planes summed into the residual; 8 is the fused decode MLP's plane count for Llama-3-8B / Phi-3 and the
    # most add_rmsnorm_dec_kernel takes
    for n_splits in (1, 3, 8):
        parts = torch.randn(n_splits, rows, hidden, device=DEV, generator=g)
        xs = x.clone()
        lib.check(lib.lib.rr_op_add_rmsnorm(P(xs), P(parts), 0, n_splits, rows * hidden, hidden, P(w), P(xn), rows, hidden,
                                            1e-5, None))
        xr = x + parts.sum(0)
        assert torch.allclose(xs, xr, atol=1e-5, rtol=1e-5), n_splits
        nr = xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5) * w.float()
        assert torch.allclose(xn.float(), nr, atol=2e-2, rtol=1e-2), n_splits      # one bf16 rounding
    # bf16 "part" (prefill orientation) and norm-only (no part)
    pb = torch.randn(rows, hidden, device=DEV, generator=g).bfloat16()
    x1 = xr.clone()
    lib.check(lib.lib.rr_op_add_rmsnorm(P(x1), P(pb), 1, 1, 0, hidden, P(w), P(xn), rows, hidden, 1e-5, None))
    assert torch.allclose(x1, xr + pb.float(), atol=1e-5, rtol=1e-5)
    x2 = xr.clone()
    lib.check(lib.lib.rr_op_add_rmsnorm(P(x2), None, 0, 1, 0, hidden, P(w), P(xn), rows, hidden, 1e-5, None))
    assert torch.equal(x2, xr) and torch.allclose(xn.float(), nr, atol=2e-2, rtol=1e-2)


def test_silu_mul():
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(1)
    rows, inter = 19, 14336
    gu = torch.randn(2, rows, 2 * inter, device=DEV, generator=g)
    act = torch.empty(rows, inter, device=DEV, dtype=torch.bfloat16)
    lib.check(lib.lib.rr_op_silu_mul(P(gu), 0, 2, rows * 2 * inter, 2 * inter, P(act), rows, inter, None))
    s = gu.sum(0)
    ref = torch.nn.functional.silu(s[:, :inter]) * s[:, inter:]
    assert torch.allclose(act.float(), ref, atol=2e-2, rtol=1e-2)
    gb = s.bfloat16()
    lib.check(lib.lib.rr_op_silu_mul(P(gb), 1, 1, 0, 2 * inter, P(act), rows, inter, None))
    ref = torch.nn.functional.silu(gb[:, :inter].float()) * gb[:, inter:].float()
    assert torch.allclose(act.float(), ref, atol=2e-2, rtol=1e-2)


def _rope_ref(x, pos, theta):
    # HF rotate_half convention on [..., 128]
    d = x.shape[-1]
    inv = 1.0 / (theta ** (torch.arange(0, d, 2, device=x.device).float() / d))
    ang = pos.float()[:, None] * inv[None, :]
    cos, sin = torch.cat([ang.cos(), ang.cos()], -1), torch.cat([ang.sin(), ang.sin()], -1)
    x1, x2 = x[..., : d // 2], x[..., d // 2:]
    rot = torch.cat([-x2, x1], -1)
    return x * cos[:, None, :] + rot * sin[:, None, :]


def test_rope_kv_append():
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(2)
    rows, H, KV, ctx_max, slots = 23, 32, 8, 640, 24
    ld = (H + 2 * KV) * 128
    qkv = torch.randn(2, rows, ld, device=DEV, generator=g)
    slot = torch.randperm(slots, device=DEV, generator=g)[:rows].int(); slot[3] = -1
    pos = torch.randint(0, ctx_max, (rows,), device=DEV, generator=g, dtype=torch.int32)
    q_out = torch.zeros(rows, H * 128, device=DEV, dtype=torch.bfloat16)
    kc = torch.zeros(slots, KV, ctx_max, 128, device=DEV, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    lib.check(lib.lib.rr_op_rope_kv(P(qkv), 0, 2, rows * ld, ld, P(q_out), P(kc), P(vc), P(slot), P(pos), rows, H, KV,
                                ctx_max, 500000.0, None))
    s = qkv.sum(0)
    q = _rope_ref(s[:, : H * 128].view(rows, H, 128), pos, 500000.0)
    k = _rope_ref(s[:, H * 128:(H + KV) * 128].view(rows, KV, 128), pos, 500000.0)
    v = s[:, (H + KV) * 128:].view(rows, KV, 128)
    for r in range(rows):
        if slot[r] < 0:
            assert q_out[r].abs().sum() == 0
            continue
        assert torch.allclose(q_out[r].float().view(H, 128), q[r], atol=3e-2, rtol=1e-2)
        assert torch.allclose(kc[slot[r], :, pos[r]].float(), k[r], atol=3e-2, rtol=1e-2)
        assert torch.allclose(vc[slot[r], :, pos[r]].float(), v[r], atol=3e-2, rtol=1e-2)
    assert kc.float().abs().sum(-1).ne(0).sum().item() == (rows - 1) * KV   # nothing else touched


def test_argmax_ties_and_inc():
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(3)
    rows, vocab = 9, 128256
    logits = torch.randn(rows, vocab, device=DEV, generator=g)
    logits[2, 77] = 50.0; logits[2, 9000] = 50.0           # tie -> lowest index
    logits[4, vocab - 1] = 60.0                            # last element (tail path)
    tok = torch.full((rows,), -7, device=DEV, dtype=torch.int32)
    val = torch.zeros(rows, device=DEV)
    active = torch.ones(rows, device=DEV, dtype=torch.int32); active[6] = -1
    pos = torch.arange(rows, device=DEV, dtype=torch.int32)
    lib.check(lib.lib.rr_op_argmax(P(logits), vocab, rows, vocab, P(tok), P(val), P(active), P(pos), None))
    ref = logits.argmax(-1).int()
    ref[2] = 77
    for r in range(rows):
        if r == 6:
            assert tok[r] == -7 and pos[r] == r
        else:
            assert tok[r] == ref[r] and pos[r] == r + 1 and val[r] == logits[r, ref[r]]


def _attn_ref(q, k, v, scale):
    # q [H, 128], k/v [KV, ctx, 128] fp32
    H, KV = q.shape[0], k.shape[0]
    G = H // KV
    out = torch.empty_like(q)
    for h in range(H):
        s = (k[h // G] @ q[h]) * scale
        p = torch.softmax(s, -1)
        out[h] = p @ v[h // G]
    return out


@pytest.mark.parametrize("H,KV,splits", [(32, 8, 1), (32, 8, 3), (8, 8, 1), (16, 2, 2), (4, 2, 1)])
def test_decode_attention(H, KV, splits):
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(H + KV + splits)
    rows, ctx_max, slots = 11, 704, 12
    kc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    vc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    q = torch.randn(rows, H * 128, device=DEV, generator=g).bfloat16()
    slot = torch.randperm(slots, device=DEV, generator=g)[:rows].int(); slot[1] = -1
    pos = torch.tensor([0, 5, 63, 64, 65, 127, 128, 300, 511, 639, 699], device=DEV, dtype=torch.int32)
    out = torch.zeros(rows, H * 128, device=DEV, dtype=torch.bfloat16)
    scale = 1 / math.sqrt(128)
    lib.check(lib.lib.rr_op_decode_attn(P(q), P(kc), P(vc), P(out), P(slot), P(pos), rows, H, KV, ctx_max, slots, scale, splits, None))
    torch.cuda.synchronize()
    for r in range(rows):
        if slot[r] < 0:
            assert out[r].abs().sum() == 0
            continue
        n = int(pos[r]) + 1
        ref = _attn_ref(q[r].float().view(H, 128), kc[slot[r], :, :n].float(), vc[slot[r], :, :n].float(), scale)
        assert torch.allclose(out[r].float().view(H, 128), ref, atol=2e-2, rtol=2e-2), (r, n)


@pytest.mark.parametrize("H,KV", [(32, 8), (8, 8), (4, 1)])
def test_prefill_attention_causal_ragged(H, KV):
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(H * 3 + KV)
    lens = [1, 17, 64, 65, 200, 512]
    slots_of = [4, 0, 5, 2, 7, 1]
    ctx_max, slots = 640, 8
    T = sum(lens)
    start = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device=DEV, dtype=torch.int32)
    seq_slot = torch.tensor(slots_of, device=DEV, dtype=torch.int32)
    q = torch.randn(T, H * 128, device=DEV, generator=g).bfloat16()
    kc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    vc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    out = torch.zeros(T, H * 128, device=DEV, dtype=torch.bfloat16)
    scale = 1 / math.sqrt(128)
    lib.check(lib.lib.rr_op_prefill_attn(P(q), P(kc), P(vc), P(out), P(start), P(seq_slot), len(lens), max(lens), H, KV,
                                     ctx_max, scale, None))
    torch.cuda.synchronize()
    G = H // KV
    for s, n in enumerate(lens):
        qs = q[int(start[s]):int(start[s]) + n].float().view(n, H, 128).transpose(0, 1)      # [H, n, 128]
        k = kc[slots_of[s], :, :n].float().repeat_interleave(G, 0)
        v = vc[slots_of[s], :, :n].float().repeat_interleave(G, 0)
        sc = (qs @ k.transpose(1, 2)) * scale
        mask = torch.ones(n, n, device=DEV, dtype=torch.bool).tril()
        sc = sc.masked_fill(~mask, float("-inf"))
        ref = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(n, H * 128)
        got = out[int(start[s]):int(start[s]) + n].float()
        assert torch.allclose(got, ref, atol=3e-2, rtol=3e-2), (s, n, (got - ref).abs().max().item())


def test_prefill_attention_rising_scores_rescale_path():
    """Online softmax of the prefill attention under rising scores: every 64-key tile beats the previous one by > 2^8
    (log2 domain), so every tile after the first rescales O and the row sum by a tiny factor; random scores barely
    exercise that path."""
    lib = L()
    H, KV, ctx_max, slots = 8, 2, 640, 3
    lens = [512, 300, 129]
    g = torch.Generator(device=DEV).manual_seed(5)
    T = sum(lens)
    start = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device=DEV, dtype=torch.int32)
    seq_slot = torch.tensor([2, 0, 1], device=DEV, dtype=torch.int32)
    q = torch.ones(T, H * 128, device=DEV).bfloat16()
    q += (torch.randn(T, H * 128, device=DEV, generator=g) * 0.05).bfloat16()
    step = 0.55 * (torch.arange(ctx_max, device=DEV) // 64).float()            # dot product jumps by ~70 per tile
    kc = (step.view(1, 1, ctx_max, 1).expand(slots, KV, ctx_max, 128)
          + torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g) * 0.02).bfloat16().contiguous()
    vc = torch.randn(slots, KV, ctx_max, 128, device=DEV, generator=g).bfloat16()
    out = torch.zeros(T, H * 128, device=DEV, dtype=torch.bfloat16)
    scale = 1 / math.sqrt(128)
    lib.check(lib.lib.rr_op_prefill_attn(P(q), P(kc), P(vc), P(out), P(start), P(seq_slot), len(lens), max(lens), H, KV,
                                         ctx_max, scale, None))
    torch.cuda.synchronize()
    G = H // KV
    for s, n in enumerate(lens):
        a0, sl = int(start[s]), int(seq_slot[s])
        qs = q[a0:a0 + n].float().view(n, H, 128).transpose(0, 1)
        k = kc[sl, :, :n].float().repeat_interleave(G, 0)
        v = vc[sl, :, :n].float().repeat_interleave(G, 0)
        sc = (qs @ k.transpose(1, 2)) * scale
        sc = sc.masked_fill(~torch.ones(n, n, device=DEV, dtype=torch.bool).tril(), float("-inf"))
        assert (sc[:, -1, 64:128].max() - sc[:, -1, :64].max()).item() * 1.4427 > 8.0 or n <= 64   # the jump is real
        ref = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(n, H * 128)
        got = out[a0:a0 + n].float()
        assert torch.isfinite(got).all()
        assert torch.allclose(got, ref, atol=3e-2, rtol=3e-2), (s, n, (got - ref).abs().max().item())
