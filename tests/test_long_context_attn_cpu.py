"""CPU: the selection operands of test_long_context_attn_gpu.py.

The selection covers every key tile of every row with 1 to 127 keys per (row, head) where the head count allows it, the
reference from running sums equals the one from comparing codes, an fp32 emulation of the kernels' online softmax (bf16
p before the PV product, exp2, kv splits merged as the combine kernel does) passes the exact check at depth, and every
wrong neighbour fails it."""
import math

import pytest
import torch

from test_long_context_attn_gpu import (PAGE, assert_neighbours_fail, code_table, exact_ok, key_ids, masked_means,
                                        neighbours, period, progression_means, query_ids, residue_codes, starts, two_hot,
                                        values)

LOG2E = 1.4426950408889634


@pytest.mark.parametrize("H,KV", [(32, 8), (16, 2), (8, 8), (32, 32)])
def test_selection_covers_every_tile(H, KV):
    M = period(H)
    p = torch.cat([torch.arange(0, 600), torch.tensor([8191, 8192, 40037, 45036, 65471, 65534, 65535])])
    st = starts(p, H)
    cnt = st // M + 1
    assert cnt.min() >= 1
    if H >= 16:
        assert cnt.max() <= 127
    for i in range(len(p)):
        sel = torch.cat([torch.arange(int(s), -1, -M) for s in st[i]])
        assert sel.max() <= p[i]
        tiles = torch.zeros(int(p[i]) // PAGE + 1, dtype=torch.bool)
        tiles[sel // PAGE] = True
        assert tiles.all(), (int(p[i]), (~tiles).nonzero().flatten()[:4].tolist())
        if H * 64 <= p[i]:                                              # the own and the next position are selected
            assert int(p[i]) in sel.tolist() and int(p[i]) + 1 - M in sel.tolist()


def _row(H, KV, hd, p, seed):
    g = torch.Generator().manual_seed(seed)
    G = H // KV
    n = min(p + 2, 65536)
    res = residue_codes(KV, H, hd, g)
    ids = key_ids(res, n)
    K = two_hot(ids, hd, code_table(hd))
    V = values(KV, n, hd, g)
    q_ids = query_ids(res, starts(torch.tensor([p]), H), G)[0]
    return res, ids, K, V, q_ids, two_hot(q_ids, hd, code_table(hd))


def emulate(q, K, V, n, G, scale, kv_splits):
    """fp32 online softmax of q [H, 128] over keys 0..n - 1 of K, V [n_kv, N, 128] as the kernels run it: 64-key tiles,
    exp2 of scaled scores less the running max, p rounded to bf16 before the PV product, splits merged at the end."""
    kv = K.shape[0]
    sc = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    s = (q.float().view(kv, G, 128) @ K[:, :n].float().transpose(1, 2)) * sc
    tiles = -(-n // PAGE)
    per = -(-tiles // kv_splits)
    parts = []
    for z in range(kv_splits):
        m = torch.full((kv, G), -math.inf)
        l = torch.zeros(kv, G)
        o = torch.zeros(kv, G, 128)
        for t in range(z * per, min(tiles, (z + 1) * per)):
            st = s[..., t * PAGE:(t + 1) * PAGE]
            mn = torch.maximum(m, st.amax(-1))
            r = torch.where(mn == -math.inf, torch.zeros_like(mn), mn)
            al = torch.exp2(m - r)
            p = torch.exp2(st - r[..., None])
            m = mn
            l = l * al + p.sum(-1)
            o = o * al[..., None] + p.bfloat16().float() @ V[:, t * PAGE:t * PAGE + p.shape[-1]].float()
        parts.append((m, l, o))
    mm = torch.stack([m for m, _, _ in parts]).amax(0)
    L, O = torch.zeros(kv, G), torch.zeros(kv, G, 128)
    for m, l, o in parts:
        f = torch.where(m == -math.inf, torch.zeros_like(m), torch.exp2(m - mm))
        L = L + l * f
        O = O + o * f[..., None]
    return (O * (1 / L)[..., None]).bfloat16().view(kv * G, 128)


@pytest.mark.parametrize("H,KV,hd", [(32, 8, 128), (16, 2, 128), (8, 8, 128), (32, 32, 96)])
@pytest.mark.parametrize("p", [8192, 45036, 65535])
def test_emulated_kernel_passes_and_every_neighbour_fails(H, KV, hd, p):
    G = H // KV
    res, ids, K, V, q_ids, q = _row(H, KV, hd, p, seed=H * 100 + KV + p)
    ref, cnt = masked_means(ids, V[..., :hd], q_ids, 0, p, G)
    assert cnt.min() >= 1 and (H < 16 or cnt.max() <= 127)
    assert torch.equal(ref, progression_means(V[..., :hd], starts(torch.tensor([p]), H), H, G)[0])
    pos0 = 40037 if p == 45036 else 0
    for ks in (1, 8):
        out = emulate(q, K, V, p + 1, G, 1 / math.sqrt(hd), ks)[:, :hd]
        ok = exact_ok(out, ref)
        assert ok.all(), (ks, int((~ok).sum()))
        assert_neighbours_fail([(out, neighbours(ids, V[..., :hd], q_ids, p, G, pos0=pos0)[1])])


def test_a_wrong_emulation_fails():
    """The check is not vacuous on the emulation either: the emulated kernel over one tile too few is refused."""
    H, KV, hd, p = 32, 8, 128, 40000
    res, ids, K, V, q_ids, q = _row(H, KV, hd, p, seed=5)
    ref, _ = masked_means(ids, V, q_ids, 0, p, H // KV)
    out = emulate(q, K, V, p + 1 - PAGE, H // KV, 1 / math.sqrt(hd), 1)
    assert not exact_ok(out, ref).all()
