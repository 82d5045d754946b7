"""CPU checks of prefill attention as the engine launches it (rr_op_prefill_attn_hd): its refusals, made before the entry
point touches the device, and the error model of test_prefill_attn_gpu.py against a host emulation of the kernel's
per-row online softmax -- 64-key tiles in absolute positions, S in fp32, c = fl(fl(1 / sqrtf(hd)) fl(log2 e)), the
exponent fmaf(s, c, -m) and exp2 computed exactly and rounded to fp32 where the kernel runs ex2.approx, p rounded to bf16
for the PV product while l sums the fp32 p, O rescaled once per visible tile, and bf16(o * (1 / l)).  The emulation
passes the bound and every close wrong answer of the GPU test lies at least 3 bounds from it somewhere in each case."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_prefill_attn_gpu import PAGE, SHAPES, chunk_layout, check_output, make_chunk, window_lo

_P = C.c_void_p(16)                # a stand-in pointer: a refused call never dereferences it

# (q, k_cache, v_cache, out, seq_start, seq_slot, seq_pos0, n_seqs, max_len, n_heads, n_kv_heads, head_dim, ctx_max,
#  page_table, pages_per_slot, n_pages, window, q_rows); the first entry is a call the checks accept
ARGS = ("q", "k_cache", "v_cache", "out", "seq_start", "seq_slot", "seq_pos0", "n_seqs", "max_len", "n_heads",
        "n_kv_heads", "head_dim", "ctx_max", "page_table", "pages_per_slot", "n_pages", "window", "q_rows")
GOOD = (_P, _P, _P, _P, _P, _P, _P, 4, 512, 32, 8, 96, 4096, _P, 64, 1000, 0, 2048)
BAD = {
    **{f"null-{a}": {a: None} for a in ARGS[:7] + ("page_table",)},
    "head_dim-48": dict(head_dim=48),
    "head_dim-72": dict(head_dim=72),
    "head_dim-120": dict(head_dim=120),
    "head_dim-144": dict(head_dim=144),
    "head_dim-0": dict(head_dim=0),
    "G-3": dict(n_heads=24, n_kv_heads=8),
    "G-16": dict(n_heads=32, n_kv_heads=2),
    "G-not-integer": dict(n_heads=12, n_kv_heads=8),
    "n_kv_heads-0": dict(n_kv_heads=0),
    "n_heads-0": dict(n_heads=0),
    "ctx_max-not-64-pages": dict(ctx_max=4032),
    "ctx_max-96": dict(ctx_max=96, pages_per_slot=1),
    "pages_per_slot-0": dict(pages_per_slot=0),
    "n_pages-0": dict(n_pages=0),
    "n_seqs-0": dict(n_seqs=0),
    "max_len-0": dict(max_len=0),
    "q_rows-below-max_len": dict(q_rows=511),
    "q_rows-0": dict(q_rows=0),
    "q_rows-negative": dict(q_rows=-1),
    "window-negative": dict(window=-1),
}


@pytest.mark.parametrize("case", list(BAD))
def test_prefill_attn_hd_refuses_before_touching_the_device(case):
    from rr_b200 import _lib
    a = dict(zip(ARGS, GOOD))
    a.update(BAD[case])
    assert _lib.lib.rr_op_prefill_attn_hd(*(a[k] for k in ARGS), None) == 4


# ------------------------------------------------------------------------------------------------ emulated kernel
def _f32(x):
    return x.float().double()


def emulate_rows(q, k, v, pos, lo, hd, scale=None):
    """Kernel arithmetic for rows at positions pos (keys lo .. pos) of q [nh, R, 128-padded hd] bf16 over k, v
    [nh, n, hd] bf16; returns bf16 [nh, R, hd].  Tiles a row does not see leave its state unchanged, as in the kernel."""
    sc = np.float32(np.float32(1.0) / np.sqrt(np.float32(hd))) if scale is None else np.float32(scale)
    sc = float(np.float32(sc * np.float32(1.4426950408889634)))
    nh, R, _ = q.shape
    qf = q.float()
    m = torch.full((nh, R, 1), -math.inf, dtype=torch.float64)
    l = torch.zeros((nh, R, 1), dtype=torch.float64)
    o = torch.zeros((nh, R, hd), dtype=torch.float64)
    for t in range(int(lo.min()) // PAGE, int(pos.max()) // PAGE + 1):
        key0 = t * PAGE
        seen = (key0 <= pos) & (key0 + PAGE > lo)
        if not seen.any():
            continue
        kt, vt = k[:, key0:key0 + PAGE], v[:, key0:key0 + PAGE]
        j = torch.arange(key0, key0 + kt.shape[1])
        vis = (j[None, :] <= pos[:, None]) & (j[None, :] >= lo[:, None])
        s = _f32(qf @ kt.float().transpose(1, 2)).masked_fill(~vis, -math.inf)   # fp32 S
        mx = _f32(s.amax(-1, keepdim=True) * sc)
        n = torch.maximum(m, mx)
        en = torch.where(n == -math.inf, torch.zeros_like(n), n)
        al = _f32(torch.exp2(_f32(m - en)))
        p = _f32(torch.exp2(_f32(s * sc - en)))                                 # fmaf, then ex2 exact and rounded
        pb = p.bfloat16().double()
        upd = seen[None, :, None]
        l = torch.where(upd, _f32(_f32(l * al) + _f32(p.sum(-1, keepdim=True))), l)
        o = torch.where(upd, _f32(_f32(o * al) + _f32(pb @ vt.double())), o)
        m = torch.where(upd, n, m)
    inv = _f32(1.0 / l)
    return _f32(o * inv).bfloat16()


def emulate_chunk(cs, scale=None, kv_of=None, hi_shift=0):
    """The whole chunk's output buffer (NaN slack) as the kernel would write it; scale, kv_of (kv head per query head) and
    hi_shift (last visible key - position) make it wrong on purpose."""
    nh, nkv, hd, ctx, W = SHAPES[cs["name"]]
    kvh = torch.arange(nh) // (nh // nkv) if kv_of is None else kv_of
    out = torch.full((cs["out_len"] + cs["slack"],), float("nan"), dtype=torch.bfloat16)
    view = out[:cs["out_len"]].view(cs["T"], nh, hd)
    st = cs["start"].tolist()
    for i, (ln, p0) in enumerate(cs["seqs"]):
        s = cs["src"][i]
        q = cs["data"][s][p0:p0 + ln].transpose(0, 1)
        k, v = cs["kd"][s][:, :p0 + ln][kvh], cs["vd"][s][:, :p0 + ln][kvh]
        pos = torch.arange(p0, p0 + ln)
        hi = (pos + hi_shift).clamp(0, p0 + ln - 1)
        view[st[i]:st[i] + ln] = emulate_rows(q, k, v, hi, window_lo(pos, W), hd, scale).transpose(0, 1)
    return out


EMU = [("tiny", "cold"), ("tiny", "pieces"), ("hd80", "cached"), ("hd64", "pieces"), ("small96", "cold"),
       ("hd112", "last"), ("tiny-sw", "pieces"), ("tiny-sw", "cached")]


@pytest.mark.parametrize("name,kind", EMU, ids=[f"{n}-{k}" for n, k in EMU])
def test_emulated_kernel_passes_and_every_neighbour_fails(name, kind):
    cs = make_chunk(name, chunk_layout(name, kind), seed=31, dev="cpu")
    stats = check_output(cs, emulate_chunk(cs))
    nh, nkv, hd, ctx, W = SHAPES[name]
    want = {"own key dropped", "key pos + 1 visible"} if kind != "last" else {"own key dropped"}
    if kind in ("cached", "pieces", "last"):
        want.add("prefix before pos0 ignored")
    if hd != 128:
        want.add("scale 1/sqrt(128)")
    if nkv > 1 and nh // nkv > 1:
        want.add("kv head h % n_kv_heads")
    if W > 0 and kind != "cold":
        want |= {"window W - 1", "window W + 1"}
    assert want <= set(stats["margins"]), (want, stats["margins"])


@pytest.mark.parametrize("wrong", ["scale 1/sqrt(128)", "kv head h % n_kv_heads", "key pos + 1 visible",
                                   "own key dropped"])
def test_a_wrong_emulation_fails_the_bound(wrong):
    """The emulated kernel made wrong in the ways the neighbours describe fails check_output."""
    name = "hd80"
    cs = make_chunk(name, chunk_layout(name, "cached"), seed=5, dev="cpu")
    nh, nkv, hd, ctx, W = SHAPES[name]
    kw = {"scale 1/sqrt(128)": dict(scale=1 / math.sqrt(128)), "kv head h % n_kv_heads": dict(kv_of=torch.arange(nh) % nkv),
          "key pos + 1 visible": dict(hi_shift=1), "own key dropped": dict(hi_shift=-1)}[wrong]
    with pytest.raises(AssertionError):
        check_output(cs, emulate_chunk(cs, **kw))
