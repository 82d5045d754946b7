"""Kernel-level parity of prefill attention (prefill_attn_tc_kernel, csrc/rr_attn_tc.cu) through rr_op_prefill_attn_hd,
which launches it exactly as run_prefill does: the true head dim with its compact output [T][n_heads * head_dim] and the
engine's scale 1 / sqrtf(head_dim) (pf_attn_layer), the page table, the window, and q mapped over q_rows > T rows.

Operands.  q rows are bf16 N(0, QSTD^2) in columns [0, head_dim) and zero in [head_dim, 128), as the engine's q buffer
is; rows T .. q_rows hold NaN.  Each sequence's V at positions 0 .. pos0 + len - 1 of its slot is bf16 N(0, 1) and its K
is N(0, KBASE^2) plus the aligned part of aligned_keys, which makes the keys that the close wrong answers add or drop
stand out at any depth; every other cache row, the pad columns [head_dim, 128) of every row and every page the table
does not name hold finite poison of magnitude 1e3..1e4 (finite: a masked key reaches the PV wgmma with p = 0, and
0 * NaN would be NaN).  Pages
are a random permutation of the pool, slots a permutation with slot != sequence, and `out` is NaN-filled with slack
past its end that a pitch of n_heads * 128 would reach.  Chunks are laid out as run_prefill lays out its sequences:
cold sequences (pos0 = 0), prefix-cache suffixes (pos0 a multiple of 64), long-prompt pieces (pos0 not a multiple of 64,
one ending at ctx_max - 1) and a single row at ctx_max - 1.

Reference, all fp64: query row at absolute position P = pos0 + i of head h sees keys lo .. P of kv head h / G, lo =
max(0, P - W + 1) (0 without a window); s_j = scale q . k_j, w = softmax(s), O = sum_j w_j v_j.  Error model of the
kernel's output before its bf16 rounding, per element d:
  * T1, the bf16 rounding of p before the PV wgmma while l sums the fp32 p: sum_j eps_j w_j v_jd, |eps_j| <= 2^-8.  With
    independent signs and sigma = 2^-9 per rounding, lambda = 6 standard deviations give lambda 2^-9 sqrt(sum_j w_j^2
    v_jd^2); the worst case 2^-8 sum_j w_j |v_jd| is used where it is smaller.  A key that is the maximum of its 64-key
    tile when that maximum is a new running maximum of the row gets p = ex2(fmaf(s, c, -fl(s c))), within 2^-23 of 1,
    which bf16 rounds to exactly 1: those keys are left out.
  * T2, the relative error mu_j of each fp32 p_j, which enters O as sum_j mu_j w_j |v_jd - O_d|:
    - the fp32 accumulation of S = q . k over 8 k16 groups of the wgmma, each of which may align and truncate:
      2^-18 scale sum_d |q_d k_jd|;
    - c = fl(fl(1 / sqrtf(hd)) fl(log2 e)) (four roundings, 2^-22 relative), the running maximum fl(max s c) and the
      rounding of fmaf(s, c, -m): 2^-21 (|s_j| + |s_max|);
    - ex2.approx.ftz.f32, whose maximum relative error the PTX ISA gives as about 2^-22 (not exp2f's): taken as 2^-21.
    ftz flushes p < 2^-126 to zero, an absolute error far below every other term (l >= 1).
  * T3, the fp32 accumulation of o and l over the row's T visible key tiles: per tile one rescale by alpha = ex2(m_old -
    m) (ex2 and the product), four k16 steps of the PV wgmma that may each truncate, 16 fp32 additions to each thread's
    l; then the quad reduction of l, 1 / l and the product: (24 T + 40) 2^-23 (sum_j w_j |v_jd| + |O_d|).
  * the bf16 rounding of the output: half the bf16 spacing at |O| + T1 + T2 + T3.
The two warpgroups of a 128-row query tile run the same arithmetic on their 64 rows each, so the model is per row.

The bound tells the reference apart from the close wrong answers listed in NEIGHBOURS: each moves the reference by at
least 3 bounds away from the kernel's output somewhere in every case where it differs from the reference at all."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_decode_attn_gpu import SHAPES as DECODE_SHAPES
from test_decode_attn_gpu import half_spacing_bf16

pytestmark = pytest.mark.gpu

DEV = "cuda"
LAMBDA = 6.0
U23 = 2.0 ** -23
PAGE = 64
QSTD = 1.5
KBASE = 0.5
S_ALIGN = 4.0
OLD_TOL = 3e-2                     # allclose(3e-2) of test_ops_gpu.py / test_prefix_cache_gpu.py: 3e-2 (1 + |ref|)

# name -> (n_heads, n_kv_heads, head_dim, ctx_max, window)
SHAPES = {n: (h, kv, hd, ctx, 0) for n, (h, kv, hd, _theta, ctx) in DECODE_SHAPES.items()}
SHAPES["mistral-7b"] = (32, 8, 128, 8192, 4096)
SHAPES["tiny-sw"] = (4, 2, 128, 640, 100)

NEIGHBOURS = ("key pos + 1 visible", "own key dropped", "prefix before pos0 ignored", "scale 1/sqrt(128)",
              "kv head h % n_kv_heads", "window W - 1", "window W + 1")


def chunk_layout(name, kind):
    """[(len, pos0)] of one chunk, in run_prefill's order."""
    _, _, _, ctx, W = SHAPES[name]
    if kind == "cold":
        return [(n, 0) for n in (1, 17, 63, 64, 65, 127, 128, 129, 300, 512)]
    if kind == "cached":                                   # prefix-cache suffixes: pos0 a multiple of 64
        return [(1, 64), (65, 128), (128, 256), (200, 320), (129, ctx - 192)]
    if kind == "pieces":                                   # long-prompt pieces: pos0 not a multiple of 64
        seqs = [(16, 1), (29, 100), (71, 229), (150, 333)]
        if W > 0 and W + 200 < ctx:
            seqs.append((200, W - 100))                    # rows on both sides of P = W
        return seqs + [(129, ctx - 130)]                  # ends at ctx_max - 1
    assert kind == "last"
    return [(1, ctx - 1)]                                  # n_heads work items: fewer than the SMs


KINDS = ("cold", "cached", "pieces", "last")
CASES = [pytest.param(n, k, id=f"{n}-{k}") for n in SHAPES for k in KINDS]


def poison(shape, g, dev):
    sign = torch.randint(0, 2, shape, device=dev, generator=g, dtype=torch.int8).float() * 2 - 1
    return (sign * (1e3 + 9e3 * torch.rand(shape, device=dev, generator=g))).bfloat16()


def aligned_keys(q, z, nkv, W):
    """bf16 K [nkv, n, hd] of a sequence with queries q [n, nh, hd]: KBASE z plus, in kv head c, s = S_ALIGN with the query
    of head c G + t at position j + off_t for off = (0, W - 1, W) (t < G; the last two with a window only).  Deep in a
    context one random key moves no output by much, so the keys the close wrong answers add or drop -- the own key, the
    first key of the window and the one before it -- are made to stand out."""
    n, nh, hd = q.shape
    G = nh // nkv
    k = KBASE * z
    qf = q.float()
    for t, off in enumerate((0, W - 1, W) if W > 0 else (0,)):
        if t >= G or off >= n:
            continue
        tgt = qf[off:, t::G]                                   # [n - off, nkv, hd]: head c G + t of position j + off
        u = tgt * (S_ALIGN * math.sqrt(hd) / (tgt * tgt).sum(-1, keepdim=True))
        k[:, :n - off] += u.transpose(0, 1)
    return k.bfloat16()


def make_chunk(name, seqs, seed, src=None, dev=DEV):
    """Buffers of one chunk.  seqs = [(len, pos0)]; src[i] names the source sequence whose q rows pos0 .. pos0 + len - 1
    and K / V rows 0 .. pos0 + len - 1 sequence i uses (default: its own), so that pieces of one sequence can be laid
    out against its cold run."""
    nh, nkv, hd, ctx, W = SHAPES[name]
    g = torch.Generator(device=dev).manual_seed(seed)
    src = list(range(len(seqs))) if src is None else src
    n_src = max(src) + 1
    need = [0] * n_src
    for (n, p0), s in zip(seqs, src):
        need[s] = max(need[s], p0 + n)
    data = [(QSTD * torch.randn(m, nh, hd, device=dev, generator=g)).bfloat16() for m in need]
    kd = [aligned_keys(d, torch.randn(nkv, d.shape[0], hd, device=dev, generator=g), nkv, W) for d in data]
    vd = [torch.randn(nkv, m, hd, device=dev, generator=g).bfloat16() for m in need]
    n = len(seqs)
    T = sum(s[0] for s in seqs)
    q_rows = T + 77
    q = torch.zeros(q_rows, nh, 128, device=dev, dtype=torch.bfloat16)
    q[T:] = float("nan")
    start = [0]
    for (ln, p0), s in zip(seqs, src):
        q[start[-1]:start[-1] + ln, :, :hd] = data[s][p0:p0 + ln]
        start.append(start[-1] + ln)
    # slots: a permutation with slot != sequence; pages: a permutation of the pool, spare pages left as poison
    n_slots = n + 2
    perm = torch.randperm(n_slots, device="cpu", generator=torch.Generator().manual_seed(seed)).tolist()
    for r in range(n_slots):
        if perm[r] == r:
            j = (r + 1) % n_slots
            perm[r], perm[j] = perm[j], perm[r]
    slots = perm[:n]
    pps = ctx // PAGE
    used = [-(-(p0 + ln) // PAGE) for ln, p0 in seqs]
    n_pages = sum(used) + 8
    pages = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed + 1)).tolist()
    spare = pages[sum(used):]
    table = torch.tensor([[spare[(r + c) % len(spare)] for c in range(pps)] for r in range(n_slots)], dtype=torch.int32)
    kp, vp = poison((n_pages, nkv, PAGE, 128), g, dev), poison((n_pages, nkv, PAGE, 128), g, dev)
    at = 0
    for i, ((ln, p0), s) in enumerate(zip(seqs, src)):
        m = p0 + ln
        for c in range(used[i]):
            pg = pages[at + c]
            table[slots[i], c] = pg
            r = min(PAGE, m - c * PAGE)
            kp[pg, :, :r, :hd] = kd[s][:, c * PAGE:c * PAGE + r]
            vp[pg, :, :r, :hd] = vd[s][:, c * PAGE:c * PAGE + r]
        at += used[i]
    i32 = dict(device=dev, dtype=torch.int32)
    return dict(name=name, seqs=seqs, src=src, T=T, q_rows=q_rows, q=q, kp=kp, vp=vp, table=table.to(dev),
                n_pages=n_pages, pps=pps, data=data, kd=kd, vd=vd, start=torch.tensor(start, **i32),
                slot=torch.tensor(slots, **i32), pos0=torch.tensor([p0 for _, p0 in seqs], **i32),
                max_len=max(ln for ln, _ in seqs), out_len=T * nh * hd, slack=T * nh * (128 - hd) + nh * 128)


def P(t):
    return C.c_void_p(t.data_ptr())


def run(cs, window=None, q=None, sync=True):
    """One rr_op_prefill_attn_hd launch; returns the NaN-filled output buffer, slack included."""
    from rr_b200 import _lib
    nh, nkv, hd, ctx, W = SHAPES[cs["name"]]
    out = torch.full((cs["out_len"] + cs["slack"],), float("nan"), device=DEV, dtype=torch.bfloat16)
    rc = _lib.lib.rr_op_prefill_attn_hd(P(cs["q"] if q is None else q), P(cs["kp"]), P(cs["vp"]), P(out), P(cs["start"]),
                                        P(cs["slot"]), P(cs["pos0"]), len(cs["seqs"]), cs["max_len"], nh, nkv, hd, ctx,
                                        P(cs["table"]), cs["pps"], cs["n_pages"], W if window is None else window,
                                        cs["q_rows"], None)
    _lib.check(rc, "rr_op_prefill_attn_hd")
    if sync:
        torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------ reference and bound
def attention(q, k, v, pos, lo, scale):
    """fp64 attention of q [nh, R, hd] (row r at position pos[r]) over k, v [nh, n, hd], keys lo[r] .. pos[r] visible:
    (O [nh, R, hd], s [nh, R, n] with -inf where masked, w)."""
    j = torch.arange(k.shape[1], device=q.device)
    vis = (j[None, :] <= pos[:, None]) & (j[None, :] >= lo[:, None])
    s = (scale * (q @ k.transpose(1, 2))).masked_fill(~vis, -math.inf)
    w = torch.softmax(s, -1)
    return w @ v, s, w


def exact_p_keys(s):
    """Mask [.., n] of the keys whose p the kernel computes as exactly 1 after its bf16 rounding: the maximum of a 64-key
    tile when it is a new running maximum of the row (ties: one of them; leaving the others in only widens the bound)."""
    n = s.shape[-1]
    nt = -(-n // PAGE)
    sp = torch.nn.functional.pad(s, (0, nt * PAGE - n), value=-math.inf).view(*s.shape[:-1], nt, PAGE)
    tm, ta = sp.max(-1)
    before = torch.cat([torch.full_like(tm[..., :1], -math.inf), tm.cummax(-1).values[..., :-1]], -1)
    rec = (tm >= before) & (tm > -math.inf)
    idx = torch.where(rec, torch.arange(nt, device=s.device) * PAGE + ta, nt * PAGE)
    mask = torch.zeros(*s.shape[:-1], nt * PAGE + 1, dtype=torch.bool, device=s.device)
    mask.scatter_(-1, idx, True)
    return mask[..., :n]


def attention_bound(q, k, v, pos, lo, scale):
    """(O, bound) per element of the module docstring's error model; q [nh, R, hd], k / v [nh, n, hd] (kv head per query
    head already gathered), fp64."""
    o, s, w = attention(q, k, v, pos, lo, scale)
    va = v.abs()
    wx = w.masked_fill(exact_p_keys(s), 0.0)
    t1 = torch.minimum(LAMBDA * 2.0 ** -9 * ((wx * wx) @ (v * v)).sqrt(), 2.0 ** -8 * (wx @ va))
    sf = torch.where(w > 0, s, torch.zeros_like(s)).abs()
    mu = (2.0 ** -18 * scale * (q.abs() @ k.abs().transpose(1, 2)) + 2.0 ** -21 * (sf + s.amax(-1, keepdim=True).abs())
          + 2.0 ** -21)
    wm = w * mu
    t2 = wm @ va + wm.sum(-1, keepdim=True) * o.abs()
    tiles = (pos // PAGE - lo // PAGE + 1).double()[None, :, None]
    t3 = (24 * tiles + 40) * U23 * (w @ va + o.abs())
    e = t1 + t2 + t3
    return o, e + half_spacing_bf16(o.abs() + e)


def seq_operands(cs, i, dev=DEV):
    """fp64 q [nh, len, hd], k / v [nkv, pos0 + len, hd] and row positions of sequence i."""
    ln, p0 = cs["seqs"][i]
    s = cs["src"][i]
    q = cs["data"][s][p0:p0 + ln].double().transpose(0, 1)
    k = cs["kd"][s][:, :p0 + ln].double()
    v = cs["vd"][s][:, :p0 + ln].double()
    return q, k, v, torch.arange(p0, p0 + ln, device=dev)


def window_lo(pos, W):
    return (pos - W + 1).clamp(min=0) if W > 0 else torch.zeros_like(pos)


def neighbour_refs(name, q, k, v, pos, lo, p0, end, kvh, scale):
    """The close wrong answers that differ from the reference on these rows: what -> O [nh, R, hd] (rows where it does not
    differ are NaN)."""
    nh, nkv, hd, ctx, W = SHAPES[name]
    kk, vv = k[kvh], v[kvh]
    alts = {}

    def rows(mask, o):
        return torch.where(mask[None, :, None], o, torch.full_like(o, math.nan))

    nxt = pos + 1 < end                                    # key pos + 1 holds data of this sequence
    if nxt.any():
        alts[NEIGHBOURS[0]] = rows(nxt, attention(q, kk, vv, torch.minimum(pos + 1, torch.full_like(pos, end - 1)), lo,
                                                  scale)[0])
    own = pos - 1 >= lo
    if own.any():
        alts[NEIGHBOURS[1]] = rows(own, attention(q, kk, vv, (pos - 1).clamp(min=0), lo, scale)[0])
    if p0 > 0:
        lo2 = lo.clamp(min=p0)
        alts[NEIGHBOURS[2]] = rows(lo2 > lo, attention(q, kk, vv, pos, lo2, scale)[0])
    if hd != 128:
        alts[NEIGHBOURS[3]] = attention(q, kk, vv, pos, lo, 1 / math.sqrt(128))[0]
    alt_kvh = torch.arange(nh, device=q.device) % nkv
    if not torch.equal(alt_kvh, kvh):
        o = attention(q, k[alt_kvh], v[alt_kvh], pos, lo, scale)[0]
        alts[NEIGHBOURS[4]] = torch.where((alt_kvh != kvh)[:, None, None], o, torch.full_like(o, math.nan))
    if W > 0:
        for what, w2 in ((NEIGHBOURS[5], W - 1), (NEIGHBOURS[6], W + 1)):
            lo2 = window_lo(pos, w2)
            if (lo2 != lo).any():
                alts[what] = rows(lo2 != lo, attention(q, kk, vv, pos, lo2, scale)[0])
    return alts


def check_output(cs, out_flat, row_block=64):
    """Every written element within its bound of the fp64 reference, nothing else written; every applicable neighbour
    at least 3 bounds from the output somewhere.  Returns stats."""
    nh, nkv, hd, ctx, W = SHAPES[cs["name"]]
    G = nh // nkv
    scale = 1.0 / math.sqrt(hd)
    assert torch.isnan(out_flat[cs["out_len"]:]).all(), "out written past T x n_heads x head_dim"
    out = out_flat[:cs["out_len"]].view(cs["T"], nh, hd)
    assert torch.isfinite(out).all(), "output not written or not finite"
    kvh = torch.arange(nh, device=out.device) // G
    worst, worst_at, margins, rel = 0.0, None, {}, []
    st = cs["start"].tolist()
    for i, (ln, p0) in enumerate(cs["seqs"]):
        q, k, v, pos = seq_operands(cs, i, out.device)
        for r0 in range(0, ln, row_block):
            r1 = min(ln, r0 + row_block)
            qb, pb = q[:, r0:r1], pos[r0:r1]
            lo = window_lo(pb, W)
            o_ref, bound = attention_bound(qb, k[kvh], v[kvh], pb, lo, scale)
            got = out[st[i] + r0:st[i] + r1].double().transpose(0, 1)
            ratio = ((got - o_ref).abs() / bound)
            rmax = ratio.max().item()
            if rmax > worst:
                worst, worst_at = rmax, (i, p0 + r0 + int(ratio.amax((0, 2)).argmax()))
            rel.append((bound / (OLD_TOL * (1 + o_ref.abs()))).flatten())
            for what, alt in neighbour_refs(cs["name"], qb, k, v, pb, lo, p0, p0 + ln, kvh, scale).items():
                m = ((alt - got).abs() / bound).nan_to_num(nan=0.0).max().item()
                margins[what] = max(margins.get(what, 0.0), m)
            del o_ref, bound, got, ratio
    assert worst <= 1.0, f"worst |out - ref| / bound = {worst:.3g} at (sequence, position) {worst_at}"
    for what, m in margins.items():
        assert m >= 3.0, f"{what}: at most {m:.3g} bounds from the output"
    rel = torch.cat(rel)
    return dict(worst=worst, worst_at=worst_at, margins=margins, median_bound_vs_old=rel.median().item())


@pytest.mark.parametrize("name,kind", CASES)
def test_prefill_attn_matches_fp64(name, kind):
    i = list(SHAPES).index(name)
    cs = make_chunk(name, chunk_layout(name, kind), seed=100 * i + KINDS.index(kind))
    stats = check_output(cs, run(cs))
    assert stats["median_bound_vs_old"] <= 0.1, stats
    print(f"\n[{name} {kind}] worst/bound {stats['worst']:.3f} at {stats['worst_at']}, median bound / old tol "
          f"{stats['median_bound_vs_old']:.4f}, margins " + ", ".join(f"{w}: {m:.1f}" for w, m in stats["margins"].items()))


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("name", list(SHAPES))
def test_prefill_attn_bits(name):
    """Repeated launches, stale q rows of NaN against zeros, window >= ctx_max against window 0, pieces of a sequence at
    pos0 > 0 against its cold run, and at head dim 128 rr_op_prefill_attn_cached_paged at the engine's scale: all bit
    for bit."""
    from rr_b200 import _lib
    nh, nkv, hd, ctx, W = SHAPES[name]
    i = list(SHAPES).index(name)
    cs = make_chunk(name, chunk_layout(name, "pieces"), seed=7000 + i)
    base = run(cs)
    again = [run(cs, sync=False) for _ in range(2)]
    torch.cuda.synchronize()
    for o in again:
        assert torch.equal(_bits(o), _bits(base)), "repeated launch differs"
    q0 = cs["q"].clone()
    q0[cs["T"]:] = 0
    assert torch.equal(_bits(run(cs, q=q0)), _bits(base)), "stale q rows change the output"
    if W == 0:
        assert torch.equal(_bits(run(cs, window=ctx)), _bits(base)), "window ctx_max != window 0"
    else:
        assert torch.equal(_bits(run(cs, window=ctx)), _bits(run(cs, window=0))), "window ctx_max != window 0"
    if hd == 128:
        scale = float(np.float32(1.0) / np.sqrt(np.float32(hd)))
        ref = torch.full_like(base, float("nan"))
        rc = _lib.lib.rr_op_prefill_attn_window(P(cs["q"]), P(cs["kp"]), P(cs["vp"]), P(ref), P(cs["start"]), P(cs["slot"]),
                                                P(cs["pos0"]), len(cs["seqs"]), cs["max_len"], nh, nkv, ctx, scale,
                                                P(cs["table"]), cs["pps"], cs["n_pages"], W, None)
        _lib.check(rc, "rr_op_prefill_attn_window")
        torch.cuda.synchronize()
        assert torch.equal(_bits(ref), _bits(base)), "head dim 128 differs from rr_op_prefill_attn_window"
    # one 600-row sequence cold, and as pieces at pos0 > 0 (multiples of 64 and not) in one chunk, each piece in its own
    # slot whose cache ends at the piece's last row
    n = min(600, ctx - 1)
    cuts = [0, 1, 100, 128, 229, 300, 511, n]
    pieces = [(b - a, a) for a, b in zip(cuts, cuts[1:])]
    both = make_chunk(name, [(n, 0)] + pieces, seed=9000 + i, src=[0] * (1 + len(pieces)))
    out = run(both).view(-1)[:both["out_len"]].view(both["T"], nh * hd)
    assert torch.equal(_bits(out[n:]), _bits(out[:n])), "pieces differ from the cold run"


# ------------------------------------------------------------------------------------------------ engines at new head dims
def _engine_spec(name):
    """2-layer models at head dims no model spec uses, hidden = n_heads x head_dim."""
    from rr_b200.models import ModelSpec
    nh, nkv, hd = {"hd64-g1": (8, 8, 64), "hd80-g2": (8, 4, 80), "hd112-g4": (8, 2, 112)}[name]
    return ModelSpec(name, 1024, nh * hd, 1024, 2, nh, nkv, hd, 10000.0, 1e-5)


ENGINE_SPECS = ("hd64-g1", "hd80-g2", "hd112-g4")


@pytest.mark.parametrize("name", ENGINE_SPECS)
def test_engine_at_new_head_dims_matches_oracle(name):
    """One prefill chunk of several prompts and 3 decode steps against oracle/llama_ref, as test_engine_matches_oracle
    runs the model specs."""
    from oracle import llama_ref
    from rr_b200.engine import Engine
    from rr_b200.models import make_weights
    from test_engine_gpu import _cmp
    spec = _engine_spec(name)
    w = make_weights(spec, seed=3, sigma=0.03, device="cuda", norm_jitter=0.1)
    eng = Engine(w, max_batch=8, ctx_max=640, max_prefill_tokens=2048, use_cuda_graph=False)
    try:
        g = torch.Generator().manual_seed(5)
        lens = [3, 64, 129, 300, 512]
        prompts = [torch.randint(0, spec.vocab, (n,), generator=g).tolist() for n in lens]
        slots = [7, 0, 5, 2, 3]
        first, logits = eng.prefill(prompts, slots, want_logits=True)
        worst = max(_cmp(logits[i], llama_ref.forward_logits(w, p)[-1], f"prefill {name} len={len(p)}")
                    for i, p in enumerate(prompts))
        toks = [list(p) for p in prompts]
        cur = [int(t) for t in first]
        for j in range(3):
            pos = [len(t) for t in toks]
            for t, c in zip(toks, cur):
                t.append(c)
            nxt, lg = eng.decode_step(slots, cur, pos, want_logits=True)
            for i in range(len(lens)):
                worst = max(worst, _cmp(lg[i], llama_ref.forward_logits(w, toks[i])[-1], f"decode {name} step {j} seq {i}"))
            cur = [int(t) for t in nxt]
        print(f"\n[{name}] worst rms(dlogit)/std = {worst:.4f}")
    finally:
        eng.close()


@pytest.mark.parametrize("name", ENGINE_SPECS)
def test_engine_at_new_head_dims_pieces_equal_one_chunk(name):
    """A 600-token prompt prefilled in pieces of 200 tokens (pos0 200 and 400: not multiples of 64) gives the tokens and
    logprobs of one chunk, bit for bit."""
    from rr_b200.engine import Engine
    from rr_b200.models import make_weights
    from test_long_prompts_gpu import _run
    spec = _engine_spec(name)
    w = make_weights(spec, seed=11, sigma=0.05, device="cuda")
    p = np.random.RandomState(600).randint(3, spec.vocab, size=600).tolist()
    out = []
    for T in (1024, 200):
        eng = Engine(w, max_batch=2, ctx_max=1024, max_prefill_tokens=T, use_cuda_graph=True)
        try:
            out.append(_run(eng, [(p, 4, dict(top_logprobs=5))]))
            assert eng.stats()["prefill_chunks"] == -(-600 // T)
        finally:
            eng.close()
    assert out[0] == out[1]
