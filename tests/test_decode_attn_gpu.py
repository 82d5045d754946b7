"""Kernel-level parity of decode attention (decode_attn_mma_kernel + decode_attn_combine_kernel, csrc/rr_attn_decode.cu)
through rr_op_decode_attn_qkv, which runs it exactly as the engine does: RoPE and the KV append fused in, q / k / v summed
from the QKV GEMM's fp32 split-K planes, the engine's scale, kv-split rule and RoPE table.

Operands.  Every q, k and v plane is N(0, 1 / n_splits), so their sums are N(0, 1).  Cache rows before `pos` of a row's
slot are bf16 N(0, 1); every other cache row, row `pos` itself, and the padding columns [head_dim, 128) of every row hold
finite poison of magnitude 1e3..1e4 (finite: a masked token reaches the PV mma with p = 0, and 0 * NaN would be NaN).
Slots are a permutation with slot != row, a few rows are inactive, and `out` is NaN-filled with slack past its end.
References are fp64.

Appends.  v = bf16 of the fp32 sum ((0 + p0) + p1) + ... in plane order (the kernel's order), bit for bit.  k = bf16 of the
fp32 rotation of that sum with the engine's table (inv_freq = theta^(-i / (head_dim / 2)) in double, angle
float(pos) * float(inv_freq) in fp32, cos / sin in double, stored as fp32).  The fp32 rotation lo * c - hi * s (or an FMA
form of it) is within eps = 2^-23 (|lo c| + |hi s|) of the exact value y; that error is relative to the operands, not to
y, because the subtraction can cancel.  The cached k must be the bf16 rounding of some value within eps of y: exact
unless a bf16 rounding midpoint lies within eps of y, where either neighbour passes.

Attention output.  Reference: q = bf16 of the fp64 rotated q, K and V as the kernel left them in the cache (rows <= pos),
w_j = p_j / sum p, O = sum w_j v_j, all fp64.  Error model of the kernel's output before its bf16 rounding, per element d:
  * T1, bf16 rounding of p before the PV mma while l sums the fp32 p: sum_j eps_j w_j v_jd, |eps_j| <= 2^-8.  With
    independent signs and sigma = 2^-9 per rounding (the relative error of a bf16 rounding spread over a binade has
    standard deviation 2^-9.3), lambda = 6 standard deviations give lambda 2^-9 sqrt(sum_j w_j^2 v_jd^2); the worst case
    2^-8 sum_j w_j |v_jd| is used where it is smaller (short contexts).  Tokens that become the running maximum of their
    warp (16 of every 64 tokens) within their kv split when their tile arrives are left out: their p is exp2f(0) = 1.
  * T2, relative error mu_j of each fp32 p_j, which enters O as sum_j mu_j w_j |v_jd - O_d|:
    - the fp32 accumulation of S = q . k on the tensor core (which may align and truncate each k16 group): 2^-18 scale
      sum_d |q_d k_jd|;
    - the scale, log2(e) and max subtractions (2^-21 (|s_j| + |s_max|)) and exp2f (2^-21);
    - q elements whose bf16 rounding is ambiguous as for k above: the kernel may hold the other neighbour, which moves
      s_j by up to scale sum_(ambiguous d') spacing_d' |k_jd'|.
  * T3, fp32 accumulation of o and l: one mma per tile and warp whose 16 products and running sum may each be truncated,
    the per-tile rescale, the 4-warp merge, the split combine and 1 / l: (24 T + 40) 2^-23 sum_j w_j |v_jd|, with T the
    tiles per split.
  * the bf16 rounding of the output: half the bf16 spacing at |O| + T1 + T2 + T3.
The bound tells the reference apart from three close neighbours, on rows with 1 <= pos and ctx <= 128: dropping token
`pos` moves it by at least 3 bounds somewhere in every such row; leaving the new key unrotated, or rotating it at pos - 1,
by at least 3 bounds somewhere in the case.  In every case the median bound is at most a tenth of 2e-2 (1 + |ref|), the
tolerance test_ops_gpu.py::test_decode_attention uses for the unfused path.  At short contexts one token's bf16 p rounding
is legitimately up to 2^-8 |v| and no bound can be that tight there."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

RR_INVALID_ARGUMENT = 4
DEV = "cuda"
LAMBDA = 6.0
U23 = 2.0 ** -23

# name -> (n_heads, n_kv_heads, head_dim, theta, ctx_max)
SHAPES = {
    "llama3-8b": (32, 8, 128, 5e5, 4096),
    "phi3-mini": (32, 32, 96, 1e4, 4096),
    "small96": (8, 2, 96, 1e4, 640),
    "tiny": (4, 2, 128, 5e5, 640),
    "g8": (16, 2, 128, 1e4, 1024),
    "hd64": (8, 8, 64, 1e4, 1024),
    "hd80": (8, 4, 80, 1e4, 640),
    "hd112": (8, 2, 112, 1e4, 4096),
}
KV_SPLITS = (1, 2, 4, 8)
# QKV plane counts: shape i, kv-split index k runs PLANE_COUNTS[(i + k) % 5], so every shape sees four of them and every
# G sees a count that leaves the kernel's last plane batch (4, 3 or 2 planes for G <= 2, 4, 8) partly empty.
PLANE_COUNTS = (1, 2, 3, 5, 8)
POSITIONS = (0, 1, 47, 48, 63, 64, 100, 127, 128, 175, 191, 511, 1000, 2000)   # and ctx_max - 1
CASES = [pytest.param(n, ks, None, id=f"{n}-ks{ks}") for n in SHAPES for ks in KV_SPLITS]
CASES.append(pytest.param("tiny", 1, 256, id="tiny-ks1-rows256"))               # the engine's largest batch


def kv_splits_rule(rows, n_kv_heads, sms):
    """The engine's rule (pick_kv_splits): double from 1 while the grid holds fewer than two CTAs per SM, up to 8."""
    ks = 1
    while rows * n_kv_heads * ks < 2 * sms and ks < 8:
        ks *= 2
    return ks


def rows_for(ks, n_kv_heads, sms):
    """A batch the rule gives `ks` for, at the edge of its range: the smallest for ks = 1, the largest otherwise."""
    rows = [r for r in range(1, 257) if kv_splits_rule(r, n_kv_heads, sms) == ks]
    if not rows:
        return None
    return rows[0] if ks == 1 else rows[-1]


def rope_table(pos, theta, head_dim):
    """(cos, sin) [len(pos), head_dim / 2] as fp64 holding the fp32 values launch_rope_table stores."""
    half = head_dim // 2
    i = torch.arange(half, dtype=torch.float64, device=pos.device)
    inv_freq = torch.full_like(i, float(torch.tensor(theta, dtype=torch.float32))) ** (-i / half)
    ang = pos.float()[:, None] * inv_freq.float()[None, :]
    return torch.cos(ang.double()).float().double(), torch.sin(ang.double()).float().double()


def rotate(x, c, s):
    """fp64 rotate_half RoPE of x [.., head_dim] with per-pair cos / sin [.., head_dim / 2]; also returns eps, the fp32
    error bound of each rotated element relative to its operands."""
    half = x.shape[-1] // 2
    lo, hi = x[..., :half].double(), x[..., half:].double()
    y = torch.cat([lo * c - hi * s, hi * c + lo * s], -1)
    eps = U23 * (1 + 2.0 ** -20) * torch.cat([(lo * c).abs() + (hi * s).abs(), (hi * c).abs() + (lo * s).abs()], -1)
    return y, eps


def bf16_edges(b):
    """The interval of reals that round to each (finite, nonzero) bf16 value of b."""
    bits = b.contiguous().view(torch.int16).int()
    x = b.double()
    e1 = (x + (bits + 1).to(torch.int16).view(torch.bfloat16).double()) / 2
    e2 = (x + (bits - 1).to(torch.int16).view(torch.bfloat16).double()) / 2
    return torch.minimum(e1, e2), torch.maximum(e1, e2)


def rounding_check(b, y, eps):
    """(ok, ambiguous): ok where b is the bf16 rounding of some value within eps of y; ambiguous where that needed the
    stated fp32 slack (y itself does not round to b)."""
    lo, hi = bf16_edges(b)
    ok = torch.maximum(lo, y - eps) <= torch.minimum(hi, y + eps)
    return ok, ok & ((y < lo) | (y > hi))


def attention(q, k, v, scale):
    """fp64 attention of q [nkv, G, hd] over k, v [nkv, n, hd]: (O [nkv, G, hd], s [nkv, G, n], w = softmax weights)."""
    s = scale * (q @ k.transpose(1, 2))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    w = p / p.sum(-1, keepdim=True)
    return w @ v, s, w


def exact_p_tokens(s, kv_splits):
    """Mask [.., n] of the tokens whose p the kernel computes as exactly 1 (bf16-exact): those that become the running
    maximum of their warp (16 of every 64 tokens) within their kv split when their tile arrives."""
    n = s.shape[-1]
    n_tiles = -(-n // 64)
    tp = -(-n_tiles // kv_splits)
    ns = -(-n_tiles // tp)
    sp = torch.nn.functional.pad(s, (0, ns * tp * 64 - n), value=-math.inf).view(*s.shape[:-1], ns, tp, 4, 16)
    cm, ca = sp.max(-1)                                              # max of each (split, tile, warp) chunk
    before = torch.cat([torch.full_like(cm[..., :1, :], -math.inf), cm.cummax(-2).values[..., :-1, :]], -2)
    rec = (cm >= before) & (cm > -math.inf)
    first = (torch.arange(ns * tp, device=s.device).view(ns, tp, 1) * 64 + 16 * torch.arange(4, device=s.device))
    idx = torch.where(rec, first + ca, ns * tp * 64)                 # non-records go to a spare slot
    mask = torch.zeros(*s.shape[:-1], ns * tp * 64 + 1, dtype=torch.bool, device=s.device)
    mask.scatter_(-1, idx.flatten(-3), True)
    return mask[..., :n]


def attention_bound(q, dq, k, v, scale, kv_splits):
    """(O, bound) per element, the error model of the module docstring; dq = spacing of ambiguous q elements, else 0."""
    o, s, w = attention(q, k, v, scale)
    va = v.abs()
    tiles = -(-((k.shape[1] + 63) // 64) // kv_splits)               # tiles per split
    wx = w.masked_fill(exact_p_tokens(s, kv_splits), 0.0)
    t1 = torch.minimum(LAMBDA * 2.0 ** -9 * ((wx * wx) @ (v * v)).sqrt(), 2.0 ** -8 * (wx @ va))
    mu = (2.0 ** -18 * scale * (q.abs() @ k.abs().transpose(1, 2)) + 2.0 ** -21 * (s.abs() + s.amax(-1, keepdim=True).abs())
          + 2.0 ** -21 + 1.01 * scale * (dq @ k.abs().transpose(1, 2)))
    wm = w * mu
    t2 = wm @ va + wm.sum(-1, keepdim=True) * o.abs()                 # sum_j mu_j w_j (|v_jd| + |O_d|)
    t3 = (24 * tiles + 40) * U23 * (w @ va)
    e = t1 + t2 + t3
    return o, e + half_spacing_bf16(o.abs() + e)


def half_spacing_bf16(m):
    """Half the bf16 spacing at magnitude m: the largest round-to-nearest error of a value of magnitude <= m."""
    return torch.ldexp(torch.ones_like(m), torch.frexp(m).exponent - 9)


def make_case(name, rows, n_splits, seed):
    """Seeded planes, caches, slots and positions of one case, on the GPU."""
    nh, nkv, hd, theta, ctx_max = SHAPES[name]
    dev = DEV
    g = torch.Generator(device=dev).manual_seed(seed)
    nqkv = (nh + 2 * nkv) * hd
    ld = nqkv + 6
    planes = torch.randn(n_splits, rows + 1, ld, device=dev, generator=g) / math.sqrt(n_splits)
    planes[:, :, nqkv:] = float("nan")                              # columns and the row past the operands: never read
    planes[:, rows] = float("nan")
    n_slots = rows + 3
    perm = torch.randperm(n_slots, device=dev, generator=g).tolist()
    for r in range(n_slots):                                         # no row keeps its own index as slot
        if perm[r] == r:
            j = (r + 1) % n_slots
            perm[r], perm[j] = perm[j], perm[r]
    slot = perm[:rows]
    active = [r for r in range(rows) if r % 6 != 4]
    for r in range(rows):
        if r % 6 == 4:
            slot[r] = -1
    plist = [p for p in POSITIONS if p < ctx_max] + [ctx_max - 1]
    pos = [0] * rows
    for j, r in enumerate(active):
        if len(active) >= len(plist):
            pos[r] = plist[j % len(plist)]
        elif len(active) == 1:
            pos[r] = plist[-1]
        else:                                                        # few rows: spread over the list, both ends included
            pos[r] = plist[round(j * (len(plist) - 1) / (len(active) - 1))]

    def cache():
        sign = torch.randint(0, 2, (n_slots, nkv, ctx_max, 128), device=dev, generator=g, dtype=torch.int8).float() * 2 - 1
        c = (sign * (1e3 + 9e3 * torch.rand(n_slots, nkv, ctx_max, 128, device=dev, generator=g))).bfloat16()
        for r in active:
            c[slot[r], :, :pos[r], :hd] = torch.randn(nkv, pos[r], hd, device=dev, generator=g).bfloat16()
        return c

    kc, vc = cache(), cache()
    return dict(name=name, shape=SHAPES[name], rows=rows, n_splits=n_splits, ld=ld, planes=planes, kc=kc, vc=vc,
                n_slots=n_slots, slot=torch.tensor(slot, device=dev, dtype=torch.int32), pos=torch.tensor(pos, device=dev, dtype=torch.int32),
                active=active, out_len=rows * nh * hd, slack=nh * hd + 64)


def run(cs, kc, vc, sync=True):
    """One call on caches kc / vc (modified in place); returns (out_flat, kv_splits)."""
    from rr_b200 import _lib
    nh, nkv, hd, theta, ctx_max = SHAPES[cs["name"]]
    out = torch.full((cs["out_len"] + cs["slack"],), float("nan"), device=DEV, dtype=torch.bfloat16)
    ks = C.c_int32(-1)
    p = cs["planes"]
    rc = _lib.lib.rr_op_decode_attn_qkv(p.data_ptr(), cs["n_splits"], p.stride(0), cs["ld"], kc.data_ptr(), vc.data_ptr(),
                                        out.data_ptr(), cs["slot"].data_ptr(), cs["pos"].data_ptr(), cs["rows"], nh, nkv, hd,
                                        ctx_max, cs["n_slots"], theta, C.byref(ks), None)
    _lib.check(rc, "rr_op_decode_attn_qkv")
    if sync:
        torch.cuda.synchronize()
    return out, ks.value


def plane_sums(cs):
    """fp32 sums of the planes in the kernel's order: ((0 + p0) + p1) + ..."""
    rows = cs["rows"]
    acc = torch.zeros_like(cs["planes"][0, :rows])
    for z in range(cs["n_splits"]):
        acc = acc + cs["planes"][z, :rows]
    return acc


def check_appends(cs, k_new, v_new):
    """The rows a call appended at each active row's pos, k_new / v_new [active rows, n_kv_heads, head_dim]: v bit-exact,
    k the bf16 rounding of the rotation up to the stated fp32 ambiguity; returns stats."""
    nh, nkv, hd, theta, _ = cs["shape"]
    act = torch.tensor(cs["active"], device=DEV)
    ps = cs["pos"][act].long()
    acc = plane_sums(cs)[act]
    ksum = acc[:, nh * hd:(nh + nkv) * hd].view(-1, nkv, hd)
    vsum = acc[:, (nh + nkv) * hd:(nh + 2 * nkv) * hd].view(-1, nkv, hd)
    c, s = rope_table(ps, theta, hd)
    assert torch.equal(v_new.contiguous().view(torch.int16), vsum.bfloat16().view(torch.int16)), "appended v differs"
    yk, ek = rotate(ksum, c[:, None, :], s[:, None, :])
    ok, amb = rounding_check(k_new, yk, ek)
    ok = torch.where(k_new == 0, yk.abs() <= ek, ok)                 # bf16_edges takes nonzero values only
    bad = (~ok).nonzero()
    assert bad.numel() == 0, f"appended k: {bad.shape[0]} elements off, first (row, kv head, dim) {bad[0].tolist()}"
    return {"k_ambiguous": int(amb.sum())}


def check_output(cs, kv_splits, out_flat, slot_kv):
    """Attention output of one call against the fp64 reference and its bound, with slot_kv(slot, n) -> (k, v), the first n
    cache rows of a slot after the call as [n_kv_heads, n, head_dim]; returns stats."""
    nh, nkv, hd, theta, _ = cs["shape"]
    G, rows = nh // nkv, cs["rows"]
    scale = 1.0 / math.sqrt(hd)
    act = torch.tensor(cs["active"], device=DEV)
    sl, ps = cs["slot"][act].long(), cs["pos"][act].long()
    acc = plane_sums(cs)[act]
    qsum = acc[:, : nh * hd].view(-1, nh, hd)
    ksum = acc[:, nh * hd:(nh + nkv) * hd].view(-1, nkv, hd)
    c, s = rope_table(ps, theta, hd)
    c, s = c[:, None, :], s[:, None, :]
    stats = {}
    out = out_flat[: cs["out_len"]].view(rows, nh, hd)
    inactive = [r for r in range(rows) if r not in set(cs["active"])]
    assert torch.isnan(out[inactive]).all(), "inactive rows written"
    assert torch.isnan(out_flat[cs["out_len"]:]).all(), "out written past rows x n_heads x head_dim"
    assert torch.isfinite(out[act]).all(), "active output not finite"

    # ---- attention output per active row
    yq, eq = rotate(qsum, c, s)
    q_ref = yq.bfloat16()
    lo, hi = bf16_edges(q_ref)
    q_amb = (yq - eq < lo) | (yq + eq > hi)
    dq = torch.where(q_amb, 2 * torch.maximum(hi - q_ref.double(), q_ref.double() - lo), torch.zeros_like(yq))
    stats["q_ambiguous"] = int(q_amb.sum())
    worst, worst_at, shifts = 0.0, None, {}
    bounds, olds = [], []
    for j, r in enumerate(cs["active"]):
        p_r, s_r = int(ps[j]), int(sl[j])
        n = p_r + 1
        k, v = (t.double() for t in slot_kv(s_r, n))
        qj = q_ref[j].double().view(nkv, G, hd)
        dqj = dq[j].view(nkv, G, hd)
        o_ref, bound = attention_bound(qj, dqj, k, v, scale, kv_splits)
        got = out[r].double().view(nkv, G, hd)
        ratio = ((got - o_ref).abs() / bound).max().item()
        if ratio > worst:
            worst, worst_at = ratio, (r, p_r)
        assert ratio <= 1.0, f"row {r} (pos {p_r}): worst |out - ref| / bound = {ratio:.3g}"
        bounds.append(bound.flatten())
        olds.append(2e-2 * (1 + o_ref.abs().flatten()))
        if p_r == 0:                                                  # p = 1, l = 1: out is the appended v row
            want = v[:, 0].bfloat16().repeat_interleave(G, 0)
            assert torch.equal(out[r].view(torch.int16), want.contiguous().view(torch.int16)), f"row {r}: pos 0 != v"
        if 1 <= p_r and n <= 128:                                    # the bound tells close neighbours apart
            c1, s1 = rope_table(ps[j:j + 1] - 1, theta, hd)
            alts = {"token pos dropped": (k[:, :-1], v[:, :-1])}
            for what, kp in (("new key unrotated", ksum[j]), ("new key rotated at pos - 1", rotate(ksum[j], c1, s1)[0])):
                k2 = k.clone()
                k2[:, -1] = kp.bfloat16().double()
                alts[what] = (k2, v)
            for what, (ka, vb) in alts.items():
                shift = ((attention(qj, ka, vb, scale)[0] - o_ref).abs() / bound).max().item()
                shifts.setdefault(what, []).append(shift)
                if what == "token pos dropped":
                    assert shift >= 3, f"row {r} (pos {p_r}): {what} moves the reference by only {shift:.3g} bounds"
        del k, v
    # A one-step RoPE error moves the new key only in its high-frequency pairs, and the unrotated key may lie close to
    # the rotated one; where the new token's weight is small in every head of a row, no bound that admits the kernel's
    # bf16 rounding of p separates those two by 3 in that row.  Each still fails the case by at least 3 bounds.
    for what, sh in shifts.items():
        assert max(sh) >= 3, f"{what} moves the reference by at most {max(sh):.3g} bounds in every row"
    bounds, olds = torch.cat(bounds), torch.cat(olds)
    stats.update(out_worst=worst, out_worst_at=worst_at, shifts={w: (min(sh), max(sh)) for w, sh in shifts.items()},
                 median_bound=bounds.median().item(),
                 median_bound_vs_old=(bounds / olds).median().item())
    return stats


def check_case(cs, kv_splits, kc0, vc0, kc, vc, out_flat):
    """Appends, untouched bytes and attention output of one call on slot-contiguous caches (before: kc0 / vc0, after:
    kc / vc); returns the worst ratios seen."""
    hd = cs["shape"][2]
    act = torch.tensor(cs["active"], device=DEV)
    sl, ps = cs["slot"][act].long(), cs["pos"][act].long()
    stats = check_appends(cs, kc[sl, :, ps, :hd], vc[sl, :, ps, :hd])
    # ---- nothing else written
    for name, before, after in (("k", kc0, kc), ("v", vc0, vc)):
        fixed = after.clone()
        fixed[sl, :, ps, :hd] = before[sl, :, ps, :hd]
        assert torch.equal(fixed.view(torch.int16), before.view(torch.int16)), f"{name} cache written outside row pos"
        del fixed
    stats.update(check_output(cs, kv_splits, out_flat, lambda s, n: (kc[s, :, :n, :hd], vc[s, :, :n, :hd])))
    rel = stats["median_bound_vs_old"]
    assert rel <= 0.1, f"median bound is {rel:.3g} of the unfused test's 2e-2 (1 + |ref|)"
    return stats


def case_setup(name, ks, rows):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nkv = SHAPES[name][1]
    if rows is None:
        rows = rows_for(ks, nkv, sms)
        if rows is None:
            pytest.skip(f"kv_splits {ks} unreachable for {nkv} kv heads on {sms} SMs")
    assert kv_splits_rule(rows, nkv, sms) == ks
    i = list(SHAPES).index(name)
    n_splits = PLANE_COUNTS[(i + KV_SPLITS.index(ks)) % len(PLANE_COUNTS)]
    return make_case(name, rows, n_splits, seed=1000 * i + 10 * ks + rows), ks


@pytest.fixture
def default_path(monkeypatch):
    """The engine's default: the last tile of a row is loaded as 16-row boxes."""
    monkeypatch.delenv("RR_ATTN_NO_TRIM", raising=False)
    return monkeypatch


@pytest.mark.parametrize("name,ks,rows", CASES)
def test_decode_attn_appends_and_output_match_fp64(name, ks, rows, default_path):
    cs, ks_want = case_setup(name, ks, rows)
    kc, vc = cs["kc"].clone(), cs["vc"].clone()
    out, ks_got = run(cs, kc, vc)
    assert ks_got == ks_want
    check_case(cs, ks_got, cs["kc"], cs["vc"], kc, vc, out)


@pytest.mark.parametrize("name,ks,rows", CASES)
def test_decode_attn_is_bit_identical_across_repeats_and_tail_loads(name, ks, rows, default_path):
    """Two calls back to back on one stream (host sync after both), and whole last tiles (RR_ATTN_NO_TRIM=1) against
    16-row boxes: masked rows contribute exactly 0, so outputs and caches agree to the bit."""
    cs, _ = case_setup(name, ks, rows)
    base_k, base_v = cs["kc"].clone(), cs["vc"].clone()
    base_out, _ = run(cs, base_k, base_v)

    def same(out, kc, vc, what):
        assert torch.equal(out.view(torch.int16), base_out.view(torch.int16)), f"out differs: {what}"
        assert torch.equal(kc.view(torch.int16), base_k.view(torch.int16)), f"k cache differs: {what}"
        assert torch.equal(vc.view(torch.int16), base_v.view(torch.int16)), f"v cache differs: {what}"

    calls = []
    for _ in range(2):
        kc, vc = cs["kc"].clone(), cs["vc"].clone()
        calls.append((run(cs, kc, vc, sync=False)[0], kc, vc))
    torch.cuda.synchronize()
    for i, (out, kc, vc) in enumerate(calls):
        same(out, kc, vc, f"back-to-back call {i}")
    del calls
    default_path.setenv("RR_ATTN_NO_TRIM", "1")
    kc, vc = cs["kc"].clone(), cs["vc"].clone()
    same(run(cs, kc, vc)[0], kc, vc, "whole last tiles")


def _reject_args():
    """Valid arguments of a small shape, with buffers large enough for every rejected variant below."""
    nh, nkv, hd, ctx_max, rows, n_slots, n_splits, ld = 8, 2, 128, 128, 4, 4, 2, 4096
    planes = torch.randn(n_splits, rows, ld, device=DEV)
    kc = torch.randn(n_slots, 4, ctx_max, 128, device=DEV).bfloat16()
    vc = torch.randn(n_slots, 4, ctx_max, 128, device=DEV).bfloat16()
    out = torch.full((rows * 32 * 144,), float("nan"), device=DEV, dtype=torch.bfloat16)
    slot = torch.tensor([1, 0, 3, 2], device=DEV, dtype=torch.int32)
    pos = torch.tensor([0, 5, 63, 100], device=DEV, dtype=torch.int32)
    bufs = dict(qkv=planes, k_cache=kc, v_cache=vc, out=out, slot=slot, pos=pos)
    args = dict(n_splits=n_splits, split_stride=rows * ld, ld=ld, rows=rows, n_heads=nh, n_kv_heads=nkv, head_dim=hd,
                ctx_max=ctx_max, n_slots=n_slots, theta=1e4)
    return bufs, args


REJECT = [
    *[pytest.param({b: None}, id=f"null-{b}") for b in ("qkv", "k_cache", "v_cache", "out", "slot", "pos", "kv_splits")],
    pytest.param({"rows": 0}, id="rows0"),
    pytest.param({"n_slots": 0}, id="n_slots0"),
    pytest.param({"n_heads": 12, "n_kv_heads": 4}, id="G3"),
    pytest.param({"n_heads": 6, "n_kv_heads": 4}, id="G-not-integer"),
    pytest.param({"n_heads": 32, "n_kv_heads": 2}, id="G16"),
    pytest.param({"n_kv_heads": 0}, id="n_kv_heads0"),
    pytest.param({"head_dim": 48}, id="head_dim48"),
    pytest.param({"head_dim": 144}, id="head_dim144"),
    pytest.param({"head_dim": 72}, id="head_dim72"),
    pytest.param({"ctx_max": 0}, id="ctx_max0"),
    pytest.param({"ctx_max": 96}, id="ctx_max96"),
    pytest.param({"n_splits": 0}, id="n_splits0"),
    pytest.param({"ld": (8 + 4) * 128 - 2}, id="ld-short"),
    pytest.param({"ld": 4095}, id="ld-odd"),
    pytest.param({"split_stride": 4 * 4096 + 1}, id="split_stride-odd"),
]


@pytest.mark.parametrize("change", REJECT)
def test_decode_attn_rejects_what_the_engine_does_not_run(change, default_path):
    """Rejected before any launch: every buffer stays untouched and *kv_splits keeps its value."""
    from rr_b200 import _lib
    bufs, args = _reject_args()
    before = {k: t.clone() for k, t in bufs.items()}
    ptr = {k: t.data_ptr() for k, t in bufs.items()}
    ks = C.c_int32(-1)
    ks_ptr = C.byref(ks)
    for k, v in change.items():
        if k == "kv_splits":
            ks_ptr = None
        elif k in ptr:
            ptr[k] = v
        else:
            args[k] = v
    a = args
    rc = _lib.lib.rr_op_decode_attn_qkv(ptr["qkv"], a["n_splits"], a["split_stride"], a["ld"], ptr["k_cache"],
                                        ptr["v_cache"], ptr["out"], ptr["slot"], ptr["pos"], a["rows"], a["n_heads"],
                                        a["n_kv_heads"], a["head_dim"], a["ctx_max"], a["n_slots"], a["theta"], ks_ptr, None)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT
    assert ks.value == -1
    for k, t in bufs.items():
        assert torch.equal(t.view(torch.uint8), before[k].view(torch.uint8)), f"{k} touched"
