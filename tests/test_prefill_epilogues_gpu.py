"""Kernel-level parity of the prefill projections as the engine runs them (gemm_pf_wgmma epilogues, csrc/rr_gemm.cu;
add_rmsnorm_kernel and rope_kv_kernel, csrc/rr_elementwise.cu), through rr_op_add_rmsnorm_pf, rr_op_prefill_qkv and
rr_op_prefill_gemm: plans made for plan_rows rows and launched for the first T, the deferred-norm fields filled by the
engine's helpers, RoPE fused into the QKV epilogue at head_dim 128 and run by rope_kv_kernel from a bf16 qkv matrix
(with the engine's table) otherwise.

Operands.  An operand row t is xhat_t = bf16(s_t z), z ~ N(0, 1), s_t log-uniform in [0.3, 3]; every 7th row (row 0
included) has s_t^2 ~ eps, so eps moves its 1 / rms by 8 % or more.  Its partial sums of squares add up to
hidden s_t^2 (0.7 .. 1.4) and are split unequally (weights uniform in [0.25, 1.75]), so a kernel reading only partial 0,
or n_part - 1 of them, or another row's, gets another scale.  Weights are bf16 with sigma 1 / sqrt(fan-in).  Rows
T .. plan_rows of every operand and of rowss are NaN, output rows >= T are NaN, KV caches hold finite poison
(1e3 .. 1e4).  Tokens are ragged sequences as run_prefill lays them out: permuted slots, positions pos0 + t with
pos0 >= 1, the last sequence ending at ctx_max - 1.  References are fp64 of the operands the kernel read.

Error model (u = 2^-24, the fp32 unit roundoff).
  * Accumulation.  A bf16 x bf16 product is exact in fp32; the wgmma main loop rounds (or truncates) its running sum, at
    most one fp32 ulp per step, with independent signs; running sums are at most twice the largest |result| M_t of their
    row.  Eight standard deviations: e_acc = 16 * 2^-23 * sqrt(K) * M_t (test_decode_mlp_gpu.py uses the same model).
  * Deferred scale.  r = rsqrtf(fl(fl(sum_p rowss_p) * fl(1 / hidden)) + eps): the n_part - 1 additions of positive
    partials, the two roundings of the scaling and the one of + eps give a relative error of (n_part + 2) u in the
    argument, half of it in r; rsqrtf adds 2 ulp.  delta_r = 1.01 ((n_part + 2) / 2 + 4) u.
  * Consumer output before its bf16 rounding, v = fl(acc * r):  |v - y| <= E = e_acc r + |y| (delta_r + u), y the fp64
    reference (xhat . w) r_64.
      - BF16 mode: out = bf16(v).
      - SILU mode: act = bf16(fl(g / (1 + __expf(-g))) * u) from g, u as above.  |silu'| <= 1.1, so
        E_act = 1.1 |u| E_g + |silu(g)| E_u + E_g E_u + (8 + 1.2 |g|) 2^-23 |act| (__expf: 2 + 1.16 |g| ulp,
        __fdividef 2 ulp, the product 1).
      - QKV.  q and k are rotated in fp32, l c - h s and h c + l s with the table's fp32 (cos, sin): the pre-rotation
        errors propagate as |c| E_l + |s| E_h, and the rotation adds 1.01 * 2^-23 (|l c| + |h s|) (relative to the
        operands: the subtraction can cancel).  At head_dim != 128 the pre-rotation values were rounded to bf16 first
        (the qkv matrix rope_kv_kernel reads): E_l grows by half a bf16 spacing.
    The kernel's bf16 output b passes where it is the round-to-nearest-even of some value within the bound of the
    reference: the interval of reals that round to b meets [y - E, y + E].  gap(b, y) = distance from y to that interval
    over E; the check is gap <= 1.
  * Producer (RESID).  x = fl(x_in + acc): |x - y| <= e_acc + 1.01 u |y|.  A partial sum of 128 squares in the
    epilogue's fixed order: at most 12 roundings deep, all terms positive: |got - ref| <= 2^-20 ref.  xhat is checked bit
    for bit as bf16(x_kernel * gamma), one fp32 product rounded to nearest even.
  * Layer-0 norm.  rowss[r][0] = sum of hidden squares, each thread summing hidden / 256 float4 groups (4 roundings
    each) before the block reduction: |got - ref| <= (hidden / 64 + 16) u ref.  xn = bf16(x * w) bit for bit.
  * Deferred form vs the textbook RMSNorm (RMSNorm(x) gamma, then W): the operand is bf16(x gamma) instead of
    bf16(x r gamma), so against an unrounded fp64 operand each product carries one bf16 rounding, |delta| <= 2^-9, with
    independent signs.  With sigma = 2^-9 and lambda = 6 standard deviations:  T1 = 6 * 2^-9 r sqrt(sum_k (x_k gamma_k
    w_k)^2); the kernel's sum of squares adds (its own bound) / 2 to delta_r.

Close wrong answers each check must reject (the kernel's output sits >= 3 bounds from each somewhere in the case, the
gap computed against the wrong answer with the reference's bound): 1 / rms = 1 (norm skipped); 1 / rms from partial 0
only; from the first n_part - 1 partials; the neighbouring row's 1 / rms; eps dropped (on the rows where it matters);
RoPE at pos - 1; RoPE pairs (i, i + 1) instead of (i, i + hd / 2); at head_dim 96, a table built for head_dim 128; each
sum-of-squares partial over columns shifted by 64.  Each case also reports its median bound as a fraction of the
tolerance the older tests use for the same op (6e-3 max|ref| for the bf16 GEMM, 2e-2 (max|ref| + |ref|) for SiLU,
1e-3 max|ref| + 1e-4 |ref| for the residual add, 3e-2 + 1e-2 |ref| for RoPE) and asserts it is below a quarter."""
import ctypes as C
import math
import random

import pytest
import torch

from test_decode_attn_gpu import bf16_edges, half_spacing_bf16, rope_table
from test_gemm_gpu import _interleave64

pytestmark = pytest.mark.gpu

DEV = "cuda"
RR_INVALID_ARGUMENT = 4
MODE_BF16, MODE_SILU, MODE_RESID = 0, 3, 5
U = 2.0 ** -24
EPS = 1e-5
EPS32 = float(torch.tensor(EPS, dtype=torch.float32))
LAMBDA = 6.0
MARGIN = 3.0
PLAN_SLACK = 45                       # plan_rows = T + PLAN_SLACK

# name -> (hidden, n_heads, n_kv_heads, head_dim, inter, theta, ctx_max); None: that projection is not run for the shape
SHAPES = {
    "llama-3-8b": (4096, 32, 8, 128, 14336, 5e5, 4096),      # ROPE epilogue; the benchmarked shape
    "phi-3-mini": (3072, 32, 32, 96, 8192, 1e4, 4096),       # BF16 qkv + rope_kv with the table
    "tiny96": (384, 4, 4, 96, 1024, 1e4, 2048),               # 1.5 residual tiles: n_part = 3, partial 3 not written
    "odd-heads": (384, 3, 3, 128, None, 5e5, 2048),           # 9 heads: the last QKV tile holds one v head
    "hidden320": (320, None, None, None, 384, None, None),    # n_part = 3, the last partial covers 64 columns
    "hidden8192": (8192, None, None, None, None, None, None),  # norm only: add_rmsnorm_kernel<256, 8>, n_part = 64
}
TS = (1, 63, 64, 65, 127, 129, 300, 1000)
QKV_SHAPES = [n for n, s in SHAPES.items() if s[1]]
MLP_SHAPES = [n for n, s in SHAPES.items() if s[4]]
RESID_SHAPES = [n for n, s in SHAPES.items() if s[4] or s[1]]


def parts(hidden):
    """pf_norm_parts: one partial sum of squares per 128 columns."""
    return (hidden + 127) // 128


def lib():
    from rr_b200 import _lib
    return _lib


# ---------------------------------------------------------------- fp64 reference helpers (device-agnostic)
def edges(b):
    """Interval of reals that round to each bf16 value of b (zero included)."""
    lo, hi = bf16_edges(b)
    z = b.double() == 0
    tiny = 2.0 ** -134
    return torch.where(z, -tiny, lo), torch.where(z, tiny, hi)


def gap(b, y, e):
    """Distance from y to the rounding interval of b, in units of e (<= 1: b is the rounding of a value within e of y)."""
    lo, hi = edges(b)
    return torch.clamp(torch.maximum(lo - y, y - hi), min=0.0) / e


def delta_r(n_part):
    return 1.01 * ((n_part + 2) / 2 + 4) * U


def rinv64(rowss, hidden):
    """fp64 1 / rms from the partial sums the kernel read."""
    return (rowss.double().sum(-1) / hidden + EPS32) ** -0.5


def e_acc(y0, K):
    """Accumulation bound of each row of an fp64 product y0 [T, N] over K."""
    return 16 * 2.0 ** -23 * math.sqrt(K) * y0.abs().amax(-1, keepdim=True)


def consumer_ref(a64, w64, r, n_part, extra=None):
    """(y0, y, E): the unscaled product, the scaled reference and the bound of fl(acc * r) (extra: T1 of the textbook
    comparison and a relative term for the sum of squares)."""
    y0 = a64 @ w64.t()
    y = y0 * r[:, None]
    ea = e_acc(y0, a64.shape[1])
    rel = delta_r(n_part) + U
    if extra is not None:
        t1, rel_ss = extra
        ea = ea + t1
        rel = rel + rel_ss
    return y0, y, 1.01 * (ea * r[:, None] + y.abs() * rel)


def silu_ref(g, u, eg, eu):
    act = g * u / (1.0 + torch.exp(-g))
    sg = g / (1.0 + torch.exp(-g))
    e = 1.1 * u.abs() * eg + sg.abs() * eu + eg * eu + (8 + 1.2 * g.abs()) * 2.0 ** -23 * act.abs()
    return act, 1.01 * e


def rot(x, c, s):
    """rotate_half RoPE of x [.., hd] with per-pair (cos, sin) [.., hd / 2]."""
    h = x.shape[-1] // 2
    lo, hi = x[..., :h], x[..., h:]
    return torch.cat([lo * c - hi * s, hi * c + lo * s], -1)


def rot_bound(x, e, c, s):
    h = x.shape[-1] // 2
    lo, hi, el, eh = x[..., :h], x[..., h:], e[..., :h], e[..., h:]
    ca, sa = c.abs(), s.abs()
    prop = torch.cat([ca * el + sa * eh, ca * eh + sa * el], -1)
    fp = 1.01 * 2.0 ** -23 * torch.cat([(lo * c).abs() + (hi * s).abs(), (hi * c).abs() + (lo * s).abs()], -1)
    return 1.01 * (prop + fp + (e + x.abs()) * 2.0 ** -40)


def rot_pairs_adjacent(x, c, s):
    """The wrong pairing: (2j, 2j + 1) rotated with frequency j."""
    xe, xo = x[..., 0::2], x[..., 1::2]
    return torch.stack([xe * c - xo * s, xo * c + xe * s], -1).flatten(-2)


def rows_deferred(n, hidden, g):
    """Operand rows xhat [n, hidden] bf16 and their partial sums rowss [n, n_part] fp32 (module docstring)."""
    s = torch.empty(n, device=g.device, dtype=torch.float64).uniform_(math.log(0.3), math.log(3.0), generator=g).exp()
    small = torch.arange(n, device=g.device) % 7 == 0
    s_small = math.sqrt(EPS) * torch.empty(n, device=g.device, dtype=torch.float64).uniform_(0.5, 2.0, generator=g)
    s = torch.where(small, s_small, s)
    xhat = (torch.randn(n, hidden, device=g.device, generator=g, dtype=torch.float64) * s[:, None]).bfloat16()
    total = hidden * s * s * torch.empty(n, device=g.device, dtype=torch.float64).uniform_(0.7, 1.4, generator=g)
    w = torch.empty(n, parts(hidden), device=g.device, dtype=torch.float64).uniform_(0.25, 1.75, generator=g)
    rowss = (total[:, None] * w / w.sum(1, keepdim=True)).float()
    return xhat, rowss, small


def wrong_scales(rowss, hidden, small):
    """Close wrong 1 / rms per row: name -> (r', rows it applies to)."""
    n = rowss.shape[0]
    r = rinv64(rowss, hidden)
    ss = rowss.double()
    alts = {"rinv = 1": (torch.ones_like(r), None),
            "rinv from partial 0": ((ss[:, 0] / hidden + EPS32) ** -0.5, None),
            "eps dropped": ((ss.sum(1) / hidden) ** -0.5, small)}
    if ss.shape[1] > 1:
        alts["rinv from n_part - 1 partials"] = ((ss[:, :-1].sum(1) / hidden + EPS32) ** -0.5, None)
    if n > 1:
        nb = torch.cat([r[1:], r[-2:-1]])
        alts["neighbouring row's rinv"] = (nb, None)
    return alts


def margin(b, y_alt, e, rows=None):
    """Largest gap of the kernel's output b from a wrong answer y_alt, over the given rows."""
    gp = gap(b, y_alt, e)
    if rows is not None:
        gp = gp[rows]
    return gp.max().item() if gp.numel() else float("inf")


def report(name, T, what, stats):
    print(f"STATS {name} T={T} {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                                      for k, v in stats.items()))


# ---------------------------------------------------------------- operands and calls
_OPS = {}


def operands(name):
    """Seeded weights of one shape (the last shape is cached; cases run shape by shape)."""
    if name not in _OPS:
        _OPS.clear()
        hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
        g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
        op = dict(gamma=(1 + 0.1 * torch.randn(hidden, device=DEV, generator=g)).bfloat16())

        def w(n, k):
            return (torch.randn(n, k, device=DEV, generator=g) / math.sqrt(k)).bfloat16()
        if H:
            op["wqkv"] = w((H + 2 * KV) * hd, hidden)
            op["wqkv64"] = op["wqkv"].double()
            # K cache slots 0..6, V cache slots 7..13 (tokens() uses at most 7 slots)
            sign = torch.randint(0, 2, (14, KV, ctx, 128), device=DEV, generator=g, dtype=torch.int8).float() * 2 - 1
            op["poison"] = (sign * (1e3 + 9e3 * torch.rand(sign.shape, device=DEV, generator=g))).bfloat16()
        if inter:
            op["wgu"] = w(2 * inter, hidden)
            op["wgu_il"] = _interleave64(op["wgu"], inter)
            op["wgu64"] = op["wgu"].double()
        K = inter or (H * hd if H else None)
        if K:
            op["wres"] = w(hidden, K)
            op["wres64"] = op["wres"].double()
        op["K_res"] = K
        _OPS[name] = op
    return _OPS[name]


def tokens(T, ctx_max, seed):
    """(slot [T], pos [T], n_slots): ragged sequences, permuted slots, pos0 >= 1, the last one ending at ctx_max - 1."""
    rnd = random.Random(seed)
    n_seqs = min(T, 5)
    cuts = sorted(rnd.sample(range(1, T), n_seqs - 1)) if n_seqs > 1 else []
    bounds = [0] + cuts + [T]
    n_slots = n_seqs + 2
    perm = list(range(n_slots))
    rnd.shuffle(perm)
    slot, pos = [], []
    for i in range(n_seqs):
        L = bounds[i + 1] - bounds[i]
        p0 = ctx_max - L if i == n_seqs - 1 else rnd.randint(1, ctx_max - L)
        slot += [perm[i]] * L
        pos += list(range(p0, p0 + L))
    return (torch.tensor(slot, device=DEV, dtype=torch.int32), torch.tensor(pos, device=DEV, dtype=torch.int32), n_slots)


def nan_rows(t, T):
    t[T:] = float("nan")
    return t


def call_norm(x, w, xn, rowss, T, hidden):
    L = lib()
    rc = L.lib.rr_op_add_rmsnorm_pf(x.data_ptr(), w.data_ptr(), xn.data_ptr(), T, hidden, EPS, rowss.data_ptr(),
                                    parts(hidden), None)
    L.check(rc, "rr_op_add_rmsnorm_pf")


def call_qkv(name, xhat, rowss, T, slot, pos, q_out, kc, vc):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    L = lib()
    fused = C.c_int32(-1)
    rc = L.lib.rr_op_prefill_qkv(xhat.data_ptr(), rowss.data_ptr(), xhat.shape[0], T, hidden,
                                 operands(name)["wqkv"].data_ptr(), H, KV, hd, ctx, theta, EPS, slot.data_ptr(),
                                 pos.data_ptr(), q_out.data_ptr(), kc.data_ptr(), vc.data_ptr(), C.byref(fused), None)
    L.check(rc, "rr_op_prefill_qkv")
    return fused.value


def call_gemm(A, T, W, out, ldo, mode, rowss=None, hidden=0, gamma=None, xhat=None, rowss_out=None):
    L = lib()
    n_part = parts(hidden) if rowss is not None else 0
    rc = L.lib.rr_op_prefill_gemm(A.data_ptr(), A.shape[0], T, A.stride(0), W.data_ptr(), W.shape[0], A.shape[1],
                                  out.data_ptr(), ldo, mode, rowss.data_ptr() if rowss is not None else None, n_part,
                                  hidden, EPS, gamma.data_ptr() if gamma is not None else None,
                                  xhat.data_ptr() if xhat is not None else None,
                                  rowss_out.data_ptr() if rowss_out is not None else None,
                                  parts(W.shape[0]) if xhat is not None else 0, None)
    L.check(rc, "rr_op_prefill_gemm")


def deferred_operand(hidden, T, seed):
    """xhat / rowss of plan_rows = T + PLAN_SLACK rows, rows >= T NaN; and the `small` mask of the first T rows."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    xhat, rowss, small = rows_deferred(T + PLAN_SLACK, hidden, g)
    return nan_rows(xhat, T), nan_rows(rowss, T), small[:T]


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


# ---------------------------------------------------------------- 1. deferred-norm consumer: BF16 and SILU modes
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("name", MLP_SHAPES)
@pytest.mark.parametrize("mode", [MODE_BF16, MODE_SILU], ids=["bf16", "silu"])
def test_consumer_modes_match_fp64(name, T, mode):
    hidden, inter = SHAPES[name][0], SHAPES[name][4]
    op = operands(name)
    xhat, rowss, small = deferred_operand(hidden, T, 17 * T + mode)
    N = 2 * inter
    width = inter if mode == MODE_SILU else N
    out = torch.full((T + PLAN_SLACK, width), float("nan"), device=DEV, dtype=torch.bfloat16)
    call_gemm(xhat, T, op["wgu_il"] if mode == MODE_SILU else op["wgu"], out, width, mode, rowss=rowss, hidden=hidden)
    torch.cuda.synchronize()
    assert torch.isnan(out[T:].float()).all(), "rows >= T written"
    got = out[:T]
    assert torch.isfinite(got.float()).all()
    n_part = parts(hidden)
    a64, r = xhat[:T].double(), rinv64(rowss[:T], hidden)
    y0, y, e = consumer_ref(a64, op["wgu64"], r, n_part)

    def finish(yy, ee):
        if mode == MODE_BF16:
            return yy, ee
        return silu_ref(yy[:, :inter], yy[:, inter:], ee[:, :inter], ee[:, inter:])
    ref, bound = finish(y, e)
    worst = gap(got, ref, bound).max().item()
    assert worst <= 1.0, f"worst gap {worst:.3g} bounds"
    stats = {"worst": worst}
    for what, (r_alt, rows) in wrong_scales(rowss[:T], hidden, small).items():
        m = margin(got, finish(y0 * r_alt[:, None], e)[0], bound, rows)
        stats[what] = m
        assert m >= MARGIN, f"{what}: the output is only {m:.3g} bounds from it"
    allowed = bound + half_spacing_bf16(ref.abs() + bound)
    mx = ref.abs().max().item()
    old = 6e-3 * mx + 1e-4 if mode == MODE_BF16 else 2e-2 * (mx + ref.abs())
    stats["median_bound_vs_old"] = (allowed / old).median().item()
    assert stats["median_bound_vs_old"] <= 0.25
    report(name, T, "bf16" if mode == MODE_BF16 else "silu", stats)


# ---------------------------------------------------------------- 2. QKV: deferred norm, RoPE, KV append
def qkv_case(name, T, seed):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    op = operands(name)
    xhat, rowss, small = deferred_operand(hidden, T, seed)
    slot, pos, n_slots = tokens(T, ctx, seed)
    kc0, vc0 = op["poison"][:n_slots], op["poison"][7:7 + n_slots]
    return dict(xhat=xhat, rowss=rowss, small=small, slot=slot, pos=pos, kc0=kc0, vc0=vc0)


def run_qkv(name, cs, T):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    q_out = torch.full((T + PLAN_SLACK, H * 128), float("nan"), device=DEV, dtype=torch.bfloat16)
    kc, vc = cs["kc0"].clone(), cs["vc0"].clone()
    fused = call_qkv(name, cs["xhat"], cs["rowss"], T, cs["slot"], cs["pos"], q_out, kc, vc)
    torch.cuda.synchronize()
    return q_out, kc, vc, fused


def qkv_outputs(name, T, slot, pos, q_out, kc, vc):
    """q [T, H, hd], k / v [T, KV, hd] as the kernel left them, and the padded cache rows [T, KV, 128]."""
    hidden, H, KV, hd = SHAPES[name][:4]
    sl, ps = slot.long(), pos.long()
    q = q_out[:T].view(T, H, 128)
    return q[..., :hd], kc[sl, :, ps, :hd], vc[sl, :, ps, :hd], kc[sl, :, ps], vc[sl, :, ps]


def split_qkv(t, H, KV, hd):
    T = t.shape[0]
    return (t[:, :H * hd].view(T, H, hd), t[:, H * hd:(H + KV) * hd].view(T, KV, hd),
            t[:, (H + KV) * hd:].view(T, KV, hd))


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("name", QKV_SHAPES)
def test_qkv_rope_and_kv_append_match_fp64(name, T):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    op = operands(name)
    cs = qkv_case(name, T, 31 * T + hd)
    q_out, kc, vc, fused = run_qkv(name, cs, T)
    assert fused == (1 if hd == 128 else 0)
    sl, ps = cs["slot"].long(), cs["pos"].long()
    q, k, v, krow, vrow = qkv_outputs(name, T, cs["slot"], cs["pos"], q_out, kc, vc)

    # ---- nothing else written: q pad columns and rows >= T, every cache byte outside columns [0, hd) of the new rows
    qv = q_out.view(-1, H, 128)
    assert torch.isnan(qv[:T, :, hd:].float()).all(), "q pad columns written"
    assert torch.isnan(q_out[T:].float()).all(), "q rows >= T written"
    for what, before, after in (("k", cs["kc0"], kc), ("v", cs["vc0"], vc)):
        fixed = after.clone()
        fixed[sl, :, ps, :hd] = before[sl, :, ps, :hd]
        assert same_bits(fixed, before), f"{what} cache written outside columns [0, hd) of the tokens' rows"

    # ---- v (and at head_dim != 128 the q / k operands of rope_kv_kernel) against the same GEMM in BF16 mode
    nqkv = (H + 2 * KV) * hd
    plain = torch.full((T + PLAN_SLACK, nqkv), float("nan"), device=DEV, dtype=torch.bfloat16)
    call_gemm(cs["xhat"], T, op["wqkv"], plain, nqkv, MODE_BF16, rowss=cs["rowss"], hidden=hidden)
    torch.cuda.synchronize()
    pq, pk, pv = split_qkv(plain[:T], H, KV, hd)
    assert same_bits(v, pv), "appended v differs from the BF16-mode v columns"

    # ---- fp64 reference
    n_part = parts(hidden)
    a64, r = cs["xhat"][:T].double(), rinv64(cs["rowss"][:T], hidden)
    y0, y, e = consumer_ref(a64, op["wqkv64"], r, n_part)
    e_pre = e if fused else e + half_spacing_bf16(y.abs() + e)
    c, s = rope_table(ps, theta, hd)
    c, s = c[:, None], s[:, None]

    def rotated(yy, cc, ss):
        qy, ky, vy = split_qkv(yy, H, KV, hd)
        return rot(qy, cc, ss), rot(ky, cc, ss), vy
    eq, ek, ev = split_qkv(e_pre, H, KV, hd)
    qy, ky, vy = split_qkv(y, H, KV, hd)
    bq, bk, bv = rot_bound(qy, eq, c, s), rot_bound(ky, ek, c, s), split_qkv(e, H, KV, hd)[2]
    rq, rk, rv = rotated(y, c, s)
    stats = {}
    for what, got, ref, bd in (("q", q, rq, bq), ("k", k, rk, bk), ("v", v, rv, bv)):
        w = gap(got, ref, bd).max().item()
        stats[f"worst_{what}"] = w
        assert w <= 1.0, f"{what}: worst gap {w:.3g} bounds"
    if not fused:
        # rope_kv_kernel from the bf16 matrix: the rounding of the fp32 rotation of those exact values
        for what, got, x in (("q", q, pq), ("k", k, pk)):
            x64 = x.double()
            w = gap(got, rot(x64, c, s), rot_bound(x64, torch.zeros_like(x64), c, s)).max().item()
            assert w <= 1.0, f"{what}: not the rotation of the bf16 qkv matrix ({w:.3g})"

    # ---- close wrong answers
    def worst_alt(alt, rows=None):
        aq, ak, av = alt
        return max(margin(q, aq, bq, rows), margin(k, ak, bk, rows))
    for what, (r_alt, rows) in wrong_scales(cs["rowss"][:T], hidden, cs["small"]).items():
        aq, ak, av = rotated(y0 * r_alt[:, None], c, s)
        m = max(worst_alt((aq, ak, av), rows), margin(v, av, bv, rows))
        stats[what] = m
        assert m >= MARGIN, f"{what}: the output is only {m:.3g} bounds from it"
    c1, s1 = rope_table(ps - 1, theta, hd)
    alts = {"RoPE at pos - 1": rotated(y, c1[:, None], s1[:, None]),
            "RoPE pairs (i, i + 1)": (rot_pairs_adjacent(qy, c, s), rot_pairs_adjacent(ky, c, s), vy)}
    if hd != 128:
        c2, s2 = rope_table(ps, theta, 128)
        alts["head_dim-128 table"] = rotated(y, c2[:, None, : hd // 2], s2[:, None, : hd // 2])
    for what, alt in alts.items():
        m = worst_alt(alt)
        stats[what] = m
        assert m >= MARGIN, f"{what}: the output is only {m:.3g} bounds from it"
    allowed = torch.cat([(bd + half_spacing_bf16(ref.abs() + bd)).flatten() for ref, bd in ((rq, bq), (rk, bk))])
    refs = torch.cat([rq.flatten(), rk.flatten()])
    stats["median_bound_vs_old"] = (allowed / (3e-2 + 1e-2 * refs.abs())).median().item()
    av = bv + half_spacing_bf16(rv.abs() + bv)
    stats["v_median_bound_vs_old"] = (av / (6e-3 * rv.abs().max() + 1e-4)).median().item()
    assert stats["median_bound_vs_old"] <= 0.25 and stats["v_median_bound_vs_old"] <= 0.25
    report(name, T, "qkv", stats)


# ---------------------------------------------------------------- 3. deferred-norm producer: RESID with xhat
def resid_case(name, T, seed):
    hidden = SHAPES[name][0]
    op = operands(name)
    K = op["K_res"]
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = T + PLAN_SLACK
    A = nan_rows(torch.randn(P, K, device=DEV, generator=g).bfloat16(), T)
    x_in = nan_rows(2 * torch.randn(P, hidden, device=DEV, generator=g), T)
    return A, x_in


def run_resid(name, A, x_in, T, defer=True):
    hidden = SHAPES[name][0]
    op = operands(name)
    P = A.shape[0]
    x = x_in.clone()
    if not defer:
        call_gemm(A, T, op["wres"], x, hidden, MODE_RESID)
        torch.cuda.synchronize()
        return x, None, None
    xhat = torch.full((P, hidden), float("nan"), device=DEV, dtype=torch.bfloat16)
    rs_flat = torch.full((P * parts(hidden) + 8,), float("nan"), device=DEV)
    call_gemm(A, T, op["wres"], x, hidden, MODE_RESID, gamma=op["gamma"], xhat=xhat, rowss_out=rs_flat)
    torch.cuda.synchronize()
    return x, xhat, rs_flat


def partial_sums(x64, hidden, shift=0):
    """sum of x^2 over columns [128 p + shift, 128 p + shift + 128) of each row (zero past hidden)."""
    n = parts(hidden)
    sq = torch.nn.functional.pad(x64 * x64, (0, n * 128 + shift - hidden))[:, shift:]
    return sq.view(x64.shape[0], n, 128).sum(-1)


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("name", RESID_SHAPES)
def test_resid_producer_matches_fp64(name, T):
    hidden = SHAPES[name][0]
    op = operands(name)
    A, x_in = resid_case(name, T, 7 * T + hidden)
    x, xhat, rs_flat = run_resid(name, A, x_in, T)
    x_plain, _, _ = run_resid(name, A, x_in, T, defer=False)
    n = parts(hidden)
    assert same_bits(x, x_plain), "x differs from the launch without xhat"
    assert torch.isnan(x[T:]).all() and torch.isnan(xhat[T:].float()).all(), "rows >= T written"
    rs = rs_flat[: (T + PLAN_SLACK) * n].view(-1, n)
    assert torch.isnan(rs[T:]).all() and torch.isnan(rs_flat[-8:]).all(), "partials of rows >= T written"

    # ---- x against fp64
    y = x_in[:T].double() + A[:T].double() @ op["wres64"].t()
    bound = e_acc(y - x_in[:T].double(), op["K_res"]) + 1.01 * U * y.abs()
    err = (x[:T].double() - y).abs()
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"x: worst |x - ref| / bound = {worst:.3g}"
    # ---- xhat = bf16(x * gamma) of the kernel's own x, bit for bit
    assert same_bits(xhat[:T], (x[:T] * op["gamma"].float()).bfloat16()), "xhat != bf16(x * gamma)"
    # ---- each partial on its own
    x64 = x[:T].double()
    ref = partial_sums(x64, hidden)
    pb = 2.0 ** -20 * ref + 1e-30
    got = rs[:T].double()
    worst_p = ((got - ref).abs() / pb).max().item()
    assert worst_p <= 1.0, f"partials: worst {worst_p:.3g} bounds"
    m = ((got - partial_sums(x64, hidden, 64)).abs() / pb).max().item()
    assert m >= MARGIN
    old = 1e-3 * y.abs().max() + 1e-4 * y.abs()
    report(name, T, "resid", {"x_worst": worst, "partials_worst": worst_p, "partials shifted by 64": m,
                              "median_bound_vs_old": (bound / old).median().item()})
    assert (bound / old).median().item() <= 0.25


# ---------------------------------------------------------------- 4. layer-0 norm in the deferred form
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_layer0_norm_deferred_form(name, T):
    hidden = SHAPES[name][0]
    op = operands(name)
    g = torch.Generator(device=DEV).manual_seed(3 * T + hidden)
    P, n = T + PLAN_SLACK, parts(hidden)
    scale = torch.empty(P, 1, device=DEV).uniform_(0.01, 3.0, generator=g)
    x = nan_rows(torch.randn(P, hidden, device=DEV, generator=g) * scale, T)
    x0 = x.clone()
    xn = torch.full((P, hidden), float("nan"), device=DEV, dtype=torch.bfloat16)
    rs = torch.full((P, n), float("nan"), device=DEV)
    call_norm(x, op["gamma"], xn, rs, T, hidden)
    torch.cuda.synchronize()
    assert same_bits(x, x0), "x written"
    assert torch.isnan(xn[T:].float()).all() and torch.isnan(rs[T:]).all(), "rows >= T written"
    assert same_bits(xn[:T], (x[:T] * op["gamma"].float()).bfloat16()), "xn != bf16(x * w)"
    ref = (x[:T].double() ** 2).sum(1)
    b = (hidden / 64 + 16) * U * ref
    worst = ((rs[:T, 0].double() - ref).abs() / b).max().item()
    assert worst <= 1.0, f"sum of squares: worst {worst:.3g} bounds"
    assert (rs[:T, 1:] == 0).all() and not torch.signbit(rs[:T, 1:]).any(), "partials 1.. not +0"
    report(name, T, "norm", {"worst": worst})


# ---------------------------------------------------------------- 5. the deferred form is an RMSNorm
def t1_term(xg64, w64):
    """lambda sigma sqrt(sum_k (x_k gamma_k w_k)^2) for sigma = 2^-9 (one bf16 rounding per operand element)."""
    return LAMBDA * 2.0 ** -9 * ((xg64 * xg64) @ (w64 * w64).t()).sqrt()


@pytest.mark.parametrize("T", (65, 300))
@pytest.mark.parametrize("name", QKV_SHAPES)
def test_norm_then_qkv_is_textbook_rmsnorm(name, T):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    op = operands(name)
    g = torch.Generator(device=DEV).manual_seed(5 * T + hidden)
    P = T + PLAN_SLACK
    scale = torch.empty(P, 1, device=DEV).uniform_(0.01, 3.0, generator=g)
    x = nan_rows(torch.randn(P, hidden, device=DEV, generator=g) * scale, T)
    xn = torch.full((P, hidden), float("nan"), device=DEV, dtype=torch.bfloat16)
    rs = torch.full((P, parts(hidden)), float("nan"), device=DEV)
    call_norm(x, op["gamma"], xn, rs, T, hidden)
    slot, pos, n_slots = tokens(T, ctx, T)
    cs = dict(xhat=xn, rowss=rs, slot=slot, pos=pos, kc0=op["poison"][:n_slots], vc0=op["poison"][7:7 + n_slots])
    q_out, kc, vc, fused = run_qkv(name, cs, T)
    q, k, v, _, _ = qkv_outputs(name, T, slot, pos, q_out, kc, vc)
    x64 = x[:T].double()
    r = ((x64 * x64).mean(1) + EPS32) ** -0.5
    xg = x64 * op["gamma"].double()
    t1 = t1_term(xg, op["wqkv64"])
    rel_ss = (hidden / 64 + 16) * U / 2
    _, y, e = consumer_ref(xn[:T].double(), op["wqkv64"], r, parts(hidden), extra=(t1, rel_ss))
    y = (xg * r[:, None]) @ op["wqkv64"].t()                        # the textbook form, unrounded operand
    e_pre = e if fused else e + half_spacing_bf16(y.abs() + e)
    c, s = rope_table(pos.long(), theta, hd)
    c, s = c[:, None], s[:, None]
    qy, ky, vy = split_qkv(y, H, KV, hd)
    eq, ek, _ = split_qkv(e_pre, H, KV, hd)
    ev = split_qkv(e, H, KV, hd)[2]
    stats = {}
    for what, got, ref, bd in (("q", q, rot(qy, c, s), rot_bound(qy, eq, c, s)),
                               ("k", k, rot(ky, c, s), rot_bound(ky, ek, c, s)), ("v", v, vy, ev)):
        w = gap(got, ref, bd).max().item()
        stats[what] = w
        assert w <= 1.0, f"{what}: worst gap {w:.3g} bounds from the textbook RMSNorm"
    report(name, T, "norm->qkv", stats)


@pytest.mark.parametrize("T", (65, 300))
@pytest.mark.parametrize("name", MLP_SHAPES)
def test_resid_then_gate_up_is_textbook_rmsnorm(name, T):
    hidden, inter = SHAPES[name][0], SHAPES[name][4]
    op = operands(name)
    A, x_in = resid_case(name, T, 11 * T + hidden)
    x, xhat, rs_flat = run_resid(name, A, x_in, T)
    n = parts(hidden)
    rs = rs_flat[: (T + PLAN_SLACK) * n].view(-1, n)
    act = torch.full((T + PLAN_SLACK, inter), float("nan"), device=DEV, dtype=torch.bfloat16)
    call_gemm(xhat, T, op["wgu_il"], act, inter, MODE_SILU, rowss=rs, hidden=hidden)
    torch.cuda.synchronize()
    x64 = x[:T].double()
    r = ((x64 * x64).mean(1) + EPS32) ** -0.5
    xg = x64 * op["gamma"].double()
    t1 = t1_term(xg, op["wgu64"])
    rel_ss = 2.0 ** -20 + n * U
    _, _, e = consumer_ref(xhat[:T].double(), op["wgu64"], r, n, extra=(t1, rel_ss))
    y = (xg * r[:, None]) @ op["wgu64"].t()
    ref, bound = silu_ref(y[:, :inter], y[:, inter:], e[:, :inter], e[:, inter:])
    w = gap(act[:T], ref, bound).max().item()
    assert w <= 1.0, f"act: worst gap {w:.3g} bounds from the textbook RMSNorm"
    report(name, T, "resid->gate/up", {"worst": w})


# ---------------------------------------------------------------- 6. a row's bits do not depend on its chunk
OFFSETS = (0, 1, 8, 63, 64, 129)
PAD_AFTER = (0, 50, 7, 100, 1, 20)
R = 300


def placements(R_rows, pool, seed):
    """Chunks holding the rows R_rows at each offset, padded before and after with rows of `pool`."""
    out = []
    for i, (o, pa) in enumerate(zip(OFFSETS, PAD_AFTER)):
        T = o + R + pa
        idx = torch.randperm(pool.shape[0], generator=torch.Generator().manual_seed(seed + i))[: T + PLAN_SLACK]
        t = pool[idx.to(pool.device)].clone()
        t[o:o + R] = R_rows
        out.append((o, T, t))
    return out


@pytest.mark.parametrize("name", ["llama-3-8b", "phi-3-mini", "tiny96", "odd-heads", "hidden320"])
def test_row_bits_do_not_depend_on_the_chunk(name):
    hidden, H, KV, hd, inter, theta, ctx = SHAPES[name]
    op = operands(name)
    g = torch.Generator(device=DEV).manual_seed(99)
    n_pool = 129 + R + 100 + PLAN_SLACK + 64
    xhat_p, rowss_p, _ = rows_deferred(n_pool + R, hidden, g)
    xs, rss = placements(xhat_p[:R], xhat_p[R:], 1), placements(rowss_p[:R], rowss_p[R:], 1)

    def check(what, outs):
        base = outs[0]
        for i, o in enumerate(outs[1:], 1):
            assert same_bits(o, base), f"{what}: rows at offset {OFFSETS[i]} differ from offset 0"

    # deferred-norm consumers
    if inter:
        for mode, W, width in ((MODE_BF16, op["wgu"], 2 * inter), (MODE_SILU, op["wgu_il"], inter)):
            outs = []
            for (o, T, xh), (_, _, rs) in zip(xs, rss):
                out = torch.empty(xh.shape[0], width, device=DEV, dtype=torch.bfloat16)
                call_gemm(xh, T, W, out, width, mode, rowss=rs, hidden=hidden)
                outs.append(out[o:o + R])
            torch.cuda.synchronize()
            check(f"mode {mode}", outs)
    # QKV: the 300 rows are one sequence in slot 0 at positions 37 .. 336; padding rows are slot 1, positions 400..
    if H:
        outs_q, outs_k, outs_v = [], [], []
        for (o, T, xh), (_, _, rs) in zip(xs, rss):
            slot = torch.ones(T, dtype=torch.int32, device=DEV)
            pos = 400 + torch.arange(T, dtype=torch.int32, device=DEV)
            slot[o:o + R] = 0
            pos[o:o + R] = 37 + torch.arange(R, dtype=torch.int32, device=DEV)
            q_out = torch.empty(xh.shape[0], H * 128, device=DEV, dtype=torch.bfloat16)
            kc, vc = op["poison"][:2].clone(), op["poison"][7:9].clone()
            call_qkv(name, xh, rs, T, slot, pos, q_out, kc, vc)
            outs_q.append(q_out[o:o + R].view(R, H, 128)[..., :hd])
            outs_k.append(kc[0, :, 37:37 + R])
            outs_v.append(vc[0, :, 37:37 + R])
        torch.cuda.synchronize()
        check("q", outs_q)
        check("k", outs_k)
        check("v", outs_v)
    # RESID producer: x, xhat, rowss
    K = op["K_res"]
    if K:
        A_p = torch.randn(n_pool + R, K, device=DEV, generator=g).bfloat16()
        x_p = 2 * torch.randn(n_pool + R, hidden, device=DEV, generator=g)
        As, xins = placements(A_p[:R], A_p[R:], 2), placements(x_p[:R], x_p[R:], 2)
        ox, oh, orr = [], [], []
        for (o, T, A), (_, _, x_in) in zip(As, xins):
            x, xhat, rs_flat = run_resid(name, A, x_in, T)
            n = parts(hidden)
            ox.append(x[o:o + R])
            oh.append(xhat[o:o + R])
            orr.append(rs_flat[: A.shape[0] * n].view(-1, n)[o:o + R])
        check("x", ox)
        check("xhat", oh)
        check("rowss_out", orr)
    # layer-0 norm: xn, rowss
    x_p =torch.randn(n_pool + R, hidden, device=DEV, generator=g)
    on, orr = [], []
    for o, T, x in placements(x_p[:R], x_p[R:], 3):
        xn = torch.empty(x.shape[0], hidden, device=DEV, dtype=torch.bfloat16)
        rs = torch.empty(x.shape[0], parts(hidden), device=DEV)
        call_norm(x, op["gamma"], xn, rs, T, hidden)
        on.append(xn[o:o + R])
        orr.append(rs[o:o + R])
    torch.cuda.synchronize()
    check("xn", on)
    check("norm rowss", orr)


# ---------------------------------------------------------------- rejections
def _small_bufs():
    P, hidden = 72, 384
    return dict(x=torch.randn(P, hidden, device=DEV), w=torch.ones(hidden, device=DEV).bfloat16(),
                xn=torch.zeros(P, hidden, device=DEV).bfloat16(), rs=torch.zeros(P, 3, device=DEV),
                wqkv=torch.zeros(12 * 96, hidden, device=DEV).bfloat16(), q=torch.zeros(P, 4 * 128, device=DEV).bfloat16(),
                kc=torch.zeros(2, 4, 128, 128, device=DEV).bfloat16(), vc=torch.zeros(2, 4, 128, 128, device=DEV).bfloat16(),
                slot=torch.zeros(P, device=DEV, dtype=torch.int32), pos=torch.ones(P, device=DEV, dtype=torch.int32),
                wo=torch.zeros(hidden, 256, device=DEV).bfloat16(), a=torch.zeros(P, 256, device=DEV).bfloat16())


NORM_REJECT = [pytest.param(dict(rows=0), id="rows0"), pytest.param(dict(hidden=320 + 32), id="hidden%64"),
               pytest.param(dict(hidden=8256, n_part=65), id="hidden>8192"), pytest.param(dict(n_part=4), id="n_part"),
               pytest.param(dict(rs=None), id="null-rowss")]


@pytest.mark.parametrize("change", NORM_REJECT)
def test_norm_rejects(change):
    b = _small_bufs()
    before = {k: v.clone() for k, v in b.items()}
    a = dict(rows=64, hidden=384, n_part=3, rs=b["rs"].data_ptr())
    a.update(change)
    rc = lib().lib.rr_op_add_rmsnorm_pf(b["x"].data_ptr(), b["w"].data_ptr(), b["xn"].data_ptr(), a["rows"], a["hidden"],
                                        EPS, a["rs"], a["n_part"], None)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT
    assert all(same_bits(b[k], before[k]) for k in b)


QKV_REJECT = [pytest.param(dict(T=0), id="T0"), pytest.param(dict(T=73), id="T>plan_rows"),
              pytest.param(dict(hd=72), id="head_dim72"), pytest.param(dict(hd=144), id="head_dim144"),
              pytest.param(dict(H=12, KV=4), id="G3"), pytest.param(dict(ctx=100), id="ctx_max100"),
              pytest.param(dict(hidden=352), id="hidden%64"), pytest.param(dict(slot=None), id="null-slot"),
              pytest.param(dict(fused=None), id="null-fused")]


@pytest.mark.parametrize("change", QKV_REJECT)
def test_qkv_rejects(change):
    b = _small_bufs()
    before = {k: v.clone() for k, v in b.items()}
    a = dict(T=64, hidden=384, H=4, KV=4, hd=96, ctx=128, slot=b["slot"].data_ptr(), fused=True)
    a.update(change)
    fused = C.c_int32(-1)
    rc = lib().lib.rr_op_prefill_qkv(b["xn"].data_ptr(), b["rs"].data_ptr(), 72, a["T"], a["hidden"], b["wqkv"].data_ptr(),
                                     a["H"], a["KV"], a["hd"], a["ctx"], 1e4, EPS, a["slot"], b["pos"].data_ptr(),
                                     b["q"].data_ptr(), b["kc"].data_ptr(), b["vc"].data_ptr(),
                                     C.byref(fused) if a["fused"] else None, None)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT and fused.value == -1
    assert all(same_bits(b[k], before[k]) for k in b)


GEMM_REJECT = [pytest.param(dict(T=0), id="T0"), pytest.param(dict(T=73), id="T>plan_rows"),
               pytest.param(dict(mode=1), id="mode-transposed"), pytest.param(dict(mode=4), id="mode-rope"),
               pytest.param(dict(n_part=3, rowss=True), id="consumer-in-resid"),
               pytest.param(dict(mode=0, ldo=384, n_part=2, rowss=True, xhat=False), id="consumer-wrong-n_part"),
               pytest.param(dict(mode=0, ldo=384, n_part=3, xhat=False), id="consumer-null-rowss"),
               pytest.param(dict(n_part_out=4), id="producer-wrong-n_part_out"),
               pytest.param(dict(gamma=False), id="producer-null-gamma"),
               pytest.param(dict(mode=0, ldo=384), id="producer-not-resid")]


@pytest.mark.parametrize("change", GEMM_REJECT)
def test_gemm_rejects(change):
    b = _small_bufs()
    before = {k: v.clone() for k, v in b.items()}
    a = dict(T=64, mode=MODE_RESID, ldo=384, n_part=0, rowss=False, gamma=True, xhat=True, n_part_out=3)
    a.update(change)
    rc = lib().lib.rr_op_prefill_gemm(b["a"].data_ptr(), 72, a["T"], 256, b["wo"].data_ptr(), 384, 256,
                                      b["x"].data_ptr(), a["ldo"], a["mode"], b["rs"].data_ptr() if a["rowss"] else None,
                                      a["n_part"], 384, EPS, b["w"].data_ptr() if a["gamma"] else None,
                                      b["xn"].data_ptr() if a["xhat"] else None, b["rs"].data_ptr(), a["n_part_out"], None)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT
    assert all(same_bits(b[k], before[k]) for k in b)
