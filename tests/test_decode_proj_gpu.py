"""Kernel-level parity of the unfused decode projections (gemm_bf16_wgmma, csrc/rr_gemm.cu) through rr_op_decode_proj,
which plans and launches each one exactly as the engine does for a decode working set of `rows` rows: tile width
pick_bn(rows), plane pitch rows, the engine's split-K rule, the TMA-store epilogue where the engine uses one.  Every
projection of every model family the engine serves (QKV, O, gate/up, down, lm_head), at batch widths 1..256: every tile
width, full and ragged tiles, one and two 128-row batch tiles.  Gate/up runs what the engine runs at that width: the fused
SiLU epilogue over 64-row interleaved weights where the engine interleaves them (one gate/up plane, rows > 16), else fp32
planes over [gate; up].  The same planes also feed the kernels between the projections: the residual add + RMSNorm
(rr_op_add_rmsnorm) and SiLU * up over `small`'s two gate/up planes (rr_op_silu_mul).  The prefill's trimmed last layer
runs O, gate/up, down and lm_head through these same plans, so this also covers the first token of every request.

Operands as the engine sees them: xn ~ N(0, 1) in bf16, weights bf16 with sigma = 1 / sqrt(K) (K = fan-in), gate/up
interleaved as engine.py does.  References are fp64, computed in blocks of weight rows.

Bounds.
  * Planes.  Plane z sums the k-blocks [kb * z / n, kb * (z + 1) / n) (kb = K / 64, n planes): K_z terms.  A bf16 x bf16
    product is exact in fp32, so the only error is the fp32 accumulation.  Each add, in any order, errs by at most one
    ulp of its result (2^-23 relative: round to nearest or truncation), and every partial sum is at most
    S_z = sum over the plane's k-range of |x[b, k] * w[n, k]|.  An adder that aligns a k16 group's 16 products and the
    accumulator to the largest exponent truncates 17 times per 16 terms, so, with the second-order terms, elementwise
        |got - ref_z| <= 2.2 * K_z * 2^-24 * S_z.
    That worst case grows like K_z and alone would let an output rounded to bf16 (2^-9 relative) through.  Each plane is
    therefore also held to the accumulation model of test_decode_mlp_gpu.py (one rounding of at most one ulp per step,
    independent signs, running sums at most twice the final magnitude, 8 standard deviations):
        max|got - ref_z| <= 16 * 2^-23 * sqrt(K_z) * max|ref_z|     (1.2e-4 of max|ref_z| at K_z = 4096).
    Boundary power: one k-block (64 terms) moves an output by about 8 / sqrt(K) (one standard deviation), while the
    elementwise bound stays below a fifth of that at these shapes (K_z <= 4096).  The test asserts that adding or
    dropping the first or the last k-block of any plane moves at least half of its outputs by more than twice their
    bound, so a k-range off by one block cannot pass.
  * SiLU epilogue: act = bf16(silu(g) * u) elementwise against fp64, with test_decode_mlp_gpu.py's bound
        |act - ref| <= 2^-8 |ref| + tau_act * max|ref|,  tau_act = (1 + 2^-8) (34 * 2^-23 sqrt(K) G^2 / max|ref| + 2^-20),
    G = max(max|g|, max|u|): accumulation errors of g and u, __expf / __fdividef, then the bf16 rounding.
  * rr_op_add_rmsnorm over n planes: its comment pins acc = ((p0 + p1) + ...) + p_{n-1}, then x + acc, each an IEEE fp32
    add, so the residual is compared bit for bit with the same adds in torch.  xn = bf16(x * inv * w), inv =
    rsqrtf(ss / hidden + eps), ss = the sum of x^2 in the kernel's order.  Relative to fp64 on the kernel's residual: ss
    errs by at most (hidden + 1) 2^-24 (positive terms, any order, and the squares), inv by half that, plus the division
    and the eps add (2^-24 each), rsqrtf (2 ulp, 2^-22) and the two products (2^-24 each), so
        delta = (0.51 (hidden + 1) + 8) 2^-24,   |xn - ref| <= (2^-8 (1 + delta) + delta) |ref|.
  * rr_op_silu_mul over planes p0, p1: g = p0 + p1 and u likewise in fp32 (2^-24 relative each; |silu'| <= 1.1), __expf
    (2 + 1.16 |g| ulp), the add, __fdividef (2 ulp) and the product with u, then the bf16 rounding:
        e = 2^-23 ((8 + 1.16 |g|) |ref| + 1.1 |u| |g| + |silu(g)| |u|),   |act - ref| <= 2^-8 (|ref| + e) + e.
Bit for bit: FP8 weights (rr_op_quantize_fp8_weight) against bf16 on their dequantized values, the TMA-store epilogue
against RR_NO_TMA_EPI=1 (tile width <= 64), two launches.  NaN guards before and after every output stay NaN: no writes
past `rows`, past `rows_w` or from the second batch tile.  n_splits is the split rule recomputed here from the SM count,
and engine.py's mirror of that rule agrees with it for gate/up."""
import ctypes as C
import math
import zlib

import pytest
import torch

from test_gemm_gpu import _interleave64

pytestmark = pytest.mark.gpu

RR_INVALID_ARGUMENT = 4
F32, SILU = 1, 2
U23, U24 = 2.0 ** -23, 2.0 ** -24
ROWS = (1, 8, 16, 17, 32, 33, 64, 65, 128, 129, 200, 256)
FAMILIES = ("llama-3-8b", "phi-3-mini", "small", "small96", "tiny", "tiny96")
HEADS = FAMILIES + ("mistral-7b",)
PROJ = ("qkv", "o", "gu", "down")
GUARD = 64                        # leading guard elements (keeps the output 16-byte aligned for the TMA-store epilogue)
BLK = 8192                        # weight rows per block of the fp64 references


def _head_rows(fam):
    return (1, 17, 65, 129, 256) if fam == "llama-3-8b" else ROWS


CASES = [pytest.param(f, p, r, id=f"{f}-{p}-rows{r}") for f in FAMILIES for p in PROJ for r in ROWS]
HEAD_CASES = [pytest.param(f, r, id=f"{f}-rows{r}") for f in HEADS for r in _head_rows(f)]


def _L():
    from rr_b200 import _lib
    return _lib


def _spec(fam):
    from rr_b200.models import SPECS
    return SPECS[fam]


def _shape(fam, proj):
    """(rows_w, K) of a projection."""
    s = _spec(fam)
    nq, nkv = s.n_heads * s.head_dim, s.n_kv_heads * s.head_dim
    return {"qkv": (nq + 2 * nkv, s.hidden), "o": (s.hidden, nq), "gu": (2 * s.inter, s.hidden),
            "down": (s.hidden, s.inter), "lm_head": (s.vocab, s.hidden)}[proj]


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _split_rule(rows_w, K):
    """The engine's split-K rule: one (128-row weight tile, plane) item per SM, at most 8 planes of at least 8 k-blocks."""
    s = max(1, min(8, _n_sm() // ((rows_w + 127) // 128)))
    while s > 1 and (K // 64) // s < 8:
        s -= 1
    return s


def _gu_fused(fam, rows):
    """engine.py interleaves gate/up (and the engine runs the SiLU epilogue) with one gate/up plane and rows > 16."""
    rows_w, K = _shape(fam, "gu")
    return _split_rule(rows_w, K) == 1 and rows > 16


def _k_ranges(K, n):
    kb = K // 64
    return [(64 * (kb * z // n), 64 * (kb * (z + 1) // n)) for z in range(n)]


_W = {}


def _weights(fam, proj):
    """Seeded bf16 weight of one projection ([gate; up] for gate/up), cached per family."""
    if _W.get("fam") != fam:
        _W.clear()
        _W["fam"] = fam
    if proj not in _W:
        rows_w, K = _shape(fam, proj)
        g = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"{fam}/{proj}".encode()))
        _W[proj] = (torch.randn(rows_w, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    return _W[proj]


def _kernel_weight(fam, proj, fused):
    w = _weights(fam, proj)
    if not fused:
        return w
    key = proj + "-il"
    if key not in _W:
        _W[key] = _interleave64(w, w.shape[0] // 2)
    return _W[key]


def _fp8(fam, proj, fused):
    """(q, scale, dequantized) of the kernel weight: e4m3 rows and their scales, and bf16(q * scale)."""
    key = proj + ("-il" if fused else "") + "-fp8"
    if key not in _W:
        L = _L()
        w = _kernel_weight(fam, proj, fused)
        q = torch.empty(w.shape, dtype=torch.float8_e4m3fn, device="cuda")
        s = torch.empty(w.shape[0], dtype=torch.float32, device="cuda")
        L.check(L.lib.rr_op_quantize_fp8_weight(w.data_ptr(), w.shape[0], w.shape[1], w.shape[1], q.data_ptr(),
                                                s.data_ptr(), None), "rr_op_quantize_fp8_weight")
        d = torch.empty(w.shape, dtype=torch.bfloat16, device="cuda")
        L.check(L.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), s.data_ptr(), w.shape[0], w.shape[1], d.data_ptr(),
                                                  w.shape[1], None), "rr_op_dequantize_fp8_weight")
        _W[key] = (q, s, d)
    return _W[key]


_X = {}


def _xn(K, rows):
    if K not in _X:
        g = torch.Generator(device="cuda").manual_seed(K)
        _X[K] = torch.randn(256, K, device="cuda", generator=g).bfloat16()
    return _X[K][:rows]


def _out_shape(rows_w, rows, mode, n):
    return (n, rows, rows_w) if mode == F32 else (rows, rows_w // 2)


def _call(w, scale, rows_w, K, x, rows, mode, lm_head, n_expect):
    """One rr_op_decode_proj call into a NaN buffer with GUARD elements before the output and a whole 128-row batch tile
    after it.  Returns (rc, n_splits, buffer, output view)."""
    L = _L()
    shape = _out_shape(rows_w, rows, mode, n_expect)
    n_el = math.prod(shape)
    tail = 128 * shape[-1]
    buf = torch.full((GUARD + n_el + tail,), float("nan"), device="cuda",
                     dtype=torch.float32 if mode == F32 else torch.bfloat16)
    ns = C.c_int32(-1)
    rc = L.lib.rr_op_decode_proj(w.data_ptr(), None if scale is None else scale.data_ptr(), rows_w, K, x.data_ptr(), rows,
                                 buf[GUARD:].data_ptr(), mode, lm_head, C.byref(ns), None)
    return rc, ns.value, buf, buf[GUARD:GUARD + n_el].view(shape)


def _run(w, scale, rows_w, K, x, rows, mode, lm_head, n_expect):
    rc, ns, buf, out = _call(w, scale, rows_w, K, x, rows, mode, lm_head, n_expect)
    _L().check(rc, "rr_op_decode_proj")
    torch.cuda.synchronize()
    assert ns == n_expect, f"n_splits {ns}, the engine's rule gives {n_expect}"
    assert torch.isnan(buf[:GUARD]).all(), "written before the output"
    assert torch.isnan(buf[GUARD + out.numel():]).all(), "written past the output (rows, rows_w or a batch tile)"
    assert not torch.isnan(out).any(), "output not written everywhere"
    return buf, out


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


def _case(fam, proj, rows):
    """(kernel weight, rows_w, K, mode, lm_head, n_splits the engine uses, fused gate/up)."""
    rows_w, K = _shape(fam, proj)
    if proj == "lm_head":
        return _weights(fam, proj), rows_w, K, F32, 1, 1, False
    fused = proj == "gu" and _gu_fused(fam, rows)
    mode = SILU if fused else F32
    return _kernel_weight(fam, proj, fused), rows_w, K, mode, 0, _split_rule(rows_w, K), fused


def _check_planes(w, x, got, n):
    """Each plane against fp64, in blocks of weight rows: the elementwise bound, the boundary power of the k-blocks at
    and next to each end of its k-range, and the plane-wide accumulation bound (module docstring)."""
    K = x.shape[1]
    ranges = _k_ranges(K, n)
    x64 = x.double()
    err_max, ref_max = [0.0] * n, [0.0] * n
    for r0 in range(0, w.shape[0], BLK):
        w64 = w[r0:r0 + BLK].double()
        for z, (k0, k1) in enumerate(ranges):
            ref = x64[:, k0:k1] @ w64[:, k0:k1].t()
            bound = 2.2 * (k1 - k0) * U24 * (x64[:, k0:k1].abs() @ w64[:, k0:k1].abs().t())
            err = (got[z, :, r0:r0 + BLK].double() - ref).abs()
            bad = (err > bound).sum().item()
            assert bad == 0, f"plane {z} (k {k0}:{k1}), weight rows from {r0}: {bad} outputs past the elementwise bound"
            err_max[z] = max(err_max[z], err.max().item())
            ref_max[z] = max(ref_max[z], ref.abs().max().item())
            for a in {k0 - 64, k0, k1 - 64, k1} - {-64, K}:      # a range one block longer or shorter at either end
                shift = (x64[:, a:a + 64] @ w64[:, a:a + 64].t()).abs()
                frac = (shift > 2 * bound).double().mean().item()
                assert frac >= 0.5, f"plane {z}: the k-block at {a} moves only {frac:.2f} of the outputs past the bound"
    for z, (k0, k1) in enumerate(ranges):
        tol = 16 * U23 * math.sqrt(k1 - k0) * ref_max[z]
        assert err_max[z] <= tol, f"plane {z} (k {k0}:{k1}): max err {err_max[z]:.3g} > {tol:.3g}"


def _check_silu(w_plain, x, act):
    inter = w_plain.shape[0] // 2
    K = x.shape[1]
    y = x.double() @ w_plain.double().t()
    g, u = y[:, :inter], y[:, inter:]
    ref = g * u / (1.0 + torch.exp(-g))
    m = ref.abs().max().item()
    G = max(g.abs().max().item(), u.abs().max().item())
    tau_act = (1 + 2.0 ** -8) * (34 * U23 * math.sqrt(K) * G * G / m + 2.0 ** -20)
    assert tau_act < 2e-3
    err = (act.double() - ref).abs()
    worst = (err / (2.0 ** -8 * ref.abs() + tau_act * m)).max().item()
    assert worst <= 1.0, f"act: worst err / bound = {worst:.3g} (tau_act {tau_act:.3g}, max|ref| {m:.3g})"


@pytest.fixture
def default_path(monkeypatch):
    """The engine's default: TMA-store epilogues where the tile width allows them."""
    monkeypatch.delenv("RR_NO_TMA_EPI", raising=False)
    return monkeypatch


def _matches_fp64(fam, proj, rows):
    w, rows_w, K, mode, lm_head, n, fused = _case(fam, proj, rows)
    x = _xn(K, rows)
    _, out = _run(w, None, rows_w, K, x, rows, mode, lm_head, n)
    if mode == SILU:
        _check_silu(_weights(fam, proj), x, out)
    else:
        _check_planes(w, x, out, n)


def _bit_identical(fam, proj, rows, monkeypatch, fp8=True):
    w, rows_w, K, mode, lm_head, n, fused = _case(fam, proj, rows)
    x = _xn(K, rows)
    _, base = _run(w, None, rows_w, K, x, rows, mode, lm_head, n)
    # two launches back to back on one stream, one host sync after both
    calls = [_call(w, None, rows_w, K, x, rows, mode, lm_head, n) for _ in range(2)]
    torch.cuda.synchronize()
    for rc, ns, _, out in calls:
        assert rc == 0 and ns == n and torch.equal(_bits(out), _bits(base)), "two launches differ"
    if mode == F32 and rows <= 64:        # tile width <= 64: the TMA-store epilogue against per-thread stores
        monkeypatch.setenv("RR_NO_TMA_EPI", "1")
        _, out = _run(w, None, rows_w, K, x, rows, mode, lm_head, n)
        monkeypatch.delenv("RR_NO_TMA_EPI")
        assert torch.equal(_bits(out), _bits(base)), "per-thread store epilogue differs from the TMA store"
    if fp8:
        q, s, d = _fp8(fam, proj, fused)
        _, o8 = _run(q, s, rows_w, K, x, rows, mode, 0, n)
        _, od = _run(d, None, rows_w, K, x, rows, mode, 0, n)
        assert torch.equal(_bits(o8), _bits(od)), "FP8 weights differ from bf16 on the dequantized weights"


@pytest.mark.parametrize("fam,proj,rows", CASES)
def test_decode_proj_each_plane_matches_fp64(fam, proj, rows, default_path):
    _matches_fp64(fam, proj, rows)


@pytest.mark.parametrize("fam,rows", HEAD_CASES)
def test_lm_head_matches_fp64(fam, rows, default_path):
    _matches_fp64(fam, "lm_head", rows)


@pytest.mark.parametrize("fam,proj,rows", CASES)
def test_decode_proj_fp8_tma_and_repeats_are_bit_identical(fam, proj, rows, default_path):
    _bit_identical(fam, proj, rows, default_path)


@pytest.mark.parametrize("fam,rows", HEAD_CASES)
def test_lm_head_tma_and_repeats_are_bit_identical(fam, rows, default_path):
    _bit_identical(fam, "lm_head", rows, default_path, fp8=False)


@pytest.mark.parametrize("fam", FAMILIES)
def test_gate_up_splits_match_the_engine_mirror(fam, default_path):
    """n_splits reported for gate/up equals engine.py's mirror of the split rule, which decides the gate/up layout; with one
    plane the SiLU epilogue is accepted from 17 rows on, with more it is refused as the engine would not fuse it."""
    from rr_b200.engine import pick_splits
    rows_w, K = _shape(fam, "gu")
    x = _xn(K, 33)
    rc, ns, _, _ = _call(_weights(fam, "gu"), None, rows_w, K, x, 33, F32, 0, 8)
    assert rc == 0 and ns == pick_splits(rows_w, K, _n_sm()) == _split_rule(rows_w, K)
    rc, ns2, buf, _ = _call(_kernel_weight(fam, "gu", True), None, rows_w, K, x, 33, SILU, 0, 1)
    torch.cuda.synchronize()
    if ns == 1:
        assert rc == 0 and ns2 == 1
    else:
        assert rc == RR_INVALID_ARGUMENT and ns2 == -1 and torch.isnan(buf).all()


@pytest.mark.parametrize("args,why", [
    (dict(rows=16, mode=SILU), "SiLU on a 16-row tile"),
    (dict(rows=257), "more rows than the engine's largest batch"),
    (dict(lm_head=1, mode=SILU), "lm_head through the SiLU epilogue"),
    (dict(K=500), "K not a multiple of 8"),
])
def test_decode_proj_refusals_leave_the_output_untouched(args, why, default_path):
    a = dict(rows=33, mode=F32, lm_head=0, K=512)
    a.update(args)
    w = _kernel_weight("tiny", "gu", True)                       # [2048, 512]
    x = torch.randn(a["rows"], 512, device="cuda").bfloat16()
    rc, ns, buf, _ = _call(w, None, 2048, a["K"], x, a["rows"], a["mode"], a["lm_head"], 1)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT and ns == -1 and torch.isnan(buf).all(), why


# ---- the kernels between the projections ----------------------------------------------------------------------------------
# the fused MLP runs at 17..128 rows, for every family but `small` (two gate/up planes at 132 SMs)
NORM_CASES = [pytest.param(f, src, r, id=f"{f}-{src}-rows{r}") for f in FAMILIES for src in ("o", "down", "mlp")
              for r in ROWS if src != "mlp" or (f != "small" and 17 <= r <= 128)]


def _mlp_planes(fam, rows):
    """The fused decode MLP's K-slice planes (rr_op_decode_mlp) on the family's gate/up and down weights."""
    L = _L()
    s = _spec(fam)
    x = _xn(s.hidden, rows)
    wgu_il, wd = _kernel_weight(fam, "gu", True), _weights(fam, "down")
    act = torch.empty(rows, s.inter, device="cuda", dtype=torch.bfloat16)
    planes = torch.full((8, rows, s.hidden), float("nan"), device="cuda", dtype=torch.float32)
    ns, skb = C.c_int32(-1), C.c_int32(-1)
    L.check(L.lib.rr_op_decode_mlp(wgu_il.data_ptr(), wd.data_ptr(), x.data_ptr(), rows, s.hidden, s.inter, act.data_ptr(),
                                   planes.data_ptr(), rows, C.byref(ns), C.byref(skb), None), "rr_op_decode_mlp")
    torch.cuda.synchronize()
    return planes[:ns.value]


@pytest.mark.parametrize("fam,src,rows", NORM_CASES)
def test_add_rmsnorm_over_the_planes(fam, src, rows, default_path):
    """Residual bit for bit in the kernel's stated association, xn within the module docstring's bound, over the planes the
    engine hands the norm: O's and down's split-K planes, and the fused MLP's K slices."""
    L = _L()
    s = _spec(fam)
    hidden = s.hidden
    if src == "mlp":
        if _split_rule(*_shape(fam, "gu")) != 1:
            pytest.skip("the engine does not fuse this family's MLP (two gate/up planes)")
        planes = _mlp_planes(fam, rows)
    else:
        w, rows_w, K, mode, lm_head, n, _ = _case(fam, src, rows)
        planes = _run(w, None, rows_w, K, _xn(K, rows), rows, mode, lm_head, n)[1]
    n = planes.shape[0]
    assert 1 <= n <= 8
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + hidden)
    x = 4 * torch.randn(rows, hidden, device="cuda", generator=g)
    nw = (1 + 0.1 * torch.randn(hidden, device="cuda", generator=g)).bfloat16()
    eps = s.rms_eps
    xd = x.clone()
    xn = torch.full((rows + 1, hidden), float("nan"), device="cuda", dtype=torch.bfloat16)
    L.check(L.lib.rr_op_add_rmsnorm(xd.data_ptr(), planes.data_ptr(), 0, n, rows * hidden, hidden, nw.data_ptr(),
                                    xn.data_ptr(), rows, hidden, eps, None), "rr_op_add_rmsnorm")
    torch.cuda.synchronize()
    acc = planes[0].clone()
    for z in range(1, n):
        acc = acc + planes[z]
    want = x + acc
    assert torch.equal(_bits(xd), _bits(want)), "residual differs from x + (((p0 + p1) + ...) in fp32"
    assert torch.isnan(xn[rows:]).all(), "xn written past rows"
    r64 = want.double()
    ref = r64 * torch.rsqrt(r64.pow(2).mean(1, keepdim=True) + eps) * nw.double()
    delta = (0.51 * (hidden + 1) + 8) * U24
    err = (xn[:rows].double() - ref).abs()
    worst = (err / ((2.0 ** -8 * (1 + delta) + delta) * ref.abs())).max().item()
    assert worst <= 1.0, f"xn: worst err / bound = {worst:.3g}"


@pytest.mark.parametrize("rows", ROWS)
def test_silu_mul_over_small_gate_up_planes(rows, default_path):
    """`small` runs gate/up as two fp32 planes over [gate; up], then rr_op_silu_mul sums them and applies SiLU * up."""
    L = _L()
    w, rows_w, K, mode, lm_head, n, fused = _case("small", "gu", rows)
    assert mode == F32 and not fused
    if n != 2:
        pytest.skip(f"two gate/up planes at 132 SMs; this GPU's rule gives {n}")
    planes = _run(w, None, rows_w, K, _xn(K, rows), rows, mode, lm_head, n)[1]
    inter = rows_w // 2
    act = torch.full((rows + 1, inter), float("nan"), device="cuda", dtype=torch.bfloat16)
    L.check(L.lib.rr_op_silu_mul(planes.data_ptr(), 0, n, rows * rows_w, rows_w, act.data_ptr(), rows, inter, None),
            "rr_op_silu_mul")
    torch.cuda.synchronize()
    assert torch.isnan(act[rows:]).all(), "act written past rows"
    p = planes.double()
    g = p[0, :, :inter] + p[1, :, :inter]
    u = p[0, :, inter:] + p[1, :, inter:]
    sg = g / (1 + torch.exp(-g))
    ref = sg * u
    e = U23 * ((8 + 1.16 * g.abs()) * ref.abs() + 1.1 * u.abs() * g.abs() + sg.abs() * u.abs())
    err = (act[:rows].double() - ref).abs()
    worst = (err / (2.0 ** -8 * (ref.abs() + e) + e)).max().item()
    assert worst <= 1.0, f"act: worst err / bound = {worst:.3g}"
