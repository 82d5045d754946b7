"""Kernel-level parity of the fused decode MLP (gemm_mlp_wgmma, csrc/rr_gemm.cu) through rr_op_decode_mlp, which runs it
exactly as the engine does: same tile width, K slices, grid and schedule.

Operands are built the way the engine sees them: xn is bf16 N(0, 1), and the gate, up and down weights are bf16 with
sigma = 1 / sqrt(K), where K is their fan-in, so g = xn . gate, u = xn . up, act and the planes are all O(1).  Gate/up rows are
interleaved in 64-row blocks as engine.py does.  References are fp64.

Tolerances.  A bf16 x bf16 product is exact in fp32, so before the output rounding the only error is the fp32 accumulation
of the wgmma main loop.  Model for a length-K dot product: one rounding of the running sum s_j per k16 step, or per internal
alignment, each at most one fp32 ulp (2^-23 |s_j|, which also allows truncation), with independent signs, and running sums
bounded by twice the final magnitude.  lambda = 8 standard deviations of that sum gives
    |err| <= 8 * 2^-23 * sqrt(K) * max_j |s_j| <= 16 * 2^-23 * sqrt(K) * max|final|.
  * planes: the reference takes the kernel's own act, so only the down GEMM's accumulation over the slice's
    K_z = 64 * (k-blocks of slice z) columns is left:  tau_plane = 16 * 2^-23 * sqrt(K_z), applied as tau_plane * max|ref_z|
    (8.1e-5 at the 1792 columns of a Llama-3-8B slice).
  * act = bf16(y) with y = silu(g) * u computed in fp32 from g and u.  With G = max(max|g|, max|u|), both accumulation errors
    are at most e = 16 * 2^-23 * sqrt(hidden) * G.  |dy/dg| = |silu'(g) u| <= 1.1 G and |dy/du| = |silu(g)| <= G, so
    |y - ref| <= 2.1 G e, plus 2^-20 |y| for __expf / __fdividef.  The bf16 rounding adds 2^-8 |y| (round to nearest), so
        |act - ref| <= 2^-8 |ref| + tau_act * max|ref|,  tau_act = (1 + 2^-8) * (34 * 2^-23 * sqrt(hidden) * G^2 / max|ref| + 2^-20)
    (6e-4 to 8e-4 for Llama-3-8B, where G^2 / max|ref| is 2 to 2.7).
The act check is elementwise.  Dropping one k-block (64 act columns) from a plane moves its reference by far more than the
plane tolerance, and the test asserts this, so a slice boundary off by one k-block cannot pass."""
import ctypes as C
import math

import pytest
import torch

from test_gemm_gpu import _interleave64

pytestmark = pytest.mark.gpu

RR_INVALID_ARGUMENT = 4
MAX_PLANES = 8                       # the engine's limit on K slices (and add_rmsnorm_dec_kernel's on planes)
U32 = 2.0 ** -23

# (hidden, inter) -> (n_slices, slice_kb) under the engine's slice rule
SHAPES = {
    (4096, 14336): (8, 28),          # Llama-3-8B / Mistral-7B
    (3072, 8192): (8, 16),           # Phi-3-mini
    (1024, 2816): (3, 15),           # `small`: slices 15 / 15 / 14, the last one ragged
    (768, 2048): (2, 16),
    (512, 1024): (1, 16),            # one slice
    (384, 1024): (1, 16),            # three down tiles
    (576, 1088): (2, 9),             # hidden = 64 mod 128: half-empty last down tile; 17 gate/up tiles -> slices 9 + 8
}
ROWS = (17, 32, 33, 64, 65, 128)     # tile widths 32 / 64 / 128, full tiles and tiles with 31 or 63 zero-filled rows
CASES = [pytest.param(h, i, r, id=f"{h}x{i}-rows{r}") for (h, i) in SHAPES for r in ROWS]


def _bn(rows):
    return 32 if rows <= 32 else (64 if rows <= 64 else 128)


_OPS = {}


def _operands(hidden, inter):
    """Seeded operands of one shape; the last shape is cached (the tests run shape by shape)."""
    key = (hidden, inter)
    if key not in _OPS:
        _OPS.clear()
        g = torch.Generator(device="cuda").manual_seed(hidden * 131 + inter)
        x = torch.randn(129, hidden, device="cuda", generator=g).bfloat16()
        wgu = (torch.randn(2 * inter, hidden, device="cuda", generator=g) / math.sqrt(hidden)).bfloat16()   # [gate; up]
        wd = (torch.randn(hidden, inter, device="cuda", generator=g) / math.sqrt(inter)).bfloat16()
        _OPS[key] = dict(x=x, wgu_il=_interleave64(wgu, inter), wd=wd, wgu64=wgu.double(), wd64=wd.double())
    return _OPS[key]


def _buffers(rows, hidden, inter, ld_rows):
    """NaN-filled outputs: act with room for a whole batch tile past `rows`, planes for MAX_PLANES slices."""
    act_flat = torch.full(((_bn(rows) + 1) * inter,), float("nan"), device="cuda", dtype=torch.bfloat16)
    planes = torch.full((MAX_PLANES, ld_rows, hidden), float("nan"), device="cuda", dtype=torch.float32)
    return act_flat, planes


def _call(op, rows, hidden, inter, act_flat, planes, ld_rows):
    from rr_b200 import _lib
    ns, skb = C.c_int32(-1), C.c_int32(-1)
    rc = _lib.lib.rr_op_decode_mlp(op["wgu_il"].data_ptr(), op["wd"].data_ptr(), op["x"].data_ptr(), rows, hidden, inter,
                                   act_flat.data_ptr(), planes.data_ptr(), ld_rows, C.byref(ns), C.byref(skb), None)
    return rc, ns.value, skb.value


def _run(op, rows, hidden, inter, ld_rows):
    act_flat, planes = _buffers(rows, hidden, inter, ld_rows)
    from rr_b200 import _lib
    rc, ns, skb = _call(op, rows, hidden, inter, act_flat, planes, ld_rows)
    _lib.check(rc, "rr_op_decode_mlp")
    torch.cuda.synchronize()
    return act_flat, planes, ns, skb


def _slice_cols(z, skb, inter):
    kb1n = inter // 64
    return 64 * z * skb, 64 * min((z + 1) * skb, kb1n)


@pytest.fixture
def default_path(monkeypatch):
    """The engine's default choices: dynamic down-item schedule, TMA-store epilogues where the tile width allows them."""
    monkeypatch.delenv("RR_MLP_STATIC", raising=False)
    monkeypatch.delenv("RR_NO_TMA_EPI", raising=False)
    return monkeypatch


@pytest.mark.parametrize("hidden,inter,rows", CASES)
def test_decode_mlp_act_and_each_plane_match_fp64(hidden, inter, rows, default_path):
    op = _operands(hidden, inter)
    ld_rows = rows + 3
    act_flat, planes, ns, skb = _run(op, rows, hidden, inter, ld_rows)
    assert (ns, skb) == SHAPES[(hidden, inter)]
    act = act_flat[: rows * inter].view(rows, inter)

    # ---- nothing out of bounds, everything in bounds written
    assert torch.isfinite(act).all()
    assert torch.isfinite(planes[:ns, :rows]).all()
    assert torch.isnan(planes[:ns, rows:]).all(), "plane rows >= rows written"
    assert torch.isnan(planes[ns:]).all(), "planes >= n_slices written"
    assert torch.isnan(act_flat[rows * inter:]).all(), "act written past rows x inter"

    # ---- act against fp64 silu(x Wg^T) * (x Wu^T)
    y = op["x"][:rows].double() @ op["wgu64"].t()
    g, u = y[:, :inter], y[:, inter:]
    ref = g * u / (1.0 + torch.exp(-g))
    m = ref.abs().max().item()
    G = max(g.abs().max().item(), u.abs().max().item())
    tau_act = (1 + 2.0 ** -8) * (34 * U32 * math.sqrt(hidden) * G * G / m + 2.0 ** -20)
    assert tau_act < 2e-3
    err = (act.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + tau_act * m
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"act: worst err / bound = {worst:.3g} (tau_act {tau_act:.3g}, max|ref| {m:.3g})"

    # ---- each plane on its own, against the kernel's own act
    a64 = act.double()
    for z in range(ns):
        k0, k1 = _slice_cols(z, skb, inter)
        ref_z = a64[:, k0:k1] @ op["wd64"][:, k0:k1].t()
        tol = 16 * U32 * math.sqrt(k1 - k0) * ref_z.abs().max().item()
        e = (planes[z, :rows].double() - ref_z).abs().max().item()
        assert e <= tol, f"plane {z} (act cols {k0}:{k1}): max err {e:.3g} > {tol:.3g}"
        # the tolerance tells the slice apart from one a k-block longer or shorter at either end
        for kb0 in {k0, k1 - 64}:
            shift = (a64[:, kb0:kb0 + 64] @ op["wd64"][:, kb0:kb0 + 64].t()).abs().max().item()
            assert shift >= 10 * tol, (z, kb0, shift, tol)


@pytest.mark.parametrize("hidden,inter,rows", CASES)
def test_decode_mlp_is_bit_identical_across_schedules_epilogues_and_repeats(hidden, inter, rows, default_path):
    """Dynamic vs static down-item schedule, TMA vs per-thread store epilogues (tile width <= 64; 128 always stores per
    thread) and two back-to-back calls on one stream: which CTA computes an item, and how its tile is stored, must not
    change a bit.  act must also equal the standalone SiLU GEMM (RR_OUT_TRANSPOSED_SILU) at the same tile width: both run
    the same main loop over the full K range and the same SiLU."""
    from rr_b200 import _lib
    op = _operands(hidden, inter)
    ld_rows = rows + 3
    base_act, base_planes, ns, _ = _run(op, rows, hidden, inter, ld_rows)

    def same(act_flat, planes, what):
        assert torch.equal(act_flat[: rows * inter], base_act[: rows * inter]), f"act differs: {what}"
        assert torch.equal(planes[:ns, :rows], base_planes[:ns, :rows]), f"planes differ: {what}"

    # two calls back to back on one stream, host sync only after both
    bufs = [_buffers(rows, hidden, inter, ld_rows) for _ in range(2)]
    for act_flat, planes in bufs:
        _lib.check(_call(op, rows, hidden, inter, act_flat, planes, ld_rows)[0], "rr_op_decode_mlp")
    torch.cuda.synchronize()
    for k, (act_flat, planes) in enumerate(bufs):
        same(act_flat, planes, f"back-to-back call {k}")

    default_path.setenv("RR_MLP_STATIC", "1")
    same(*_run(op, rows, hidden, inter, ld_rows)[:2], "static schedule")
    default_path.delenv("RR_MLP_STATIC")
    if _bn(rows) <= 64:
        default_path.setenv("RR_NO_TMA_EPI", "1")
        same(*_run(op, rows, hidden, inter, ld_rows)[:2], "per-thread store epilogues")
        default_path.delenv("RR_NO_TMA_EPI")

    act2 = torch.full((rows, inter), float("nan"), device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib.rr_gemm_bf16(op["wgu_il"].data_ptr(), 2 * inter, hidden, op["x"].data_ptr(), rows, hidden, hidden,
                                     act2.data_ptr(), inter, 0, 1, 2, _bn(rows), None), "rr_gemm_bf16")
    torch.cuda.synchronize()
    assert torch.equal(act2, base_act[: rows * inter].view(rows, inter)), "act differs from the standalone SiLU GEMM"


@pytest.mark.parametrize("rows,hidden,inter,ld_rows", [
    (16, 512, 1024, 16),      # tile width 16: the engine does not fuse the MLP
    (129, 512, 1024, 129),    # wider than one batch tile
    (33, 520, 1024, 33),      # hidden % 64 != 0
    (33, 512, 1056, 33),      # inter % 64 != 0
    (33, 512, 1024, 32),      # plane pitch below rows
])
def test_decode_mlp_rejects_what_the_engine_does_not_fuse(rows, hidden, inter, ld_rows, default_path):
    """Rejected before any launch: buffers sized for the claimed shape stay untouched and the out values are not set."""
    from rr_b200 import _lib
    x = torch.randn(rows, hidden, device="cuda").bfloat16()
    wgu = (torch.randn(2 * inter, hidden, device="cuda") / math.sqrt(hidden)).bfloat16()
    wd = (torch.randn(hidden, inter, device="cuda") / math.sqrt(inter)).bfloat16()
    op = dict(x=x, wgu_il=wgu, wd=wd)
    act_flat = torch.full(((rows + 1) * inter,), float("nan"), device="cuda", dtype=torch.bfloat16)
    planes = torch.full((MAX_PLANES, max(ld_rows, rows), hidden), float("nan"), device="cuda", dtype=torch.float32)
    rc, ns, skb = _call(op, rows, hidden, inter, act_flat, planes, ld_rows)
    torch.cuda.synchronize()
    assert rc == RR_INVALID_ARGUMENT
    assert (ns, skb) == (-1, -1)
    assert torch.isnan(act_flat).all() and torch.isnan(planes).all()
