"""Parity of the wgmma GEMM (rr_gemm_bf16) against a torch fp32 reference of the same op.
Tolerance: bf16 inputs are exact in both; fp32 accumulation order differs -> |err| <= 2e-3 * sqrt(K)
relative to |a||b| scale for fp32 out, plus one bf16 rounding (2^-8 relative) for bf16 out."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _gemm(A, B, mode, bn, splits=1, ld_rows=None):
    from rr_b200 import _lib
    rowsA, K = A.shape
    rowsB = B.shape[0]
    if mode == 0:
        out = torch.full((rowsA, rowsB), float("nan"), device="cuda", dtype=torch.bfloat16)
        ldo, ldr = rowsB, 0
    else:
        ldr = ld_rows or rowsB
        out = torch.full((splits, ldr, rowsA), float("nan"), device="cuda", dtype=torch.float32)
        ldo = rowsA
    rc = _lib.lib.rr_gemm_bf16(A.data_ptr(), rowsA, A.stride(0), B.data_ptr(), rowsB, B.stride(0),
                               K, out.data_ptr(), ldo, ldr, splits, mode, bn, None)
    _lib.check(rc, "rr_gemm_bf16")
    torch.cuda.synchronize()
    return out


CASES_T = [  # decode orientation: rowsA = weight rows, rowsB = batch
    (128, 16, 64, 16, 1), (256, 64, 512, 64, 1), (384, 33, 4096, 64, 3), (4096, 64, 4096, 64, 4),
    (1000, 7, 320, 16, 2), (6144, 64, 4096, 64, 3), (512, 128, 1024, 128, 2), (640, 20, 14336, 32, 7),
]


@pytest.mark.parametrize("rowsA,rowsB,K,bn,splits", CASES_T)
def test_gemm_transposed_f32(rowsA, rowsB, K, bn, splits):
    g = torch.Generator(device="cuda").manual_seed(rowsA * 7 + rowsB)
    A = (torch.randn(rowsA, K, device="cuda", generator=g) * 0.05).bfloat16()
    B = torch.randn(rowsB, K, device="cuda", generator=g).bfloat16()
    out = _gemm(A, B, 1, bn, splits)
    got = out.sum(0)                      # [rowsB, rowsA]
    ref = B.float() @ A.float().t()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 1e-3 * scale + 1e-4, (err, scale)


@pytest.mark.parametrize("rowsA,rowsB,K,bn,splits,ld_rows", [(384, 33, 512, 64, 3, 64), (1000, 7, 320, 16, 2, 8), (6144, 64, 4096, 64, 3, 64),
                                                          (4096, 20, 1024, 32, 4, 32)])
def test_decode_gemm_tma_store_epilogue_equals_lsu_epilogue_and_clips(rowsA, rowsB, K, bn, splits, ld_rows, monkeypatch):
    """Decode orientation: the planes tile goes out as ONE TMA store per item (3-D tensor map [split][row][feature]).  It must
    write exactly the bits of the per-thread store epilogue (RR_NO_TMA_EPI=1, read when the plan is built) and must not touch
    plane rows >= rowsB (the map's row extent is rowsB, not the plane pitch)."""
    g = torch.Generator(device="cuda").manual_seed(rowsA + 31 * rowsB)
    A = (torch.randn(rowsA, K, device="cuda", generator=g) * 0.05).bfloat16()
    B = torch.randn(rowsB, K, device="cuda", generator=g).bfloat16()
    monkeypatch.delenv("RR_NO_TMA_EPI", raising=False)
    tma = _gemm(A, B, 1, bn, splits, ld_rows=ld_rows)
    monkeypatch.setenv("RR_NO_TMA_EPI", "1")
    lsu = _gemm(A, B, 1, bn, splits, ld_rows=ld_rows)
    assert torch.isfinite(tma[:, :rowsB]).all()
    assert torch.equal(tma[:, :rowsB], lsu[:, :rowsB])
    if ld_rows > rowsB:
        assert torch.isnan(tma[:, rowsB:]).all() and torch.isnan(lsu[:, rowsB:]).all()


CASES_R = [(128, 256, 64, 256), (512, 6144, 4096, 256), (1000, 520, 256, 128), (2048, 4096, 4096, 256),
           (130, 72, 128, 64), (4096, 28672, 4096, 256),
           # ragged shapes with bn 256 (run as 128-wide tiles): partial tiles on both axes
           (1000, 520, 256, 256), (300, 304, 192, 256), (257, 8200, 64, 256), (8192, 1024, 4096, 256)]


@pytest.mark.parametrize("rowsA,rowsB,K,bn", CASES_R)
def test_gemm_rowmajor_bf16(rowsA, rowsB, K, bn):
    g = torch.Generator(device="cuda").manual_seed(rowsA + rowsB)
    A = torch.randn(rowsA, K, device="cuda", generator=g).bfloat16()
    B = (torch.randn(rowsB, K, device="cuda", generator=g) * 0.05).bfloat16()
    got = _gemm(A, B, 0, bn).float()
    ref = A.float() @ B.float().t()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 6e-3 * scale + 1e-4, (err, scale)


def test_gemm_exact_small_integers():
    """Integer-valued operands: every product and partial sum is exact in fp32 -> bit-exact."""
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randint(-4, 5, (256, 512), device="cuda", generator=g).bfloat16()
    B = torch.randint(-4, 5, (64, 512), device="cuda", generator=g).bfloat16()
    got = _gemm(A, B, 1, 64, 2).sum(0)
    ref = B.float() @ A.float().t()
    assert torch.equal(got, ref)


def _interleave64(w, inter):
    g, u = w[:inter].view(-1, 64, w.shape[1]), w[inter:].view(-1, 64, w.shape[1])
    return torch.stack([g, u], 1).reshape(2 * inter, w.shape[1]).contiguous()


@pytest.mark.parametrize("inter,K,B,bn", [(14336, 4096, 64, 64), (1024, 512, 37, 64), (2816, 1024, 20, 32), (1024, 512, 128, 128)])
def test_gemm_fused_silu_decode_orientation(inter, K, B, bn):
    from rr_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(inter + B)
    W = (torch.randn(2 * inter, K, device="cuda", generator=g) * 0.05).bfloat16()        # [gate; up]
    X = torch.randn(B, K, device="cuda", generator=g).bfloat16()
    Wil = _interleave64(W, inter)
    act = torch.full((B, inter), float("nan"), device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib.rr_gemm_bf16(Wil.data_ptr(), 2 * inter, K, X.data_ptr(), B, K, K, act.data_ptr(), inter, 0, 1, 2, bn, None))
    torch.cuda.synchronize()
    y = X.float() @ W.float().t()
    ref = torch.nn.functional.silu(y[:, :inter]) * y[:, inter:]
    assert torch.isfinite(act.float()).all()
    assert torch.allclose(act.float(), ref, atol=2e-2 * ref.abs().max().item(), rtol=2e-2)


@pytest.mark.parametrize("inter,K,T", [(14336, 4096, 1024), (1024, 512, 300), (2816, 1024, 130)])
def test_gemm_fused_silu_prefill_orientation(inter, K, T):
    from rr_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(inter + T)
    W = (torch.randn(2 * inter, K, device="cuda", generator=g) * 0.05).bfloat16()
    X = torch.randn(T, K, device="cuda", generator=g).bfloat16()
    Wil = _interleave64(W, inter)
    act = torch.full((T, inter), float("nan"), device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib.rr_gemm_bf16(X.data_ptr(), T, K, Wil.data_ptr(), 2 * inter, K, K, act.data_ptr(), inter, 0, 1, 3, 256, None))
    torch.cuda.synchronize()
    y = X.float() @ W.float().t()
    ref = torch.nn.functional.silu(y[:, :inter]) * y[:, inter:]
    assert torch.isfinite(act.float()).all()
    assert torch.allclose(act.float(), ref, atol=2e-2 * ref.abs().max().item(), rtol=2e-2)


def test_gemm_residual_epilogue():
    """OUT_ROWMAJOR_RESID: fp32 residual += A @ B^T (prefill O / down projections)."""
    from rr_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(77)
    T, N, K = 1000, 4096, 512
    A = torch.randn(T, K, device="cuda", generator=g).bfloat16()
    B = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    x = torch.randn(T, N, device="cuda", generator=g)
    ref = x + A.float() @ B.float().t()
    _lib.check(_lib.lib.rr_gemm_bf16(A.data_ptr(), T, K, B.data_ptr(), N, K, K, x.data_ptr(), N, 0, 1, 5, 256, None))
    torch.cuda.synchronize()
    assert torch.allclose(x, ref, atol=1e-3 * ref.abs().max().item(), rtol=1e-4)
