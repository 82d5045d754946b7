"""Prefill-orientation GEMM (128 x 256 tiles, two consumer warpgroups) at the edges of its tiling: token-tile counts that
leave the last CTA of a wave alone, weight-row counts that end in half a 256-wide tile, K that ends in a partial k-block,
and back-to-back launches of the persistent grid.  References are torch fp32 of the same op."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MODE_BF16, MODE_SILU, MODE_RESID = 0, 3, 5


def _lib():
    from rr_b200 import _lib
    return _lib


def _launch(A, B, out, ldo, mode):
    L = _lib()
    rc = L.lib.rr_gemm_bf16(A.data_ptr(), A.shape[0], A.stride(0), B.data_ptr(), B.shape[0], B.stride(0), A.shape[1],
                            out.data_ptr(), ldo, 0, 1, mode, 256, None)
    L.check(rc, "rr_gemm_bf16")


def _operands(T, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(T, K, device="cuda", generator=g).bfloat16()
    B = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    return A, B, g


def _interleave64(w, inter):
    g, u = w[:inter].view(-1, 64, w.shape[1]), w[inter:].view(-1, 64, w.shape[1])
    return torch.stack([g, u], 1).reshape(2 * inter, w.shape[1]).contiguous()


# rowsA: 2, 3 and 8 token tiles; rowsB = 128 mod 256; K = 64 k + {8, 40}
SHAPES = [(130, 384, 200), (257, 640, 72), (1000, 4224, 1000), (257, 128, 520)]


@pytest.mark.parametrize("T,N,K", SHAPES)
def test_prefill_gemm_bf16_ragged(T, N, K):
    A, B, _ = _operands(T, N, K, T + N + K)
    out = torch.full((T, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    _launch(A, B, out, N, MODE_BF16)
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    got = out.float()
    assert torch.isfinite(got).all()
    assert (got - ref).abs().max().item() <= 6e-3 * ref.abs().max().item() + 1e-4


@pytest.mark.parametrize("T,N,K", SHAPES)
def test_prefill_gemm_silu_ragged(T, N, K):
    inter = N // 2                                  # N = 128 mod 256: the last tile holds one gate/up pair
    A, B, _ = _operands(T, 2 * inter, K, 3 * T + K)
    act = torch.full((T, inter), float("nan"), device="cuda", dtype=torch.bfloat16)
    _launch(A, _interleave64(B, inter), act, inter, MODE_SILU)
    torch.cuda.synchronize()
    y = A.float() @ B.float().t()
    ref = torch.nn.functional.silu(y[:, :inter]) * y[:, inter:]
    assert torch.isfinite(act.float()).all()
    assert torch.allclose(act.float(), ref, atol=2e-2 * ref.abs().max().item(), rtol=2e-2)


@pytest.mark.parametrize("T,N,K", SHAPES)
def test_prefill_gemm_residual_ragged(T, N, K):
    A, B, g = _operands(T, N, K, 5 * T + N)
    x = torch.randn(T, N + 8, device="cuda", generator=g)       # pitch wider than N: columns >= N stay untouched
    ref = x.clone()
    ref[:, :N] += A.float() @ B.float().t()
    _launch(A, B, x, N + 8, MODE_RESID)
    torch.cuda.synchronize()
    assert torch.equal(x[:, N:], ref[:, N:])
    assert torch.allclose(x, ref, atol=1e-3 * ref.abs().max().item(), rtol=1e-4)


def test_prefill_gemm_back_to_back_launches():
    """Two launches on one stream without a host sync in between: the second one's CTAs reuse the persistent grid and
    read the residual the first one wrote."""
    T, N, K = 1000, 4224, 1000
    A, B, g = _operands(T, N, K, 11)
    x = torch.randn(T, N, device="cuda", generator=g)
    ref = x + 2.0 * (A.float() @ B.float().t())
    _launch(A, B, x, N, MODE_RESID)
    _launch(A, B, x, N, MODE_RESID)
    torch.cuda.synchronize()
    assert torch.allclose(x, ref, atol=2e-3 * ref.abs().max().item(), rtol=1e-4)
