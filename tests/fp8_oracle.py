"""Reference of the FP8 weight rule (csrc/rr_fp8.cu): per-row power-of-two scale, e4m3 round-to-nearest-even through
torch.float8_e4m3fn, and the exact dequantization bf16(Q * s).  Device-agnostic torch code: it runs on CPU tensors, or on
the GPU for the large projection shapes."""
import torch

E_MIN, E_MAX = -117, 127


def row_exponents(w: torch.Tensor) -> torch.Tensor:
    """e[n] = the smallest integer with max_k |w[n, k]| <= 448 * 2^e, clamped to [E_MIN, E_MAX]; 0 for a zero row."""
    a = w.double().abs().amax(1)
    _, E = torch.frexp(a)                       # a = m 2^E, m in [0.5, 1)
    e = E.long() - 9
    e = e + (a > torch.ldexp(torch.full_like(a, 448.0), e)).long()
    e = e.clamp(E_MIN, E_MAX)
    return torch.where(a > 0, e, torch.zeros_like(e))


def quantize(w: torch.Tensor):
    """bf16 [N, K] -> (Q float8_e4m3fn [N, K], scale fp32 [N])."""
    e = row_exponents(w)
    q = (w.double() * torch.ldexp(torch.ones_like(e, dtype=torch.float64), -e)[:, None]).to(torch.float8_e4m3fn)
    return q, torch.ldexp(torch.ones_like(e, dtype=torch.float64), e).float()


def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """bf16(Q * s), exact."""
    return (q.double() * scale.double()[:, None]).bfloat16()
