"""Model descriptors and seeded synthetic weights for the on-box replicas that replace the
reference's `litellm_params.model: bedrock/...` deployments (reference config/config.yaml:39-91).

No checkpoints or tokenizers exist on the box (SURVEY.md §0.4), so replicas are instantiated at the
exact architecture shapes with seeded random weights (BASELINE.md §3: manual_seed(0), sigma 0.02,
bf16).  Weight layout is what librr_b200.so consumes: torch nn.Linear convention
[out_features, in_features], q/k/v fused row-wise into `wqkv`, gate/up fused into `wgu`.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch


@dataclass(frozen=True)
class ModelSpec:
    name: str
    vocab: int
    hidden: int
    inter: int
    n_layers: int
    n_heads: int
    n_kv_heads: int
    head_dim: int = 128
    rope_theta: float = 500000.0
    rms_eps: float = 1e-5
    # sliding-window attention W (0: full causal): position q attends to positions max(0, q - W + 1) .. q
    sliding_window: int = 0

    @property
    def n_params(self) -> int:
        per_layer = (self.hidden * (self.n_heads + 2 * self.n_kv_heads) * self.head_dim
                     + self.n_heads * self.head_dim * self.hidden + 3 * self.hidden * self.inter
                     + 2 * self.hidden)
        return 2 * self.vocab * self.hidden + self.n_layers * per_layer + self.hidden

    @property
    def weight_bytes_per_decode_step(self) -> int:
        """bf16 bytes streamed once per decode step: every layer + final norm + lm_head
        (the embedding table is gathered, not streamed) — BASELINE.md §4."""
        per_layer = (self.hidden * (self.n_heads + 2 * self.n_kv_heads) * self.head_dim
                     + self.n_heads * self.head_dim * self.hidden + 3 * self.hidden * self.inter
                     + 2 * self.hidden)
        return 2 * (self.n_layers * per_layer + self.hidden + self.vocab * self.hidden)

    @property
    def kv_bytes_per_token(self) -> int:
        return 2 * self.n_layers * self.n_kv_heads * self.head_dim * 2

    @property
    def prefill_flops_per_token(self) -> int:
        """2 * (matmul parameters touched per token), attention excluded (<1 % at 512 tokens)."""
        per_layer = (self.hidden * (self.n_heads + 2 * self.n_kv_heads) * self.head_dim
                     + self.n_heads * self.head_dim * self.hidden + 3 * self.hidden * self.inter)
        return 2 * (self.n_layers * per_layer + self.vocab * self.hidden)


SPECS: Dict[str, ModelSpec] = {
    "llama-3-8b": ModelSpec("llama-3-8b", 128256, 4096, 14336, 32, 32, 8, 128, 500000.0, 1e-5),
    # Mistral-7B-v0.1: MistralConfig().sliding_window = 4096
    "mistral-7b": ModelSpec("mistral-7b", 32000, 4096, 14336, 32, 32, 8, 128, 10000.0, 1e-5, 4096),
    # Phi-3-mini-4k: fused qkv / gate_up are layout only (our layout is fused anyway); head_dim 96, MHA
    "phi-3-mini": ModelSpec("phi-3-mini", 32064, 3072, 8192, 32, 32, 32, 96, 10000.0, 1e-5),
    # small shapes for parity tests / smoke (same kernels, same code path)
    "tiny": ModelSpec("tiny", 1024, 512, 1024, 2, 4, 2, 128, 500000.0, 1e-5),
    "small": ModelSpec("small", 4096, 1024, 2816, 4, 8, 2, 128, 10000.0, 1e-5),
    "llama-3-8b-2l": ModelSpec("llama-3-8b-2l", 128256, 4096, 14336, 2, 32, 8, 128, 500000.0, 1e-5),
    "phi-3-mini-2l": ModelSpec("phi-3-mini-2l", 32064, 3072, 8192, 2, 32, 32, 96, 10000.0, 1e-5),
    "mistral-7b-2l": ModelSpec("mistral-7b-2l", 32000, 4096, 14336, 2, 32, 8, 128, 10000.0, 1e-5, 4096),
    # the tiny shape with a 100-token window (not a multiple of 64), for window tests that run past W in seconds
    "tiny-sw": ModelSpec("tiny-sw", 1024, 512, 1024, 2, 4, 2, 128, 500000.0, 1e-5, 100),
    "tiny96": ModelSpec("tiny96", 1024, 384, 1024, 2, 4, 4, 96, 10000.0, 1e-5),
    "small96": ModelSpec("small96", 4096, 768, 2048, 3, 8, 2, 96, 10000.0, 1e-5),
}


def ring_pages(sliding_window: int, max_prefill_tokens: int) -> int:
    """64-token KV pages a windowed engine's ring request reserves per choice: ceil((W + Tmax - 2) / 64) + 1, the most
    pages the W + Tmax - 1 positions a prefill piece reads or writes can touch, Tmax the engine's prefill chunk
    (rr_engine.cu ring_pages); 0 without a window.  A choice reserves min(ceil(reach / 64), ring)."""
    if sliding_window <= 0:
        return 0
    tmax = max(16, max_prefill_tokens if max_prefill_tokens > 0 else 8192)
    return -(-(sliding_window + tmax - 2) // 64) + 1


def resolve_spec(model: str) -> ModelSpec:
    """`b200/llama-3-8b`, `llama-3-8b`, ... -> ModelSpec."""
    key = model.split("/", 1)[-1].split("@", 1)[0].lower()
    if key not in SPECS:
        raise KeyError(f"unknown local model {model!r}; known: {sorted(SPECS)}")
    return SPECS[key]


@dataclass
class Weights:
    spec: ModelSpec
    embed: torch.Tensor
    lm_head: torch.Tensor
    final_norm: torch.Tensor
    wqkv: List[torch.Tensor] = field(default_factory=list)
    wo: List[torch.Tensor] = field(default_factory=list)
    wgu: List[torch.Tensor] = field(default_factory=list)
    wdown: List[torch.Tensor] = field(default_factory=list)
    norm_attn: List[torch.Tensor] = field(default_factory=list)
    norm_mlp: List[torch.Tensor] = field(default_factory=list)
    flat: Optional[torch.Tensor] = None      # the one allocation every tensor above is a view of (make_weights); None after .to()

    def tensors(self) -> List[torch.Tensor]:
        out = [self.embed, self.lm_head, self.final_norm]
        for lst in (self.wqkv, self.wo, self.wgu, self.wdown, self.norm_attn, self.norm_mlp):
            out.extend(lst)
        return out

    def to(self, device) -> "Weights":
        mv = lambda t: t.to(device)
        return Weights(self.spec, mv(self.embed), mv(self.lm_head), mv(self.final_norm),
                       [mv(t) for t in self.wqkv], [mv(t) for t in self.wo],
                       [mv(t) for t in self.wgu], [mv(t) for t in self.wdown],
                       [mv(t) for t in self.norm_attn], [mv(t) for t in self.norm_mlp])

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.tensors())


def make_weights(spec: ModelSpec, seed: int = 0, sigma: float = 0.02, device="cuda",
                 norm_jitter: float = 0.0, allocate_only: bool = False) -> Weights:
    """Seeded N(0, sigma^2) bf16 weights (norm weights 1 + norm_jitter * N(0,1)).

    The generator lives on `device`, so values are reproducible per (torch version, device type);
    parity tests share the tensors with the oracle instead of regenerating them.
    `allocate_only` leaves the values uninitialised (ranks > 0 before the start-up NCCL broadcast).
    """
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(seed)
    nq, nkv = spec.n_heads * spec.head_dim, spec.n_kv_heads * spec.head_dim
    # ONE flat allocation, every tensor a 256-byte-aligned view of it: the start-up weight broadcast is then a single
    # ncclBroadcast instead of 195 small ones (broadcast_weights)
    shapes = [(spec.vocab, spec.hidden), (spec.vocab, spec.hidden), (spec.hidden,)]
    for _ in range(spec.n_layers):
        shapes += [(nq + 2 * nkv, spec.hidden), (spec.hidden, nq), (2 * spec.inter, spec.hidden), (spec.hidden, spec.inter),
                   (spec.hidden,), (spec.hidden,)]
    offs, total = [], 0
    for sh in shapes:
        n = 1
        for d in sh:
            n *= d
        offs.append(total)
        total += (n + 127) // 128 * 128
    flat = torch.empty(total, device=dev, dtype=torch.bfloat16)
    views = iter([flat[o: o + torch.Size(sh).numel()].view(*sh) for o, sh in zip(offs, shapes)])

    def rnd(*shape):
        out = next(views)
        assert tuple(out.shape) == tuple(shape)
        if allocate_only:
            return out
        rows = shape[0]
        step = max(1, (1 << 26) // max(1, shape[1]))      # bound the fp32 temporary to 256 MB
        for r0 in range(0, rows, step):
            r1 = min(rows, r0 + step)
            out[r0:r1] = (torch.randn(r1 - r0, shape[1], device=dev, generator=g) * sigma).bfloat16()
        return out

    def norm():
        out = next(views)
        if allocate_only:
            return out
        w = torch.ones(spec.hidden, device=dev)
        if norm_jitter:
            w = w + norm_jitter * torch.randn(spec.hidden, device=dev, generator=g)
        out.copy_(w.bfloat16())
        return out

    w = Weights(spec, rnd(spec.vocab, spec.hidden), rnd(spec.vocab, spec.hidden), norm())
    for _ in range(spec.n_layers):
        w.wqkv.append(rnd(nq + 2 * nkv, spec.hidden))
        w.wo.append(rnd(spec.hidden, nq))
        w.wgu.append(rnd(2 * spec.inter, spec.hidden))
        w.wdown.append(rnd(spec.hidden, spec.inter))
        w.norm_attn.append(norm())
        w.norm_mlp.append(norm())
    w.flat = flat
    return w


@dataclass
class Fp8Weights:
    """Weights with e4m3 layer projections (`litellm_params.quantization: fp8`): each of wqkv / wo / wgu / wdown is
    Q [N, K] torch.float8_e4m3fn with one fp32 row scale s[n] = 2^e[n] (`*_scale`, [N]); embed, lm_head and the norms
    stay bf16.  The engine computes exactly what a bf16 engine computes on dequantize() = bf16(Q * s)
    (include/rr_b200.h, RR_WEIGHTS_FP8_E4M3)."""
    spec: ModelSpec
    embed: torch.Tensor
    lm_head: torch.Tensor
    final_norm: torch.Tensor
    wqkv: List[torch.Tensor] = field(default_factory=list)
    wo: List[torch.Tensor] = field(default_factory=list)
    wgu: List[torch.Tensor] = field(default_factory=list)
    wdown: List[torch.Tensor] = field(default_factory=list)
    norm_attn: List[torch.Tensor] = field(default_factory=list)
    norm_mlp: List[torch.Tensor] = field(default_factory=list)
    wqkv_scale: List[torch.Tensor] = field(default_factory=list)
    wo_scale: List[torch.Tensor] = field(default_factory=list)
    wgu_scale: List[torch.Tensor] = field(default_factory=list)
    wdown_scale: List[torch.Tensor] = field(default_factory=list)

    PROJ = ("wqkv", "wo", "wgu", "wdown")

    def tensors(self) -> List[torch.Tensor]:
        out = [self.embed, self.lm_head, self.final_norm]
        for name in self.PROJ:
            out.extend(getattr(self, name))
            out.extend(getattr(self, name + "_scale"))
        out.extend(self.norm_attn)
        out.extend(self.norm_mlp)
        return out

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.tensors())

    def dequantize(self) -> Weights:
        """bf16(Q * s) of every projection (rr_op_dequantize_fp8_weight), exact; embed, lm_head and the norms are shared."""
        from . import _lib
        stream = torch.cuda.current_stream(self.embed.device).cuda_stream
        w = Weights(self.spec, self.embed, self.lm_head, self.final_norm,
                    norm_attn=list(self.norm_attn), norm_mlp=list(self.norm_mlp))
        for name in self.PROJ:
            for q, sc in zip(getattr(self, name), getattr(self, name + "_scale")):
                d = torch.empty(q.shape, dtype=torch.bfloat16, device=q.device)
                _lib.check(_lib.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), sc.data_ptr(), q.shape[0], q.shape[1],
                                                                d.data_ptr(), q.shape[1], stream),
                           "rr_op_dequantize_fp8_weight")
                getattr(w, name).append(d)
        return w


def quantize_fp8(w: Weights) -> Fp8Weights:
    """Per-row power-of-two e4m3 quantization of the layer projections on the GPU (rr_op_quantize_fp8_weight): row n gets
    e[n] = the smallest integer with max |W[n]| <= 448 * 2^e, clamped to [-117, 127] (0 for a zero row), and
    Q = e4m3_rne(W / 2^e).  embed, lm_head and the norms are cloned into allocations of their own, so the result keeps no
    reference to `w` and dropping `w` frees all of its memory.  Raises for a row with Inf or NaN."""
    from . import _lib
    stream = torch.cuda.current_stream(w.embed.device).cuda_stream
    out = Fp8Weights(w.spec, w.embed.clone(), w.lm_head.clone(), w.final_norm.clone(),
                     norm_attn=[t.clone() for t in w.norm_attn], norm_mlp=[t.clone() for t in w.norm_mlp])
    for name in Fp8Weights.PROJ:
        for t in getattr(w, name):
            assert t.dtype == torch.bfloat16 and t.is_contiguous() and t.dim() == 2
            q = torch.empty(t.shape, dtype=torch.float8_e4m3fn, device=t.device)
            sc = torch.empty(t.shape[0], dtype=torch.float32, device=t.device)
            _lib.check(_lib.lib.rr_op_quantize_fp8_weight(t.data_ptr(), t.shape[0], t.shape[1], t.shape[1], q.data_ptr(),
                                                          sc.data_ptr(), stream), "rr_op_quantize_fp8_weight")
            getattr(out, name).append(q)
            getattr(out, name + "_scale").append(sc)
    return out


def broadcast_weights(w: Weights, src: int = 0, group=None) -> None:
    """Start-up weight broadcast (K12): rank `src` -> every replica of the model group over
    NCCL/NVLink.  The only collective on the path; requests never cross GPUs afterwards.
    Weights made by make_weights live in one flat buffer: ONE ncclBroadcast of 16 GB (round 1 issued 195 per-tensor calls
    and reached ~70 % of the link rate)."""
    import torch.distributed as dist
    if w.flat is not None:
        dist.broadcast(w.flat, src=src, group=group)
        return
    for t in w.tensors():
        dist.broadcast(t, src=src, group=group)
