"""Prefill-orientation GEMM timing at the Llama-3-8B chunk shapes (8192 tokens): plain bf16 epilogue, fused SiLU epilogue
(mode 3, gate/up only), and torch.matmul (cuBLAS) at the same shape as the reachable-rate yardstick on the same card."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rr_b200 import _lib
lib = _lib.lib


def timed(f, iters):
    for _ in range(3): f()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(T, N, K, mode, iters=20):
    A = torch.randn(T, K, device="cuda").bfloat16(); B = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    if mode == "cublas":
        ms = timed(lambda: torch.matmul(A, B.t()), iters)
    else:
        ncol = N // 2 if mode == 3 else N
        out = torch.empty(T, ncol, device="cuda", dtype=torch.bfloat16)
        f = lambda: lib.rr_gemm_bf16(A.data_ptr(), T, K, B.data_ptr(), N, K, K, out.data_ptr(), ncol, 0, 1, mode, 256, None)
        assert f() == 0
        ms = timed(f, iters)
    return ms, 2.0 * T * N * K / ms / 1e9


for name, T, N, K in [("gate_up", 8192, 28672, 4096), ("down", 8192, 4096, 14336), ("qkv", 8192, 6144, 4096), ("o", 8192, 4096, 4096)]:
    for mode in ([0, 3, "cublas"] if name == "gate_up" else [0, "cublas"]):
        ms, tf = run(T, N, K, mode)
        label = "cuBLAS " if mode == "cublas" else f"mode {mode}"
        print(f"{name:8s} {label}: {ms:7.3f} ms  {tf:6.0f} TFLOP/s")
