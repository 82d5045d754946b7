"""How fast can a SUBSET of the SMs stream weights?  Decode-orientation GEMM (rr_gemm_bf16, OUT_TRANSPOSED_F32, 64 batch
rows, no split-K) with exactly n_tiles 128-row weight tiles = n_tiles CTAs, K = 4096..16384: bytes / time / n_tiles =
per-SM streaming rate.  Decides whether a projection can skip split-K (fewer, longer CTAs) without losing bandwidth."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tools.gemm_probe import time_gemm
for K in (4096, 14336):
    for n_tiles in (16, 32, 64, 96, 128, 132):
        N = n_tiles * 128
        nc = max(2, int(300e6 / (N * K * 2)) + 1)
        ms = time_gemm(N, 64, K, 1, 64, 1, iters=20, ncopies=min(nc, 24))
        gb = N * K * 2 / ms / 1e6
        print(f"K={K:5d} CTAs={n_tiles:3d}: {ms*1e3:7.1f} us  total {gb:6.0f} GB/s  per SM {gb / n_tiles:6.1f} GB/s")
