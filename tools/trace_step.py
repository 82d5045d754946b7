"""In-graph timeline of one decode step (CTA-0 globaltimer stamps, rr_debug_trace_*): per kernel type the time
CTA 0 is resident, and the gap between consecutive kernels' starts/ends — shows what the CUDA-graph + PDL
execution really looks like (ncu serialises launches)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from rr_b200 import _lib
from rr_b200.models import SPECS, make_weights
from rr_b200.engine import Engine
NAMES = {1: "gemm_dec", 2: "gemm_pf", 3: "attn_dec", 4: "attn_pf", 5: "norm", 6: "rope", 7: "silu", 8: "embed", 9: "argmax"}
spec = SPECS["llama-3-8b"]
w = make_weights(spec, seed=0, device="cuda")
eng = Engine(w, max_batch=64, ctx_max=640, max_prefill_tokens=8192)
ids = np.random.RandomState(0).randint(0, spec.vocab, size=(64, 512)).astype(np.int32)
start = np.arange(0, 64 * 512 + 1, 512, dtype=np.int32)
eng.run_batch(ids.reshape(-1), start, 8)                      # warm-up + graph capture
N = 6000
_lib.check(_lib.lib.rr_debug_trace_start(N))
eng.run_batch(ids.reshape(-1), start, 6)
buf = (C.c_uint64 * (4 * N))(); n = C.c_int32()
_lib.check(_lib.lib.rr_debug_trace_stop(buf, N, C.byref(n)))
a = np.frombuffer(buf, dtype=np.uint64)[: 4 * n.value].reshape(-1, 4).astype(np.int64)
a = a[np.argsort(a[:, 1])]
L = spec.n_layers
layer_names = ["gemm_qkv", "attn(+rope)", "gemm_o", "norm_mlp", "mlp(gate_up+down)", "norm_next"]   # 64 rows: fused MLP
PER = len(layer_names)
n_step = 2 + PER * L + 2
dec = a[-n_step:]                                               # last decode step
t0 = dec[0, 1]
print(f"{n.value} kernels traced; last decode step ({n_step} launches): {(dec[-1, 3] - t0) / 1e3:.1f} us first start -> last end")
# critical-path segment of kernel k = (dependency of kernel k+1 resolved) - (dependency of kernel k resolved):
# griddepcontrol.wait returns when the WHOLE preceding grid has completed and flushed.
agg = {}
for i in range(len(dec) - 1):
    kid, s_, d, e = dec[i]
    seg = (dec[i + 1, 2] - d) / 1e3
    if i < 2: name = ["embed", "norm0"][i]
    elif i < 2 + PER * L: name = layer_names[(i - 2) % PER]
    else: name = "gemm_lm_head"
    a_ = agg.setdefault(name, [0, 0.0, 0.0]); a_[0] += 1; a_[1] += seg; a_[2] += (e - d) / 1e3
tot = sum(v[1] for v in agg.values())
print("kernel          n   critical-path us (sum)  share   avg us   avg CTA0 body us")
for k, (c, seg, body) in sorted(agg.items(), key=lambda x: -x[1][1]):
    print(f"{k:14s} {c:3d}   {seg:10.1f}          {100 * seg / tot:5.1f}%  {seg / c:6.1f}   {body / c:6.1f}")
print(f"total {tot:.1f} us (+ argmax)")
eng.close()
