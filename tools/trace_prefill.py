"""In-situ timeline of one prefill chunk (16 x 512 tokens): critical-path segment per kernel type
(dependency-resolved stamps, see tools/trace_step.py)."""
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
g = torch.Generator().manual_seed(0)
prompts = [torch.randint(0, spec.vocab, (512,), generator=g).tolist() for _ in range(16)]
eng.prefill(prompts, list(range(16)))
N = 1000
_lib.check(_lib.lib.rr_debug_trace_start(N))
eng.prefill(prompts, list(range(16)))
buf = (C.c_uint64 * (4 * N))(); n = C.c_int32()
_lib.check(_lib.lib.rr_debug_trace_stop(buf, N, C.byref(n)))
a = np.frombuffer(buf, dtype=np.uint64)[: 4 * n.value].reshape(-1, 4).astype(np.int64)
a = a[np.argsort(a[:, 1])]
print(f"{n.value} kernels; chunk span {(a[-1, 3] - a[0, 1]) / 1e6:.2f} ms")
# per layer (after embed, norm0): deferred RMSNorm, so no norm kernels inside the layers
names = ["gemm_qkv(+rope,*rinv)", "attn", "gemm_o(+resid,xhat)", "gemm_gate_up(+silu,*rinv)", "gemm_down(+resid,xhat)"]
PER = len(names)
agg = {}
for i in range(len(a) - 1):
    kid, s, d, e = a[i]
    seg = (a[i + 1, 2] - d) / 1e3
    if i < 2: nm = ["embed", "norm0"][i]
    elif i < 2 + PER * spec.n_layers: nm = names[(i - 2) % PER]
    else: nm = "tail(" + NAMES.get(int(kid), str(kid)) + ")"
    x = agg.setdefault(nm, [0, 0.0, 0.0]); x[0] += 1; x[1] += seg; x[2] += (e - d) / 1e3
tot = sum(v[1] for v in agg.values())
for k, (c, seg, body) in sorted(agg.items(), key=lambda x: -x[1][1]):
    print(f"{k:26s} n={c:3d}  critical {seg / 1e3:8.2f} ms  {100 * seg / tot:5.1f}%  avg {seg / c:8.1f} us  (CTA0 body {body / c:8.1f} us)")
print(f"total {tot / 1e3:.2f} ms")
eng.close()
