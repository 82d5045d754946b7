"""Cost of logprobs on the GPU: the card, then CUDA-event time of rr_op_logprobs alone (64 x 128256 fp32 logits, k = 20)
and the Llama-3-8B decode step (64 rows, 512-token prompts) with 0 and with 64 logprobs rows.

    python tools/logprobs_probe.py [--model llama-3-8b] [--new 48] [--iters 200]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rr_b200 import _lib  # noqa: E402
from rr_b200.engine import Engine  # noqa: E402
from rr_b200.models import SPECS, make_weights  # noqa: E402


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def kernel_us(rows: int, vocab: int, k: int, iters: int) -> float:
    x = torch.randn(rows, vocab, device="cuda") * 3
    top = torch.full((rows,), k, dtype=torch.int32, device="cuda")
    lp = torch.empty(rows, 20, device="cuda")
    ids = torch.empty(rows, 20, dtype=torch.int32, device="cuda")
    args = [C.c_void_p(x.data_ptr()), vocab, rows, vocab, C.c_void_p(top.data_ptr()), 20, C.c_void_p(lp.data_ptr()),
            C.c_void_p(ids.data_ptr()), None]
    flush = torch.empty(64 << 20, dtype=torch.int8, device="cuda")   # 64 MB: the logits leave L2 between calls
    times = []
    for i in range(iters + 10):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(_lib.lib.rr_op_logprobs(*args), "rr_op_logprobs")
        b.record()
        if i >= 10:
            times.append((a, b))
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in times])) * 1e3


def step_ms(eng: Engine, spec, batch: int, new: int, top) -> float:
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=512).tolist() for _ in range(batch)]
    eng.wait(eng.submit(prompts[0], 4, top_logprobs=top))         # warm both graphs
    eng.reset_stats()
    tk = [eng.submit(p, new, top_logprobs=top) for p in prompts]
    for t in tk:
        eng.wait(t)
    st = eng.stats()
    return st["decode_ms_total"] / st["decode_steps"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--new", type=int, default=48)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(f"card: {card()}")
    print(f"rr_op_logprobs {a.batch} x 128256, k = 20, logits from HBM: {kernel_us(a.batch, 128256, 20, a.iters):.1f} us (median)")
    spec = SPECS[a.model]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=a.batch, ctx_max=640, max_prefill_tokens=8192)
    for rep in range(2):
        plain = step_ms(eng, spec, a.batch, a.new, None)
        lp = step_ms(eng, spec, a.batch, a.new, 20)
        print(f"{a.model} decode step, {a.batch} rows, rep {rep}: {plain:.3f} ms without logprobs, {lp:.3f} ms with "
              f"{a.batch} logprobs rows (k = 20): +{(lp - plain) * 1e3:.1f} us")
    eng.close()


if __name__ == "__main__":
    main()
