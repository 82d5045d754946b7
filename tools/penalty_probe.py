"""Cost of frequency / presence penalties and logit bias on the GPU: the card and its power limit, then the time of
rr_op_logit_penalties at 64 x 128256 fp32 logits with 128, 1024 and 4096-token histories and 300-entry bias lists on every
row, and the Llama-3-8B decode step (64 rows, 512-token prompts) with 0 and with 64 processed rows, alternated in this one
process.

    python tools/penalty_probe.py [--model llama-3-8b] [--new 48] [--iters 200] [--reps 3]
"""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rr_b200 import _lib  # noqa: E402
from rr_b200.engine import Engine  # noqa: E402
from rr_b200.models import SPECS, make_weights  # noqa: E402
from tools.logprobs_probe import card  # noqa: E402

BIAS = 300


def kernel_us(rows: int, vocab: int, hist_len: int, iters: int):
    g = torch.Generator(device="cuda").manual_seed(hist_len)
    x = torch.randn(rows, vocab, device="cuda", generator=g) * 3
    hist = torch.randint(0, vocab, (rows, hist_len), dtype=torch.int32, device="cuda", generator=g)
    hl = torch.full((rows,), hist_len, dtype=torch.int32, device="cuda")
    fp = torch.full((rows,), 0.5, device="cuda")
    pp = torch.full((rows,), 0.25, device="cuda")
    ids = torch.stack([torch.randperm(vocab, device="cuda", generator=g)[:BIAS] for _ in range(rows)]).to(torch.int32)
    vals = torch.rand(rows, BIAS, device="cuda", generator=g) * 200 - 100
    nb = torch.full((rows,), BIAS, dtype=torch.int32, device="cuda")
    args = [C.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else t
            for t in (x, vocab, rows, vocab, hist, hist_len, hl, fp, pp, ids, vals, BIAS, nb)] + [None]
    flush = torch.empty(64 << 20, dtype=torch.int8, device="cuda")   # 64 MB: the logits leave L2 between calls
    times = []
    for i in range(iters + 10):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(_lib.lib.rr_op_logit_penalties(*args), "rr_op_logit_penalties")
        b.record()
        if i >= 10:
            times.append((a, b))
    torch.cuda.synchronize()
    window = float(np.median([a.elapsed_time(b) for a, b in times])) * 1e3
    # the event window also holds the entry point's workspace allocation and zeroing (rows x vocab int32; the engine
    # allocates and zeroes its workspace once, and the kernel leaves it zero).  The kernel alone from the profiler's
    # device timestamps:
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            flush.zero_()
            _lib.check(_lib.lib.rr_op_logit_penalties(*args), "rr_op_logit_penalties")
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "logit_penalties" in e.name]
    assert len(ev) == iters, len(ev)
    return window, float(np.median([e.time_range.end - e.time_range.start for e in ev]))


def step_ms(eng: Engine, spec, batch: int, new: int, processed: bool) -> float:
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=512).tolist() for _ in range(batch)]
    kw = {}
    if processed:
        bias = dict(zip(rng.choice(spec.vocab, BIAS, replace=False).tolist(), rng.uniform(-5, 5, BIAS).tolist()))
        kw = dict(frequency_penalty=0.5, presence_penalty=0.25, logit_bias=bias)
    eng.wait(eng.submit(prompts[0], 4, **kw))                     # warm the graph
    eng.reset_stats()
    tk = [eng.submit(p, new, **kw) for p in prompts]
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
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(f"card: {card()}")
    for h in (128, 1024, 4096):
        window, kern = kernel_us(a.batch, 128256, h, a.iters)
        print(f"rr_op_logit_penalties {a.batch} x 128256, {h}-token histories, {BIAS} bias entries per row, logits from "
              f"HBM: kernel {kern:.1f} us (median), call {window:.1f} us (median event window, workspace allocation and "
              f"zeroing included)")
    spec = SPECS[a.model]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=a.batch, ctx_max=640, max_prefill_tokens=8192)
    for rep in range(a.reps):
        plain = step_ms(eng, spec, a.batch, a.new, False)
        pen = step_ms(eng, spec, a.batch, a.new, True)
        print(f"{a.model} decode step, {a.batch} rows, rep {rep}: {plain:.3f} ms plain, {pen:.3f} ms with {a.batch} "
              f"processed rows (both penalties, {BIAS} bias entries): {(pen - plain) * 1e3:+.1f} us")
    eng.close()
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
