"""Cost of seeded sampling on the GPU: the card, then CUDA-event time of rr_op_sample alone (64 x 128256 and 64 x 32064 fp32
logits, top_p 1 and 0.9, flat and peaked rows) and the Llama-3-8B decode step (64 rows, 512-token prompts) with 0 and
with 64 sampled rows.

    python tools/sampling_probe.py [--model llama-3-8b] [--new 48] [--iters 200]
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


def kernel_us(rows: int, vocab: int, top_p: float, sigma: float, iters: int) -> float:
    """sigma 0.02: the flat rows the synthetic weights give; sigma 3: peaked rows."""
    x = torch.randn(rows, vocab, device="cuda") * sigma
    temp = torch.full((rows,), 1.0, device="cuda")
    top = torch.full((rows,), top_p, device="cuda")
    seed = torch.arange(rows, dtype=torch.int64, device="cuda")
    pos = torch.full((rows,), 600, dtype=torch.int32, device="cuda")
    tok = torch.empty(rows, dtype=torch.int32, device="cuda")
    args = [C.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else t
            for t in (x, vocab, rows, vocab, temp, top, seed, pos, tok)] + [None]
    flush = torch.empty(64 << 20, dtype=torch.int8, device="cuda")   # 64 MB: the logits leave L2 between calls
    times = []
    for i in range(iters + 10):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(_lib.lib.rr_op_sample(*args), "rr_op_sample")
        b.record()
        if i >= 10:
            times.append((a, b))
    torch.cuda.synchronize()
    window = float(np.median([a.elapsed_time(b) for a, b in times])) * 1e3
    # the event window also holds rr_op_sample's stream-ordered workspace allocation (the engine allocates its workspace
    # once).  The kernels alone: from the start of the threshold kernel to the end of the merge kernel of each call, from
    # the profiler's device timestamps (a sum of kernel durations would count twice the time a PDL launch spends
    # resident while it waits for its predecessor)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            flush.zero_()
            _lib.check(_lib.lib.rr_op_sample(*args), "rr_op_sample")
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if "sample_" in e.name), key=lambda e: e.time_range.start)
    starts = [e.time_range.start for e in ev if "sample_threshold" in e.name]
    ends = [e.time_range.end for e in ev if "sample_merge" in e.name]
    assert len(starts) == len(ends) == iters, (len(starts), len(ends))
    return window, float(np.median(np.array(ends) - np.array(starts)))


def step_ms(eng: Engine, spec, batch: int, new: int, temperature) -> float:
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=512).tolist() for _ in range(batch)]
    kw = dict(temperature=temperature, top_p=0.9, seed=1) if temperature else {}
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
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(f"card: {card()}")
    for vocab in (128256, 32064):
        for top_p in (1.0, 0.9):
            for name, sigma in (("flat", 0.02), ("peaked", 3.0)):
                window, kern = kernel_us(a.batch, vocab, top_p, sigma, a.iters)
                print(f"rr_op_sample {a.batch} x {vocab}, top_p {top_p}, {name} rows, logits from HBM: kernels {kern:.1f} us "
                      f"(median, threshold start to merge end), call {window:.1f} us (median event window, workspace allocation included)")
    spec = SPECS[a.model]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=a.batch, ctx_max=640, max_prefill_tokens=8192)
    for rep in range(2):
        plain = step_ms(eng, spec, a.batch, a.new, None)
        samp = step_ms(eng, spec, a.batch, a.new, 1.0)
        print(f"{a.model} decode step, {a.batch} rows, rep {rep}: {plain:.3f} ms greedy, {samp:.3f} ms with {a.batch} "
              f"sampled rows (T = 1, top_p = 0.9): +{(samp - plain) * 1e3:.1f} us")
    eng.close()


if __name__ == "__main__":
    main()
