"""Prompt prefix caching on a full-size model: a burst of 64 requests sharing a 448-token prefix (64 distinct tokens each,
128 out) through an engine with prefix_cache on and one without, alternated in one process, plus CUDA-event timing of the
KV prefix copy kernel for one 448-token prefix.

    python tools/prefix_cache_probe.py [--model llama-3-8b] [--reps 3] [--json out.json]

Per arm: prefill ms (CUDA events on the engine stream), TTFT p50 / p99, completions/s, prefill tokens counted by the
engine, and whether the generated tokens equal the other arm's.  Every repetition uses a fresh shared prefix, so the
caching arm starts cold each time.  The copy kernel is HBM-bound: 2 x 448 x bytes-per-token moved (read + write); the
floor at the H100 SXM data-sheet 3.35 TB/s is printed beside the measured time, as a bound, not a measurement."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def burst(eng, prompts, n_new):
    eng.reset_stats()
    t0 = time.perf_counter()
    tk = [eng.submit(p, n_new) for p in prompts]
    recs = [eng.wait(t) for t in tk]
    wall = time.perf_counter() - t0
    st = eng.stats()
    ttft = np.array([r.ttft for r in recs]) * 1e3
    assert all(r.status == 0 for r in recs)
    return {"prefill_ms": st["prefill_ms_total"], "prefill_tokens": st["prefill_tokens"],
            "prefill_chunks": st["prefill_chunks"], "prefix_hits": st["prefix_hits"], "kv_copy_tokens": st["kv_copy_tokens"],
            "ttft_p50_ms": float(np.percentile(ttft, 50)), "ttft_p99_ms": float(np.percentile(ttft, 99)),
            "completions_per_s": len(prompts) / wall}, [r.tokens for r in recs]


def time_copy(spec, n_tok=448, iters=200):
    from rr_b200 import _lib
    slots, ctx = 2, 512
    shape = (spec.n_layers, slots, spec.n_kv_heads, ctx, 128)
    kc = torch.randn(shape, device="cuda").bfloat16()
    vc = torch.randn(shape, device="cuda").bfloat16()
    one = lambda v: (C.c_int32 * 1)(v)                                             # noqa: E731

    def run():
        _lib.check(_lib.lib.rr_op_kv_copy_prefix(C.c_void_p(kc.data_ptr()), C.c_void_p(vc.data_ptr()), spec.n_layers,
                                                 slots, spec.n_kv_heads, ctx, one(0), one(1), one(n_tok), 1, None), "copy")
    for _ in range(10):
        run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1e3 / iters
    assert torch.equal(kc[:, 1, :, :n_tok], kc[:, 0, :, :n_tok]) and torch.equal(vc[:, 1, :, :n_tok], vc[:, 0, :, :n_tok])
    moved = 2 * n_tok * spec.n_layers * spec.n_kv_heads * 128 * 2 * 2              # K and V, read + write
    return {"tokens": n_tok, "us": us, "bytes_moved": moved, "gb_per_s": moved / us / 1e3,
            "floor_us_at_3350_gbs": moved / 3350e9 * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--shared", type=int, default=448)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    print("card:", card(), flush=True)
    spec = SPECS[a.model]
    w = make_weights(spec, seed=0, device="cuda")
    kw = dict(max_batch=a.requests, ctx_max=1024, max_prefill_tokens=8192, use_cuda_graph=True)
    arms = {"off": Engine(w, **kw), "on": Engine(w, prefix_cache=True, **kw)}
    rng = np.random.RandomState(0)
    warm = [rng.randint(3, spec.vocab, size=a.shared + a.distinct).tolist() for _ in range(a.requests)]
    for e in arms.values():
        burst(e, warm, 4)
    rows = []
    for rep in range(a.reps):
        shared = rng.randint(3, spec.vocab, size=a.shared).tolist()
        prompts = [shared + rng.randint(3, spec.vocab, size=a.distinct).tolist() for _ in range(a.requests)]
        toks = {}
        for name in (("off", "on") if rep % 2 == 0 else ("on", "off")):
            r, toks[name] = burst(arms[name], prompts, a.max_new)
            r.update(arm=name, rep=rep)
            rows.append(r)
        for r in rows[-2:]:
            r["tokens_equal"] = toks["on"] == toks["off"]
            print(json.dumps(r), flush=True)
    summary = {}
    for name in ("off", "on"):
        rs = [r for r in rows if r["arm"] == name]
        summary[name] = {k: float(np.median([r[k] for r in rs])) for k in
                         ("prefill_ms", "ttft_p50_ms", "ttft_p99_ms", "completions_per_s", "prefill_tokens")}
    summary["tokens_equal"] = all(r["tokens_equal"] for r in rows)
    summary["copy"] = time_copy(spec)
    summary["card"] = card()
    print(json.dumps(summary), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"rows": rows, "summary": summary}, f, indent=1)
    for e in arms.values():
        e.close()


if __name__ == "__main__":
    main()
