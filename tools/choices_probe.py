"""Several choices per request (`n`) against the same choices as separate requests, on the full-size model.

8 distinct 512-token prompts, temperature 1, 128 tokens out.  Arm "n": 8 requests with n = 8; arm "sep": 64 requests,
prompt j with seeds seed + i.  Both arms run in one process, alternated --rounds times after one warm-up each.  Reports
per arm: prefill ms per burst (CUDA events, engine stats), TTFT p50 / p99 over the 64 choices, choices/s, and whether the
two arms generated the same tokens.  The fan-out's KV copy is timed apart with CUDA events around rr_op_kv_copy_prefix at
the arm's shape (7 copies of each 512-token prompt into fresh slots of the engine's cache layout).

    python tools/choices_probe.py --out choices_probe.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rr_b200 import _lib  # noqa: E402
from rr_b200.engine import Engine  # noqa: E402
from rr_b200.models import SPECS, make_weights  # noqa: E402


def burst(eng, prompts, n, max_new, seed):
    """Submit the whole burst, wait for all -> (per-choice token lists [prompt][choice], ttfts, wall s, prefill ms)."""
    eng.reset_stats()
    t0 = time.perf_counter()
    if n > 1:
        tks = [eng.submit(p, max_new, temperature=1.0, seed=seed, n=n) for p in prompts]
    else:
        tks = [eng.submit(p, max_new, temperature=1.0, seed=seed + i) for p in prompts for i in range(N_CHOICES)]
    recs = [eng.wait(t) for t in tks]
    wall = time.perf_counter() - t0
    assert all(r.status == 0 for r in recs)
    if n > 1:
        toks = [r.choices for r in recs]
        ttft = [r.ttft for r in recs for _ in range(n)]
    else:
        toks = [[recs[j * N_CHOICES + i].tokens for i in range(N_CHOICES)] for j in range(len(prompts))]
        ttft = [r.ttft for r in recs]
    st = eng.stats()
    return toks, ttft, wall, st["prefill_ms_total"], st["kv_copy_tokens"]


def kv_copy_ms(spec, B, ctx, n_src, n_choices, L, reps=20):
    """CUDA-event time of one rr_op_kv_copy_prefix launch copying each of n_src L-token prompts to n_choices - 1 slots."""
    shape = (spec.n_layers, B, spec.n_kv_heads, ctx, 128)
    k = torch.zeros(shape, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros_like(k)
    src = [j for j in range(n_src) for _ in range(n_choices - 1)]
    dst = list(range(n_src, n_src + len(src)))
    arr = lambda a: (C.c_int32 * len(a))(*a)  # noqa: E731
    args = (C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()), spec.n_layers, B, spec.n_kv_heads, ctx, arr(src),
            arr(dst), arr([L] * len(src)), len(src), None)
    for _ in range(3):
        _lib.check(_lib.lib.rr_op_kv_copy_prefix(*args), "rr_op_kv_copy_prefix")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(torch.cuda.default_stream())
    for _ in range(reps):
        _lib.lib.rr_op_kv_copy_prefix(*args)
    e1.record(torch.cuda.default_stream())
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    moved = 2 * 2 * len(src) * L * 128 * 2 * spec.n_layers * spec.n_kv_heads        # K and V, read and written
    del k, v
    torch.cuda.empty_cache()
    return ms, moved / (ms * 1e-3) / 1e12


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:        # the record says so rather than guessing
        return f"unavailable ({e})"


N_CHOICES = 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--prompts", type=int, default=8)
    ap.add_argument("--prompt-len", type=int, default=512)
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    spec = SPECS[a.model]
    B, ctx = a.prompts * N_CHOICES, 1024
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=a.prompt_len).tolist() for _ in range(a.prompts)]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=B, ctx_max=ctx, max_prefill_tokens=8192)
    arms = {"n": N_CHOICES, "sep": 1}
    res = {k: {"prefill_ms": [], "ttft_p50_ms": [], "ttft_p99_ms": [], "choices_per_s": [], "kv_copy_tokens": []}
           for k in arms}
    toks = {}
    for k, n in arms.items():                                     # warm-up: graphs, first launches
        burst(eng, prompts, n, a.max_new, a.seed)
    for _ in range(a.rounds):
        for k, n in arms.items():
            t, ttft, wall, pf_ms, kvt = burst(eng, prompts, n, a.max_new, a.seed)
            toks[k] = t
            r = res[k]
            r["prefill_ms"].append(pf_ms)
            r["ttft_p50_ms"].append(1e3 * float(np.percentile(ttft, 50)))
            r["ttft_p99_ms"].append(1e3 * float(np.percentile(ttft, 99)))
            r["choices_per_s"].append(len(ttft) / wall)
            r["kv_copy_tokens"].append(kvt)
    eng.close()
    del eng
    torch.cuda.empty_cache()
    copy_ms, copy_tbs = kv_copy_ms(spec, B, ctx, a.prompts, N_CHOICES, a.prompt_len)
    out = {"gpu": gpu_info(), "model": a.model, "prompts": a.prompts, "n": N_CHOICES, "prompt_len": a.prompt_len,
           "max_new": a.max_new, "rounds": a.rounds,
           "arms": {k: {m: [round(x, 3) for x in v] for m, v in r.items()} for k, r in res.items()},
           "kv_copy_ms": round(copy_ms, 4), "kv_copy_tb_per_s": round(copy_tbs, 3),
           "tokens_equal": toks["n"] == toks["sep"]}
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
