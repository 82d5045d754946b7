"""Sliding-window attention on full Mistral-7B: an engine with the model's window (W = 4096) against one without (W = 0)
on the same weights, created and measured alternately, --reps times in one process.

    python tools/sliding_window_probe.py [--reps 3] [--json out.json]

Per arm and repetition:
  * TTFT of one 32768-token prompt (64 decode rows, context window 32768 + 64, a 262144-token pool, 8192-token chunks, CUDA
    graphs): the engine's submit-to-first-token time, and the prefill ms of its four chunks (CUDA events);
  * how many 32768-token requests (32704 in, 64 out) the 262144-token pool holds at once: the pages one such request
    reserves, read from rr_engine_kv_usage while it runs alone, into the pool's 4096 pages;
  * decode attention at 64 rows deep in context (positions 16384 .. 30000, Mistral-7B's 32 heads / 8 kv heads, one layer's
    pool of scattered pages): CUDA-event time of rr_op_decode_attn_qkv_window with the arm's window over 200 launches,
    and that time x 32 layers, the attention share of a decode step.  Everything else in the step is the same kernels on
    the same shapes in both arms.  A W = 0 engine cannot hold 64 rows that deep (1.5 M tokens of KV), so this is measured
    at kernel level.
Prints the card and its power limit, read in the same process."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def ttft_and_fit(w, prompt, long_req):
    from rr_b200.engine import Engine
    eng = Engine(w, max_batch=64, ctx_max=32768 + 64, kv_cache_tokens=262144)
    try:
        eng.reset_stats()
        r = eng.wait(eng.submit(prompt, 1), timeout=900)
        assert r.status == 0
        st = eng.stats()
        out = dict(ttft_ms=1e3 * r.ttft, prefill_ms=st["prefill_ms_total"], chunks=st["prefill_chunks"])
        t = eng.submit(long_req, 64)
        for _ in range(6000):
            got, done, _ = eng.peek(t, 1, timeout=0.5)
            if got or done:
                break
        total, free = eng.kv_usage()
        assert not done
        eng.wait(t, timeout=900)
        out["pages_per_request"] = total - free
        out["requests_that_fit"] = total // (total - free)
        return out
    finally:
        eng.close()


def decode_attn_us(window, reps=200):
    """Decode attention of one Mistral-7B layer at 64 rows, positions 16384 .. 30000, over scattered pages."""
    import torch
    from rr_b200 import _lib
    nh, nkv, hd, ctx, rows = 32, 8, 128, 32768, 64
    g = torch.Generator().manual_seed(3)
    pos = torch.linspace(16384, 30000, rows).round().int()
    need = [int(p) // 64 + 1 for p in pos]
    n_pages = sum(need) + 8
    perm = torch.randperm(n_pages, generator=g)
    table = torch.zeros(rows, ctx // 64, dtype=torch.int32)
    at = 0
    for r, n in enumerate(need):
        table[r, :n] = perm[at:at + n].int()
        at += n
    k = torch.randn(n_pages, nkv, 64, 128, device="cuda").bfloat16()
    v = torch.randn(n_pages, nkv, 64, 128, device="cuda").bfloat16()
    nqkv = (nh + 2 * nkv) * hd
    planes = torch.randn(1, rows, nqkv, device="cuda")
    out = torch.empty(rows * nh * hd, device="cuda", dtype=torch.bfloat16)
    slot, dpos, dtab = torch.arange(rows, dtype=torch.int32).cuda(), pos.cuda(), table.cuda()
    ks = C.c_int32()
    P = lambda t: C.c_void_p(t.data_ptr())                                          # noqa: E731

    def call():
        _lib.check(_lib.lib.rr_op_decode_attn_qkv_window(P(planes), 1, planes.stride(0), nqkv, P(k), P(v), P(out), P(slot),
                                                         P(dpos), rows, nh, nkv, hd, ctx, rows, 10000.0, C.byref(ks),
                                                         P(dtab), ctx // 64, n_pages, window, None), "decode_attn_window")
    for _ in range(10):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps, ks.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import dataclasses
    import torch
    from rr_b200 import SPECS, make_weights
    spec = SPECS["mistral-7b"]
    assert spec.sliding_window == 4096
    print("card:", card(), flush=True)
    w = make_weights(spec, seed=0, device="cuda")
    arms = {"W=4096": w, "W=0": dataclasses.replace(w, spec=dataclasses.replace(spec, sliding_window=0))}
    rs = np.random.RandomState(0)
    prompt = rs.randint(3, spec.vocab, size=32768).tolist()
    long_req = rs.randint(3, spec.vocab, size=32704).tolist()
    res = {k: [] for k in arms}
    for rep in range(a.reps):
        for name, ww in arms.items():
            r = ttft_and_fit(ww, prompt, long_req)
            r["decode_attn_us"], r["kv_splits"] = decode_attn_us(ww.spec.sliding_window)
            r["decode_attn_step_ms"] = 32 * r["decode_attn_us"] / 1e3
            res[name].append(r)
            print(rep, name, json.dumps({k: round(x, 3) if isinstance(x, float) else x for k, x in r.items()}), flush=True)
            torch.cuda.empty_cache()
    summary = {name: {k: statistics.median(r[k] for r in rows) for k in rows[0]} for name, rows in res.items()}
    print("card:", card())
    print("medians:", json.dumps(summary, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), runs=res, medians=summary), f, indent=1)


if __name__ == "__main__":
    main()
