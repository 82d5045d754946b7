"""Long prompts on full Llama-3-8B: one replica of 64 rows, a 65536-token context window, a 262144-token pool and prefill
chunks of 8192 tokens.

    python tools/long_prompt_probe.py [--model llama-3-8b] [--json out.json]

1. TTFT of one prompt alone at 8192 / 16384 / 32768 / 65535 tokens (pieces of 8192), the time of each piece (CUDA events
   around every chunk), the prefill attention's share of the 65535-token prompt's kernel time (the in-situ trace of
   tools/trace_prefill.py: critical-path segment per kernel) and TFLOP/s on executed FLOPs: the projections of every
   token through every layer it runs, lm_head for the last token, and causal attention (QK^T and PV over keys 0..p for
   the query at position p) in every layer that runs it.  A non-final piece skips the last layer after its QKV projection.
2. 63 rows decoding while a 65528-token prompt is prefilled: the largest gap between two tokens of a decoding row, seen by
   a reader that streams it, against one chunk's time.
Prints the card and its power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

PIECE = 8192
ATTN_PF = 4                       # kernel id of prefill attention in the debug trace (tools/trace_prefill.py)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def flops(spec, n):
    """(projection, attention) FLOPs executed for an n-token prompt prefilled in pieces of PIECE"""
    d, L = spec, spec.n_layers
    nq, nkv = d.n_heads * d.head_dim, d.n_kv_heads * d.head_dim
    qkv = 2 * d.hidden * (nq + 2 * nkv)
    rest = 2 * nq * d.hidden + 2 * d.hidden * 2 * d.inter + 2 * d.inter * d.hidden
    proj = attn = 0
    for a in range(0, n, PIECE):
        b = min(n, a + PIECE)
        t, last = b - a, b == n
        keys = sum(range(a + 1, b + 1))                                   # query p attends keys 0..p
        proj += t * qkv * L + t * rest * (L - 1) + (rest + 2 * d.hidden * d.vocab if last else 0)
        attn += 4 * d.head_dim * d.n_heads * keys * (L if last else L - 1)
    return proj, attn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from rr_b200 import SPECS, _lib, make_weights
    from rr_b200.engine import Engine
    spec = SPECS[a.model]
    w = make_weights(spec, seed=0, device="cuda")
    rng = np.random.RandomState(0)

    def toks(n):
        return rng.randint(3, spec.vocab, size=n).tolist()
    out = {"card": card(), "model": a.model, "piece": PIECE}
    eng = Engine(w, max_batch=64, ctx_max=65536, max_prefill_tokens=PIECE, kv_cache_tokens=262144)
    try:
        eng.wait(eng.submit(toks(100), 4))                                    # warm-up: graphs captured
        eng.wait(eng.submit(toks(2 * PIECE + 5), 1))
        ttft = {}
        for n in (8192, 16384, 32768, 65535):
            eng.reset_stats()
            r = eng.wait(eng.submit(toks(n), 1))
            st = eng.stats()
            proj, attn = flops(spec, n)
            pf_s = st["prefill_ms_total"] / 1e3
            ttft[n] = {"ttft_s": r.t_first_token - r.t_submit, "pieces": st["prefill_chunks"],
                       "prefill_s": pf_s, "ms_per_piece_mean": 1e3 * pf_s / st["prefill_chunks"],
                       "proj_tflop": proj / 1e12, "attn_tflop": attn / 1e12,
                       "tflops_executed": (proj + attn) / pf_s / 1e12}
        out["ttft"] = ttft
        # per piece and attention share: the in-situ kernel trace of the 65535-token prompt
        N = 8192
        _lib.check(_lib.lib.rr_debug_trace_start(N), "trace")
        eng.reset_stats()
        eng.wait(eng.submit(toks(65535), 1))
        buf = (C.c_uint64 * (4 * N))()
        n = C.c_int32()
        _lib.check(_lib.lib.rr_debug_trace_stop(buf, N, C.byref(n)), "trace")
        tr = np.frombuffer(buf, dtype=np.uint64)[: 4 * n.value].reshape(-1, 4).astype(np.int64)
        tr[:, 0] &= 0xff                                                        # kernel id (sample CTA above it)
        tr = tr[np.argsort(tr[:, 1])]
        seg = np.append(tr[1:, 2] - tr[:-1, 2], tr[-1, 3] - tr[-1, 2]) / 1e6    # ms from one kernel's start to the next
        starts = np.flatnonzero(tr[:, 0] == 8)                                  # embed opens every chunk
        bounds = list(starts) + [len(tr)]
        out["trace_kernels"] = int(n.value)
        out["piece_ms_trace"] = [float(seg[bounds[i]:bounds[i + 1] - 1].sum()) for i in range(len(starts))]
        out["attn_share_65535"] = float(seg[tr[:, 0] == ATTN_PF].sum() / seg.sum())
        # decode while a long prompt is prefilled
        short = [eng.submit(toks(128), 1024) for _ in range(63)]
        eng.peek(short[-1], 0, timeout=60)
        stamps = []

        def reader():
            have = 0
            while True:
                got, done, _ = eng.peek(short[0], have, timeout=60)
                if len(got) > have:
                    stamps.append(time.perf_counter())
                    have = len(got)
                if done:
                    return
        th = threading.Thread(target=reader)
        th.start()
        time.sleep(0.5)
        eng.reset_stats()
        t0 = time.perf_counter()
        rl = eng.wait(eng.submit(toks(65528), 8))
        t1 = time.perf_counter()
        st = eng.stats()
        th.join()
        for t in short:
            eng.wait(t)
        during = [b - a for a, b in zip(stamps, stamps[1:]) if b >= t0 and a <= t1]
        out["decode_during_long"] = {"max_gap_ms": 1e3 * max(during) if during else None, "gaps": len(during),
                                     "long_ttft_s": rl.t_first_token - rl.t_submit,
                                     "chunk_ms_mean": st["prefill_ms_total"] / max(1, st["prefill_chunks"]),
                                     "decode_ms_mean": st["decode_ms_total"] / max(1, st["decode_steps"])}
    finally:
        eng.close()
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
