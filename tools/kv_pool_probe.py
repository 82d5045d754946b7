"""The paged KV cache on full Llama-3-8B: one replica of 64 rows with an 8192-token context window and a 262144-token pool
serves 64 requests of 512 in / 128 out together with 4 requests of a 7680-token prompt and 256 new tokens.

    python tools/kv_pool_probe.py [--model llama-3-8b] [--json out.json]

Reports completions/s of the mix, decode ms/step without the long rows (the mean over a separate run of the 64 short
requests alone) and with them (the mean over every decode step of the mix), the long requests' TTFT,
torch.cuda.mem_get_info after creation, and decode ms/step at the bench shape (64 x 512 in / 128 out) on a fresh engine
against one whose free list was scattered by earlier traffic.  With a
slot-contiguous cache this mix needs ctx_max = 8192 on every row: 64 x 8192 x 131072 B = 68.7 GB of KV beside 16.06 GB of
weights, more than the card holds (arithmetic; not tried).  Prints the card and its power limit."""
import argparse
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


def run(eng, reqs):
    """-> (wall s, records, decode ms/step) of submitting every (prompt, max_new) at once"""
    eng.reset_stats()
    t0 = time.perf_counter()
    tk = [eng.submit(p, m) for p, m in reqs]
    recs = [eng.wait(t) for t in tk]
    wall = time.perf_counter() - t0
    st = eng.stats()
    return wall, recs, st["decode_ms_total"] / max(1, st["decode_steps"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS[a.model]
    w = make_weights(spec, seed=0, device="cuda")
    rng = np.random.RandomState(0)

    def toks(n):
        return rng.randint(3, spec.vocab, size=n).tolist()
    out = {"card": card()}
    eng = Engine(w, max_batch=64, ctx_max=8192, max_prefill_tokens=8192, kv_cache_tokens=262144)
    try:
        free, total = torch.cuda.mem_get_info()
        out["mem_free_gb_after_create"], out["mem_total_gb"] = free / 1e9, total / 1e9
        short = [(toks(512), 128) for _ in range(64)]
        run(eng, short[:8])                                            # warm-up: graphs captured
        _, _, out["decode_ms_short_only"] = run(eng, short)
        long = [(toks(7680), 256) for _ in range(4)]
        wall, recs, out["decode_ms_mix"] = run(eng, short + long)
        out["mix_completions_per_s"] = len(recs) / wall
        out["long_ttft_s"] = [r.ttft for r in recs[64:]]
        out["pages_after_mix"] = eng.kv_usage()
    finally:
        eng.close()
    # bench shape: fresh free list against one scattered by mixed-length traffic
    bench = [(toks(512), 128) for _ in range(64)]
    eng = Engine(w, max_batch=64, ctx_max=640, max_prefill_tokens=8192)
    try:
        run(eng, bench[:8])
        _, fresh, out["decode_ms_bench_fresh"] = run(eng, bench)
        run(eng, [(toks(int(n)), int(m)) for n, m in zip(rng.randint(16, 500, 96), rng.randint(1, 130, 96))])
        _, scat, out["decode_ms_bench_scattered"] = run(eng, bench)
        out["bench_tokens_equal"] = [r.tokens for r in fresh] == [r.tokens for r in scat]
    finally:
        eng.close()
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
