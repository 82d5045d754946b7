"""Embeddings on full Llama-3-8B (synthetic weights), arms alternated --reps times in one process.

    python tools/embeddings_probe.py [--reps 3] [--json out.json]

  * throughput: 64 inputs of 512 tokens submitted at once as embedding requests (rr_engine_submit_embed) against the same
    prompts as generation requests with max_tokens = 1: requests/s (wall clock, submit to last result), prefill chunks and
    ms per chunk (CUDA events, rr_engine_stats.prefill_ms_total);
  * interference: 32 rows decoding 256 tokens each, alone, with 32 embedding requests of 512 tokens submitted while they
    decode, and with the same 32 prompts as generation requests of max_tokens = 1 instead: decode ms per step (CUDA
    events, decode_ms_total / decode_steps); the spread of each arm over the reps is the run-to-run noise the arms are
    judged against.
Prints the card and its power limit, read in the same process."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def burst(eng, prompts, embed):
    eng.reset_stats()
    t0 = time.perf_counter()
    if embed:
        ts = [eng.submit_embedding(p) for p in prompts]
        for t in ts:
            eng.embedding(t, timeout=900)
            assert eng.wait(t, timeout=900).status == 0
    else:
        ts = [eng.submit(p, 1) for p in prompts]
        for t in ts:
            assert eng.wait(t, timeout=900).status == 0
    dt = time.perf_counter() - t0
    st = eng.stats()
    return {"req_per_s": len(prompts) / dt, "chunks": st["prefill_chunks"],
            "ms_per_chunk": st["prefill_ms_total"] / max(1, st["prefill_chunks"])}


def decode_arm(eng, gen_prompts, side_prompts, embed=True):
    eng.reset_stats()
    ts = [eng.submit(p, 256) for p in gen_prompts]
    while eng.stats()["decode_steps"] < 8:       # every generation row is decoding before the side traffic arrives
        time.sleep(0.001)
    es = [eng.submit_embedding(p) if embed else eng.submit(p, 1) for p in side_prompts]
    for t in es:
        if embed:
            eng.embedding(t, timeout=900)
        eng.wait(t, timeout=900)
    for t in ts:
        assert eng.wait(t, timeout=900).status == 0
    st = eng.stats()
    return {"decode_ms_per_step": st["decode_ms_total"] / st["decode_steps"], "steps": st["decode_steps"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    from rr_b200 import Engine, SPECS
    spec = SPECS["llama-3-8b"]
    eng = Engine.synthetic(spec, seed=0, max_batch=64, ctx_max=1024, max_prefill_tokens=8192)
    g = torch.Generator().manual_seed(0)

    def prompt(n):
        return [1] + torch.randint(3, spec.vocab, (n - 1,), generator=g).tolist()

    prompts = [prompt(512) for _ in range(64)]
    gen_prompts, emb_prompts = [prompt(512) for _ in range(32)], [prompt(512) for _ in range(32)]
    burst(eng, prompts[:8], True)                # warm-up: buffers, graphs
    burst(eng, prompts[:8], False)
    decode_arm(eng, gen_prompts[:4], [])
    out = {"card": card(), "throughput": [], "decode": []}
    for _ in range(a.reps):
        out["throughput"].append({"embed": burst(eng, prompts, True), "max_tokens_1": burst(eng, prompts, False)})
        out["decode"].append({"plain": decode_arm(eng, gen_prompts, []),
                              "with_embeddings": decode_arm(eng, gen_prompts, emb_prompts),
                              "with_max_tokens_1": decode_arm(eng, gen_prompts, emb_prompts, embed=False)})
    eng.close()
    print(out["card"])
    for i, (t, d) in enumerate(zip(out["throughput"], out["decode"])):
        print(f"rep {i}: embeddings {t['embed']['req_per_s']:.1f}/s, {t['embed']['ms_per_chunk']:.2f} ms/chunk "
              f"({t['embed']['chunks']} chunks) | max_tokens=1 {t['max_tokens_1']['req_per_s']:.1f}/s, "
              f"{t['max_tokens_1']['ms_per_chunk']:.2f} ms/chunk ({t['max_tokens_1']['chunks']} chunks) | decode "
              f"{d['plain']['decode_ms_per_step']:.3f} ms/step plain, {d['with_embeddings']['decode_ms_per_step']:.3f} "
              f"with embeddings, {d['with_max_tokens_1']['decode_ms_per_step']:.3f} with the same prompts at "
              f"max_tokens=1")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
