"""FP8 weights against bf16 on full Llama-3-8B: one engine with e4m3 projections (models.quantize_fp8) and one bf16 engine
on the same weights dequantized (Fp8Weights.dequantize), so the two arms must produce the same tokens.  Both have 64 decode
rows, prefill chunks of 8192 tokens and CUDA graphs, and run alternately, --reps times in one process.

    python tools/fp8_probe.py [--model llama-3-8b] [--reps 3] [--json out.json]

Per arm and repetition:
  * the bench.py-shaped burst, 64 prompts x 512 tokens in / 128 out: completions/s (wall clock), mean and p50 TTFT, and the
    decode step in ms (the engine's CUDA events around every step / steps);
  * the prefill chunk of one 8192-token and of one 512-token prompt alone (CUDA events around the chunk);
  * the tokens of the burst, which must equal the other arm's.
Once per arm after the timed repetitions: a torch.profiler trace of a short burst, kernel time per decode step by kernel
name and the weight GB/s of the projection kernels (algorithmic weight bytes from the shapes over their kernel time).
fp8 arm only: the dequantize of all 32 layers' projections (rr_op_dequantize_fp8_weight, CUDA events), the share of a
prefill chunk it costs.  Prints the card and its power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def burst(eng, prompts, max_new):
    eng.reset_stats()
    t0 = time.perf_counter()
    tk = [eng.submit(p, max_new) for p in prompts]
    recs = [eng.wait(t, timeout=600) for t in tk]
    wall = time.perf_counter() - t0
    st = eng.stats()
    assert all(r.status == 0 for r in recs)
    ttft = [1e3 * r.ttft for r in recs]
    return dict(completions_per_s=len(prompts) / wall, ttft_ms_mean=statistics.mean(ttft),
                ttft_ms_p50=statistics.median(ttft), decode_step_ms=st["decode_ms_total"] / max(1, st["decode_steps"]),
                decode_steps=st["decode_steps"]), [r.tokens for r in recs]


def chunk_ms(eng, prompt):
    eng.reset_stats()
    r = eng.wait(eng.submit(prompt, 1), timeout=600)
    assert r.status == 0
    st = eng.stats()
    assert st["prefill_chunks"] == 1, st
    return st["prefill_ms_total"]


def kernel_table(eng, prompts, spec, fp8):
    """kernel time per decode step by kernel name (torch.profiler, CUDA activities) and the weight GB/s of the projections"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.reset_stats()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tk = [eng.submit(p, 16) for p in prompts]
        for t in tk:
            eng.wait(t, timeout=600)
        torch.cuda.synchronize()
    steps = max(1, eng.stats()["decode_steps"])
    agg = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        a = agg.setdefault(ev.name, [0, 0.0])
        a[0] += 1
        a[1] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
    L, H = spec.n_layers, spec.hidden
    nqkv = (spec.n_heads + 2 * spec.n_kv_heads) * spec.head_dim
    b = 1 if fp8 else 2
    # weight bytes per decode step of the projection kernels (the prefill's decode-orientation tail is a few launches)
    mlp_bytes = L * 3 * spec.inter * H * b
    proj_bytes = L * (nqkv + spec.n_heads * spec.head_dim) * H * b
    head_bytes = 2 * spec.vocab * H
    rows = []
    for name, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        if us / steps < 5:
            continue
        row = dict(kernel=name[:90], launches_per_step=round(n / steps, 2), us_per_step=round(us / steps, 1))
        # the decode launches of the projection kernels (QKV and O: 2 per layer, + lm_head in the bf16 instantiation); the
        # prefill tail's few decode-orientation launches are counted in their time, so the rates are lower bounds
        if "gemm_mlp_wgmma" in name:
            row["weight_GBps"] = round(mlp_bytes / (us / steps) / 1e3, 1)
        elif "gemm_bf16_wgmma<64, 1, 8" in name and n / steps >= 2 * L:
            wb = proj_bytes if fp8 else proj_bytes + head_bytes
            row["weight_GBps"] = round(wb / (us / steps) / 1e3, 1)
        rows.append(row)
    return dict(decode_steps=steps, rows=rows)


def dequant_ms(q, reps=5):
    import torch
    from rr_b200 import _lib
    mats = [(t, s) for name in q.PROJ for t, s in zip(getattr(q, name), getattr(q, name + "_scale"))]
    outs = [torch.empty(t.shape, dtype=torch.bfloat16, device="cuda") for t, _ in mats]
    st = torch.cuda.current_stream().cuda_stream

    def run():
        for (t, s), o in zip(mats, outs):
            _lib.check(_lib.lib.rr_op_dequantize_fp8_weight(t.data_ptr(), s.data_ptr(), t.shape[0], t.shape[1],
                                                            o.data_ptr(), t.shape[1], st))
    run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    from rr_b200.models import quantize_fp8
    spec = SPECS[a.model]
    w = make_weights(spec, seed=0, device="cuda")
    q = quantize_fp8(w)
    del w
    torch.cuda.empty_cache()
    d = q.dequantize()
    out = {"card": card(), "model": a.model}
    kw = dict(max_batch=64, ctx_max=8256, max_prefill_tokens=8192, kv_cache_tokens=65536)
    arms = {"fp8": Engine(q, **kw), "bf16": Engine(d, **kw)}
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=512).tolist() for _ in range(64)]
    long8k, short = rng.randint(3, spec.vocab, size=8192).tolist(), rng.randint(3, spec.vocab, size=512).tolist()
    try:
        for eng in arms.values():                                     # warm-up: graphs captured, every shape seen
            burst(eng, prompts[:8], 8)
            chunk_ms(eng, long8k)
        runs = {k: [] for k in arms}
        for rep in range(a.reps):
            toks = {}
            for k, eng in arms.items():
                r, toks[k] = burst(eng, prompts, 128)
                r["prefill_8192_ms"] = chunk_ms(eng, long8k)
                r["prefill_512_ms"] = chunk_ms(eng, short)
                runs[k].append(r)
                print(k, rep, json.dumps(r), flush=True)
            assert toks["fp8"] == toks["bf16"], f"repetition {rep}: the arms' tokens differ"
        out["runs"] = runs
        out["tokens_equal"] = True
        med = {k: {m: statistics.median(r[m] for r in v) for m in v[0]} for k, v in runs.items()}
        out["median"] = med
        out["decode_step_ratio_fp8_over_bf16"] = med["fp8"]["decode_step_ms"] / med["bf16"]["decode_step_ms"]
        out["dequantize_all_layers_ms"] = dequant_ms(q)
        out["dequantize_share_of_chunk"] = {
            n: out["dequantize_all_layers_ms"] / med["fp8"][f"prefill_{n}_ms"] for n in (8192, 512)}
        out["kernels"] = {k: kernel_table(eng, prompts[:64], spec, k == "fp8") for k, eng in arms.items()}
    finally:
        for eng in arms.values():
            eng.close()
    s = json.dumps(out, indent=1)
    print(s)
    if a.json:
        with open(a.json, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
