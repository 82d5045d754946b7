"""Cost of prompt logprobs on full Llama-3-8B (synthetic weights): prefill with and without scoring, alternated --reps
times in one process, and the scoring kernels timed alone.

    python tools/prompt_logprobs_probe.py [--reps 3] [--json out.json]

  * one 8192-token prompt in one 8192-token chunk: the chunk's CUDA-event time (rr_engine_stats.prefill_ms_total) of a
    plain request against one with prompt logprobs (k = 5, what `echo` + `logprobs: 5` asks for);
  * one 65536-token prompt over eight 8192-token pieces: the same, summed over its chunks;
  * per kernel, CUDA events over --iters launches on the engine's shapes: the last layer's O, gate/up and down GEMMs over
    8192 rows (rr_op_prefill_gemm), lm_head over one 1024-row block (RR_OUT_ROWMAJOR_F32) and the log-softmax / top-k of
    that block (rr_op_logprobs), the last two times the 8 blocks of a chunk.
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def chunk_ms(eng, prompt, score):
    eng.reset_stats()
    t = eng.submit(prompt, 1, prompt_logprobs=5 if score else None)
    if score:
        eng.prompt_logprobs(t, timeout=900)
    r = eng.wait(t, timeout=900)
    assert r.status == 0
    st = eng.stats()
    return st["prefill_ms_total"], st["prefill_chunks"]


def kernels(iters):
    import torch
    from rr_b200 import _lib
    T, H, I, V, S = 8192, 4096, 14336, 128256, 1024
    dev = "cuda"
    bf = torch.bfloat16
    x = torch.randn(T, H, device=dev).to(bf)
    act = torch.randn(T, I, device=dev).to(bf)
    wo, wgu, wd = (torch.randn(H, H, device=dev) * 0.02).to(bf), (torch.randn(2 * I, H, device=dev) * 0.02).to(bf), \
        (torch.randn(H, I, device=dev) * 0.02).to(bf)
    head = (torch.randn(V, H, device=dev) * 0.02).to(bf)
    res = torch.zeros(T, H, device=dev)
    xhat = torch.empty(T, H, device=dev, dtype=bf)
    rowss = torch.rand(T, H // 128, device=dev) + 0.5
    rowss_out = torch.empty_like(rowss)
    gamma = torch.ones(H, device=dev, dtype=bf)
    logits = torch.empty(S, V, device=dev)
    top = torch.full((S,), 5, dtype=torch.int32, device=dev)
    lp, ids = torch.empty(S, 20, device=dev), torch.empty(S, 20, dtype=torch.int32, device=dev)
    L = _lib.lib
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731

    def o():
        _lib.check(L.rr_op_prefill_gemm(p(x), T, T, H, p(wo), H, H, p(res), H, 5, None, 0, 0, 0.0, p(gamma), p(xhat),
                                        p(rowss_out), H // 128, None), "o")

    def gu():
        _lib.check(L.rr_op_prefill_gemm(p(x), T, T, H, p(wgu), 2 * I, H, p(act), I, 3, p(rowss), H // 128, H, 1e-5,
                                        None, None, None, 0, None), "gu")

    def down():
        _lib.check(L.rr_op_prefill_gemm(p(act), T, T, I, p(wd), H, I, p(res), H, 5, None, 0, 0, 0.0, p(gamma), p(xhat),
                                        p(rowss_out), H // 128, None), "down")

    def lm_head():
        _lib.check(L.rr_op_prefill_gemm(p(x), S, S, H, p(head), V, H, p(logits), V, 6, p(rowss), H // 128, H, 1e-5,
                                        None, None, None, 0, None), "lm_head")

    def logprobs():
        _lib.check(L.rr_op_logprobs(p(logits), V, S, V, p(top), 20, p(lp), p(ids), None), "logprobs")

    out = {}
    for name, fn in (("o", o), ("gate_up", gu), ("down", down), ("lm_head_1024", lm_head), ("logprobs_1024", logprobs)):
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        out[name + "_ms"] = a.elapsed_time(b) / iters
    out["lm_head_1024_tflops"] = 2 * S * H * V / (out["lm_head_1024_ms"] * 1e-3) / 1e12
    out["last_layer_ms"] = out["o_ms"] + out["gate_up_ms"] + out["down_ms"]
    out["lm_head_8192_ms"] = 8 * out["lm_head_1024_ms"]
    out["logprobs_8192_ms"] = 8 * out["logprobs_1024_ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--skip-long", action="store_true", help="leave out the 65536-token prompt")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    print("card:", card(), flush=True)
    spec = SPECS["llama-3-8b"]
    w = make_weights(spec, seed=0, device="cuda")
    g = torch.Generator().manual_seed(0)
    result = {"card": card()}
    cases = [("8192", 8192, 8192 + 64)] + ([] if a.skip_long else [("65536", 65536, 65536 + 64)])
    for label, n, ctx in cases:
        prompt = [1] + torch.randint(3, spec.vocab, (n - 1,), generator=g).tolist()
        eng = Engine(w, max_batch=2, ctx_max=ctx, max_prefill_tokens=8192, kv_cache_tokens=ctx)
        try:
            chunk_ms(eng, prompt, True)                 # warm-up of both arms (and the scoring buffers)
            chunk_ms(eng, prompt, False)
            plain, scored = [], []
            for _ in range(a.reps):
                plain.append(chunk_ms(eng, prompt, False)[0])
                scored.append(chunk_ms(eng, prompt, True)[0])
            r = dict(plain_ms=plain, scored_ms=scored, ratio=statistics.median(scored) / statistics.median(plain))
            result[label] = r
            print(f"{label}-token prompt: plain {statistics.median(plain):.1f} ms, scored {statistics.median(scored):.1f} ms,"
                  f" {r['ratio']:.3f}x  (plain {plain}, scored {scored})", flush=True)
        finally:
            eng.close()
            torch.cuda.empty_cache()
    del w
    torch.cuda.empty_cache()
    k = kernels(a.iters)
    result["kernels"] = k
    for name, v in k.items():
        print(f"  {name}: {v:.3f}", flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
