"""Stop sequences on the full-size model: what the match costs and what an early end gives back.

(a) kernel: rr_op_stop_match at 64 rows with 4 x 64-byte sequences each over 512-token histories, CUDA events over many
    launches.
(b) step: a Llama-3-8B decode step with all 64 rows carrying 4 x 64-byte stop sequences that never hit, against the plain
    step, alternated in one process (decode_ms_total / decode_steps of the engine's CUDA events).
(c) queue: 256 requests of 512 tokens in / 128 max out on 64 rows, temperature 1, seed = the request's index.  Arm "stop":
    each request's stop sequence is two bytes of its own free-running reply chosen so that it hits around token 32;
    arm "plain": the same queue without stop.
    Alternated --rounds times after one warm-up each: completions/s, decode steps and generated tokens from the engine
    stats, and whether every kept reply equals the oracle cut of the plain arm's.

    python tools/stop_probe.py --out stop_probe.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rr_b200 import _lib  # noqa: E402
from rr_b200.engine import Engine  # noqa: E402
from rr_b200.models import SPECS, make_weights  # noqa: E402
from stop_oracle import stop_cut  # noqa: E402

NEVER = [bytes([250 + i]) * 64 for i in range(4)]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:        # the record says so rather than guessing
        return f"unavailable ({e})"


def kernel_us(rows=64, hist_len=512, reps=2000):
    rng = np.random.RandomState(0)
    hist = torch.from_numpy(rng.randint(3, 259, size=(rows, hist_len + 8)).astype(np.int32)).cuda()
    tok = torch.from_numpy(rng.randint(3, 259, size=rows).astype(np.int32)).cuda()
    gen0 = torch.zeros(rows, dtype=torch.int32).cuda()
    pos = torch.full((rows,), hist_len, dtype=torch.int32).cuda()
    n = torch.full((rows,), 4, dtype=torch.int32).cuda()
    ln = torch.full((rows, 4), 64, dtype=torch.uint8).cuda()
    by = torch.from_numpy(rng.randint(0, 256, size=(rows, 4, 64)).astype(np.uint8)).cuda()
    cut, hold = torch.zeros(rows, dtype=torch.int32).cuda(), torch.zeros(rows, dtype=torch.int32).cuda()
    st = torch.cuda.current_stream().cuda_stream
    args = (hist.data_ptr(), hist_len + 8, tok.data_ptr(), pos.data_ptr(), None, n.data_ptr(), gen0.data_ptr(),
            ln.data_ptr(), by.data_ptr(), cut.data_ptr(), hold.data_ptr(), rows, st)
    for _ in range(20):
        _lib.check(_lib.lib.rr_op_stop_match(*args), "rr_op_stop_match")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        _lib.lib.rr_op_stop_match(*args)
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps            # back-to-back launches: includes the launch gap


def run_queue(eng, prompts, max_new, stops, sampled=False):
    """sampled: temperature 1 with the request's index as its seed, so the replies differ and do not repeat themselves."""
    eng.reset_stats()
    t0 = time.perf_counter()
    tks = [eng.submit(p, max_new, stop=s, **(dict(temperature=1.0, seed=i) if sampled else {}))
           for i, (p, s) in enumerate(zip(prompts, stops))]
    recs = [eng.wait(t) for t in tks]
    wall = time.perf_counter() - t0
    assert all(r.status == 0 for r in recs)
    st = eng.stats()
    return recs, wall, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--rows", type=int, default=64)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--prompt-len", type=int, default=512)
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--hit-at", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    spec = SPECS[a.model]
    out = {"gpu": gpu_info(), "model": a.model, "rows": a.rows, "requests": a.requests, "prompt_len": a.prompt_len,
           "max_new": a.max_new, "rounds": a.rounds, "kernel_us_64rows_4x64B": round(kernel_us(), 3)}
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=a.prompt_len).tolist() for _ in range(a.requests)]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=a.rows, ctx_max=1024, max_prefill_tokens=8192)
    # (b) one full batch, every row with stop sequences that never hit, against the same batch plain
    step = {"plain": [], "stop": []}
    first = prompts[: a.rows]
    for arm in ("plain", "stop", "plain", "stop"):                # warm-up: graphs of both modes
        run_queue(eng, first, 8, [NEVER if arm == "stop" else None] * a.rows)
    same = True
    for _ in range(a.rounds):
        toks = {}
        for arm in ("plain", "stop"):
            recs, _, st = run_queue(eng, first, a.max_new, [NEVER if arm == "stop" else None] * a.rows)
            step[arm].append(st["decode_ms_total"] / st["decode_steps"])
            toks[arm] = [r.tokens for r in recs]
        same = same and toks["plain"] == toks["stop"]
    out["step_ms"] = {k: [round(x, 4) for x in v] for k, v in step.items()}
    out["step_tokens_equal"] = same
    # (c) the queue: stop sequences from each request's own free-running reply
    free, _, _ = run_queue(eng, prompts, a.max_new, [None] * a.requests, True)
    stops = []
    for r in free:
        t = r.tokens
        i = next((i for i in range(a.hit_at, len(t) - 1) if t[i] >= 3 and t[i + 1] >= 3), a.hit_at)
        stops.append([bytes((x - 3) % 256 for x in t[i: i + 2])])
    arms = {"plain": [None] * a.requests, "stop": stops}
    res = {k: {"completions_per_s": [], "decode_steps": [], "generated_tokens": [], "returned_tokens": []} for k in arms}
    equal = True
    for _ in range(a.rounds):
        for k, st_list in arms.items():
            recs, wall, st = run_queue(eng, prompts, a.max_new, st_list, True)
            r = res[k]
            r["completions_per_s"].append(round(a.requests / wall, 2))
            r["decode_steps"].append(st["decode_steps"])
            r["generated_tokens"].append(st["generated_tokens"])
            r["returned_tokens"].append(sum(len(x.tokens) for x in recs))
            if k == "stop":
                equal = equal and all(x.tokens == f.tokens[: stop_cut(f.tokens, s)[0]]
                                      for x, f, s in zip(recs, free, stops))
            else:
                equal = equal and all(x.tokens == f.tokens for x, f in zip(recs, free))
    eng.close()
    out["queue"] = res
    out["queue_kept_tokens_equal_oracle_cut"] = equal
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
