"""JSON mode on the full-size model: what the grammar mask costs and what an early end gives back.

(a) kernels: rr_op_json_mask at 64 x 128256 with every row inside a string (few columns written) and with every row after
    '{' (nearly every column written), and rr_op_json_advance at 64 rows; CUDA events over many back-to-back launches.
(b) step: a Llama-3-8B decode step with all 64 rows in JSON mode against the same rows plain, alternated --rounds times in
    one process (decode_ms_total / decode_steps of the engine's CUDA events).  Both arms carry the same logit bias, which
    keeps the JSON rows inside one long string so that none ends before max_new: the arms differ by the two JSON
    launches and the 4-byte readback only.
(c) queue: 256 requests of 512 tokens in / 128 max out on 64 rows, temperature 1, seed = the request's index, with a small
    bias towards '}' so that objects close early.  Arm "json" asks for json_object, arm "plain" does not; alternated
    --rounds times after one warm-up: completions/s, decode steps, returned tokens, and how many JSON replies closed
    their object (and parse as a dict).

    python tools/json_probe.py --out json_probe.json
"""
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

from rr_b200 import _lib  # noqa: E402
from rr_b200.engine import Engine  # noqa: E402
from rr_b200.models import SPECS, make_weights  # noqa: E402

JS = {"type": "json_object"}
B = lambda ch: 3 + ord(ch)                                        # noqa: E731  the byte tokenizer's id of a character


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:        # the record says so rather than guessing
        return f"unavailable ({e})"


def _timed(fn, reps):
    for _ in range(20):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps            # back-to-back launches: includes the launch gap


def kernel_us(rows=64, vocab=128256, reps=500):
    st = torch.cuda.current_stream().cuda_stream
    x = torch.zeros((rows, vocab), dtype=torch.float32, device="cuda")
    fmt = torch.ones(rows, dtype=torch.int32, device="cuda")
    state = torch.zeros((rows, 16), dtype=torch.uint8, device="cuda")
    done = torch.zeros(rows, dtype=torch.int32, device="cuda")
    out = {}
    for name, byte in (("after_open_brace", "{"), ("in_string", '"')):
        state.zero_()
        tok = torch.full((rows,), B("{"), dtype=torch.int32, device="cuda")
        _lib.check(_lib.lib.rr_op_json_advance(rows, fmt.data_ptr(), None, tok.data_ptr(), None, state.data_ptr(), None,
                                               done.data_ptr(), st), "rr_op_json_advance")
        if byte == '"':
            tok.fill_(B('"'))
            _lib.check(_lib.lib.rr_op_json_advance(rows, fmt.data_ptr(), None, tok.data_ptr(), state.data_ptr(),
                                                   state.data_ptr(), None, done.data_ptr(), st), "rr_op_json_advance")
        out[f"mask_us_{name}"] = round(_timed(lambda: _lib.lib.rr_op_json_mask(
            x.data_ptr(), vocab, rows, vocab, fmt.data_ptr(), None, state.data_ptr(), st), reps), 3)
    nxt = torch.zeros_like(state)
    tok = torch.full((rows,), B("a"), dtype=torch.int32, device="cuda")
    out["advance_us"] = round(_timed(lambda: _lib.lib.rr_op_json_advance(
        rows, fmt.data_ptr(), None, tok.data_ptr(), state.data_ptr(), nxt.data_ptr(), None, done.data_ptr(), st), reps), 3)
    return out


def run_queue(eng, prompts, max_new, sampled=False, **kw):
    eng.reset_stats()
    t0 = time.perf_counter()
    tks = [eng.submit(p, max_new, **kw, **(dict(temperature=1.0, seed=i) if sampled else {}))
           for i, p in enumerate(prompts)]
    recs = [eng.wait(t) for t in tks]
    wall = time.perf_counter() - t0
    assert all(r.status == 0 for r in recs)
    return recs, wall, eng.stats()


def _closed(tokens):
    try:
        return isinstance(json.loads(bytes((t - 3) % 256 for t in tokens).decode("utf-8")), dict)
    except ValueError:
        return False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3-8b")
    ap.add_argument("--rows", type=int, default=64)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--prompt-len", type=int, default=512)
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--close-bias", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    spec = SPECS[a.model]
    out = {"gpu": gpu_info(), "model": a.model, "rows": a.rows, "requests": a.requests, "prompt_len": a.prompt_len,
           "max_new": a.max_new, "rounds": a.rounds, "kernels_64x128256": kernel_us()}
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, spec.vocab, size=a.prompt_len).tolist() for _ in range(a.requests)]
    eng = Engine(make_weights(spec, seed=0, device="cuda"), max_batch=a.rows, ctx_max=1024, max_prefill_tokens=8192)
    # (b) one full batch in one long string, JSON mode against plain with the same bias
    string_bias = {B("{"): 50.0, B('"'): 50.0, B("a"): 100.0}      # '{' lies inside strings too: below 'a'
    step = {"plain": [], "json": []}
    first = prompts[: a.rows]
    for arm in ("plain", "json", "plain", "json"):                # warm-up: graphs of both modes
        run_queue(eng, first, 8, logit_bias=string_bias, response_format=JS if arm == "json" else None)
    for _ in range(a.rounds):
        for arm in ("plain", "json"):
            recs, _, st = run_queue(eng, first, a.max_new, logit_bias=string_bias,
                                    response_format=JS if arm == "json" else None)
            assert all(len(r.tokens) == a.max_new for r in recs)
            step[arm].append(st["decode_ms_total"] / st["decode_steps"])
    out["step_ms"] = {k: [round(x, 4) for x in v] for k, v in step.items()}
    # (c) the queue: JSON replies that close their object early against the same queue plain
    bias = {B("}"): a.close_bias}
    res = {k: {"completions_per_s": [], "decode_steps": [], "returned_tokens": [], "closed": []} for k in ("plain", "json")}
    for arm in ("plain", "json"):
        run_queue(eng, prompts[: a.rows], 16, True, logit_bias=bias, response_format=JS if arm == "json" else None)
    for _ in range(a.rounds):
        for arm in ("plain", "json"):
            recs, wall, st = run_queue(eng, prompts, a.max_new, True, logit_bias=bias,
                                       response_format=JS if arm == "json" else None)
            r = res[arm]
            r["completions_per_s"].append(round(a.requests / wall, 2))
            r["decode_steps"].append(st["decode_steps"])
            r["returned_tokens"].append(sum(len(x.tokens) for x in recs))
            r["closed"].append(sum(x.finish_reasons == ["stop"] and _closed(x.tokens) for x in recs))
    eng.close()
    out["queue"] = res
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
