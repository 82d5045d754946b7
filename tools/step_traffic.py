"""profiles/r02_decode_step_traffic.json from the ncu_summary records of tools/profile_r02.sh's decode captures:
DRAM bytes of one decode step = (layer 0's six kernels) x n_layers + embed + first norm + lm_head + argmax.
  python tools/ncu_summary.py --json /tmp/recs.json profiles/r02_decode_layer0.ncu-rep profiles/r02_decode_head.ncu-rep
  python tools/step_traffic.py /tmp/recs.json profiles/r02_decode_step_traffic.json"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
src, dst = sys.argv[1], sys.argv[2]
recs = json.load(open(src))
lay = [r for r in recs if "decode_layer0" in r["file"]]
head = [r for r in recs if "decode_head" in r["file"]]
assert len(lay) == 8 and len(head) == 2, (len(lay), len(head))
labels = ["embed_kernel", "add_rmsnorm (layer 0 input norm)", "gemm_bf16_tcgen05<64,1> QKV projection", "decode_attn_mma_kernel<4>",
          "gemm_bf16_tcgen05<64,1> O projection", "add_rmsnorm (after O)", "gemm_mlp_tcgen05<64>", "add_rmsnorm (after MLP)",
          "gemm_bf16_tcgen05<64,1> lm_head", "argmax_kernel"]
L, rows, prompt_len, ctx = 32, 64, 512, 577
per = lambda r: r["dram_read_bytes"] + r["dram_write_bytes"]
total = per(lay[0]) + per(lay[1]) + L * sum(per(r) for r in lay[2:8]) + per(head[0]) + per(head[1])
# algorithmic bytes at the same context (models.py: weights streamed once + KV of ctx tokens per row)
import importlib.util
spec = importlib.util.spec_from_file_location("_m", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                                  "sample-resilient-llm-inference_b200", "models.py"))
m = importlib.util.module_from_spec(spec); sys.modules["_m"] = m; spec.loader.exec_module(m)
s = m.SPECS["llama-3-8b"]
alg = s.weight_bytes_per_decode_step + rows * ctx * s.kv_bytes_per_token
out = {"model": "llama-3-8b", "rows": rows, "prompt_len": prompt_len, "ctx": ctx, "dram_bytes_per_step": int(total),
       "algorithmic_bytes_same_ctx": int(alg),
       "source": "ncu --set full --clock-control none over one eager decode step of the final code (tools/profile_r02.sh): sum over "
                 "the step's 196 kernels of dram__bytes_read.sum + dram__bytes_write.sum (layer 0's six kernels x 32 + embed, first norm, "
                 "lm_head, argmax); profiles/r02_ncu_full_summary.txt; tools/step_traffic.py.  ncu flushes the caches between kernels, so the "
                 "small consumers (norm planes, logits for argmax) show DRAM reads that are L2 hits inside the real step: an upper bound.",
       "kernels": [{"kernel": lb, "time_us_isolated": r["time_us"], "dram_read_bytes": r["dram_read_bytes"],
                    "dram_write_bytes": r["dram_write_bytes"], "tensor_pipe_pct": r["tensor_pipe_pct"],
                    "dram_pct_of_ncu_peak": r["dram_pct"]} for lb, r in zip(labels, lay + head)]}
json.dump(out, open(dst, "w"), indent=1)
print(f"{total / 1e9:.3f} GB per step = {total / alg:.3f} x algorithmic ({alg / 1e9:.3f} GB)")
