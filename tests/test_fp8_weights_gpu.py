"""GPU: FP8 weights (e4m3 projections with power-of-two row scales), from the kernels up to the engine.

D = bf16(Q * s) is exact, and the fp8 decode kernels convert each e4m3 tile into exactly the bf16 tile the bf16 kernels
read, then run the same wgmma sequence, splits and epilogues.  So every check here is bit for bit against the bf16 path on
D, never a tolerance: the quantizer against tests/fp8_oracle.py, rr_gemm_fp8w against rr_gemm_bf16, rr_op_decode_mlp_fp8
against rr_op_decode_mlp, and an fp8 engine against a bf16 engine built on Fp8Weights.dequantize()."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import fp8_oracle as ref
from test_gemm_gpu import _interleave64

pytestmark = pytest.mark.gpu
RR_INVALID_ARGUMENT = 4


def _lib():
    from rr_b200 import _lib
    return _lib


def _quantize(w):
    L = _lib()
    q = torch.empty(w.shape, dtype=torch.float8_e4m3fn, device="cuda")
    s = torch.empty(w.shape[0], dtype=torch.float32, device="cuda")
    rc = L.lib.rr_op_quantize_fp8_weight(w.data_ptr(), w.shape[0], w.shape[1], w.stride(0), q.data_ptr(), s.data_ptr(), None)
    return rc, q, s


def _dequantize(q, s):
    L = _lib()
    d = torch.full(q.shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    L.check(L.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), s.data_ptr(), q.shape[0], q.shape[1], d.data_ptr(),
                                              q.shape[1], None), "rr_op_dequantize_fp8_weight")
    torch.cuda.synchronize()
    return d


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32 if t.element_size() == 4 else torch.uint8)


# ---- quantizer / dequantizer ----------------------------------------------------------------------------------------------
SHAPES_Q = {
    "llama-3-8b": [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)],
    "phi-3-mini": [(9216, 3072), (3072, 3072), (16384, 3072), (3072, 8192)],
    "tiny96": [(1152, 384), (384, 384), (2048, 384), (384, 1024)],
    "ragged": [(1, 64), (7, 16), (33, 208), (129, 4096)],
}


def _planted(rows, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(rows, K, device="cuda", generator=g) * 0.02).bfloat16()
    if rows >= 8:
        w[1] = 0                                                   # zero row: e = 0, Q = 0
        w[2] = (torch.randn(K, device="cuda", generator=g) * 2.0 ** -128).bfloat16()   # below the clamp: e = -117
        w[3] = 0; w[3, ::5] = 448.0 * 2.0 ** -20                   # amax exactly at a bound
        w[4] = 2.0 ** torch.randint(-30, 5, (K,), device="cuda", generator=g).float()  # powers of two
        w[5] *= 1e-3; w[5, 0] = 3.0                                # many subnormal codes
        w[6, 0] = -0.0
    return w


@pytest.mark.parametrize("model,rows,K", [pytest.param(m, r, k, id=f"{m}-{r}x{k}") for m in SHAPES_Q for r, k in SHAPES_Q[m]])
def test_quantize_equals_reference_bit_for_bit(model, rows, K):
    w = _planted(rows, K, rows * 7 + K)
    rc, q, s = _quantize(w)
    assert rc == 0
    torch.cuda.synchronize()
    q_ref, s_ref = ref.quantize(w)                                 # torch on the GPU tensors (the same code runs on CPU)
    assert torch.equal(s, s_ref)
    assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8))
    if rows <= 4096 and K <= 4096:                                 # and the CPU run of the reference agrees
        q_cpu, s_cpu = ref.quantize(w.cpu())
        assert torch.equal(q_cpu.view(torch.uint8), q.cpu().view(torch.uint8)) and torch.equal(s_cpu, s.cpu())
    d = _dequantize(q, s)
    assert torch.equal(_bits(d), _bits(ref.dequantize(q, s)))
    assert torch.equal(d.double(), q.double() * s.double()[:, None])   # exact


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_quantize_refuses_a_row_with_nan_or_inf(bad):
    w = _planted(64, 256, 5)
    w[37, 100] = bad
    rc, _, _ = _quantize(w)
    assert rc == RR_INVALID_ARGUMENT
    rc, _, _ = _quantize(_planted(64, 256, 5))                     # and the next call is fine
    assert rc == 0


def test_quantize_and_dequantize_refuse_bad_arguments():
    L = _lib()
    w = _planted(16, 64, 1)
    q = torch.empty(16, 64, dtype=torch.float8_e4m3fn, device="cuda")
    s = torch.empty(16, dtype=torch.float32, device="cuda")
    assert L.lib.rr_op_quantize_fp8_weight(w.data_ptr(), 16, 40, 64, q.data_ptr(), s.data_ptr(), None) == RR_INVALID_ARGUMENT
    assert L.lib.rr_op_quantize_fp8_weight(w.data_ptr(), 16, 64, 64, q.data_ptr() + 8, s.data_ptr(), None) == RR_INVALID_ARGUMENT
    assert L.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), None, 16, 64, w.data_ptr(), 64, None) == RR_INVALID_ARGUMENT
    assert L.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), s.data_ptr(), 16, 64, w.data_ptr(), 60, None) == RR_INVALID_ARGUMENT


# ---- decode GEMM ----------------------------------------------------------------------------------------------------------
def _weight(rows, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(rows, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    rc, q, s = _quantize(w)
    assert rc == 0
    return q, s, _dequantize(q, s)


def _gemm(fp8, A, s, B, mode, bn, splits, ld_rows, ldo):
    L = _lib()
    rowsA, K = A.shape
    rowsB = B.shape[0]
    if mode == 1:
        out = torch.full((splits, ld_rows, ldo), float("nan"), device="cuda", dtype=torch.float32)
    else:
        out = torch.full((ld_rows, ldo), float("nan"), device="cuda", dtype=torch.bfloat16)
    if fp8:
        rc = L.lib.rr_gemm_fp8w(A.data_ptr(), s.data_ptr(), rowsA, K, B.data_ptr(), rowsB, K, K, out.data_ptr(), ldo,
                                ld_rows, splits, mode, bn, None)
    else:
        rc = L.lib.rr_gemm_bf16(A.data_ptr(), rowsA, K, B.data_ptr(), rowsB, K, K, out.data_ptr(), ldo, ld_rows, splits,
                                mode, bn, None)
    L.check(rc, "rr_gemm_fp8w" if fp8 else "rr_gemm_bf16")
    torch.cuda.synchronize()
    return out


GEMM_CASES = [  # rowsA, K, rowsB, bn, splits
    (128, 64, 1, 16, 1), (6144, 4096, 64, 64, 3), (4096, 4096, 16, 16, 4), (4096, 14336, 64, 64, 8),
    (1000, 320, 7, 16, 2), (384, 4096, 33, 64, 5), (640, 1024, 20, 32, 7), (512, 1024, 128, 128, 2),
    (1152, 384, 100, 128, 1), (4096, 1024, 32, 32, 6), (300, 4096, 64, 64, 8), (256, 512, 65, 128, 3),
]


@pytest.mark.parametrize("tma_epi", [True, False], ids=["tma-store", "per-thread"])
@pytest.mark.parametrize("rowsA,K,rowsB,bn,splits", GEMM_CASES)
def test_gemm_fp8w_f32_equals_bf16_on_dequantized(rowsA, K, rowsB, bn, splits, tma_epi, monkeypatch):
    if tma_epi:
        monkeypatch.delenv("RR_NO_TMA_EPI", raising=False)
    else:
        monkeypatch.setenv("RR_NO_TMA_EPI", "1")
    q, s, d = _weight(rowsA, K, rowsA + K)
    g = torch.Generator(device="cuda").manual_seed(rowsB)
    x = torch.randn(rowsB, K, device="cuda", generator=g).bfloat16()
    ld_rows = rowsB + 2
    a = _gemm(True, q, s, x, 1, bn, splits, ld_rows, rowsA)
    b = _gemm(False, d, None, x, 1, bn, splits, ld_rows, rowsA)
    n = min(splits, (K + 63) // 64)
    assert torch.equal(_bits(a[:n, :rowsB]), _bits(b[:n, :rowsB]))
    assert torch.isfinite(a[:n, :rowsB]).all()
    assert torch.isnan(a[:, rowsB:]).all() and torch.isnan(a[n:]).all(), "written past rows / planes"
    again = _gemm(True, q, s, x, 1, bn, splits, ld_rows, rowsA)
    assert torch.equal(_bits(again), _bits(a))


@pytest.mark.parametrize("inter,K,rowsB,bn", [(1024, 512, 17, 32), (14336, 4096, 64, 64), (8192, 3072, 128, 128),
                                               (1024, 384, 40, 64), (2048, 768, 32, 32)])
def test_gemm_fp8w_silu_equals_bf16_on_dequantized(inter, K, rowsB, bn):
    q, s, d = _weight(2 * inter, K, inter + K)
    g = torch.Generator(device="cuda").manual_seed(rowsB)
    x = torch.randn(rowsB, K, device="cuda", generator=g).bfloat16()
    a = _gemm(True, q, s, x, 2, bn, 1, rowsB + 1, inter)
    b = _gemm(False, d, None, x, 2, bn, 1, rowsB + 1, inter)
    assert torch.equal(_bits(a[:rowsB]), _bits(b[:rowsB])) and torch.isfinite(a[:rowsB]).all()
    assert torch.isnan(a[rowsB:]).all()


def test_gemm_fp8w_refuses_rowmajor_modes_and_null_scale():
    L = _lib()
    q, s, d = _weight(256, 256, 3)
    x = torch.randn(16, 256, device="cuda").bfloat16()
    out = torch.empty(256 * 256, device="cuda")
    for mode in (0, 3, 4, 5):
        assert L.lib.rr_gemm_fp8w(q.data_ptr(), s.data_ptr(), 256, 256, x.data_ptr(), 16, 256, 256, out.data_ptr(), 256,
                                  16, 1, mode, 16, None) == RR_INVALID_ARGUMENT
    assert L.lib.rr_gemm_fp8w(q.data_ptr(), None, 256, 256, x.data_ptr(), 16, 256, 256, out.data_ptr(), 256, 16, 1, 1, 16,
                              None) == RR_INVALID_ARGUMENT


# ---- fused decode MLP ------------------------------------------------------------------------------------------------------
MLP_SHAPES = [(4096, 14336), (3072, 8192), (1024, 2816), (768, 2048), (512, 1024), (384, 1024), (576, 1088)]


@pytest.mark.parametrize("static", [False, True], ids=["dynamic", "static"])
@pytest.mark.parametrize("hidden,inter", MLP_SHAPES)
def test_decode_mlp_fp8_equals_bf16_on_dequantized(hidden, inter, static, monkeypatch):
    L = _lib()
    if static:
        monkeypatch.setenv("RR_MLP_STATIC", "1")
    else:
        monkeypatch.delenv("RR_MLP_STATIC", raising=False)
    g = torch.Generator(device="cuda").manual_seed(hidden + inter)
    wgu = (torch.randn(2 * inter, hidden, device="cuda", generator=g) / math.sqrt(hidden)).bfloat16()
    wd = (torch.randn(hidden, inter, device="cuda", generator=g) / math.sqrt(inter)).bfloat16()
    rc, qgu, sgu = _quantize(wgu)
    rc2, qd, sd = _quantize(wd)
    assert rc == 0 and rc2 == 0
    dgu, dd = _dequantize(qgu, sgu), _dequantize(qd, sd)
    qgu_il = _interleave64(qgu.view(torch.uint8), inter)
    sgu_il = _interleave64(sgu[:, None], inter)[:, 0].contiguous()
    dgu_il = _interleave64(dgu, inter)
    for rows in (17, 64, 65, 128):
        x = torch.randn(rows, hidden, device="cuda", generator=g).bfloat16()
        outs = []
        for fp8 in (True, True, False):
            act = torch.full(((rows + 64) * inter,), float("nan"), device="cuda", dtype=torch.bfloat16)
            planes = torch.full((8, rows + 3, hidden), float("nan"), device="cuda", dtype=torch.float32)
            ns, skb = C.c_int32(-1), C.c_int32(-1)
            if fp8:
                rc = L.lib.rr_op_decode_mlp_fp8(qgu_il.data_ptr(), sgu_il.data_ptr(), qd.data_ptr(), sd.data_ptr(),
                                                x.data_ptr(), rows, hidden, inter, act.data_ptr(), planes.data_ptr(),
                                                rows + 3, C.byref(ns), C.byref(skb), None)
            else:
                rc = L.lib.rr_op_decode_mlp(dgu_il.data_ptr(), dd.data_ptr(), x.data_ptr(), rows, hidden, inter,
                                            act.data_ptr(), planes.data_ptr(), rows + 3, C.byref(ns), C.byref(skb), None)
            L.check(rc, "decode mlp")
            torch.cuda.synchronize()
            outs.append((act, planes, ns.value))
        (a8, p8, n8), (a8b, p8b, _), (ab, pb, nb) = outs
        assert n8 == nb
        assert torch.equal(_bits(a8[: rows * inter]), _bits(ab[: rows * inter])), f"act rows={rows}"
        assert torch.equal(_bits(p8[:n8, :rows]), _bits(pb[:nb, :rows])), f"planes rows={rows}"
        assert torch.isfinite(p8[:n8, :rows]).all() and torch.isnan(p8[:n8, rows:]).all()
        assert torch.equal(_bits(a8), _bits(a8b)) and torch.equal(_bits(p8), _bits(p8b)), "two calls differ"


# ---- engine ---------------------------------------------------------------------------------------------------------------
def _pair(name, max_batch=64, **kw):
    """An fp8 engine and a bf16 engine on its dequantized weights."""
    from rr_b200.engine import Engine
    from rr_b200.models import SPECS, make_weights, quantize_fp8
    spec = SPECS[name]
    w = make_weights(spec, seed=5, sigma=0.05, device="cuda", norm_jitter=0.1)
    q = quantize_fp8(w)
    d = q.dequantize()
    e8 = Engine(q, max_batch=max_batch, **kw)
    eb = Engine(d, max_batch=max_batch, **kw)
    return spec, w, q, d, e8, eb


def _res(r):
    assert r.status == 0, r.status
    lp = None if r.choice_logprobs is None else [[[(i, np.float32(v).view(np.int32).item()) for i, v in row] for row in c]
                                                 for c in r.choice_logprobs]
    return r.choices, r.finish_reasons, lp


def _run(eng, reqs):
    tk = [eng.submit(p, m, **kw) for p, m, kw in reqs]
    return [_res(eng.wait(t, timeout=600)) for t in tk]


def _prompts(spec, n, lo, hi, seed):
    rs = np.random.RandomState(seed)
    return [rs.randint(3, spec.vocab, size=rs.randint(lo, hi)).tolist() for _ in range(n)]


@pytest.mark.parametrize("name,max_batch", [pytest.param("tiny", 64, id="tiny"), pytest.param("tiny96", 64, id="tiny96"),
                                            pytest.param("llama-3-8b-2l", 64, id="llama-3-8b-2l"),
                                            # two batch tiles per weight tile, MLP unfused
                                            pytest.param("tiny", 256, id="tiny-256")])
def test_engine_fp8_equals_bf16_engine_on_dequantized_weights(name, max_batch):
    from oracle import llama_ref
    spec, w, q, d, e8, eb = _pair(name, max_batch, ctx_max=1024, max_prefill_tokens=2048, prefix_cache=True)
    try:
        # low-level prefill / decode logits
        ps = _prompts(spec, 4, 5, 200, 1)
        f8, l8 = e8.prefill(ps, [0, 1, 2, 3], want_logits=True)
        fb, lb = eb.prefill(ps, [0, 1, 2, 3], want_logits=True)
        assert np.array_equal(f8, fb) and np.array_equal(l8.view(np.int32), lb.view(np.int32))
        pos = [len(p) for p in ps]
        n8, m8 = e8.decode_step([0, 1, 2, 3], f8, pos, want_logits=True)
        nb, mb = eb.decode_step([0, 1, 2, 3], fb, pos, want_logits=True)
        assert np.array_equal(n8, nb) and np.array_equal(m8.view(np.int32), mb.view(np.int32))
        # teacher-forced logits against the fp32 reference model on D (test_engine_gpu.py's tolerance), and the rms
        # deviation from the original bf16 weights (informational, loose)
        ref_d = llama_ref.forward_logits(d, ps[0])[-1].float().cpu().numpy()
        dev, std = l8[0] - ref_d, float(np.std(ref_d))
        assert np.sqrt(np.mean(dev ** 2)) <= 0.02 * std and np.abs(dev).max() <= 0.08 * std   # test_engine_gpu.py's bounds
        ref_w = llama_ref.forward_logits(w, ps[0])[-1].float().cpu().numpy()
        rms = float(np.sqrt(np.mean((l8[0] - ref_w) ** 2)) / (np.std(ref_w) + 1e-12))
        print(f"{name}: rms(fp8 logits - bf16-weight logits) / std = {rms:.4f}")
        assert rms < 0.3                                              # measured on an H100: 0.16 tiny, 0.10 tiny96, 0.22 8b-2l
        # serving: greedy + logprobs, seeded sampling, n = 3, stop, JSON mode, a 64-request burst, a prefix hit
        base = _prompts(spec, 64, 8, 300, 2)
        reqs = [(p, 24, {}) for p in base[:40]]
        reqs += [(p, 16, dict(top_logprobs=20)) for p in base[40:48]]
        reqs += [(p, 16, dict(temperature=0.8, top_p=0.9, seed=11 + i, top_logprobs=3)) for i, p in enumerate(base[48:56])]
        reqs += [(base[56], 12, dict(n=3, temperature=1.0, seed=3, top_logprobs=2))]
        reqs += [(base[57], 40, dict(stop=["a", "\x05"])), (base[58], 40, dict(response_format={"type": "json_object"}))]
        reqs += [(p, 8, {}) for p in base[59:64]]
        assert _run(e8, reqs) == _run(eb, reqs)
        # a prefix-cache hit: the second prompt shares 130 leading tokens with the first, which has finished
        shared = base[0][:8] + list(range(3, 3 + 122))
        for eng in (e8, eb):
            eng.reset_stats()
        assert _run(e8, [(shared + [7, 8, 9], 10, {})]) == _run(eb, [(shared + [7, 8, 9], 10, {})])
        hit = [(shared + [11, 12], 10, dict(top_logprobs=5))]
        assert _run(e8, hit) == _run(eb, hit)
        assert e8.stats()["prefix_hits"] == eb.stats()["prefix_hits"] == 1
        assert e8.stats()["prefix_cached_tokens"] == eb.stats()["prefix_cached_tokens"] >= 64
    finally:
        e8.close(); eb.close()


@pytest.mark.parametrize("name", ["tiny", "llama-3-8b-2l"])
def test_engine_fp8_prompt_in_pieces_equals_bf16(name):
    """max_prefill_tokens small: long prompts run over several chunks (PDL on), each chunk dequantizing every layer into
    the scratch between the previous layer's GEMMs and this layer's."""
    spec, w, q, d, e8, eb = _pair(name, ctx_max=2048, max_prefill_tokens=128)
    try:
        ps = _prompts(spec, 12, 200, 900, 4)
        reqs = [(p, 16, dict(top_logprobs=4)) for p in ps[:10]] + [(ps[10], 16, dict(n=2, temperature=0.7, seed=1))]
        reqs += [(ps[11], 16, dict(response_format={"type": "json_object"}))]
        assert _run(e8, reqs) == _run(eb, reqs)
    finally:
        e8.close(); eb.close()


def test_engine_fp8_resident_bytes_and_kv_usage():
    from rr_b200.engine import Engine
    from rr_b200.models import SPECS
    spec = SPECS["llama-3-8b-2l"]
    # 64 rows, as served: the gate/up rows are interleaved, and the engine holds that copy beside the caller's weights
    e8 = Engine.synthetic(spec, quantization="fp8", max_batch=64, ctx_max=1024, kv_cache_tokens=4096)
    eb = Engine.synthetic(spec, max_batch=64, ctx_max=1024, kv_cache_tokens=4096)
    try:
        nqkv = (spec.n_heads + 2 * spec.n_kv_heads) * spec.head_dim
        proj = nqkv * spec.hidden + spec.hidden * spec.n_heads * spec.head_dim + 3 * spec.inter * spec.hidden
        rows = nqkv + spec.hidden + 2 * spec.inter + spec.hidden
        want = spec.n_layers * (proj + 4 * rows + 4 * spec.hidden) + 2 * 2 * spec.vocab * spec.hidden + 2 * spec.hidden
        assert e8.weights.nbytes() == want
        il = sum(t.numel() * t.element_size() for t in e8._wgu_il + e8._wgu_scale_il)
        assert il == spec.n_layers * (2 * spec.inter * spec.hidden + 4 * 2 * spec.inter)
        assert e8.kv_usage() == eb.kv_usage()
        p = list(range(3, 300))
        assert _run(e8, [(p, 8, {})]) and e8.kv_usage() == eb.kv_usage()
    finally:
        e8.close(); eb.close()
    with pytest.raises(ValueError):
        Engine.synthetic(spec, quantization="int8")


def test_full_llama_3_8b_fp8_equals_bf16_on_dequantized():
    """32 layers, 8 rows x 512-token prompts, 32 greedy tokens."""
    from rr_b200.engine import Engine
    from rr_b200.models import SPECS, make_weights, quantize_fp8
    spec = SPECS["llama-3-8b"]
    w = make_weights(spec, seed=0, device="cuda")
    q = quantize_fp8(w)
    del w
    torch.cuda.empty_cache()
    d = q.dequantize()
    ps = _prompts(spec, 8, 512, 513, 9)
    reqs = [(p, 32, {}) for p in ps]
    e8 = Engine(q, max_batch=64, ctx_max=1024)
    r8 = _run(e8, reqs)
    e8.close()
    eb = Engine(d, max_batch=64, ctx_max=1024)
    rb = _run(eb, reqs)
    eb.close()
    assert r8 == rb


# ---- gateway ---------------------------------------------------------------------------------------------------------------
def _server(router):
    import os
    import threading
    import time
    import uvicorn
    from rr_b200.server import create_app
    port = 23000 + os.getpid() % 1000
    server = uvicorn.Server(uvicorn.Config(create_app(router), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(200):
        if server.started:
            break
        time.sleep(0.05)
    return server, th, port


def test_gateway_fp8_deployment_over_http_equals_the_engine_level_run():
    """An fp8 deployment built by build_backends (Engine.synthetic(quantization="fp8")) against a bf16 replica on the same
    weights dequantized, through the OpenAI SDK, streamed and non-streamed; and Router.completion against the Engine-level
    fp8 run."""
    import openai
    from rr_b200 import EngineBackend, Router, SPECS, make_weights
    from rr_b200.config import build_config
    from rr_b200.engine import Engine
    from rr_b200.models import quantize_fp8
    from rr_b200.server import build_backends
    ml = [{"model_name": "fp8", "litellm_params": {"model": "b200/tiny", "gpu": 0, "quantization": "fp8"}},
          {"model_name": "ref", "litellm_params": {"model": "b200/tiny", "gpu": 1}}]
    backends = build_backends(build_config(ml[:1]), stub=False, max_batch=8)
    assert backends[0].engine.weights.__class__.__name__ == "Fp8Weights"
    q = quantize_fp8(make_weights(SPECS["tiny"], seed=0, device="cuda"))     # build_backends' weights, quantized alike
    ref_eng, e8 = Engine(q.dequantize(), max_batch=8), Engine(q, max_batch=8)
    backends[1] = EngineBackend(ref_eng)
    r = Router(model_list=ml, backends=backends, default_max_tokens=24, seed=0)
    server, th, port = _server(r)
    try:
        for k in range(3):
            p = _prompts(SPECS["tiny"], 1, 20, 200, 30 + k)[0]
            o = r.completion(model="fp8", prompt_ids=p, max_tokens=12)
            assert o._token_ids == e8.wait(e8.submit(p, 12)).tokens
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        for turn in ("hello there", "what is fp8?", "{\"a\": 1}"):
            msgs = [{"role": "user", "content": turn}]
            a = client.chat.completions.create(model="fp8", messages=msgs, timeout=60)
            b = client.chat.completions.create(model="ref", messages=msgs, timeout=60)
            assert a.choices[0].message.content == b.choices[0].message.content
            assert a.usage.completion_tokens == b.usage.completion_tokens > 0
            sa = "".join(c.choices[0].delta.content or "" for c in
                         client.chat.completions.create(model="fp8", messages=msgs, stream=True, timeout=60) if c.choices)
            assert sa == a.choices[0].message.content
    finally:
        server.should_exit = True
        th.join(10)
        r.close(); backends[0].engine.close(); ref_eng.close(); e8.close()


def test_gateway_fp8_fallback_replays_through_the_oracle_router():
    from rr_b200 import EngineBackend, Router, SPECS, make_weights
    from rr_b200.engine import Engine
    from rr_b200.models import quantize_fp8
    from test_gateway_gpu import _replay
    spec = SPECS["tiny"]
    q = quantize_fp8(make_weights(spec, seed=0, sigma=0.05, device="cuda"))
    kw = dict(max_batch=4, ctx_max=1024)
    bad, good, ref_eng = Engine(q, fail_prob=0.5, fail_seed=42, **kw), Engine(q, **kw), Engine(q.dequantize(), **kw)
    ml = [{"model_name": "primary", "litellm_params": {"model": "b200/tiny", "gpu": 0, "quantization": "fp8"}},
          {"model_name": "backup", "litellm_params": {"model": "b200/tiny", "gpu": 1, "quantization": "fp8"}}]
    r = Router(model_list=ml, routing_strategy="simple-shuffle", fallbacks=[{"primary": ["backup"]}], allowed_fails=1000,
               cooldown_time=15, backends={0: EngineBackend(bad), 1: EngineBackend(good)}, seed=0, clock=lambda: 7000.0)
    r.record_trace = 4096
    try:
        fell = 0
        for k in range(12):
            p = _prompts(spec, 1, 30, 400, 50 + k)[0]
            want = ref_eng.wait(ref_eng.submit(p, 6))
            o = r.completion(model="primary", prompt_ids=p, max_tokens=6)
            assert o._token_ids == want.tokens
            fell += o._fell_back
        assert 0 < fell < 12
        assert _replay(r, r.gateway_trace()) == 12 + fell
    finally:
        r.close(); bad.close(); good.close(); ref_eng.close()


def test_quantize_refuses_a_row_whose_codes_leave_the_bf16_range():
    w = _planted(16, 64, 9)
    w[5, 3] = 3.3e38                                            # amax within 2^-4 of bf16's largest value: 256 * 2^120 = inf
    rc, _, _ = _quantize(w)
    assert rc == RR_INVALID_ARGUMENT
    w[5, 3] = 3.0e38                                            # 226 * 2^120 rounds down to 224 * 2^120: accepted
    rc, q, s = _quantize(w)
    assert rc == 0
    d = _dequantize(q, s)
    assert torch.isfinite(d.float()).all() and torch.equal(d.double(), q.double() * s.double()[:, None])
