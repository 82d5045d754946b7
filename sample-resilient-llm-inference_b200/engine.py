"""Python handle on one model replica (rr_engine in librr_b200.so).

Thin by design: torch provides device memory for the weights and the current device; every
computation happens in the CUDA library.  Replaces one `bedrock/...` deployment of the reference
(config/config.yaml:39-91) — the thing `litellm` would call over the network.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .models import Fp8Weights, ModelSpec, Weights, make_weights, quantize_fp8
from .router import FINISH_REASONS, check_response_format, check_stop, gen_args, logprob_pairs


@dataclass
class CompletionRecord:
    ticket: int
    status: int
    n_prompt: int
    tokens: List[int]
    t_submit: float
    t_first_token: float
    t_done: float
    # submit(top_logprobs=k): per generated token the max(1, k) most likely (token id, logprob) pairs, best first; with
    # temperature > 0 followed by the generated token's own pair
    logprobs: Optional[List[List[Tuple[int, float]]]] = None
    # prompt tokens whose KV came from the prefix cache (Engine(prefix_cache=True)); 0 otherwise
    n_cached: int = 0
    # submit(n=k): every choice's tokens and, with top_logprobs, pairs ([k][tokens]); tokens / logprobs are choice 0's
    choices: List[List[int]] = field(default_factory=list)
    choice_logprobs: Optional[List[List[List[Tuple[int, float]]]]] = None
    # every choice's finish reason: "stop" when a stop sequence of submit(stop=) cut it (its tokens end before the match),
    # else "length"; with `stop` the choices have their own lengths
    finish_reasons: List[str] = field(default_factory=list)

    @property
    def ttft(self) -> float:
        return self.t_first_token - self.t_submit

    @property
    def latency(self) -> float:
        return self.t_done - self.t_submit


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32))


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def pick_splits(rows_w: int, K: int, n_sm: int) -> int:
    """Split-K planes of a decode projection of rows_w weight rows over K inputs on a GPU with n_sm SMs; mirrors
    pick_splits() in csrc/rr_gemm.cu."""
    tiles, kb = (rows_w + 127) // 128, (K + 63) // 64
    s = max(1, min(8, n_sm // tiles))
    while s > 1 and kb // s < 8:
        s -= 1
    return s


class Engine:
    def __init__(self, weights: Union[Weights, Fp8Weights], device: int = 0, max_batch: int = 64, ctx_max: int = 1024,
                 max_prefill_tokens: int = 8192, use_cuda_graph: bool = True,
                 fail_prob: float = 0.0, fail_seed: int = 0, prefix_cache: bool = False,
                 kv_cache_tokens: Optional[int] = None):
        """prefix_cache=True: a KV slot keeps the prompt its last prefill wrote, and a prompt that shares at least 64
        leading tokens with one is prefilled from there on (tokens and logits bit-identical to a cold prefill).  Off by
        default: a resident prefix is a timing side channel between the engine's users.

        kv_cache_tokens: the KV cache, a pool of 64-token pages the decode rows share; None = max_batch x ctx_max (the pool
        never binds).  Otherwise a multiple of 64 in [ctx_max, max_batch x ctx_max].  ctx_max is then the limit of one
        request (prompt + max_new_tokens), and each choice reserves ceil((prompt + max_new_tokens) / 64) pages while it
        runs; a request that does not fit waits, and one that never could is refused at submit.

        weights: bf16 Weights, or Fp8Weights (models.quantize_fp8): e4m3 layer projections, computing exactly what a bf16
        engine computes on weights.dequantize().  Prefill then also holds a bf16 scratch of one layer's projections."""
        if not torch.cuda.is_available():
            raise RuntimeError("rr_b200.Engine needs a CUDA device (no CPU fallback)")
        self.spec: ModelSpec = weights.spec
        self.weights = weights          # keep the tensors alive
        self.device = device
        self.max_batch = max_batch
        self.ctx_max = ctx_max
        self.max_prefill_tokens = max_prefill_tokens
        self.prefix_cache = bool(prefix_cache)
        self.kv_cache_tokens = int(kv_cache_tokens or max_batch * ctx_max)
        s = self.spec
        desc = _lib.ModelDesc(s.vocab, s.hidden, s.inter, s.n_layers, s.n_heads, s.n_kv_heads,
                              s.head_dim, s.rope_theta, s.rms_eps)
        L = s.n_layers

        def arr(ts):
            return (C.c_void_p * L)(*[t.data_ptr() for t in ts])

        # Engine-owned layout of the gate/up weights: rows interleaved in 64-row gate/up blocks so that the GEMM
        # epilogue can apply SiLU(gate) * up itself (csrc/rr_gemm.cu, OUT_*_SILU).  Needs one gate/up plane at this
        # batch size (no split-K for gate/up) and batch tiles >= 32 rows; otherwise the [gate; up] layout is kept.
        n_sm = torch.cuda.get_device_properties(device).multi_processor_count
        gu_splits = pick_splits(2 * s.inter, s.hidden, n_sm)
        interleave = s.inter % 64 == 0 and gu_splits == 1 and max_batch > 16
        fp8 = isinstance(weights, Fp8Weights)
        wgu = weights.wgu
        wgu_scale = weights.wgu_scale if fp8 else []

        def il(t):                  # [gate; up] -> 64-row blocks [g0..g63, u0..u63, ...] (rows, or their scales)
            g, u = t[: s.inter].reshape(-1, 64, *t.shape[1:]), t[s.inter:].reshape(-1, 64, *t.shape[1:])
            return torch.stack([g, u], 1).reshape(2 * s.inter, *t.shape[1:]).contiguous()

        if interleave:
            self._wgu_il = [il(t.view(torch.uint8)).view(t.dtype) if fp8 else il(t) for t in weights.wgu]
            wgu = self._wgu_il
            if fp8:
                self._wgu_scale_il = [il(t) for t in weights.wgu_scale]
                wgu_scale = self._wgu_scale_il
        self._arrs = [arr(weights.wqkv), arr(weights.wo), arr(wgu), arr(weights.wdown),
                      arr(weights.norm_attn), arr(weights.norm_mlp)]
        dtypes = (torch.bfloat16, torch.float8_e4m3fn, torch.float32) if fp8 else (torch.bfloat16,)
        for t in weights.tensors():
            assert t.is_cuda and t.dtype in dtypes and t.is_contiguous()
        scales = [None] * 4
        if fp8:
            self._arrs += [arr(weights.wqkv_scale), arr(weights.wo_scale), arr(wgu_scale), arr(weights.wdown_scale)]
            scales = self._arrs[6:]
        flags = (_lib.RR_WEIGHTS_WGU_INTERLEAVED64 if interleave else 0) | (_lib.RR_WEIGHTS_FP8_E4M3 if fp8 else 0)
        mw = _lib.ModelWeights(weights.embed.data_ptr(), weights.lm_head.data_ptr(),
                               weights.final_norm.data_ptr(), *self._arrs[:6], flags, s.sliding_window, *scales)
        opts = _lib.EngineOpts(device, max_batch, ctx_max, max_prefill_tokens,
                               1 if use_cuda_graph else 0, fail_seed, fail_prob,
                               int(kv_cache_tokens or 0), (C.c_int32 * 3)(),
                               1 if prefix_cache else 0)
        torch.cuda.synchronize(device)   # weights were produced on torch's stream
        self._lp_k: Dict[int, int] = {}     # ticket -> pairs per token of a request submitted with top_logprobs
        self._n: Dict[int, int] = {}        # ticket -> choices of a request submitted with n > 1
        self._score: Dict[int, Tuple[int, int]] = {}    # ticket -> (prompt length, pairs per position) of a scoring request
        self._h = C.c_void_p()
        _lib.check(_lib.lib.rr_engine_create(C.byref(desc), C.byref(mw), C.byref(opts),
                                             C.byref(self._h)), "rr_engine_create")

    @classmethod
    def synthetic(cls, spec: ModelSpec, seed: int = 0, device: int = 0, quantization: Optional[str] = None,
                  **kw) -> "Engine":
        """An engine on the seeded weights of make_weights.  quantization="fp8": those weights through quantize_fp8, the
        bf16 copy freed before the engine is created (peak memory while quantizing: both copies, about 16 + 9.5 GB for
        Llama-3-8B)."""
        if quantization not in (None, "fp8"):
            raise ValueError(f"quantization must be None or 'fp8', got {quantization!r}")
        w = make_weights(spec, seed=seed, device=f"cuda:{device}")
        if quantization == "fp8":
            q = quantize_fp8(w)
            del w
            torch.cuda.empty_cache()     # the engine allocates its buffers with cudaMalloc, outside torch's cache
            w = q
        return cls(w, device=device, **kw)

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib.rr_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- low-level synchronous steps (parity tests) ---------------------------------------------
    def prefill(self, prompts: Sequence[Sequence[int]], slots: Sequence[int], want_logits=False):
        ids = _i32([t for p in prompts for t in p])
        start = _i32(np.concatenate([[0], np.cumsum([len(p) for p in prompts])]))
        sl = _i32(slots)
        n = len(prompts)
        first = np.zeros(n, dtype=np.int32)
        logits = np.zeros((n, self.spec.vocab), dtype=np.float32) if want_logits else None
        lp = logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None
        _lib.check(_lib.lib.rr_engine_prefill(self._h, _p(ids), _p(start), _p(sl), n, _p(first), lp),
                   "rr_engine_prefill")
        return first, logits

    def decode_step(self, slots, toks, pos, want_logits=False):
        sl, tk, ps = _i32(slots), _i32(toks), _i32(pos)
        n = len(sl)
        nxt = np.zeros(n, dtype=np.int32)
        logits = np.zeros((n, self.spec.vocab), dtype=np.float32) if want_logits else None
        lp = logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None
        _lib.check(_lib.lib.rr_engine_decode_step(self._h, _p(sl), _p(tk), _p(ps), n, _p(nxt), lp),
                   "rr_engine_decode_step")
        return nxt, logits

    # ---- serving interface ----------------------------------------------------------------------
    def submit(self, prompt_ids: Sequence[int], max_new_tokens: int, top_logprobs: Optional[int] = None,
               temperature: Optional[float] = None, top_p: Optional[float] = None, seed: Optional[int] = None,
               frequency_penalty: Optional[float] = None, presence_penalty: Optional[float] = None,
               logit_bias: Optional[Dict[int, float]] = None, n: int = 1, stop=None, response_format=None,
               prompt_logprobs: Optional[int] = None) -> int:
        """top_logprobs = k in 0..20: also record the max(1, k) most likely tokens and their logprobs at every step
        (the generated tokens do not change).  temperature in (0, 2]: draw every token from the top_p (default 1)
        nucleus of softmax(logits / temperature) with `seed` (taken modulo 2^64; a random one when None), see
        rr_engine_submit; None or 0 is greedy.  frequency_penalty / presence_penalty in [-2, 2] and logit_bias
        {token id: bias in [-100, 100]} (at most 300 entries): applied to the logits before every token is picked, the
        penalties over the tokens generated so far; None, 0 or {} change nothing.
        n in 1..max_batch: n choices of the prompt, prefilled once; choice i is drawn with seed + i.  wait() returns
        them all; peek() is for n = 1 only.
        stop: a string or up to 4 strings (or bytes) of 1..64 bytes each: a choice ends where its reply text (the bytes of
        its tokens) would contain one, returns the tokens before the match and frees its decode row at once.  The
        tokens are a prefix of the same request's without `stop`.
        response_format {"type": "json_object"}: JSON mode: every token is picked from the logits masked to the JSON
        grammar, and a choice ends with finish reason "stop" on the token that closes its top-level object.  None and
        {"type": "text"} change nothing (check_response_format).
        prompt_logprobs = k in 0..20: also score the prompt (rr_engine_submit_scored); read the scores with
        prompt_logprobs() before wait()."""
        ids = _i32(prompt_ids)
        bias = logit_bias or {}
        stops = stop if isinstance(stop, (list, tuple)) and all(isinstance(b, bytes) for b in stop) else check_stop(stop)
        gen = gen_args(top_logprobs, temperature, top_p, seed, frequency_penalty, presence_penalty, list(bias.keys()),
                       list(bias.values()), stop=stops, json_object=check_response_format(response_format), n=n)
        t = C.c_uint64()
        if prompt_logprobs is None:
            _lib.check(_lib.lib.rr_engine_submit(self._h, _p(ids), len(ids), max_new_tokens, C.byref(gen.params),
                                                 C.byref(t)), "rr_engine_submit")
        else:
            _lib.check(_lib.lib.rr_engine_submit_scored(self._h, _p(ids), len(ids), max_new_tokens, C.byref(gen.params),
                                                        int(prompt_logprobs), C.byref(t)), "rr_engine_submit_scored")
            self._score[t.value] = (len(ids), max(1, int(prompt_logprobs)))
        if n > 1:
            self._n[t.value] = n
        if gen.width:
            self._lp_k[t.value] = gen.width
        return t.value

    def _lp_bufs(self, ticket: int, max_tokens: int, n: int = 1):
        k = self._lp_k.get(ticket)
        if k is None:
            return None, None, None, None
        lp, ids = np.zeros((n, max_tokens, k), dtype=np.float32), np.zeros((n, max_tokens, k), dtype=np.int32)
        return lp, ids, lp.ctypes.data_as(C.POINTER(C.c_float)), _p(ids)

    def prompt_logprobs(self, ticket: int, timeout: float = 0.0):
        """The scores of a request submitted with prompt_logprobs=k, once it is done (the ticket stays for wait()):
        (target [n_prompt - 1] float32, logprobs [n_prompt - 1][max(1, k)] float32, ids int32 alike); row t - 1 is prompt
        position t.  Raises RRError when the request did not end RR_OK."""
        n, k = self._score[ticket]
        tgt = np.zeros(max(0, n - 1), dtype=np.float32)
        lp, ids = np.zeros((max(0, n - 1), k), dtype=np.float32), np.zeros((max(0, n - 1), k), dtype=np.int32)
        f32 = C.POINTER(C.c_float)
        _lib.check(_lib.lib.rr_engine_prompt_logprobs(self._h, ticket, float(timeout), tgt.ctypes.data_as(f32),
                                                      lp.ctypes.data_as(f32), _p(ids)), "rr_engine_prompt_logprobs")
        return tgt, lp, ids

    def submit_embedding(self, prompt_ids: Sequence[int]) -> int:
        """An embedding request (rr_engine_submit_embed): the prompt is prefilled and its last position's final-norm row
        pooled and L2-normalised; no token is generated.  Read it with embedding(), then finish with wait()."""
        ids = _i32(prompt_ids)
        t = C.c_uint64()
        _lib.check(_lib.lib.rr_engine_submit_embed(self._h, _p(ids), len(ids), C.byref(t)), "rr_engine_submit_embed")
        return t.value

    def embedding(self, ticket: int, timeout: float = 0.0) -> np.ndarray:
        """The embedding of a request from submit_embedding(), once it is done (the ticket stays for wait()): float32
        [hidden].  Raises RRError when the request did not end RR_OK."""
        out = np.zeros(self.spec.hidden, dtype=np.float32)
        dim = C.c_int32()
        _lib.check(_lib.lib.rr_engine_embedding(self._h, ticket, float(timeout), out.ctypes.data_as(C.POINTER(C.c_float)),
                                                len(out), C.byref(dim)), "rr_engine_embedding")
        return out[: dim.value]

    def wait(self, ticket: int, timeout: float = 0.0, max_tokens: int = 4096) -> CompletionRecord:
        c = _lib.Completion()
        nc = self._n.get(ticket, 1)
        buf = np.zeros((nc, max_tokens), dtype=np.int32)
        lp, ids, lp_p, ids_p = self._lp_bufs(ticket, max_tokens, nc)
        n_tok, fin = (C.c_int32 * nc)(), (C.c_int32 * nc)()
        rc = _lib.lib.rr_engine_wait(self._h, ticket, float(timeout), C.byref(c), _p(buf), max_tokens, lp_p, ids_p, n_tok,
                                     fin)
        if rc != 6:
            self._lp_k.pop(ticket, None)
            self._n.pop(ticket, None)
            self._score.pop(ticket, None)
        if rc not in (0, 6, 7):
            _lib.check(rc, "rr_engine_wait")
        ns = [min(k, max_tokens) for k in n_tok]
        toks = [row[:k].tolist() for row, k in zip(buf, ns)]
        pairs = [logprob_pairs(a, b, 0, k) for a, b, k in zip(lp, ids, ns)] if lp is not None else None
        return CompletionRecord(ticket, rc, c.n_prompt, toks[0], c.t_submit_s, c.t_first_token_s, c.t_done_s,
                                pairs[0] if pairs else None, c.n_cached, toks, pairs, [FINISH_REASONS[f] for f in fin])

    def peek(self, ticket: int, have: int, timeout: float = 0.05, max_tokens: int = 4096):
        """Streaming: wait until more than `have` tokens exist (or done / timeout). -> (tokens so far, done, ttft_s), and
        for a request submitted with top_logprobs a fourth element: the per-token pairs so far (see CompletionRecord)."""
        buf = np.zeros(max_tokens, dtype=np.int32)
        n, done, ttft = C.c_int32(), C.c_int32(), C.c_double()
        lp, ids, lp_p, ids_p = self._lp_bufs(ticket, max_tokens)
        lp, ids = (None, None) if lp is None else (lp[0], ids[0])
        _lib.check(_lib.lib.rr_engine_peek(self._h, ticket, have, float(timeout), _p(buf), max_tokens, C.byref(n),
                                           C.byref(done), C.byref(ttft), lp_p, ids_p), "rr_engine_peek")
        if lp is None:
            return buf[: n.value].tolist(), bool(done.value), ttft.value
        m = min(n.value, max_tokens)
        return buf[: n.value].tolist(), bool(done.value), ttft.value, logprob_pairs(lp, ids, 0, m)

    def run_batch(self, prompt_ids: np.ndarray, prompt_start: np.ndarray, max_new_tokens: int):
        """Closed burst: submit every prompt, wait for all.  `prompt_ids` is a host buffer; the
        H2D copies happen inside the library.  -> (completions, tokens [n, max_new])."""
        ids, start = _i32(prompt_ids), _i32(prompt_start)
        n = len(start) - 1
        comps = (_lib.Completion * n)()
        toks = np.zeros((n, max_new_tokens), dtype=np.int32)
        rc = _lib.lib.rr_engine_run_batch(self._h, _p(ids), _p(start), n, max_new_tokens, comps, _p(toks))
        if rc not in (0, 7):
            _lib.check(rc, "rr_engine_run_batch")
        recs = [CompletionRecord(c.ticket, c.status, c.n_prompt, toks[i, :c.n_generated].tolist(),
                                 c.t_submit_s, c.t_first_token_s, c.t_done_s, n_cached=c.n_cached)
                for i, c in enumerate(comps)]
        return recs, toks

    def now(self) -> float:
        return _lib.lib.rr_engine_now(self._h)

    def kv_usage(self) -> Tuple[int, int]:
        """(pages_total, pages_free) of the KV page pool (64 tokens a page)."""
        tot, free = C.c_int32(), C.c_int32()
        _lib.check(_lib.lib.rr_engine_kv_usage(self._h, C.byref(tot), C.byref(free)), "rr_engine_kv_usage")
        return tot.value, free.value

    def stats(self) -> dict:
        s = _lib.EngineStats()
        _lib.check(_lib.lib.rr_engine_get_stats(self._h, C.byref(s)), "stats")
        return {k: getattr(s, k) for k, _ in s._fields_}

    def reset_stats(self):
        _lib.check(_lib.lib.rr_engine_reset_stats(self._h), "reset_stats")
