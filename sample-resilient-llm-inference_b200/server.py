"""OpenAI-compatible HTTP front of the router (SURVEY.md §8f-1).

Restores the reference's real client boundary: the demos talk to `http://0.0.0.0:<litellm.port>` with the
OpenAI SDK and POST `<base_url>/chat/completions` (reference src/demo_load_balancing.py:24,106-110; the
gateway itself is `litellm --config ./config/config.yaml --port $PORT --num_workers 1`,
reference bin/start-gateway.sh:54).  Rate-limited requests answer HTTP 429 so the SDK raises
`openai.RateLimitError` (reference src/demo_quota_isolation.py:80).

    python -m rr_b200_server --config config/config.yaml            # real replicas (needs the GPUs named in the config)
    python -m rr_b200_server --config config/config.yaml --stub     # mock-completion backends (plumbing only)
"""
import argparse
import time
from typing import Dict, Optional

from .config import RouterConfig, load_config
from .models import resolve_spec
from .router import (APIError, APITimeoutError, BadRequestError, EngineBackend, RateLimitError, Router,
                     StubBackend, check_embedding, check_logprobs, check_n, check_penalties, check_response_format,
                     check_sampling, check_stop, check_text_completion)


def _error_body(e: APIError, typ: str) -> dict:
    return {"error": {"message": e.message, "type": typ, "param": None, "code": str(e.status_code)}}


def create_app(router: Router):
    from fastapi import FastAPI, Request
    from fastapi.responses import JSONResponse
    from starlette.concurrency import run_in_threadpool

    app = FastAPI(title="rr_b200 gateway")
    t_start = time.time()

    @app.on_event("startup")
    async def _raise_thread_limit():
        # every in-flight request parks one worker thread in rr_gateway_wait (GIL released); the default limit of 40 would
        # cap the concurrency below one replica's 64 decode rows
        import anyio.to_thread
        anyio.to_thread.current_default_thread_limiter().total_tokens = 2048

    async def stream_completion(model, messages, body, lp_kw, samp_kw):
        """Server-sent events in the OpenAI chunk format; the first chunk leaves when the first token exists (TTFT).
        With logprobs, every chunk carries `logprobs.content` for the tokens of its delta (the closing chunk null)."""
        import json as _json
        import uuid
        from fastapi.responses import StreamingResponse
        from .router import detokenize
        gen = router.completion_stream(model=model, messages=messages, timeout=body.get("timeout"),
                                       max_tokens=body.get("max_tokens"), **lp_kw, **samp_kw)
        try:
            first = await run_in_threadpool(next, gen)            # admission errors surface before the 200
        except RateLimitError as e:
            return JSONResponse(_error_body(e, "rate_limit_error"), 429, headers={"retry-after": "1"})
        except BadRequestError as e:
            return JSONResponse(_error_body(e, "invalid_request_error"), 400)
        except APIError as e:
            return JSONResponse(_error_body(e, "api_error"), e.status_code)
        cid = "chatcmpl-" + uuid.uuid4().hex[:24]

        def chunk(item):
            label, toks, done = item[:3]
            delta = {} if done else {"role": "assistant", "content": detokenize(toks)}
            choice = {"index": 0, "delta": delta,
                      "finish_reason": (getattr(item, "finish_reason", None) or "length") if done else None}
            if lp_kw:
                choice["logprobs"] = None if done else {"content": item[4], "refusal": None}
            return "data: " + _json.dumps({"id": cid, "object": "chat.completion.chunk", "created": int(time.time()),
                                           "model": label, "choices": [choice]}) + "\n\n"

        def events():
            try:
                yield chunk(first)
                if not first[2]:
                    for item in gen:
                        yield chunk(item)
                yield "data: [DONE]\n\n"
            finally:
                gen.close()        # client gone before the last chunk: the router cancels the request and frees its decode row

        return StreamingResponse(events(), media_type="text/event-stream")

    async def chat_completions(request: Request):
        try:
            body = await request.json()
        except Exception:
            return JSONResponse(_error_body(BadRequestError("invalid JSON body"), "invalid_request_error"), 400)
        model, messages = body.get("model"), body.get("messages")
        if not isinstance(model, str) or not isinstance(messages, list):
            return JSONResponse(_error_body(BadRequestError("`model` and `messages` are required"),
                                            "invalid_request_error"), 400)
        try:
            # passed on only when asked for: a request without them reaches the router exactly as before
            lp_kw = {}
            if check_logprobs(body.get("logprobs"), body.get("top_logprobs")) is not None:
                lp_kw = {"logprobs": True, "top_logprobs": body.get("top_logprobs")}
            samp_kw = {k: body[k] for k in ("temperature", "top_p", "seed") if body.get(k) is not None}
            check_sampling(**samp_kw)
            samp_kw.update({k: body[k] for k in ("frequency_penalty", "presence_penalty", "logit_bias")
                            if body.get(k) is not None})
            check_penalties(**{k: v for k, v in samp_kw.items() if k not in ("temperature", "top_p", "seed")})
            if body.get("stop") is not None:
                check_stop(body["stop"])
                samp_kw["stop"] = body["stop"]
            if body.get("response_format") is not None and check_response_format(body["response_format"]):
                samp_kw["response_format"] = body["response_format"]      # {"type": "text"} is the default: not passed
            if "n" in body:
                samp_kw["n"] = body["n"]
                if check_n(body["n"]) > 1 and body.get("stream"):
                    raise BadRequestError("streaming is not available with `n` > 1: send the request without `stream`")
        except BadRequestError as e:
            return JSONResponse(_error_body(e, "invalid_request_error"), 400)
        if body.get("stream"):
            return await stream_completion(model, messages, body, lp_kw, samp_kw)
        try:
            resp = await run_in_threadpool(router.completion, model=model, messages=messages,
                                           timeout=body.get("timeout"), max_tokens=body.get("max_tokens"), **lp_kw,
                                           **samp_kw)
            return JSONResponse(resp.model_dump())
        except RateLimitError as e:
            return JSONResponse(_error_body(e, "rate_limit_error"), 429, headers={"retry-after": "1"})
        except BadRequestError as e:
            return JSONResponse(_error_body(e, "invalid_request_error"), 400)
        except APITimeoutError as e:
            return JSONResponse(_error_body(e, "timeout"), 408)
        except APIError as e:
            return JSONResponse(_error_body(e, "api_error"), e.status_code)

    # the SDK appends /chat/completions to base_url; both spellings are served
    app.add_api_route("/chat/completions", chat_completions, methods=["POST"])
    app.add_api_route("/v1/chat/completions", chat_completions, methods=["POST"])

    def _error(e: APIError):
        if isinstance(e, RateLimitError):
            return JSONResponse(_error_body(e, "rate_limit_error"), 429, headers={"retry-after": "1"})
        if isinstance(e, BadRequestError):
            return JSONResponse(_error_body(e, "invalid_request_error"), 400)
        if isinstance(e, APITimeoutError):
            return JSONResponse(_error_body(e, "timeout"), 408)
        return JSONResponse(_error_body(e, "api_error"), e.status_code)

    async def stream_text_completion(kw):
        """Server-sent events in the OpenAI `text_completion` chunk format (no `echo`: check_text_completion)."""
        import json as _json
        import uuid
        from fastapi.responses import StreamingResponse
        from .router import detokenize, text_offsets
        gen = router.text_completion_stream(**kw)
        try:
            first = await run_in_threadpool(next, gen)            # admission errors surface before the 200
        except APIError as e:
            return _error(e)
        cid = "cmpl-" + uuid.uuid4().hex[:24]

        def chunk(item):
            label, toks, done = item[:3]
            lp = None
            if kw.get("logprobs") is not None and not done:
                # the chunk's tokens from completion_stream's entries; text_offset counts from the chunk's text
                ents, top = item[4], []
                for e in ents:
                    d = {}
                    for t in e["top_logprobs"] + [e]:
                        if t["token"] not in d or t["logprob"] > d[t["token"]]:
                            d[t["token"]] = t["logprob"]
                    top.append(d)
                lp = {"tokens": [e["token"] for e in ents], "token_logprobs": [e["logprob"] for e in ents],
                      "top_logprobs": top, "text_offset": text_offsets(toks)[1]}
            choice = {"index": 0, "text": "" if done else detokenize(toks), "logprobs": lp,
                      "finish_reason": (getattr(item, "finish_reason", None) or "length") if done else None}
            return "data: " + _json.dumps({"id": cid, "object": "text_completion", "created": int(time.time()),
                                           "model": label, "choices": [choice]}) + "\n\n"

        def events():
            try:
                yield chunk(first)
                if not first[2]:
                    for item in gen:
                        yield chunk(item)
                yield "data: [DONE]\n\n"
            finally:
                gen.close()

        return StreamingResponse(events(), media_type="text/event-stream")

    async def text_completions(request: Request):
        """OpenAI's /v1/completions (Router.text_completion): `prompt` in any of its four forms, `echo` and `logprobs`
        0..5 (with `echo`, the prompt's tokens scored on the GPU)."""
        try:
            body = await request.json()
        except Exception:
            return JSONResponse(_error_body(BadRequestError("invalid JSON body"), "invalid_request_error"), 400)
        model = body.get("model") if isinstance(body, dict) else None
        if not isinstance(model, str) or "prompt" not in body:
            return JSONResponse(_error_body(BadRequestError("`model` and `prompt` are required"),
                                            "invalid_request_error"), 400)
        try:
            check_text_completion(body["prompt"], body.get("max_tokens"), body.get("echo"), body.get("logprobs"),
                                  body.get("stream"), body.get("best_of"), body.get("suffix"))
            if body.get("stream") and check_n(body.get("n")) > 1:
                raise BadRequestError("streaming is not available with `n` > 1: send the request without `stream`")
        except BadRequestError as e:
            return _error(e)
        # passed on only when present: absent fields take the router's defaults
        kw = {k: body[k] for k in ("max_tokens", "logprobs", "temperature", "top_p", "seed", "n", "stop",
                                   "frequency_penalty", "presence_penalty", "logit_bias", "timeout")
              if body.get(k) is not None}
        if body.get("stream"):
            return await stream_text_completion(dict(kw, model=model, prompt=body["prompt"]))
        try:
            resp = await run_in_threadpool(router.text_completion, model=model, prompt=body["prompt"],
                                           echo=bool(body.get("echo")), **kw)
            return JSONResponse(resp.model_dump())
        except APIError as e:
            return _error(e)

    app.add_api_route("/completions", text_completions, methods=["POST"])
    app.add_api_route("/v1/completions", text_completions, methods=["POST"])

    async def embeddings(request: Request):
        """OpenAI's /v1/embeddings (Router.embedding): `input` in any of its four forms, `encoding_format` "float" or
        "base64" (the OpenAI SDK's default), `dimensions` absent or the hidden size."""
        try:
            body = await request.json()
        except Exception:
            return JSONResponse(_error_body(BadRequestError("invalid JSON body"), "invalid_request_error"), 400)
        model = body.get("model") if isinstance(body, dict) else None
        if not isinstance(model, str) or "input" not in body:
            return JSONResponse(_error_body(BadRequestError("`model` and `input` are required"),
                                            "invalid_request_error"), 400)
        try:
            check_embedding(body["input"], body.get("encoding_format"), body.get("dimensions"))
        except BadRequestError as e:
            return _error(e)
        kw = {k: body[k] for k in ("encoding_format", "dimensions", "timeout", "user") if body.get(k) is not None}
        try:
            resp = await run_in_threadpool(router.embedding, model=model, input=body["input"], **kw)
            return JSONResponse(resp.model_dump())
        except APIError as e:
            return _error(e)

    app.add_api_route("/embeddings", embeddings, methods=["POST"])
    app.add_api_route("/v1/embeddings", embeddings, methods=["POST"])

    @app.get("/health")
    async def health():
        return {"status": "ok", "uptime_s": time.time() - t_start}

    async def models():
        return {"object": "list", "data": [{"id": g, "object": "model", "owned_by": "rr_b200"}
                                           for g in router.cfg.groups]}

    app.add_api_route("/v1/models", models, methods=["GET"])
    app.add_api_route("/models", models, methods=["GET"])          # the SDK appends /models to a base_url without /v1

    @app.get("/router/state")
    async def state():
        snap = await run_in_threadpool(router.snapshot)
        if router.cfg.routing_strategy == "latency-based-routing":
            lat = await run_in_threadpool(router.latency_snapshot)
            for s, (mean, n) in zip(snap, lat):
                s.update(latency_us_per_token=mean, latency_samples=n)
        return {"deployments": [dict(model_name=d.model_name, model=d.response_model, gpu=d.gpu, rpm=d.rpm,
                                     tpm=d.tpm, **s) for d, s in zip(router.cfg.deployments, snap)]}

    return app


def build_backends(cfg: RouterConfig, stub: bool, spec_override: Optional[str] = None, max_batch: int = 64,
                   ctx_max: Optional[int] = None) -> Dict[int, object]:
    """One backend per replica (GPU) named in the config; deployments on the same GPU share it.  Each engine serves the
    deployment's litellm_params.context_window (ctx_max overrides it) with its kv_cache_tokens pool (None: the full
    max_batch x context window) and its quantization (fp8: e4m3 layer projections, Engine.synthetic).  A pool outside
    [context window, max_batch x context window] raises ValueError before any engine is created."""
    backends: Dict[int, object] = {}
    for d in cfg.deployments:
        ctx = ctx_max if ctx_max is not None else d.context_window
        kv = d.kv_cache_tokens
        if not stub and kv is not None and not ctx <= kv <= max_batch * ctx:
            raise ValueError(f"model_list[{d.index}].litellm_params.kv_cache_tokens = {kv} is outside "
                             f"[{ctx}, {max_batch * ctx}] (context window {ctx}, {max_batch} decode rows)")
    for d in cfg.deployments:
        if d.gpu in backends:
            continue
        if stub:
            backends[d.gpu] = StubBackend()
            continue
        from .engine import Engine
        spec = resolve_spec(spec_override or d.model)
        ctx = ctx_max if ctx_max is not None else d.context_window
        backends[d.gpu] = EngineBackend(Engine.synthetic(spec, seed=0, device=d.gpu, max_batch=max_batch,
                                                         ctx_max=ctx, prefix_cache=d.prefix_cache,
                                                         kv_cache_tokens=d.kv_cache_tokens,
                                                         quantization=d.quantization))
    return backends


def main(argv=None):
    ap = argparse.ArgumentParser(description="rr_b200 OpenAI-compatible gateway")
    ap.add_argument("--config", default="./config/config.yaml")
    ap.add_argument("--port", type=int, default=None)
    ap.add_argument("--host", default="0.0.0.0")
    ap.add_argument("--stub", action="store_true", help="mock-completion backends instead of model replicas")
    ap.add_argument("--spec", default=None, help="override the model spec of every deployment (e.g. tiny)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-tokens", type=int, default=64)
    a = ap.parse_args(argv)
    import uvicorn
    cfg = load_config(a.config)
    router = Router(config=cfg, backends=build_backends(cfg, a.stub, a.spec), seed=a.seed,
                    default_max_tokens=a.max_tokens)
    print(f"rr_b200 gateway: {len(cfg.deployments)} deployments in {len(cfg.groups)} model groups, "
          f"routing_strategy={cfg.routing_strategy}, port {a.port or cfg.port}")
    uvicorn.run(create_app(router), host=a.host, port=a.port or cfg.port, workers=1, log_level="warning")


if __name__ == "__main__":
    main()
