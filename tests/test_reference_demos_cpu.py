"""CPU: the request streams of the reference's three gateway demo scripts, replayed over HTTP with the OpenAI SDK against
this repo's gateway (sample-resilient-llm-inference_b200/server.py) loaded from config/config.yaml.

tests/golden/reference_demo_requests.json holds every distinct request the UNMODIFIED reference scripts
(src/demo_fallback.py, src/demo_load_balancing.py, src/demo_quota_isolation.py) sent when they were run against this
gateway.  The router kernel needs a GPU, so here a RECORDING DOUBLE sits behind server.py (first-fit over the config's
rpm limits -- a test double, not the product and not the oracle): what this proves is the wire contract -- the demos'
OpenAI-SDK calls (one shared client, or one client per request with the SDK's default retries of a 429) are served,
`.model` and HTTP 429 come back as the scripts expect, and the outcomes are the reference README's counts
(README.md:167-171, 206-213, 262-264).  tests/test_reference_demos_gpu.py replays the same requests against the real
K1-backed gateway."""
import json
import os
import socket
import threading
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "reference_demo_requests.json")


class RecordingDouble:
    """First-fit admission over the YAML's rpm limits + fallbacks; records every request."""

    def __init__(self, cfg):
        from rr_b200.router import Choice, Message, ModelResponse, RateLimitError, BadRequestError, Usage
        self.cfg, self.used, self.log, self.lock = cfg, [0] * len(cfg.deployments), [], threading.Lock()
        self._t = (Choice, Message, ModelResponse, RateLimitError, BadRequestError, Usage)

    def completion(self, model, messages, timeout=None, max_tokens=None):
        Choice, Message, ModelResponse, RateLimitError, BadRequestError, Usage = self._t
        with self.lock:
            self.log.append({"model": model, "messages": messages, "timeout": timeout})
            g = self.cfg.group_index(model)
            if g < 0:
                raise BadRequestError(f"Invalid model name passed in model={model}")
            for grp in [g] + self.cfg.fallbacks.get(g, []):
                for d in self.cfg.deployments:
                    if d.group == grp and (d.rpm < 0 or self.used[d.index] < d.rpm):
                        self.used[d.index] += 1
                        return ModelResponse("chatcmpl-double", d.response_model, [Choice(0, Message("assistant", "ok"))], Usage(8, 2, 10))
            raise RateLimitError(f"No deployments available for selected model, passed model={model}")

    def snapshot(self):
        return []


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _replay_demo(reqs, tmp_path, stagger, client_per_request):
    """Serve config/config.yaml through the double; send `reqs` one thread per request like the demos' dispatch loops
    (src/demo_fallback.py:212-220, demo_quota_isolation.py:135-139).  Returns (per-request outcome, the double's log)."""
    import openai
    import uvicorn
    from rr_b200.config import load_config
    from rr_b200.server import create_app
    port = _free_port()
    dbl = RecordingDouble(load_config(os.path.join(ROOT, "config", "config.yaml")))
    server = uvicorn.Server(uvicorn.Config(create_app(dbl), host="127.0.0.1", port=port, log_level="error"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    for _ in range(200):
        if server.started:
            break
        time.sleep(0.05)
    out = [None] * len(reqs)
    try:
        shared = openai.OpenAI(api_key="demo-key", base_url=f"http://127.0.0.1:{port}")

        def work(i, r):
            c = openai.OpenAI(api_key=f"key-{i}", base_url=f"http://127.0.0.1:{port}") if client_per_request else shared
            try:
                resp = c.chat.completions.create(model=r["model"], messages=[{"role": "user", "content": r["content"]}], timeout=30)
                out[i] = resp.model
            except openai.RateLimitError:
                out[i] = 429
            except Exception as e:                                      # noqa: BLE001
                out[i] = e
        ths = []
        for i, r in enumerate(reqs):
            t = threading.Thread(target=work, args=(i, r))
            t.start(); ths.append(t)
            if stagger:
                time.sleep(stagger)
        for t in ths:
            t.join()
    finally:
        server.should_exit = True
        th.join(10)
    return out, dbl.log


def test_unmodified_reference_demos_against_this_gateway(tmp_path):
    with open(GOLD) as f:
        gold = json.load(f)
    assert sorted(gold) == ["demo_fallback", "demo_load_balancing", "demo_quota_isolation"]
    # ---- fallback demo: 10 requests 50 ms apart, primary rpm 3 -> 3 primary + 7 fallback (README.md:167-171)
    got, log = _replay_demo(gold["demo_fallback"], tmp_path, 0.05, False)
    assert len(got) == 10 and not [g for g in got if isinstance(g, Exception) or g == 429], got
    assert sum("3-5-sonnet" in g for g in got) == 7
    # ---- load-balancing demo: 3 + 3 on the two primaries, 4 on the fallback (README.md:206-213)
    got, log = _replay_demo(gold["demo_load_balancing"], tmp_path, 0.1, False)
    assert len(log) == 10 and all(r["model"] == "claude-sonnet-loadbalance-demo" for r in log)
    dist = {}
    for g in got:
        dist[g] = dist.get(g, 0) + 1
    assert 429 not in dist and sorted(dist.values()) == [3, 3, 4], dist
    # ---- quota isolation: A 3/5 (2 rate limited), B 5/5, C 5/5 (README.md:262-264)
    got, log = _replay_demo(gold["demo_quota_isolation"], tmp_path, 0.0, True)
    by = {}
    for req, g in zip(gold["demo_quota_isolation"], got):
        ok, lim = by.get(req["model"], (0, 0))
        by[req["model"]] = (ok + (g != 429), lim + (g == 429))
    assert by == {"consumer-a-model": (3, 2), "consumer-b-model": (5, 0), "consumer-c-model": (5, 0)}
    attempts = {}
    for r in log:
        attempts[r["model"]] = attempts.get(r["model"], 0) + 1
    # the OpenAI SDK retries a 429 twice by default (one client per request, reference src/demo_quota_isolation.py:42):
    # team A's two rejected requests arrive three times each
    assert attempts == {"consumer-a-model": 9, "consumer-b-model": 5, "consumer-c-model": 5}
    # every call has the shape SURVEY.md 8b states: model (group name), one user message; and the gateway saw exactly the
    # recorded requests
    for name, reqs in gold.items():
        for r in reqs:
            assert isinstance(r["model"], str) and isinstance(r["content"], str)
    assert sorted({(r["model"], r["messages"][0]["content"]) for r in log}) == \
        sorted((r["model"], r["content"]) for r in gold["demo_quota_isolation"])
    assert all(len(r["messages"]) == 1 and r["messages"][0]["role"] == "user" for r in log)
