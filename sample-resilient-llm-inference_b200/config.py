"""Loader for the reference's gateway configuration schema.

Keeps the keys the reference's config/config.yaml uses (reference config/config.yaml:31-33 `litellm.port`,
:35-94 `model_list[].{model_name, litellm_params.model, rpm, tpm}`, :100-108
`router_settings.{routing_strategy, enable_pre_call_checks, allowed_fails, cooldown_time, fallbacks}`);
YAML anchors / merge keys (`<<: *aws-defaults`, :40) are resolved by PyYAML.  AWS-only keys
(`aws_region_name`, `aws_profile_name`, the `aws:` / `cris:` sections) are accepted and ignored.
`router_settings.routing_strategy_args` takes litellm's latency-based-routing keys (`lowest_latency_buffer`,
`max_latency_list_size`, `ttl`).  Local extensions: `litellm_params.gpu: N` pins a deployment to a replica; `litellm_params.model:
b200/<spec>` names an on-box model (models.SPECS) instead of `bedrock/<id>`; `litellm_params.prefix_cache: true` turns on
prompt prefix caching in the replica; `litellm_params.context_window: N` is the longest request (prompt + max_tokens, in
tokens) the replica serves, a positive multiple of 64, default 1024; `litellm_params.kv_cache_tokens: N` sizes the replica's
KV cache, a pool of 64-token pages its decode rows share: a multiple of 64 in [context_window, max_batch x context_window],
default the full max_batch x context_window; `litellm_params.quantization: fp8` stores the replica's layer projections as
e4m3 weights with power-of-two row scales (absent or null: bf16).  Deployments on one GPU share its engine, so they must
agree on all four.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import yaml

STRATEGIES = {"simple-shuffle": 0, "least-busy": 1, "round-robin": 2, "split": 3, "random": 4,
              "latency-based-routing": 5}
_INT32_MAX = 2**31 - 1
_PROVIDER_PREFIXES = ("bedrock/", "b200/", "openai/", "azure/")


# litellm_params.quantization values: None = bf16 weights
QUANTIZATIONS = (None, "fp8")


def strip_provider(model: str) -> str:
    """`bedrock/us.anthropic...` -> `us.anthropic...` — what callers see in `response.model`
    (reference README.md:153-162; demos do the same for display, src/demo_load_balancing.py:59-60)."""
    for p in _PROVIDER_PREFIXES:
        if model.startswith(p):
            return model[len(p):]
    return model


@dataclass
class DeploymentCfg:
    index: int
    model_name: str            # model group
    model: str                 # litellm_params.model
    group: int
    rpm: int = -1
    tpm: int = -1
    weight: int = -1           # simple-shuffle weight (litellm_params.weight / rpm / tpm), -1 = unset
    gpu: int = 0
    prefix_cache: bool = False  # litellm_params.prefix_cache: the replica reuses cached prompt prefixes
    context_window: int = 1024  # litellm_params.context_window: prompt + max_tokens of one request, a multiple of 64
    kv_cache_tokens: Optional[int] = None   # litellm_params.kv_cache_tokens: the KV pool; None = max_batch x context_window
    quantization: Optional[str] = None      # litellm_params.quantization: None (bf16 weights) or "fp8" (e4m3 projections)
    params: Dict[str, Any] = field(default_factory=dict)

    @property
    def response_model(self) -> str:
        return strip_provider(self.model)


@dataclass
class RouterConfig:
    groups: List[str]
    deployments: List[DeploymentCfg]
    fallbacks: Dict[int, List[int]]
    routing_strategy: str = "simple-shuffle"
    enable_pre_call_checks: bool = False
    allowed_fails: int = 3
    cooldown_time: float = 5.0
    port: int = 4000
    # latency-based-routing (router_settings.routing_strategy_args)
    latency_list_size: int = 10          # max_latency_list_size
    latency_buffer_ppm: int = 0          # lowest_latency_buffer in millionths
    latency_ttl_ms: int = 3_600_000      # ttl

    @property
    def strategy_id(self) -> int:
        return STRATEGIES[self.routing_strategy]

    def group_index(self, name: str) -> int:
        try:
            return self.groups.index(name)
        except ValueError:
            return -1


def _int_or(v, default=-1) -> int:
    if v is None:
        return default
    if isinstance(v, bool) or not isinstance(v, (int, float)) or int(v) != v:
        raise ValueError(f"rpm/tpm/weight must be integers, got {v!r}")
    return int(v)


def _number(key: str, v) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)) or v != v or v in (float("inf"), float("-inf")):
        raise ValueError(f"routing_strategy_args.{key} must be a finite number, got {v!r}")
    return v


def parse_strategy_args(args: Optional[dict]) -> Dict[str, int]:
    """router_settings.routing_strategy_args of latency-based-routing -> the integer settings the router kernel takes:
    latency_list_size (max_latency_list_size, 1..32, default 10), latency_buffer_ppm (lowest_latency_buffer >= 0 in
    millionths, round(v * 1e6), default 0), latency_ttl_ms (ttl seconds > 0, default 3600)."""
    args = dict(args or {})
    unknown = sorted(set(args) - {"lowest_latency_buffer", "max_latency_list_size", "ttl"})
    if unknown:
        raise ValueError(f"routing_strategy_args: unsupported keys {unknown}; supported: "
                         "lowest_latency_buffer, max_latency_list_size, ttl")
    n = args.get("max_latency_list_size", 10)
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= 32:
        raise ValueError(f"routing_strategy_args.max_latency_list_size must be an integer in 1..32, got {n!r}")
    buf = _number("lowest_latency_buffer", args.get("lowest_latency_buffer", 0))
    ppm = round(buf * 1e6)
    if buf < 0 or ppm > _INT32_MAX:
        raise ValueError(f"routing_strategy_args.lowest_latency_buffer must be in [0, {_INT32_MAX / 1e6:g}], got {buf!r}")
    ttl = _number("ttl", args.get("ttl", 3600))
    ttl_ms = round(ttl * 1000)
    if ttl_ms < 1 or ttl_ms > _INT32_MAX:
        raise ValueError(f"routing_strategy_args.ttl must be in (0, {_INT32_MAX // 1000}] seconds, got {ttl!r}")
    return {"latency_list_size": n, "latency_buffer_ppm": ppm, "latency_ttl_ms": ttl_ms}


def build_config(model_list: List[dict], router_settings: Optional[dict] = None, port: int = 4000) -> RouterConfig:
    rs = dict(router_settings or {})
    groups: List[str] = []
    deps: List[DeploymentCfg] = []
    for i, entry in enumerate(model_list or []):
        name = entry["model_name"]
        lp = dict(entry.get("litellm_params") or {})
        if "model" not in lp:
            raise ValueError(f"model_list[{i}] has no litellm_params.model")
        if name not in groups:
            groups.append(name)
        # limits: top level of the entry (reference config.yaml:41-42) or inside litellm_params
        rpm = _int_or(entry.get("rpm", lp.get("rpm")))
        tpm = _int_or(entry.get("tpm", lp.get("tpm")))
        pc = lp.get("prefix_cache", False)
        if not isinstance(pc, bool):
            raise ValueError(f"model_list[{i}].litellm_params.prefix_cache must be true or false, got {pc!r}")
        cw = lp.get("context_window", 1024)
        if isinstance(cw, bool) or not isinstance(cw, int) or cw < 64 or cw % 64:
            raise ValueError(f"model_list[{i}].litellm_params.context_window must be a positive multiple of 64, got {cw!r}")
        kv = lp.get("kv_cache_tokens")
        if kv is not None and (isinstance(kv, bool) or not isinstance(kv, int) or kv < cw or kv % 64):
            raise ValueError(f"model_list[{i}].litellm_params.kv_cache_tokens must be a multiple of 64 of at least "
                             f"context_window ({cw}), got {kv!r}")
        qz = lp.get("quantization")
        if qz not in QUANTIZATIONS:
            raise ValueError(f"model_list[{i}].litellm_params.quantization must be null or one of "
                             f"{sorted(q for q in QUANTIZATIONS if q)}, got {qz!r}")
        deps.append(DeploymentCfg(index=i, model_name=name, model=lp["model"], group=groups.index(name),
                                  rpm=rpm, tpm=tpm, gpu=int(lp.get("gpu", 0)), prefix_cache=pc, context_window=cw,
                                  kv_cache_tokens=kv, quantization=qz, params=lp))
    for d in deps:                       # one engine per GPU: its deployments share the settings
        first = next(x for x in deps if x.gpu == d.gpu)
        for key in ("prefix_cache", "context_window", "kv_cache_tokens", "quantization"):
            if getattr(d, key) != getattr(first, key):
                raise ValueError(f"model_list[{first.index}] and model_list[{d.index}] share gpu {d.gpu} but disagree on "
                                 f"litellm_params.{key}")
    # simple-shuffle weights: the first of weight / rpm / tpm present in the litellm_params of the
    # group's first deployment decides the key for the whole group (oracle/router.py header).
    for g in range(len(groups)):
        members = [d for d in deps if d.group == g]
        key = next((k for k in ("weight", "rpm", "tpm") if members[0].params.get(k) is not None), None)
        for d in members:
            d.weight = _int_or(d.params.get(key), 0) if key else -1
    strategy = rs.get("routing_strategy", "simple-shuffle")
    if strategy not in STRATEGIES:
        raise ValueError(f"unsupported routing_strategy {strategy!r}; supported: {sorted(STRATEGIES)}")
    sargs = rs.get("routing_strategy_args")
    if sargs is not None and not isinstance(sargs, dict):
        raise ValueError(f"routing_strategy_args must be a mapping, got {sargs!r}")
    lat = parse_strategy_args(sargs)
    fbs: Dict[int, List[int]] = {}
    for item in rs.get("fallbacks") or []:
        for src, dst in item.items():
            if src not in groups:
                raise ValueError(f"fallbacks: unknown model group {src!r}")
            lst = []
            for d in dst:
                if d not in groups:
                    raise ValueError(f"fallbacks: unknown model group {d!r}")
                lst.append(groups.index(d))
            fbs[groups.index(src)] = lst
    return RouterConfig(groups=groups, deployments=deps, fallbacks=fbs, routing_strategy=strategy,
                        enable_pre_call_checks=bool(rs.get("enable_pre_call_checks", False)),
                        allowed_fails=int(rs.get("allowed_fails", 3)),
                        cooldown_time=float(rs.get("cooldown_time", 5.0)), port=port, **lat)


def load_config(path: str) -> RouterConfig:
    with open(path, "r") as f:
        raw = yaml.safe_load(f) or {}
    port = (raw.get("litellm") or {}).get("port", 4000)
    if not isinstance(port, int) or port < 1024 or port > 65535:   # reference bin/start-gateway.sh:18
        port = 4000
    return build_config(raw.get("model_list") or [], raw.get("router_settings") or {}, port)
