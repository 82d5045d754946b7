"""CPU restatement of latency-based-routing — TEST INFRASTRUCTURE, NOT THE PRODUCT.

Extends oracle/router.py (whose semantics, RNG and PARITY UNPINNED status apply unchanged) with the strategy
`routing_strategy: latency-based-routing`.  Only tests/ may import this module.

[UPSTREAM-RECALL router_strategy/lowest_latency.py; settings from router_settings.routing_strategy_args]

Settings:
  max_latency_list_size N (default 10, 1..32); lowest_latency_buffer resolved to millionths,
  ppm = round(v * 1e6), buffer = ppm / 1e6 (default 0); ttl in ms (default 3 600 000).

Sample sources (the event's 4th field, `chain_start`, which only ADMIT reads otherwise):
  DONE(deployment, completion tokens, latency L, now), L > 0: sample L / tokens (us per output
    token; one IEEE division), float(L) when tokens == 0.
  FAIL(deployment, timeout flag, now) with the flag == 1: sample 1e9 (litellm's 1000 s penalty).
  Any other FAIL, and a DONE with L <= 0, records nothing.  Every other strategy ignores the field.

Latency state:
  per deployment a list of samples.  Recording: if len(list) < N append, else
  list = list[:N-1] + [sample] (litellm's rule: the first N-1 samples are frozen, only the last slot
  is replaced).
  per model group a stamp = now_ms of its last write (-1 = never).  The group has expired when
  now_ms - stamp > ttl_ms; this is checked before every write and every pick in the group, and an
  expired group has every list in it cleared (the stamp stays until the next write, which sets
  stamp = now_ms).

pick(group), where the other strategies pick (inside the fallback walk), over the same eligible set
(cooldown, then the rpm / tpm pre-call checks when enabled):
  drop the group's samples if it has expired; mean = total / len per eligible deployment, total
  summed in list order from 0.0, an empty list gives 0.0 (unmeasured deployments are tried first);
  lowest = min(mean); threshold = lowest + (buffer * lowest) (two roundings);
  valid = [d for d in eligible if mean <= threshold], stably sorted by mean (ties keep config
  order); pick = random.choice(valid) (draws even when len(valid) == 1).  The debit is the common one.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

from .router import EV_DONE, EV_FAIL, Decision, Event, OracleRouter, Settings

STRATEGY_LATENCY_BASED = 5
LATENCY_TIMEOUT_PENALTY = 1e9


@dataclass
class LatencySettings(Settings):
    latency_list_size: int = 10          # max_latency_list_size
    latency_buffer_ppm: int = 0          # lowest_latency_buffer * 1e6, rounded
    latency_ttl_ms: int = 3_600_000      # ttl


class LatencyOracleRouter(OracleRouter):
    """OracleRouter plus latency-based-routing; with any other strategy it behaves exactly like OracleRouter."""

    def __init__(self, deployments, n_groups, fallbacks, settings: LatencySettings, seed: int = 0):
        super().__init__(deployments, n_groups, fallbacks, settings, seed)
        self.latencies: List[List[float]] = [[] for _ in self.deps]     # samples per deployment, oldest first
        self.lat_stamp = [-1] * n_groups

    @property
    def _latency(self) -> bool:
        return self.settings.strategy == STRATEGY_LATENCY_BASED

    def _lat_buffer(self) -> float:
        return self.settings.latency_buffer_ppm / 1e6

    def _lat_mean(self, i: int) -> float:
        total = 0.0
        for x in self.latencies[i]:
            total += x
        return total / len(self.latencies[i]) if self.latencies[i] else 0.0

    def _lat_expire(self, group: int, now_ms: int) -> None:
        if now_ms - self.lat_stamp[group] > self.settings.latency_ttl_ms:
            for i in self.by_group[group]:
                self.latencies[i] = []

    def _lat_record(self, dep: int, sample: float, now_ms: int) -> None:
        g = self.deps[dep].group
        self._lat_expire(g, now_ms)
        n = self.settings.latency_list_size
        if len(self.latencies[dep]) < n:
            self.latencies[dep].append(sample)
        else:
            self.latencies[dep] = self.latencies[dep][:n - 1] + [sample]
        self.lat_stamp[g] = now_ms

    def _eligible(self, group: int, n_tokens: int, now_ms: int) -> List[int]:
        """The eligible set of OracleRouter._pick: window roll, cooldown, then the rpm / tpm pre-call checks."""
        cands = self.by_group[group]
        for i in cands:
            self._roll(self.deps[i], now_ms)
        healthy = [i for i in cands if now_ms >= self.deps[i].cooldown_until_ms]
        if self.settings.enable_pre_call_checks:
            healthy = [i for i in healthy
                       if not (self.deps[i].rpm >= 0 and self.deps[i].req_count >= self.deps[i].rpm)
                       and not (self.deps[i].tpm >= 0 and self.deps[i].tok_count + n_tokens > self.deps[i].tpm)]
        return healthy

    def _pick(self, group: int, n_tokens: int, now_ms: int) -> Optional[int]:
        if not self._latency:
            return super()._pick(group, n_tokens, now_ms)
        healthy = self._eligible(group, n_tokens, now_ms)
        if not healthy:
            return None
        self._lat_expire(group, now_ms)
        means = {i: self._lat_mean(i) for i in healthy}
        lowest = min(means.values())
        threshold = lowest + (self._lat_buffer() * lowest)
        valid = sorted((i for i in healthy if means[i] <= threshold), key=lambda i: means[i])
        return self.rng.choice(valid)

    def process(self, events: Sequence[Event]) -> List[Decision]:
        out = []
        for e in events:
            out.extend(super().process([e]))
            if not self._latency or not 0 <= e.target < len(self.deps):
                continue
            if e.type == EV_DONE and e.chain_start > 0:
                self._lat_record(e.target, e.chain_start / e.tokens if e.tokens > 0 else float(e.chain_start), e.now_ms)
            elif e.type == EV_FAIL and e.chain_start == 1:
                self._lat_record(e.target, LATENCY_TIMEOUT_PENALTY, e.now_ms)
        return out

    def latency_snapshot(self):
        """[(mean us per output token, sample count)] per deployment, as stored (an expired group is cleared at its
        next write or pick): what rr_router_latency_snapshot returns."""
        return [(self._lat_mean(i), len(self.latencies[i])) for i in range(len(self.deps))]
