"""CPU: admission traces recorded at full size by `bench.py --config quota|fallback|fleet --trace-out ...` (the events the
native gateway fed to the K1 router kernel at BASELINE.json's full sizes, with the decisions the kernel returned) replayed
through the CPU oracle (oracle/router.py): every decision must be bit-exact.  This is the full-size half of the router
parity statement; the seeded random-trace matrix is tests/test_router_gpu.py.  Fixtures: tests/golden/trace_*.json
(written by bench.py's run_fleet; the generating command is in each file's `command` field / profiles/README.md)."""
import glob
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "trace_*.json")))


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(p) for p in FILES])
def test_recorded_hardware_trace_replays_bit_exact_through_the_oracle(path):
    from oracle import router as O
    from rr_b200.config import build_config
    with open(path) as f:
        rec = json.load(f)
    cfg = build_config(rec["model_list"], rec["router_settings"])
    deps = [O.Deployment(d.group, rpm=d.rpm, tpm=d.tpm, weight=d.weight) for d in cfg.deployments]
    orc = O.OracleRouter(deps, len(cfg.groups), dict(cfg.fallbacks),
                         O.Settings(strategy=cfg.strategy_id, enable_pre_call_checks=cfg.enable_pre_call_checks,
                                    allowed_fails=cfg.allowed_fails, cooldown_ms=int(round(cfg.cooldown_time * 1000))),
                         seed=rec.get("seed", 0))
    n_admit = n_rejected = 0
    for i, (ev, dec) in enumerate(rec["trace"]):
        want = orc.process([O.Event(*ev)])[0].as_tuple()
        if ev[0] == O.EV_ADMIT:
            assert tuple(dec) == want, (os.path.basename(path), i, ev, dec, want)
            n_admit += 1
            n_rejected += dec[0] != 0
    assert n_admit > 0
    inflight = sum(d.inflight for d in orc.deps)
    assert inflight == 0, "the recorded trace ends with every admitted request reported DONE or FAIL"
    print(f"\n{os.path.basename(path)}: {len(rec['trace'])} events, {n_admit} admissions ({n_rejected} rejected) bit-exact")


def test_fixtures_present():
    assert FILES, "no recorded traces under tests/golden/"
