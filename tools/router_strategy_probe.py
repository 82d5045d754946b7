"""Admission kernel K1: µs per event for every routing strategy, with the router state staged in shared memory and with it
in HBM (RR_ROUTER_GLOBAL_STATE=1).  One mixed 2048-event trace (ADMIT / DONE with a latency / FAIL, some of them
timeouts / BURST) over 5 model groups (8, 8, 4, 2 and 32 deployments, fallback chains), timed with CUDA events around
back-to-back rr_router_process_device launches: kernel time only, no H2D / D2H copies."""
import ctypes as C
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rr_b200 import _lib

lib = _lib.lib
N_EVENTS, ITERS = 2048, 50
NAMES = ["simple-shuffle", "least-busy", "round-robin", "split", "random", "latency-based-routing"]
SIZES = [8, 8, 4, 2, 32]
FALLBACKS = {0: [1, 4], 1: [4], 2: [3], 3: [], 4: [0]}


def trace(rng):
    n_deps, now, ev = sum(SIZES), 0, (_lib.Event * N_EVENTS)()
    for i in range(N_EVENTS):
        now += rng.choice([0, 1, 2, 5, 20])
        t = rng.choices([0, 1, 2, 3], weights=[55, 35, 5, 5])[0]
        if t == 0:
            ev[i] = _lib.Event(0, rng.randrange(len(SIZES)), rng.randrange(1, 200), 0, now)
        elif t == 1:
            ev[i] = _lib.Event(1, rng.randrange(n_deps), rng.randrange(0, 64), rng.choice([800, 1500, 4000, 9000]), now)
        elif t == 2:
            ev[i] = _lib.Event(2, rng.randrange(n_deps), 0, rng.choice([0, 1]), now)
        else:
            ev[i] = _lib.Event(3, rng.randrange(len(SIZES)), rng.randrange(1, 64), 0, now)
    return ev


def probe(strategy, ev, global_state):
    if global_state:
        os.environ["RR_ROUTER_GLOBAL_STATE"] = "1"                # read by rr_router_create
    else:
        os.environ.pop("RR_ROUTER_GLOBAL_STATE", None)
    deps = (_lib.DeploymentDesc * sum(SIZES))()
    k = 0
    for g, n in enumerate(SIZES):
        for j in range(n):
            deps[k] = _lib.DeploymentDesc(g, -1, -1, 1 + j % 3, 0, 0)
            k += 1
    offs, flat = [0], []
    for g in range(len(SIZES)):
        flat += FALLBACKS[g]
        offs.append(len(flat))
    st = _lib.RouterSettings(strategy, 1, 1000, 5000, 0, 10, 100_000, 3_600_000)
    h = C.c_void_p()
    _lib.check(lib.rr_router_create(deps, len(deps), len(SIZES), (C.c_int32 * len(offs))(*offs),
                                    (C.c_int32 * len(flat))(*flat), C.byref(st), 0, 0, C.byref(h)), "create")
    d_ev = torch.frombuffer(bytearray(bytes(ev)), dtype=torch.int32).cuda()
    d_dec = torch.empty(N_EVENTS * 4, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream()
    launch = lambda: _lib.check(lib.rr_router_process_device(h, d_ev.data_ptr(), N_EVENTS, d_dec.data_ptr(),
                                                             s.cuda_stream), "process")
    for _ in range(5):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(ITERS):
        launch()
    e1.record(s)
    torch.cuda.synchronize()
    lib.rr_router_destroy(h)
    return e0.elapsed_time(e1) * 1e3 / (ITERS * N_EVENTS)


if __name__ == "__main__":
    ev = trace(random.Random(0))
    print(f"{torch.cuda.get_device_name()}: K1 µs per event, {N_EVENTS}-event mixed trace, {ITERS} launches")
    print(f"{'strategy':24s} {'shared memory':>14s} {'HBM':>8s}")
    for s, name in enumerate(NAMES):
        print(f"{name:24s} {probe(s, ev, False):14.3f} {probe(s, ev, True):8.3f}")
