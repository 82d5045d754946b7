"""CPU checks of rr_op_decode_proj's refusals: every one below is made before the entry point touches the device (so they
run without a GPU) and leaves *n_splits alone.  The refusal that needs the SM count (a SiLU epilogue where the split rule
gives gate/up more than one plane) is checked on the GPU, in test_decode_proj_gpu.py."""
import ctypes as C

import pytest

F32, SILU = 1, 2
_P = C.c_void_p(16)              # a 16-byte aligned stand-in pointer: a refused call never dereferences it
_ODD = C.c_void_p(24)            # not 16-byte aligned


# (w, w_scale, rows_w, K, xn, rows, out, mode, lm_head); the first entry is a call the checks accept
GOOD = (_P, None, 6144, 4096, _P, 64, _P, F32, 0)
BAD = {
    "null-w": dict(w=None),
    "null-xn": dict(xn=None),
    "null-out": dict(out=None),
    "rows-0": dict(rows=0),
    "rows-negative": dict(rows=-1),
    "rows-257": dict(rows=257),
    "rows_w-0": dict(rows_w=0),
    "K-0": dict(K=0),
    "K-not-multiple-of-8": dict(K=4092),
    "mode-rowmajor-bf16": dict(mode=0),
    "mode-rowmajor-silu": dict(mode=3),
    "mode-rowmajor-f32": dict(mode=6),
    "mode-7": dict(mode=7),
    "lm_head-silu": dict(rows_w=28672, mode=SILU, lm_head=1),
    "lm_head-fp8": dict(w_scale=_P, lm_head=1),
    "silu-rows-16": dict(rows_w=28672, mode=SILU, rows=16),
    "silu-rows-1": dict(rows_w=28672, mode=SILU, rows=1),
    "silu-rows_w-not-whole-tiles": dict(rows_w=2 * 1000, mode=SILU),
    "fp8-K-not-multiple-of-16": dict(w_scale=_P, K=4088),
    "fp8-misaligned-weight": dict(w_scale=_P, w=_ODD),
}
ARGS = ("w", "w_scale", "rows_w", "K", "xn", "rows", "out", "mode", "lm_head")


@pytest.mark.parametrize("case", list(BAD))
def test_decode_proj_refuses_before_touching_the_device(case):
    from rr_b200 import _lib
    a = dict(zip(ARGS, GOOD))
    a.update(BAD[case])
    ns = C.c_int32(-7)
    rc = _lib.lib.rr_op_decode_proj(*(a[k] for k in ARGS), C.byref(ns), None)
    assert rc == 4 and ns.value == -7


def test_decode_proj_refuses_a_null_n_splits():
    from rr_b200 import _lib
    assert _lib.lib.rr_op_decode_proj(*GOOD, None, None) == 4


def test_engine_split_rule_mirror_at_132_sms():
    """engine.py's mirror of the split rule, at the SM count of an H100 SXM (132), by arithmetic: Llama-3-8B QKV 2, O 4,
    down 4, gate/up 1; Phi-3-mini O 5 and down 5 (ragged k-ranges); `small` down 5 over 44 k-blocks and gate/up 2."""
    from rr_b200.engine import pick_splits
    assert [pick_splits(n, k, 132) for n, k in [(6144, 4096), (4096, 4096), (4096, 14336), (28672, 4096)]] == [2, 4, 4, 1]
    assert [pick_splits(n, k, 132) for n, k in [(9216, 3072), (3072, 3072), (3072, 8192), (16384, 3072)]] == [1, 5, 5, 1]
    assert [pick_splits(n, k, 132) for n, k in [(1536, 1024), (1024, 1024), (1024, 2816), (5632, 1024)]] == [2, 2, 5, 2]
    assert pick_splits(128, 64, 132) == 1 and pick_splits(128, 64 * 64, 132) == 8      # one k-block; the 8-plane cap
