"""CPU checks of the hand-off between two decode steps: the refusals of rr_op_argmax (the greedy pick), rr_op_embed (the
next step's embedding gather) and rr_engine_create's vocabulary rule.  Every refusal is made before the entry point
touches the device, so they run without a GPU; the kernels themselves are checked in test_greedy_pick_gpu.py."""
import ctypes as C

import pytest

_P = C.c_void_p(16)              # a 16-byte aligned stand-in pointer: a refused call never dereferences it
_ODD = C.c_void_p(24)            # 8-byte but not 16-byte aligned
_F4 = C.c_void_p(20)             # 4-byte aligned, like a float row that starts one column late

# (logits, ld, rows, vocab, out_tok, out_val, row_active, pos_inc); the first entry is a call the checks accept
ARGMAX_GOOD = (_P, 128256, 64, 128256, _P, _P, _P, _P)
ARGMAX_ARGS = ("logits", "ld", "rows", "vocab", "out_tok", "out_val", "row_active", "pos_inc")
ARGMAX_BAD = {
    "null-logits": dict(logits=None),
    "null-out_tok": dict(out_tok=None),
    "rows-0": dict(rows=0),
    "rows-negative": dict(rows=-1),
    "vocab-0": dict(vocab=0),
    "vocab-negative": dict(vocab=-4),
    "vocab-above-ld": dict(vocab=128260),
    "vocab-one-above-ld": dict(ld=1024, vocab=1025),
    "ld-not-multiple-of-4": dict(ld=1003, vocab=1003),
    "ld-2-mod-4": dict(ld=32002, vocab=32001),
    "logits-8-byte-aligned": dict(logits=_ODD),
    "logits-4-byte-aligned": dict(logits=_F4),
}


@pytest.mark.parametrize("case", list(ARGMAX_BAD))
def test_argmax_refuses_before_touching_the_device(case):
    from rr_b200 import _lib
    a = dict(zip(ARGMAX_ARGS, ARGMAX_GOOD))
    a.update(ARGMAX_BAD[case])
    assert _lib.lib.rr_op_argmax(*(a[k] for k in ARGMAX_ARGS), None) == 4


# (ids, table, x, rows, hidden, row_active)
EMBED_GOOD = (_P, _P, _P, 256, 4096, _P)
EMBED_ARGS = ("ids", "table", "x", "rows", "hidden", "row_active")
EMBED_BAD = {
    "null-ids": dict(ids=None),
    "null-table": dict(table=None),
    "null-x": dict(x=None),
    "rows-0": dict(rows=0),
    "rows-negative": dict(rows=-3),
    "hidden-0": dict(hidden=0),
    "hidden-negative": dict(hidden=-8),
    "hidden-4": dict(hidden=4),
    "hidden-not-multiple-of-8": dict(hidden=4092),
    "table-8-byte-aligned": dict(table=_ODD),
    "x-8-byte-aligned": dict(x=_ODD),
    "x-4-byte-aligned": dict(x=_F4),
}


@pytest.mark.parametrize("case", list(EMBED_BAD))
def test_embed_refuses_before_touching_the_device(case):
    from rr_b200 import _lib
    a = dict(zip(EMBED_ARGS, EMBED_GOOD))
    a.update(EMBED_BAD[case])
    assert _lib.lib.rr_op_embed(*(a[k] for k in EMBED_ARGS), None) == 4


@pytest.mark.parametrize("vocab", [-4, 0, 1, 2, 3, 5, 1001, 1026, 1027, 32001, 128258])
def test_engine_create_refuses_a_vocabulary_the_logits_tail_cannot_read(vocab):
    """Each row of the [rows][vocab] fp32 logits is read with 16-byte loads, so vocab must be a multiple of 4 (and at least
    4).  The refusal comes before any CUDA call, with *out untouched; the model is otherwise one rr_engine_create
    accepts (test_paged_kv_cpu.py refuses only its pool)."""
    from rr_b200 import _lib
    desc = _lib.ModelDesc(vocab, 256, 512, 2, 4, 2, 64, 10000.0, 1e-5)
    w = _lib.ModelWeights()
    opts = _lib.EngineOpts(0, 4, 512, 256, 0, 0, 0.0, 0, (C.c_int32 * 3)(), 0)
    h = C.c_void_p()
    assert _lib.lib.rr_engine_create(C.byref(desc), C.byref(w), C.byref(opts), C.byref(h)) == 4
    assert h.value is None
