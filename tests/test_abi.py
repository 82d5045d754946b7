"""CPU checks of the C-ABI boundary: the library loads without a GPU, exports every function
declared in include/rr_b200.h, the ctypes table matches the header, and host-only entry points
(MT19937 seeding, tokenizer) give reference answers."""
import ctypes as C
import random
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def _declared():
    text = (ROOT / "include" / "rr_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(rr_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from rr_b200 import _lib
    names = _declared()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(_lib.lib, n)]
    assert not missing, missing
    assert not _lib.MISSING
    assert sorted(_lib.PROTOTYPES) == names


def test_struct_sizes_match_header():
    from rr_b200 import _lib
    assert C.sizeof(_lib.Event) == 24 and C.sizeof(_lib.Decision) == 16
    assert C.sizeof(_lib.DeploymentDesc) == 24 and C.sizeof(_lib.RouterSettings) == 32
    assert C.sizeof(_lib.DeploymentState) == 48
    assert C.sizeof(_lib.ModelDesc) == 36 and C.sizeof(_lib.Completion) == 48
    assert C.sizeof(_lib.StubDesc) == 16


def test_gen_params_layout_matches_header():
    """rr_gen_params is 80 bytes with these offsets on every LP64 platform; the library reads it by the header's layout."""
    from rr_b200 import _lib
    P = _lib.GenParams
    assert C.sizeof(P) == 80
    want = {"n_choices": 0, "top_logprobs": 4, "temperature": 8, "top_p": 12, "seed": 16, "frequency_penalty": 24,
            "presence_penalty": 28, "n_bias": 32, "n_stop": 36, "bias_ids": 40, "bias_vals": 48, "stop_bytes": 56,
            "stop_off": 64, "response_format": 72, "reserved": 76}
    assert {f: getattr(P, f).offset for f, _ in P._fields_} == want
    assert _lib.GatewayResult.finish.offset == 76 and C.sizeof(_lib.GatewayResult) == 80


def test_mt19937_seeding_matches_cpython():
    from rr_b200 import _lib
    for seed in [0, 1, 42, 1234, 2**31 - 1, 2**32 - 1, 2**32, 2**40 + 12345, 2**64 - 1]:
        buf = (C.c_uint32 * 625)()
        assert _lib.lib.rr_mt_seed_state(seed, buf) == 0
        want = random.Random(seed).getstate()[1]
        assert tuple(buf) == tuple(want), seed


def test_tokenizer_counts():
    from rr_b200 import _lib
    n = C.c_int32()
    s = "What is machine learning?".encode()
    assert _lib.lib.rr_count_tokens(s, len(s), C.byref(n)) == 0 and n.value == len(s) + 1
    ids = (C.c_int32 * 64)()
    assert _lib.lib.rr_tokenize(s, len(s), 128256, ids, 64, C.byref(n)) == 0
    assert n.value == len(s) + 1 and ids[0] == 1 and ids[1] == 3 + ord("W")
    assert _lib.lib.rr_tokenize(s, len(s), 128256, ids, 4, C.byref(n)) != 0   # buffer too small


def test_version_and_errors():
    from rr_b200 import _lib
    assert b"sm_90a" in _lib.lib.rr_version()
    assert b"429" in _lib.lib.rr_strerror(1)


def test_decode_mlp_entry_point_validates_before_touching_the_device():
    """rr_op_decode_mlp rejects null pointers with RR_INVALID_ARGUMENT before it touches the device (so this passes without
    one) and leaves its out values alone."""
    from rr_b200 import _lib
    ns, skb = C.c_int32(-1), C.c_int32(-1)
    rc = _lib.lib.rr_op_decode_mlp(None, None, None, 64, 4096, 14336, None, None, 64, C.byref(ns), C.byref(skb), None)
    assert rc == 4 and (ns.value, skb.value) == (-1, -1)


def test_decode_attn_entry_point_validates_before_touching_the_device():
    """rr_op_decode_attn_qkv rejects null pointers with RR_INVALID_ARGUMENT before it touches the device (so this passes
    without one) and leaves *kv_splits alone."""
    from rr_b200 import _lib
    ks = C.c_int32(-1)
    rc = _lib.lib.rr_op_decode_attn_qkv(None, 3, 64 * 6144, 6144, None, None, None, None, None, 64, 32, 8, 128, 4096, 64,
                                        5e5, C.byref(ks), None)
    assert rc == 4 and ks.value == -1


def test_prefill_norm_entry_point_validates_before_touching_the_device():
    """rr_op_add_rmsnorm_pf rejects null pointers with RR_INVALID_ARGUMENT before it touches the device."""
    from rr_b200 import _lib
    assert _lib.lib.rr_op_add_rmsnorm_pf(None, None, None, 64, 4096, 1e-5, None, 32, None) == 4


def test_prefill_qkv_entry_point_validates_before_touching_the_device():
    """rr_op_prefill_qkv rejects null pointers with RR_INVALID_ARGUMENT before it touches the device and leaves *fused
    alone."""
    from rr_b200 import _lib
    fused = C.c_int32(-1)
    rc = _lib.lib.rr_op_prefill_qkv(None, None, 128, 64, 4096, None, 32, 8, 128, 4096, 5e5, 1e-5, None, None, None, None,
                                    None, C.byref(fused), None)
    assert rc == 4 and fused.value == -1


def test_prefill_gemm_entry_point_validates_before_touching_the_device():
    """rr_op_prefill_gemm rejects null pointers with RR_INVALID_ARGUMENT before it touches the device, for the consumer
    (gate/up) and the producer (down) forms."""
    from rr_b200 import _lib
    rc = _lib.lib.rr_op_prefill_gemm(None, 128, 64, 4096, None, 28672, 4096, None, 14336, 3, None, 32, 4096, 1e-5, None,
                                     None, None, 0, None)
    assert rc == 4
    rc = _lib.lib.rr_op_prefill_gemm(None, 128, 64, 14336, None, 4096, 14336, None, 4096, 5, None, 0, 0, 0.0, None, None,
                                     None, 32, None)
    assert rc == 4


@pytest.mark.parametrize("grid,inter,hidden,slice_kb",[(148, 14336, 4096, 28), (148, 8192, 3072, 16), (132, 2816, 1024, 15),
                                                        (148, 1024, 512, 16), (7, 14336, 4096, 28)])
def test_fused_mlp_schedule_is_a_partition_and_deadlock_free(grid, inter, hidden, slice_kb):
    """Host logic of the fused decode MLP kernel (csrc/rr_gemm.cu, mlp_schedule): every gate/up tile and every
    (down tile, K-slice) appears exactly once; in every CTA's list all gate/up items precede all down items (a down
    item waits on gate/up tiles of OTHER CTAs, which therefore can never be queued behind a waiting item); slices
    cover the K range without gaps; the lists are balanced."""
    import ctypes as C
    import numpy as np
    from rr_b200 import _lib as lib
    mx = C.c_int32()
    cap = grid * 128
    buf = np.full((cap, 4), -7, dtype=np.int32)
    rc = lib.lib.rr_debug_mlp_schedule(grid, inter, hidden, slice_kb, buf.ctypes.data_as(C.POINTER(C.c_int32)), cap, C.byref(mx))
    assert rc == 0 and 1 <= mx.value <= 128
    items = buf[: grid * mx.value].reshape(grid, mx.value, 4)
    tiles0, kb0n = 2 * inter // 128, (hidden + 63) // 64
    tiles1, kb1n = (hidden + 127) // 128, inter // 64
    n_slices = (kb1n + slice_kb - 1) // slice_kb
    seen0, seen1, loads = set(), set(), []
    for c in range(grid):
        phase_seen, load, ended = 0, 0, False
        for tp, k0, k1, z in items[c]:
            if tp < 0:
                ended = True
                continue
            assert not ended                                   # no entry after the terminator
            ph, tile = tp >> 16, tp & 0xFFFF
            assert ph >= phase_seen                            # gate/up first, then down
            phase_seen = ph
            if ph == 0:
                assert (k0, k1) == (0, kb0n) and tile < tiles0 and tile not in seen0
                seen0.add(tile)
            else:
                assert tile < tiles1 and 0 <= z < n_slices and (tile, z) not in seen1
                assert k0 == z * slice_kb and k1 == min(kb1n, k0 + slice_kb)
                seen1.add((tile, z))
            load += k1 - k0
        loads.append(load)
    assert len(seen0) == tiles0 and len(seen1) == tiles1 * n_slices
    total = tiles0 * kb0n + tiles1 * kb1n
    assert sum(loads) == total
    if grid >= 64 and total // grid >= 100:                    # the production shapes: within 15 % of the mean
        assert max(loads) <= 1.15 * total / grid + slice_kb


def _prototype_arity():
    """{name: parameter count} of every function declared in include/rr_b200.h"""
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "rr_b200.h").read_text(), flags=re.S)
    out = {}
    for m in re.finditer(r"\b(rr_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text):
        params = m.group(2).strip()
        out[m.group(1)] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_ctypes_argument_counts_match_the_header():
    """Every _lib.py prototype takes as many arguments as the header declares (a missing or extra argument would shift
    every later one)."""
    from rr_b200 import _lib
    arity = _prototype_arity()
    assert sorted(arity) == sorted(_lib.PROTOTYPES)
    wrong = {n: (arity[n], len(a)) for n, (_, a) in _lib.PROTOTYPES.items() if arity[n] != len(a)}
    assert not wrong, wrong


def test_handoff_entry_points_validate_before_touching_the_device():
    """rr_op_gather_last, rr_op_activate_rows and rr_op_dequantize_fp8_jobs reject null pointers and bad shapes with
    RR_INVALID_ARGUMENT before they touch the device (so this passes without one).  The non-null addresses below are never
    dereferenced: every call is refused by its host-side checks."""
    from rr_b200 import _lib
    L = _lib.lib
    a = 1 << 20                                                          # a 16-byte aligned address, never read
    # gather_last(attn, x, last, n_rows, nq, hidden, attn_out, x_out, stream)
    assert L.rr_op_gather_last(None, a, a, 4, 4096, 4096, a, a, None) == 4
    assert L.rr_op_gather_last(a, None, a, 4, 4096, 4096, a, a, None) == 4
    assert L.rr_op_gather_last(a, a, None, 4, 4096, 4096, a, a, None) == 4
    assert L.rr_op_gather_last(a, a, a, 4, 4096, 4096, None, a, None) == 4
    assert L.rr_op_gather_last(a, a, a, 4, 4096, 4096, a, None, None) == 4
    assert L.rr_op_gather_last(a, a, a, 0, 4096, 4096, a, a, None) == 4          # n_rows < 1
    assert L.rr_op_gather_last(a, a, a, 4, 4092, 4096, a, a, None) == 4          # nq % 8
    assert L.rr_op_gather_last(a, a, a, 4, 4096, 4094, a, a, None) == 4          # hidden % 4
    assert L.rr_op_gather_last(a + 8, a, a, 4, 4096, 4096, a, a, None) == 4      # misaligned attn
    assert L.rr_op_gather_last(a, a, a, 4, 4096, 4096, a, a + 4, None) == 4      # misaligned x_out
    # activate_rows(seq_slot, first_tok, tok_pos, last, n, d_tok, d_pos, d_slot, stream)
    for k in range(7):
        args = [a] * 7
        args[k] = None
        assert L.rr_op_activate_rows(*args[:4], 8, *args[4:], None) == 4, k
    assert L.rr_op_activate_rows(a, a, a, a, 0, a, a, a, None) == 4              # n < 1
    # dequantize_fp8_jobs(q[], scale[], rows[], K[], out[], ld_out[], n_jobs, stream): four valid jobs of a Llama-3-8B
    # layer's shapes, the last one changed by `last`

    def jobs(n, **last):
        cols = {"q": [a] * n, "scale": [a] * n, "rows": [6144, 4096, 28672, 4096][:n], "K": [4096, 4096, 4096, 14336][:n],
                "out": [a] * n, "ld_out": [4096, 4096, 4096, 14336][:n]}
        for c, v in last.items():
            cols[c][-1] = v
        P = lambda v: (C.c_void_p * n)(*v)
        I = lambda v: (C.c_int32 * n)(*v)
        return [P(cols["q"]), P(cols["scale"]), I(cols["rows"]), I(cols["K"]), P(cols["out"]), I(cols["ld_out"])]

    for k in range(6):
        args = jobs(4)
        args[k] = None
        assert L.rr_op_dequantize_fp8_jobs(*args, 4, None) == 4, k
    assert L.rr_op_dequantize_fp8_jobs(*jobs(4), 0, None) == 4                    # job count outside 1..4
    assert L.rr_op_dequantize_fp8_jobs(*jobs(4), 5, None) == 4
    for bad in [{"q": None}, {"scale": None}, {"out": None}, {"q": a + 8}, {"out": a + 8}, {"rows": 0}, {"K": 14328},
                {"K": 0}, {"ld_out": 14320}, {"ld_out": 14340}]:
        assert L.rr_op_dequantize_fp8_jobs(*jobs(4, **bad), 4, None) == 4, bad
