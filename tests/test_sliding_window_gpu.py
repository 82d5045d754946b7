"""Sliding-window attention on the GPU: the two window entry points against fp64 windowed references, the KV ring of a
windowed engine, and a windowed deployment through the gateway.

Kernel operands are N(0, 1) except for "boundary" V rows of +-500: the keys just below and at a decode row's window
start, the rest of that start's key tile below it, and a random tenth of the prefill keys.  A correct output stays
within 1e-2 of the fp64 |weights| @ |V| (plus 2e-3) of the reference over the row's window; a kernel off by one key at
either end of the window, or one that leaves the first tile below the window unmasked, moves some output by about
500 x that key's weight, and each such wrong neighbour is shown to fail the same check."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_decode_attn_gpu import KV_SPLITS, SHAPES, default_path, plane_sums, rope_table, rotate  # noqa: F401
from test_long_context_attn_gpu import PAGE, _bits, decode_case, make_pool, put_rows, slot_rows

pytestmark = pytest.mark.gpu
DEV = "cuda"
BIG = 500.0
WINDOWS = (1, 64, 100, 4096)


def P(t):
    return C.c_void_p(t.data_ptr())


def set_rows(pool_t, table, s, positions, value, hd):
    for p in positions:
        pool_t[0, int(table[s, p // PAGE]), :, p % PAGE, :hd] = value


def ring_table(table, R, pps):
    """[n_slots, pps] table mapping logical page p of slot s to table[s, p % R]."""
    return table[:, torch.arange(pps) % R].contiguous()


def copy_to_ring(pool_t, table, ring, s, first_page, last_page):
    """The data of logical pages first..last of slot s, from the linear layout to where the ring table puts them (read
    all first: a ring page may be a later logical page's linear one)."""
    pages = range(first_page, last_page + 1)
    data = [pool_t[0, int(table[s, p])].clone() for p in pages]
    for p, d in zip(pages, data):
        pool_t[0, int(ring[s, p])] = d


def window_ref(q, k, v, scale):
    """fp64 attention of q [nkv, G, hd] over k, v [nkv, n, hd] -> (O, tolerance)."""
    s = scale * (q @ k.transpose(1, 2))
    w = torch.softmax(s, -1)
    return w @ v, 1e-2 * (w @ v.abs()) + 2e-3


def fails(got, ref_tol):
    o, tol = ref_tol
    return bool(((got - o).abs() > tol).any())


# ------------------------------------------------------------------------------------------------ decode
def run_decode_window(cs, k, v, window, table=None):
    from rr_b200 import _lib
    nh, nkv, hd, theta, ctx = cs["shape"]
    pool = cs["pool"]
    out = torch.full((cs["out_len"] + cs["slack"],), float("nan"), device=DEV, dtype=torch.bfloat16)
    ks = C.c_int32(-1)
    p = cs["planes"]
    dt = pool.dtable if table is None else table
    if window is None:
        fn, extra = _lib.lib.rr_op_decode_attn_qkv_paged, ()
    else:
        fn, extra = _lib.lib.rr_op_decode_attn_qkv_window, (window,)
    _lib.check(fn(P(p), cs["n_splits"], p.stride(0), cs["ld"], P(k), P(v), P(out), P(cs["slot"]), P(cs["pos"]), cs["rows"],
                  nh, nkv, hd, ctx, cs["n_slots"], theta, C.byref(ks), P(dt), pool.pps, pool.n_pages, *extra, None),
               "decode_attn_qkv_window")
    torch.cuda.synchronize()
    return out, ks.value


DEC_CASES = [pytest.param(n, ks, id=f"{n}-ks{ks}") for n in ("llama3-8b", "phi3-mini", "g8") for ks in KV_SPLITS]


@pytest.mark.parametrize("name,ks", DEC_CASES)
def test_decode_window_against_fp64(name, ks, default_path):
    """Positions 8191 .. 65535 of a 65536-token context over scattered pages, inactive rows, kv_splits 1 to 8: every
    window W in WINDOWS against its fp64 reference, the wrong neighbours refused; W = 1 gives bf16(v) of the row's own
    position exactly; W = 65536 (> every position) gives rr_op_decode_attn_qkv_paged's bits; a ring-mapped table the
    linear table's bits."""
    cs = decode_case(name, 65536, ks, "normal", seed=5 * ks + len(name))
    nh, nkv, hd, theta, ctx = cs["shape"]
    G = nh // nkv
    pool = cs["pool"]
    act = cs["active"]
    scale = 1.0 / math.sqrt(hd)
    acc = plane_sums(cs)[torch.tensor(act, device=DEV)]
    c, sn = rope_table(cs["pos"][act].long(), theta, hd)
    q_all = rotate(acc[:, : nh * hd].view(-1, nh, hd), c[:, None, :], sn[:, None, :])[0].bfloat16()
    k_lin, v_lin = pool.k.clone(), pool.v.clone()
    # W > every position: the paged call's bits
    out0, _ = run_decode_window(cs, pool.k.clone(), pool.v.clone(), None)
    out1, ks_got = run_decode_window(cs, pool.k.clone(), pool.v.clone(), 65536)
    assert ks_got == ks
    assert torch.equal(_bits(out0), _bits(out1)), "W > pos differs from the paged call"
    for W in WINDOWS:
        k, v = k_lin.clone(), v_lin.clone()
        for r in act:
            s, p = int(cs["slot"][r]), int(cs["pos"][r])
            lo = max(0, p - W + 1)
            set_rows(v, pool.table, s, range(lo // PAGE * PAGE, lo), BIG, hd)        # the first tile below the window
            set_rows(v, pool.table, s, [x for x in (lo - 1,) if x >= 0], BIG, hd)
            set_rows(v, pool.table, s, [x for x in (lo,) if x < p], -BIG, hd)
        k0, v0 = k.clone(), v.clone()
        out, _ = run_decode_window(cs, k, v, W)
        o = out[:cs["out_len"]].view(cs["rows"], nh, hd)
        inactive = [r for r in range(cs["rows"]) if r not in set(act)]
        assert torch.isnan(o[inactive]).all() and torch.isnan(out[cs["out_len"]:]).all()
        neigh = {}                                    # wrong neighbour -> refused by some row where it differs
        for j, r in enumerate(act):
            s, p = int(cs["slot"][r]), int(cs["pos"][r])
            lo = max(0, p - W + 1)
            K = slot_rows(k, pool.table, s, p + 1)[..., :hd].double()
            V = slot_rows(v, pool.table, s, p + 1)[..., :hd].double()
            qj = q_all[j].double().view(nkv, G, hd)
            got = o[r].double().view(nkv, G, hd)
            if W == 1:
                want = V[:, p:p + 1].expand(nkv, G, hd)
                assert torch.equal(got, want), f"W = 1, row {r} (pos {p}): not bf16(v) of its own position"
            ref = window_ref(qj, K[:, lo:], V[:, lo:], scale)
            assert not fails(got, ref), f"W = {W}, row {r} (pos {p}): {((got - ref[0]).abs() / ref[1]).max():.3g} x tol"
            if lo > 0:
                neigh["window W + 1"] = neigh.get("window W + 1", False) | fails(got, window_ref(qj, K[:, lo - 1:],
                                                                                                 V[:, lo - 1:], scale))
            if lo < p:
                neigh["window W - 1"] = neigh.get("window W - 1", False) | fails(got, window_ref(qj, K[:, lo + 1:],
                                                                                                 V[:, lo + 1:], scale))
            if lo % PAGE:
                t0 = lo // PAGE * PAGE
                neigh["first tile unmasked"] = neigh.get("first tile unmasked", False) | fails(
                    got, window_ref(qj, K[:, t0:], V[:, t0:], scale))
        assert all(neigh.values()) and (W == 1 or {"window W + 1", "window W - 1"} <= set(neigh)), (W, neigh)
        # the same call through a ring of R pages: the same bits
        R = -(-(W - 1) // PAGE) + 1
        ring = ring_table(pool.table, R, pool.pps)
        for r in act:
            s, p = int(cs["slot"][r]), int(cs["pos"][r])
            copy_to_ring(k0, pool.table, ring, s, max(0, p - W + 1) // PAGE, p // PAGE)
            copy_to_ring(v0, pool.table, ring, s, max(0, p - W + 1) // PAGE, p // PAGE)
        out_r, _ = run_decode_window(cs, k0, v0, W, ring.to(DEV))
        assert torch.equal(_bits(out_r), _bits(out)), f"W = {W}: the ring table changes the output"


# ------------------------------------------------------------------------------------------------ prefill
PF_CTX = 16384
PF_SEQS = [(0, 700), (3000, 1000), (9037, 300), (16383, 1)]          # (pos0, len): pieces at pos0 > 0, a partial tile


def prefill_setup(H, KV, seed):
    g = torch.Generator().manual_seed(seed)
    gd = torch.Generator(device=DEV).manual_seed(seed)
    n = len(PF_SEQS)
    need = [-(-(p0 + ln) // PAGE) for p0, ln in PF_SEQS]
    slots = torch.randperm(n, generator=g).tolist()
    pool = make_pool(KV, PF_CTX, [need[slots.index(s)] for s in range(n)], 5, g)
    kv = []
    for i, (p0, ln) in enumerate(PF_SEQS):
        m = need[i] * PAGE
        K = torch.randn(KV, m, 128, device=DEV, generator=gd).bfloat16()
        V = torch.randn(KV, m, 128, device=DEV, generator=gd)
        big = torch.rand(KV, m, 1, device=DEV, generator=gd) < 0.1
        sign = torch.randint(0, 2, (KV, m, 1), device=DEV, generator=gd).float() * 2 - 1
        V = torch.where(big, sign * BIG, V).bfloat16()
        put_rows(pool.k, pool.table, slots[i], K)
        put_rows(pool.v, pool.table, slots[i], V)
        kv.append((K, V))
    lens = [ln for _, ln in PF_SEQS]
    q = torch.randn(sum(lens), H * 128, device=DEV, generator=gd).bfloat16()
    start = torch.tensor([0] + np.cumsum(lens).tolist(), device=DEV, dtype=torch.int32)
    return dict(pool=pool, kv=kv, q=q, start=start, slots=torch.tensor(slots, device=DEV, dtype=torch.int32),
                pos0=torch.tensor([p0 for p0, _ in PF_SEQS], device=DEV, dtype=torch.int32), H=H, KV=KV, lens=lens)


def run_prefill_window(cs, window, table=None):
    from rr_b200 import _lib
    pool = cs["pool"]
    out = torch.full_like(cs["q"], float("nan"))
    dt = pool.dtable if table is None else table
    args = (P(cs["q"]), P(pool.k), P(pool.v), P(out), P(cs["start"]), P(cs["slots"]), P(cs["pos0"]), len(PF_SEQS),
            max(cs["lens"]), cs["H"], cs["KV"], PF_CTX, 1 / math.sqrt(128), P(dt), pool.pps, pool.n_pages)
    if window is None:
        _lib.check(_lib.lib.rr_op_prefill_attn_cached_paged(*args, None), "prefill_attn_cached_paged")
    else:
        _lib.check(_lib.lib.rr_op_prefill_attn_window(*args, window, None), "prefill_attn_window")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("H,KV", [(32, 8), (8, 8)])
def test_prefill_window_against_fp64(H, KV):
    """Every row of pieces at pos0 0, 3000, 9037 and 16383 against its fp64 windowed reference for W in WINDOWS, the
    wrong neighbours refused; W = 1 (a late row meets key tiles wholly below its window) gives bf16(v) of the row's own
    position exactly; W = 16384 gives rr_op_prefill_attn_cached_paged's bits; a ring-mapped table the linear one's."""
    cs = prefill_setup(H, KV, 10 * H + KV)
    G = H // KV
    scale = 1 / math.sqrt(128)
    out0 = run_prefill_window(cs, None)
    assert torch.equal(_bits(out0), _bits(run_prefill_window(cs, PF_CTX))), "W > pos differs from the paged call"
    st = cs["start"].tolist()
    for W in WINDOWS:
        out = run_prefill_window(cs, W)
        assert not torch.isnan(out).any()
        neigh = {"window W + 1": False, "window W - 1": False, "first tile unmasked": False}
        for i, (p0, ln) in enumerate(PF_SEQS):
            K, V = (t[..., :128].double() for t in cs["kv"][i])
            got_all = out[st[i]:st[i + 1]].view(ln, KV, G, 128).double()
            q_all = cs["q"][st[i]:st[i + 1]].view(ln, KV, G, 128).double()
            for r0 in range(0, ln, 128):
                r1 = min(ln, r0 + 128)
                a, b = max(0, p0 + r0 - W), p0 + r1            # keys of the block, one below the window included
                kp = torch.arange(a, b, device=DEV)
                qp = torch.arange(p0 + r0, p0 + r1, device=DEV)
                s = scale * torch.einsum("rkgd,knd->rkgn", q_all[r0:r1], K[:, a:b])
                got = got_all[r0:r1]

                def ref(first):
                    vis = (kp[None, :] <= qp[:, None]) & (kp[None, :] >= first[:, None])
                    w = torch.softmax(s.masked_fill(~vis[:, None, None, :], -math.inf), -1)
                    return (torch.einsum("rkgn,knd->rkgd", w, V[:, a:b]),
                            1e-2 * torch.einsum("rkgn,knd->rkgd", w, V[:, a:b].abs()) + 2e-3)
                lo = (qp - W + 1).clamp(min=0)
                o, tol = ref(lo)
                bad = (got - o).abs() > tol
                assert not bad.any(), f"W = {W}, seq {i}: rows {(bad.flatten(1).any(1)).nonzero().flatten()[:8].tolist()} off"
                if W == 1:
                    own = V[:, p0 + r0:p0 + r1].permute(1, 0, 2)[:, :, None, :].expand_as(got)
                    assert torch.equal(got, own), f"W = 1, seq {i}: not bf16(v) of the own position"
                if W > 1:
                    neigh["window W + 1"] |= fails(got, ref((qp - W).clamp(min=0)))
                    neigh["window W - 1"] |= fails(got, ref(torch.minimum(qp - W + 2, qp).clamp(min=0)))
                    neigh["first tile unmasked"] |= fails(got, ref(lo // PAGE * PAGE))
        if W > 1:
            assert all(neigh.values()), (W, neigh)
        # through a ring of R pages per slot: the same bits
        R = -(-(W + max(cs["lens"]) - 2) // PAGE) + 1
        if R < cs["pool"].pps:
            pool = cs["pool"]
            k_lin, v_lin = pool.k.clone(), pool.v.clone()
            ring = ring_table(pool.table, R, pool.pps)
            for i, (p0, ln) in enumerate(PF_SEQS):
                s = int(cs["slots"][i])
                for t in (pool.k, pool.v):
                    copy_to_ring(t, pool.table, ring, s, max(0, p0 - W + 1) // PAGE, (p0 + ln - 1) // PAGE)
            out_r = run_prefill_window(cs, W, ring.to(DEV))
            pool.k.copy_(k_lin); pool.v.copy_(v_lin)
            assert torch.equal(_bits(out_r), _bits(out)), f"W = {W}: the ring table changes the output"


# ------------------------------------------------------------------------------------------------ engine
def _cmp(got, ref, what):
    from test_engine_gpu import _cmp as cmp
    cmp(got, ref, what)


def _engine(spec_name="tiny-sw", seed=11, wkw=(("sigma", 0.05), ("norm_jitter", 0.1)), **kw):
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    w = make_weights(SPECS[spec_name], seed=seed, device="cuda", **dict(wkw))
    return Engine(w, **kw), w


def _prompt(spec, n, seed):
    rs = np.random.RandomState(seed)
    return rs.randint(3, spec.vocab, size=n).tolist()


def test_tiny_sw_matches_the_hf_golden_and_the_oracle_past_the_window():
    """tiny-sw (W = 100) against HF MistralForCausalLM(sliding_window=100): prefill logits of prompts of 1 .. 700 tokens
    and a teacher-forced decode step; then 400 teacher-forced decode steps from position 150 against the windowed
    oracle."""
    from test_sliding_window_cpu import golden_case
    from window_oracle import forward_logits
    spec, w_cpu, g = golden_case()
    from rr_b200.engine import Engine
    w = w_cpu.to("cuda")
    eng = Engine(w, max_batch=8, ctx_max=1024, max_prefill_tokens=1024, use_cuda_graph=False)
    try:
        prompts = g["prompts"]
        for i, p in enumerate(prompts):
            _, lg = eng.prefill([p], [i], want_logits=True)
            _cmp(lg[0], g["logits"][i][0], f"prefill len={len(p)}")
        _, lg2 = eng.decode_step(list(range(len(prompts))), [t[0] for t in g["tokens"]], [len(p) for p in prompts],
                                 want_logits=True)
        for i, p in enumerate(prompts):
            _cmp(lg2[i], g["logits"][i][1], f"decode len={len(p)}")
        seq = _prompt(spec, 550, 3)
        ref = forward_logits(w, seq)
        _, lg = eng.prefill([seq[:150]], [7], want_logits=True)
        _cmp(lg[0], ref[149], "prefill 150")
        for p in range(150, 550):
            _, lg = eng.decode_step([7], [seq[p]], [p], want_logits=True)
            _cmp(lg[0], ref[p], f"decode at {p}")
    finally:
        eng.close()


def _run(eng, reqs):
    """Submit every (prompt, max_new, kw) together, wait for all -> records."""
    tickets = [eng.submit(p, m, **kw) for p, m, kw in reqs]
    return [eng.wait(t, timeout=120.0) for t in tickets]


def test_ring_pool_equals_ample_linear_pool_and_pieces_equal_one_chunk():
    """tiny-sw, max_prefill_tokens 256: R = ceil((100 + 254) / 64) + 1 = 7 pages.  Requests reaching up to 1500
    positions (24 pages linearly) on a 16-page pool (ring requests, 7 pages each) give the tokens and logprob bits of an
    ample linear pool; prompts in pieces of 256 give the bits of one 2048-token chunk."""
    from rr_b200 import SPECS
    from rr_b200.models import ring_pages
    spec = SPECS["tiny-sw"]
    assert ring_pages(100, 256) == 7
    reqs = [(_prompt(spec, n, 40 + n), m, dict(top_logprobs=2)) for n, m in ((1200, 300), (700, 200), (90, 40), (400, 30))]
    ring, _ = _engine(max_batch=4, ctx_max=2048, max_prefill_tokens=256, kv_cache_tokens=2048)
    lin, _ = _engine(max_batch=4, ctx_max=2048, max_prefill_tokens=2048)
    try:
        a, b = _run(ring, reqs), _run(lin, reqs)
        for x, y in zip(a, b):
            assert x.status == 0 and y.status == 0
            assert x.tokens == y.tokens and len(x.tokens) > 0
            assert x.logprobs == y.logprobs
        # kv_usage: while a ring request runs alone it holds R pages
        t = ring.submit(reqs[0][0], 840)
        for _ in range(2000):
            got, done, _ = ring.peek(t, 5, timeout=0.5)
            if len(got) > 5 or done:
                break
        usage = ring.kv_usage()
        assert not done and usage == (32, 32 - 7), usage
        assert ring.wait(t, timeout=60.0).status == 0
        assert ring.kv_usage() == (32, 32)
    finally:
        ring.close(); lin.close()


def test_ring_request_choices_stop_json_and_prefix_cache():
    """n > 1, stop and JSON mode on ring requests give what an ample linear pool gives; a ring request is a prefix-cache
    miss and retains nothing, while a short windowed request still hits."""
    from rr_b200 import SPECS
    spec = SPECS["tiny-sw"]
    eng, _ = _engine(max_batch=6, ctx_max=1536, max_prefill_tokens=256, kv_cache_tokens=1536, prefix_cache=True)
    lin, _ = _engine(max_batch=6, ctx_max=1536, max_prefill_tokens=2048, prefix_cache=True)
    try:
        p = _prompt(spec, 1000, 9)
        kw = dict(temperature=0.8, seed=5, n=3)
        a, b = _run(eng, [(p, 100, kw)])[0], _run(lin, [(p, 100, kw)])[0]
        assert a.status == 0 and a.choices == b.choices and len(set(map(tuple, a.choices))) > 1
        base = _run(lin, [(p, 60, {})])[0].tokens
        stop = [bytes((t - 3) % 256 for t in base[30:32] if t >= 3)]     # the byte-level text of two reply tokens
        s1, s2 = _run(eng, [(p, 60, dict(stop=stop))])[0], _run(lin, [(p, 60, dict(stop=stop))])[0]
        assert s1.tokens == s2.tokens and s1.finish_reasons == s2.finish_reasons
        j1 = _run(eng, [(p, 80, dict(response_format={"type": "json_object"}))])[0]
        j2 = _run(lin, [(p, 80, dict(response_format={"type": "json_object"}))])[0]
        assert j1.tokens == j2.tokens and j1.finish_reasons == j2.finish_reasons
        # prefix cache: the same long prompt twice misses twice; a short prompt twice hits the second time
        eng.reset_stats()
        r1, r2 = _run(eng, [(p, 5, {})])[0], _run(eng, [(p, 5, {})])[0]
        assert r1.n_cached == 0 and r2.n_cached == 0 and eng.stats()["prefix_hits"] == 0
        assert r1.tokens == r2.tokens == base[:5]
        q = _prompt(spec, 300, 10)
        s1, s2 = _run(eng, [(q, 5, {})])[0], _run(eng, [(q, 5, {})])[0]
        assert s1.n_cached == 0 and s2.n_cached == 299 and s1.tokens == s2.tokens
        assert eng.stats()["prefix_hits"] == 1
    finally:
        eng.close(); lin.close()


def test_mistral_2l_long_prompt_matches_the_oracle():
    """mistral-7b-2l (W = 4096, a ring of 193 pages at 8192-token chunks): a 12400-token prompt, a ring request
    prefilled in two pieces, picks the oracle's first token; and teacher-forced decode logits from position 8192 to 12431
    (linear pages, low-level calls) against the windowed oracle."""
    from window_oracle import forward_logits
    from rr_b200 import SPECS
    spec = SPECS["mistral-7b-2l"]
    eng, w = _engine("mistral-7b-2l", seed=0, wkw=(), max_batch=4, ctx_max=16384, kv_cache_tokens=16384)
    try:
        seq = _prompt(spec, 12432, 77)
        ref = forward_logits(w, seq)
        rec = eng.wait(eng.submit(seq[:12400], 1), timeout=300.0)
        assert rec.status == 0 and eng.kv_usage() == (256, 256)
        top2 = ref[12399].topk(2).values
        assert rec.tokens[0] == int(ref[12399].argmax()) or (top2[0] - top2[1]).item() < 0.05 * ref[12399].std().item()
        _, lg = eng.prefill([seq[:8192]], [1], want_logits=True)
        _cmp(lg[0], ref[8191], "prefill 8192")
        for p in range(8192, 12432):
            _, lg = eng.decode_step([1], [seq[p]], [p], want_logits=p % 16 == 0 or p == 12431)
            if lg is not None:
                _cmp(lg[0], ref[p], f"decode at {p}")
    finally:
        eng.close()


def test_mistral_window_changes_nothing_below_4096_tokens():
    """A W = 4096 engine and a W = 0 engine on the same weights: the same tokens and logprob bits below 4096 tokens."""
    import dataclasses
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    spec = SPECS["mistral-7b-2l"]
    w = make_weights(spec, seed=0, device="cuda")
    w0 = dataclasses.replace(w, spec=dataclasses.replace(spec, sliding_window=0))
    reqs = [(_prompt(spec, n, n), m, dict(top_logprobs=3)) for n, m in ((4000, 95), (512, 128), (3000, 64), (17, 40))]
    a_eng, b_eng = Engine(w, max_batch=8, ctx_max=4096), Engine(w0, max_batch=8, ctx_max=4096)
    try:
        a, b = _run(a_eng, reqs), _run(b_eng, reqs)
        for x, y in zip(a, b):
            assert x.tokens == y.tokens and x.logprobs == y.logprobs
    finally:
        a_eng.close(); b_eng.close()


# ------------------------------------------------------------------------------------------------ gateway
def test_gateway_windowed_deployment_over_http():
    """b200/tiny-sw at a 16384-token context window on a 17408-token pool (272 pages; a ring is 131 pages at the default
    8192-token prefill chunk): n = 2 choices of a ~9000-token prompt (2 x 142 pages linearly) are served, through the
    OpenAI SDK, streamed and non-streamed; n = 3 (3 x 131 pages) stays a 400."""
    import openai
    from test_fp8_weights_gpu import _server
    from rr_b200 import Router
    from rr_b200.config import build_config
    from rr_b200.server import build_backends
    ml = [{"model_name": "sw", "litellm_params": {"model": "b200/tiny-sw", "gpu": 0, "context_window": 16384,
                                                  "kv_cache_tokens": 17408}}]
    backends = build_backends(build_config(ml), stub=False, max_batch=4)
    r = Router(model_list=ml, backends=backends, default_max_tokens=24, seed=0)
    server, th, port = _server(r)
    try:
        client = openai.OpenAI(api_key="k", base_url=f"http://127.0.0.1:{port}", max_retries=0)
        text = " ".join(f"w{i % 97}" for i in range(2400))                 # ~9000 bytes: byte-level tokens
        msgs = [{"role": "user", "content": text}]
        a = client.chat.completions.create(model="sw", messages=msgs, n=2, max_tokens=16, timeout=120)
        assert len(a.choices) == 2 and a.usage.prompt_tokens > 8500
        assert a.usage.prompt_tokens + 16 > 131 * 64                       # a ring request
        b = client.chat.completions.create(model="sw", messages=msgs, max_tokens=16, timeout=120)
        sb = "".join(c.choices[0].delta.content or "" for c in
                     client.chat.completions.create(model="sw", messages=msgs, max_tokens=16, stream=True, timeout=120)
                     if c.choices)
        assert sb == b.choices[0].message.content and b.usage.completion_tokens > 0
        with pytest.raises(openai.BadRequestError):
            client.chat.completions.create(model="sw", messages=msgs, n=3, max_tokens=16, timeout=120)
    finally:
        server.should_exit = True
        th.join(10)
        r.close()
        for be in backends.values():
            be.engine.close()
