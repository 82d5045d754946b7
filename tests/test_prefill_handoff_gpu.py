"""GPU, kernel level: the kernels that hand a prefill chunk's results over to decode, as run_prefill runs them.

  kv_copy_prefix_kernel   the cached-prefix copies before the first layer and the n-choices fan-out after the last one,
                          over the paged pool (rr_op_kv_copy_prefix_paged) and the slot-contiguous cache (rr_op_kv_copy_prefix)
  gather_last_kernel      the tail and embedding rows' attention output and residual into the decode buffers (rr_op_gather_last)
  activate_rows_kernel    each tail row becomes a live decode row: token, position, slot (rr_op_activate_rows)
  dequantize_fp8_kernel   an FP8 layer's QKV, O, gate/up and down weights into the prefill scratch in one launch
                          (rr_op_dequantize_fp8_jobs)

All four only move data, so every reference is exact and every check compares bits.  Whatever a kernel must not write
holds a sentinel (NaN bit patterns for bf16 / fp32, -7 for ints) that is checked afterwards.  The shapes are the engine's:
the model families' layer counts, kv heads and head dims, max_batch up to 256 (KV_COPY_MAX), max_prefill_tokens 8192,
context windows up to 65536 tokens and pools whose last layers lie past 2^31 elements."""
import ctypes as C
import gc

import pytest
import torch

from test_fp8_weights_gpu import _planted, _quantize
from test_paged_kv_gpu import PAGE, Pool

pytestmark = pytest.mark.gpu
DEV = "cuda"
RR_INVALID_ARGUMENT = 4
SENT_K, SENT_V = 0x7FA1, -0x005D            # bf16 NaN bit patterns (0x7FA1, 0xFFA3) of the KV pool's untouched rows
SENT_BF16 = 0x7FC1                          # bf16 NaN
SENT_F32 = 0x7FC00001                       # fp32 NaN
SENT_INT = -7


def _lib():
    from rr_b200 import _lib
    return _lib


def P(t):
    return C.c_void_p(t.data_ptr())


def _i32(xs):
    return (C.c_int32 * len(xs))(*xs)


def _spec(family):
    from rr_b200.models import SPECS
    return SPECS[family]


@pytest.fixture(autouse=True)
def _release_memory():
    """The largest cases hold ~10 GB; give it back to the device before the next test."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------ KV copies
class KvCopyCase:
    """A KV cache for one copy list (src slot, dst slot, n) as run_prefill launches it: every layer, every kv head, K and V.

    Paged: a Pool (test_paged_kv_gpu) whose pages a random permutation hands out, so a slot's pages are not monotonic; a
    source slot owns the pages of its n positions, a destination those of its reach (n + 1 positions, the first generated
    token included, at most ctx), and table entries past a slot's pages name unused pages.  Contiguous:
    [layers][slots][kv][ctx][128].  Source rows hold random bits (zero in the pad columns of a head_dim-96 family, as the
    engine leaves them) and every other row a NaN sentinel.  The expected cache is built one layer at a time: sentinel,
    the sources' rows regenerated from their seeds, then a gather / scatter of whole 128-wide rows through the same table."""

    def __init__(self, family, layers, ctx, copies, paged=True, seed=0, extra=8, n_pages=None):
        spec = _spec(family)
        self.KV, self.hd, self.L, self.ctx, self.copies, self.paged = spec.n_kv_heads, spec.head_dim, layers, ctx, copies, paged
        self.seed = seed
        self.n_slots = max(x for s, d, _ in copies for x in (s, d)) + 1
        self.fill = {}                                            # source slot -> positions of KV it holds
        for s, _, n in copies:
            self.fill[s] = max(self.fill.get(s, 0), n)
        if paged:
            self.pps = ctx // PAGE
            need = [0] * self.n_slots
            for s, n in self.fill.items():
                need[s] = -(-n // PAGE)
            for _, d, n in copies:
                need[d] = min(self.pps, -(-(n + 1) // PAGE))
            if n_pages is not None:
                extra = n_pages - sum(need)
            assert extra >= 1
            self.pool = Pool(layers, self.KV, ctx, need, extra, torch.Generator().manual_seed(seed))
            self.k, self.v = self.pool.k, self.pool.v
            self.table = self.pool.table.long()
            self.unit = PAGE
        else:
            shape = (layers, self.n_slots, self.KV, ctx, 128)
            self.k = torch.empty(shape, device=DEV, dtype=torch.bfloat16)
            self.v = torch.empty(shape, device=DEV, dtype=torch.bfloat16)
            self.unit = ctx
        self.k.view(torch.int16).fill_(SENT_K)
        self.v.view(torch.int16).fill_(SENT_V)
        for s in self.fill:
            for l in range(layers):
                self.k.view(torch.int16)[l, self.units(s)] = self.src_bits(s, l, 0)
                self.v.view(torch.int16)[l, self.units(s)] = self.src_bits(s, l, 1)

    def units(self, s):
        """the pages (paged) or the slot (contiguous) that hold source slot s's KV"""
        if not self.paged:
            return torch.tensor([s], device=DEV)
        return self.pool.dtable[s, :-(-self.fill[s] // PAGE)].long()

    def src_bits(self, s, l, which):
        g = torch.Generator(device=DEV).manual_seed(((self.seed * 1000 + s) * 256 + l) * 2 + which)
        n_units = 1 if not self.paged else -(-self.fill[s] // PAGE)
        r = torch.randint(-32768, 32768, (n_units, self.KV, self.unit, 128), device=DEV, dtype=torch.int16, generator=g)
        if self.hd < 128:
            r[..., self.hd:] = 0
        return r

    def rows(self, slot, n):
        """rows of positions [0, n) of slot, every kv head, in one layer's [rows][128] view"""
        p, h = torch.arange(n), torch.arange(self.KV)[:, None]
        if self.paged:
            return ((self.table[slot, p // PAGE][None] * self.KV + h) * PAGE + p % PAGE).flatten()
        return ((slot * self.KV + h) * self.ctx + p[None]).flatten()

    def launch(self, copies=None):
        L = _lib()
        copies = self.copies if copies is None else copies
        src, dst, n = (list(x) for x in zip(*copies)) if copies else ([], [], [])
        if self.paged:
            return L.lib.rr_op_kv_copy_prefix_paged(P(self.k), P(self.v), self.L, self.n_slots, self.KV, self.ctx, _i32(src),
                                                    _i32(dst), _i32(n), len(copies), P(self.pool.dtable), self.pps,
                                                    self.pool.n_pages, None)
        return L.lib.rr_op_kv_copy_prefix(P(self.k), P(self.v), self.L, self.n_slots, self.KV, self.ctx, _i32(src), _i32(dst),
                                          _i32(n), len(copies), None)

    def check(self):
        torch.cuda.synchronize()
        src = torch.cat([self.rows(s, n) for s, _, n in self.copies]).to(DEV)
        dst = torch.cat([self.rows(d, n) for _, d, n in self.copies]).to(DEV)
        for which, (t, sent) in enumerate(((self.k, SENT_K), (self.v, SENT_V))):
            for l in range(self.L):
                want = torch.full(t.shape[1:], sent, device=DEV, dtype=torch.int16)
                for s in self.fill:
                    want[self.units(s)] = self.src_bits(s, l, which)
                flat = want.view(-1, 128)
                flat[dst] = flat[src]                     # no source is a destination: the order does not matter
                assert torch.equal(t[l].view(torch.int16), want), f"{'KV'[which]} cache, layer {l}"


def _run(case):
    _lib().check(case.launch(), "kv copy")
    case.check()


FAMILIES = ["llama-3-8b", "phi-3-mini", "mistral-7b", "tiny96", "small"]
# n of the fan-out per (family, destinations): the n values of the prefix lists below spread over the cases, small enough
# for the wide fan-outs of the 32-layer families to fit their pools in about 9 GB
FANOUT_N = {
    "llama-3-8b": {1: 4097, 2: 4097, 3: 4097, 63: 128, 255: 65},
    "phi-3-mini": {1: 4097, 2: 65, 3: 127, 63: 127, 255: 63},
    "mistral-7b": {1: 1, 2: 64, 3: 4097, 63: 63, 255: 64},
    "tiny96": {1: 4160, 2: 4097, 3: 1, 63: 4160, 255: 127},
    "small": {1: 63, 2: 4160, 3: 4097, 63: 4097, 255: 128},
}
CTX = 4160                                                  # 65 pages: n up to 4097 and n = ctx_max


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("dests", [1, 2, 3, 63, 255])
def test_kv_copy_fanout(family, dests):
    """The n-choices fan-out: one source slot to the slots of a request's other `dests` choices (up to 255 with
    max_batch 256), every layer of the family, slots scattered over the batch."""
    n = FANOUT_N[family][dests]
    slots = torch.randperm(256, generator=torch.Generator().manual_seed(dests))[:dests + 1].tolist()
    case = KvCopyCase(family, _spec(family).n_layers, CTX, [(slots[0], d, n) for d in slots[1:]], seed=dests)
    _run(case)


def _prefix_list(ctx):
    """cached prefixes from three sources in one launch, n mixed so grid.x follows the largest: 1, 63, 64, 65, 127, 128,
    4097 and ctx_max; destinations on both sides of their sources"""
    return [(5, 1, ctx), (0, 7, 1), (9, 2, 63), (5, 3, 64), (0, 4, 65), (9, 6, 127), (5, 8, 128), (0, 10, 4097)]


@pytest.mark.parametrize("family", FAMILIES)
def test_kv_copy_prefix_list(family):
    _run(KvCopyCase(family, _spec(family).n_layers, CTX, _prefix_list(CTX), seed=11))


@pytest.mark.parametrize("family", ["tiny96", "small"])
@pytest.mark.parametrize("copies", ["fanout", "prefix"])
def test_kv_copy_contiguous(family, copies):
    """The slot-contiguous layout [layers][slots][kv][ctx][128] with the same lists."""
    lst = _prefix_list(CTX) if copies == "prefix" else [(17, d, 4097) for d in range(64) if d != 17]
    _run(KvCopyCase(family, _spec(family).n_layers, CTX, lst, paged=False, seed=12))


def test_kv_copy_llama_ctx_65536():
    """A whole 65536-token context copied (n = ctx_max, 1024 pages per slot) next to a 4097-token one in the same list.
    8 of Llama-3-8B's 32 layers: with all 32 the pool for two full contexts would take 17 GB."""
    _run(KvCopyCase("llama-3-8b", 8, 65536, [(2, 0, 65536), (1, 3, 4097)], seed=13))


def test_kv_copy_llama_pool_past_2_31_elements():
    """Llama-3-8B, all 32 layers, over a pool of 1152 pages: layer l starts at l x 1152 x 8 x 64 x 128 elements, so the
    copies of layers 29..31 land past 2^31 elements."""
    case = KvCopyCase("llama-3-8b", 32, CTX, [(7, 0, 4097), (7, 3, 4097), (7, 5, 4097), (2, 6, 65)], seed=14, n_pages=1152)
    layer_elems = case.pool.n_pages * case.KV * PAGE * 128
    assert case.k[31].data_ptr() - case.k.data_ptr() == 31 * layer_elems * 2
    assert 31 * layer_elems > 2 ** 31 and 29 * layer_elems > 2 ** 31 > 28 * layer_elems
    _run(case)


def test_kv_copy_refusals_leave_the_pool_unchanged():
    """The lists kv_copy_check refuses (run_prefill returns RR_INVALID_ARGUMENT for them) are refused before the launch:
    a destination listed twice, a destination that is also a source, n > ctx_max or n < 1, a slot outside the batch,
    more than 256 copies.  The pool keeps every bit."""
    case = KvCopyCase("small", 4, CTX, [(0, 1, 100), (2, 3, 64)], seed=15)
    k0, v0 = case.k.clone(), case.v.clone()
    bad = [[(0, 1, 10), (2, 1, 10)],                      # duplicate destination
           [(0, 1, 10), (1, 3, 10)],                      # a source that is also a destination
           [(0, 1, CTX + 1)],                             # n > ctx_max
           [(0, 1, 0)],                                   # n < 1
           [(0, case.n_slots, 10)],                       # slot outside [0, n_slots)
           [(0, 1 + i % 3, 10) for i in range(257)]]      # count > 256 (refused before the list is read)
    for lst in bad:
        assert case.launch(lst) == RR_INVALID_ARGUMENT, lst[:3]
    torch.cuda.synchronize()
    assert torch.equal(case.k.view(torch.int16), k0.view(torch.int16))
    assert torch.equal(case.v.view(torch.int16), v0.view(torch.int16))


# --------------------------------------------------------------------------------------------------- the tail rows
def _chunk(seqs, seed):
    """A prefill chunk's rows as run_prefill numbers them.  seqs: (len, pos0, choices) per sequence, choices 0 for an
    embedding request.  Returns the token positions [T], and per row (tail rows in sequence order, then the embedding
    rows): the index of its sequence's last token and its slot, distinct slots of a shuffled batch of 256."""
    tok_pos, last, emb_last = [], [], []
    for ln, p0, ch in seqs:
        tok_pos += range(p0, p0 + ln)
        (last if ch else emb_last).extend([len(tok_pos) - 1] * max(ch, 1))
    slots = torch.randperm(256, generator=torch.Generator().manual_seed(seed))[:len(last) + len(emb_last)].tolist()
    return tok_pos, last + emb_last, slots


def _seqs(rows, T, emb=0, seed=0):
    """Sequences over T tokens with rows - emb tail rows, about 3 / 4 as many sequences as tail rows (so several rows
    share a last token), then emb embedding requests"""
    g = torch.Generator().manual_seed(seed)
    n_tail_seqs = max(1, min(rows - emb, T - emb, 200) * 3 // 4)
    n_seq = n_tail_seqs + emb
    cuts = sorted(torch.randperm(T - 1, generator=g)[:n_seq - 1].add(1).tolist())
    lens = [b - a for a, b in zip([0] + cuts, cuts + [T])]
    choices = [1] * n_tail_seqs
    for _ in range(rows - emb - n_tail_seqs):
        choices[int(torch.randint(n_tail_seqs, (1,), generator=g))] += 1
    p0 = torch.randint(0, 4096, (n_seq,), generator=g).tolist()
    return [(lens[i], p0[i], choices[i] if i < n_tail_seqs else 0) for i in range(n_seq)]


def _rand_bits(shape, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if dtype == torch.bfloat16:
        return torch.randint(-32768, 32768, shape, device=DEV, dtype=torch.int16, generator=g).view(torch.bfloat16)
    return torch.randint(-2 ** 31, 2 ** 31, shape, device=DEV, dtype=torch.int32, generator=g).view(torch.float32)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


GATHER_WIDTHS = {"llama-3-8b": (4096, 4096), "phi-3-mini": (3072, 3072), "tiny": (512, 512), "tiny96": (384, 384),
                 "small": (1024, 1024), "small96": (768, 768)}
GATHER_ROWS = {"1": (1, 8192, 0), "2": (2, 8192, 0), "64": (64, 8192, 0), "129": (129, 5000, 0), "256": (256, 8192, 0),
               "240tail_16emb": (256, 8192, 16), "129_fanout_from_3_tokens": (129, 3, 0)}


@pytest.mark.parametrize("family", list(GATHER_WIDTHS))
@pytest.mark.parametrize("rows", list(GATHER_ROWS))
def test_gather_last(family, rows):
    """attn_out / x_out rows r < n_rows are rows last[r] of the chunk's attention output (bf16 [T][nq], nq = n_heads x
    head_dim) and residual (fp32 [T][hidden]), several rows sharing a last token (the choices of one prompt), embedding
    rows after the tail rows; the rows after n_rows of the decode buffers (max_batch + 8) keep their sentinel."""
    L = _lib()
    nq, hidden = GATHER_WIDTHS[family]
    n_rows, T, emb = GATHER_ROWS[rows]
    seqs = [(T, 0, n_rows)] if T < n_rows else _seqs(n_rows, T, emb, seed=n_rows + T)
    _, last, _ = _chunk(seqs, 0)
    assert len(last) == n_rows
    attn, x = _rand_bits((T, nq), torch.bfloat16, 1), _rand_bits((T, hidden), torch.float32, 2)
    a0, x0 = attn.clone(), x.clone()
    attn_out = torch.full((264, nq), SENT_BF16, device=DEV, dtype=torch.int16).view(torch.bfloat16)
    x_out = torch.full((264, hidden), SENT_F32, device=DEV, dtype=torch.int32).view(torch.float32)
    d_last = torch.tensor(last, device=DEV, dtype=torch.int32)
    L.check(L.lib.rr_op_gather_last(P(attn), P(x), P(d_last), n_rows, nq, hidden, P(attn_out), P(x_out), None), "gather")
    torch.cuda.synchronize()
    idx = d_last.long()
    assert torch.equal(_bits(attn_out[:n_rows]), _bits(attn.index_select(0, idx)))
    assert torch.equal(_bits(x_out[:n_rows]), _bits(x.index_select(0, idx)))
    assert bool((_bits(attn_out[n_rows:]) == SENT_BF16).all()) and bool((_bits(x_out[n_rows:]) == SENT_F32).all())
    assert torch.equal(_bits(attn), _bits(a0)) and torch.equal(_bits(x), _bits(x0))


ACTIVATE = {
    # 256 one-choice sequences whose slots are a permutation of the batch, cached prefixes of up to 4095 positions
    "perm256": lambda: [(1 + i % 37, (i * 97) % 4096, 1) for i in range(256)],
    # one prompt's 255 choices share its last token; one more sequence in the last slot
    "fanout255": lambda: [(700, 300, 255), (5, 0, 1)],
    # positions up to ctx_max - 1 = 65535: a 65000-token cached prefix, the prompt ending at 65534
    "ctx_edge": lambda: [(535, 65000, 3), (64, 65471, 1), (1, 0, 2)],
    # one row; and 129 rows (two 128-thread CTAs) of 256, the other slots live decode rows that must keep their state
    "one": lambda: [(1, 0, 1)],
    "129of256": lambda: [(3 + i % 5, i * 31, 1 + (i % 3 == 0)) for i in range(96)] + [(2, 5, 1)],
}


@pytest.mark.parametrize("case", list(ACTIVATE))
def test_activate_rows(case):
    """Tail row i: d_tok[s] = first_tok[i], d_pos[s] = tok_pos[last[i]] + 1, d_slot[s] = s for s = its slot.  Slots not
    in the list keep token, position and slot bit for bit (some hold live rows, the others the -7 sentinel)."""
    L = _lib()
    tok_pos, last, slots = _chunk(ACTIVATE[case](), seed=len(case))
    n = len(last)
    g = torch.Generator().manual_seed(n)
    first = torch.randint(0, 128256, (n,), generator=g, dtype=torch.int32)
    live = torch.rand(256, generator=g) < 0.5
    tok0 = torch.where(live, torch.randint(0, 128256, (256,), generator=g, dtype=torch.int32), SENT_INT).int()
    pos0 = torch.where(live, torch.randint(0, 65536, (256,), generator=g, dtype=torch.int32), SENT_INT).int()
    slot0 = torch.where(live, torch.arange(256, dtype=torch.int32), SENT_INT).int()
    d_tok, d_pos, d_slot = tok0.to(DEV), pos0.to(DEV), slot0.to(DEV)
    ins = [torch.tensor(xs, device=DEV, dtype=torch.int32) for xs in (slots, first.tolist(), tok_pos, last)]
    L.check(L.lib.rr_op_activate_rows(*map(P, ins), n, P(d_tok), P(d_pos), P(d_slot), None), "activate")
    torch.cuda.synchronize()
    want_tok, want_pos, want_slot = tok0.clone(), pos0.clone(), slot0.clone()
    for i, s in enumerate(slots):
        want_tok[s], want_pos[s], want_slot[s] = first[i], tok_pos[last[i]] + 1, s
    assert max(want_pos[slots].tolist()) <= 65535
    if case == "ctx_edge":
        assert max(want_pos[slots].tolist()) == 65535
    assert torch.equal(d_tok.cpu(), want_tok) and torch.equal(d_pos.cpu(), want_pos) and torch.equal(d_slot.cpu(), want_slot)


# ------------------------------------------------------------------------------------------- FP8 layer dequantize
FP8_FAMILIES = ["llama-3-8b", "phi-3-mini", "tiny96", "small96"]


def _layer_jobs(spec, last_layer):
    """(rows, K) of launch_dequant_layer's jobs, back to back in the scratch with ld_out = K: wqkv, wo, wgu, wdown; the
    last layer of a chunk that does not score has wqkv only"""
    nq, nqkv = spec.n_heads * spec.head_dim, (spec.n_heads + 2 * spec.n_kv_heads) * spec.head_dim
    jobs = [(nqkv, spec.hidden), (spec.hidden, nq), (2 * spec.inter, spec.hidden), (spec.hidden, spec.inter)]
    return jobs[:1] if last_layer else jobs


@pytest.mark.parametrize("family", FP8_FAMILIES)
@pytest.mark.parametrize("layer", ["layer", "last"])
def test_dequantize_fp8_layer_jobs(family, layer):
    """One launch over a layer's jobs equals q.double() x scale exactly and, bit for bit, one rr_op_dequantize_fp8_weight
    call per job; the scratch after the last job (the engine's scratch is exactly the four jobs long) keeps its sentinel.
    For the full layers of every family but tiny96 the chunks outnumber the capped grid's threads, so threads walk from
    one job into the next."""
    L = _lib()
    spec = _spec(family)
    jobs = _layer_jobs(spec, layer == "last")
    if layer == "layer":
        assert sum(r * k for r, k in jobs) == (jobs[0][0] + jobs[1][1] + 3 * spec.inter) * spec.hidden   # e->deq's size
    qs, ss = [], []
    for i, (r, k) in enumerate(jobs):
        rc, q, s = _quantize(_planted(r, k, 100 * i + r))
        assert rc == 0
        qs.append(q)
        ss.append(s)
    offs = [0]
    for r, k in jobs:
        offs.append(offs[-1] + r * k)
    total_chunks = offs[-1] // 16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if layer == "layer" and family != "tiny96":
        assert total_chunks > 8 * sms * 256
    tail = 4096

    def scratch():
        return torch.full((offs[-1] + tail,), SENT_BF16, device=DEV, dtype=torch.int16).view(torch.bfloat16)

    one, again, sep = scratch(), scratch(), scratch()
    for out in (one, again):
        vp = lambda xs: (C.c_void_p * len(xs))(*xs)          # noqa: E731
        L.check(L.lib.rr_op_dequantize_fp8_jobs(vp([q.data_ptr() for q in qs]), vp([s.data_ptr() for s in ss]),
                                                _i32([r for r, _ in jobs]), _i32([k for _, k in jobs]),
                                                vp([out[o:].data_ptr() for o in offs[:-1]]), _i32([k for _, k in jobs]),
                                                len(jobs), None), "dequantize jobs")
    for (r, k), q, s, o in zip(jobs, qs, ss, offs):
        L.check(L.lib.rr_op_dequantize_fp8_weight(q.data_ptr(), s.data_ptr(), r, k, sep[o:].data_ptr(), k, None), "dequantize")
    torch.cuda.synchronize()
    assert torch.equal(_bits(one), _bits(again))
    assert torch.equal(_bits(one), _bits(sep))
    assert bool((_bits(one[offs[-1]:]) == SENT_BF16).all())
    for (r, k), q, s, o in zip(jobs, qs, ss, offs):
        d = one[o:o + r * k].view(r, k)
        assert torch.equal(d.double(), q.double() * s.double()[:, None]), (r, k)


# ------------------------------------------------------------------------------------------------------ determinism
def test_handoff_ops_are_deterministic():
    """Two calls of the KV copy, the gather and the activation on the same inputs give the same bits."""
    L = _lib()
    case = KvCopyCase("small96", 3, CTX, _prefix_list(CTX), seed=16)
    _lib().check(case.launch(), "kv copy")
    k1, v1 = case.k.clone(), case.v.clone()
    _lib().check(case.launch(), "kv copy")
    torch.cuda.synchronize()
    assert torch.equal(_bits(case.k), _bits(k1)) and torch.equal(_bits(case.v), _bits(v1))
    T, nq, hidden = 8192, 4096, 4096
    _, last, slots = _chunk(_seqs(256, T, 16, seed=3), 1)
    attn, x = _rand_bits((T, nq), torch.bfloat16, 3), _rand_bits((T, hidden), torch.float32, 4)
    d_last = torch.tensor(last, device=DEV, dtype=torch.int32)
    outs = []
    for _ in range(2):
        ao = torch.empty(256, nq, device=DEV, dtype=torch.bfloat16)
        xo = torch.empty(256, hidden, device=DEV, dtype=torch.float32)
        L.check(L.lib.rr_op_gather_last(P(attn), P(x), P(d_last), 256, nq, hidden, P(ao), P(xo), None), "gather")
        outs.append((ao, xo))
    tok_pos = torch.arange(T, device=DEV, dtype=torch.int32)
    d_slots, first = torch.tensor(slots, device=DEV, dtype=torch.int32), torch.arange(256, device=DEV, dtype=torch.int32)
    rows = []
    for _ in range(2):
        st = [torch.full((256,), SENT_INT, device=DEV, dtype=torch.int32) for _ in range(3)]
        L.check(L.lib.rr_op_activate_rows(P(d_slots), P(first), P(tok_pos), P(d_last), 240, *map(P, st), None), "activate")
        rows.append(st)
    torch.cuda.synchronize()
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(outs[0], outs[1]))
    assert all(torch.equal(a, b) for a, b in zip(rows[0], rows[1]))
