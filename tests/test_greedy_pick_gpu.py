"""GPU: the hand-off between two decode steps at kernel level, as the engine runs it.  The greedy pick (rr_op_argmax, the
first kernel of the logits tail) writes one token per row; the sampler (rr_op_sample) may replace it; the next step's
embedding gather (rr_op_embed) reads table row `token` with no check.

The reference pick is exact, so every comparison is equality, never a tolerance: replace NaN by -inf, take m = the row
max, and pick the first index with x == m (-0 == +0), or 0 when m == -inf.  out_val must be that column's value bit for
bit (-inf when m is -inf).  The argmax kernel (rr_elementwise.cu) has 1024 threads, each reading 16-byte vectors 4096
columns apart, 8 of them per round (32768 columns), then a scalar tail of vocab % 4 columns; the special rows below put
the maximum, ties, signed zeros, infinities, subnormals and NaN on those seams.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sampling_oracle as O

pytestmark = pytest.mark.gpu

STRIDE = 1024 * 4                # columns between a thread's vectors
ROUND = 8 * STRIDE               # columns per round of the main loop
NAN, INF = np.float32("nan"), np.float32("inf")
TOP = np.float32(10.0)           # a planted maximum: random rows are N(0, 1), under 6.5 over 33 M draws
GUARD = 4                        # entries past `rows` in every output array, which must stay as they were


def _lib():
    from rr_b200 import _lib
    return _lib.lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def ref_pick(x):
    """x float32 [rows, vocab] -> (token int64 [rows], value float32 [rows]) of the contract."""
    y = np.where(np.isnan(x), -INF, x)
    m = y.max(axis=1)
    tok = np.argmax(y == m[:, None], axis=1)
    tok = np.where(m == -INF, 0, tok)
    val = np.where(m == -INF, -INF, x[np.arange(len(x)), tok]).astype(np.float32)
    return tok, val


# ------------------------------------------------------------------------------------------------ special rows
def _seams(vocab):
    """Columns where the kernel changes thread, warp, vector slot, round, or goes from the vector body to the scalar tail."""
    v4 = vocab & ~3
    last_round = (v4 - 1) // ROUND * ROUND
    cols = [0, 3, 4, 4095, 4096, 32767, 32768, 4 * 31, 4 * 32, 4 * 1023 + 3,
            last_round, last_round + 4, last_round + STRIDE - 1, v4 - 4, v4 - 1]
    cols += list(range(v4, vocab))                      # every scalar-tail column
    return sorted({c for c in cols if 0 <= c < vocab})


def _ties(vocab):
    """Pairs (and one triple) of columns planted with the same maximum: the lowest must win."""
    v4 = vocab & ~3
    t = [(8, 9), (8, 11), (9, 10),                      # one float4
         (4, 12), (20, 124),                            # lanes of one warp
         (0, 128), (124, 128), (128, 3968), (4092, 4096),   # warps; the last also across vector slots
         (16, 16 + STRIDE), (16 + STRIDE, 16 + 7 * STRIDE),  # vector slots of one thread
         (16, 16 + ROUND), (32767, 32768), (5, 5 + 3 * ROUND),   # rounds
         (0, vocab - 1), (v4 - 4, vocab - 1), (v4 - 1, vocab - 1),   # body and the last column
         (5, STRIDE + 5, vocab - 1)]
    if vocab % 4 >= 2:
        t.append((v4, vocab - 1))                       # inside the tail
    if vocab % 4:
        t.append((v4 - 1, v4))                          # the last vector column and the first tail column
    return [p for p in t if len(set(p)) == len(p) and 0 <= min(p) and max(p) < vocab]


def special_rows(vocab, rng):
    """[(name, row float32 [vocab])]: each row is one edge case over N(0, 1) noise.  Fixed columns past the end of a small
    vocabulary fold onto its last column; the reference is computed from the row as built, so a fold is still a case."""
    rows = []

    def at(c):
        return min(c, vocab - 1)

    def noise():
        return rng.standard_normal(vocab, dtype=np.float32)

    def neg():                                          # every value in [-6, -1]: below 0 and below every subnormal
        return np.clip(-1.0 - np.abs(noise()), -6.0, -1.0).astype(np.float32)

    for c in _seams(vocab):
        x = noise(); x[c] = TOP
        rows.append((f"max@{c}", x))
    for p in _ties(vocab):
        x = noise(); x[list(p)] = TOP
        rows.append((f"tie@{p}", x))
    rows.append(("all-equal", np.full(vocab, 1.5, np.float32)))
    rows.append(("all-equal-negative", np.full(vocab, -3.25, np.float32)))
    rows.append(("all-ninf", np.full(vocab, -INF, np.float32)))
    rows.append(("all-nan", np.full(vocab, NAN, np.float32)))
    x = np.full(vocab, -INF, np.float32); x[::2] = NAN
    rows.append(("nan-ninf-alternating", x))
    x = np.full(vocab, NAN, np.float32); x[vocab // 2:] = -INF
    rows.append(("nan-then-ninf", x))
    x = np.full(vocab, -INF, np.float32); x[at(1)] = NAN; x[vocab - 1] = NAN
    rows.append(("ninf-with-nan-at-1-and-last", x))
    for c in (0, 4096, vocab - 1):
        x = np.full(vocab, -INF, np.float32); x[at(c)] = np.float32(-1e30)
        rows.append((f"ninf-but-one@{at(c)}", x))
    x = np.full(vocab, -INF, np.float32); x[: vocab - 1: 3] = NAN; x[vocab - 1] = np.float32(-1e30)
    rows.append(("ninf-nan-but-last", x))
    # signed zeros tie: the first of them wins, with its own sign bit
    a, b = at(4), at(STRIDE + 4)
    x = neg(); x[b] = np.float32(0.0); x[a] = np.float32(-0.0)
    rows.append(("-0-then-+0", x))
    x = neg(); x[b] = np.float32(-0.0); x[a] = np.float32(0.0)
    rows.append(("+0-then--0", x))
    x = neg(); x[vocab - 1] = np.float32(-0.0); x[vocab // 3] = np.float32(-0.0)
    rows.append(("-0-twice", x))
    # infinities
    x = noise(); x[at(vocab - 2)] = INF
    rows.append(("+inf", x))
    x = noise(); x[at(7)] = INF; x[at(3)] = INF
    rows.append(("+inf-tie", x))
    x = np.full(vocab, NAN, np.float32); x[: vocab // 4] = -INF; x[vocab // 2] = INF
    rows.append(("+inf-among-nan", x))
    # subnormal maxima: with flush-to-zero compares they would tie with 0 or with each other
    tiny = np.float32(1.4e-45)
    x = neg(); x[at(STRIDE + 1)] = tiny; x[at(2)] = np.float32(0.0)
    rows.append(("subnormal-above-0", x))
    x = neg(); x[at(1)] = tiny; x[vocab - 1] = np.float32(2.8e-45)
    rows.append(("larger-subnormal-last", x))
    x = neg(); x[0] = np.float32(-2.8e-45); x[vocab - 1] = -tiny
    rows.append(("negative-subnormals", x))
    x = neg(); x[at(vocab // 2 + 1)] = np.float32(1.1754942e-38); x[vocab // 2] = np.float32(1.17549435e-38)
    rows.append(("smallest-normal-vs-largest-subnormal", x))
    # maxima near the ends of the finite range
    x = noise() * np.float32(1e37); x[0] = np.float32(2.9999998e38); x[vocab - 1] = np.float32(3e38)
    rows.append(("+3e38", x))
    x = np.full(vocab, np.float32(-3.4028235e38), np.float32); x[::5] = -INF
    x[vocab // 3] = np.float32(-3e38); x[vocab - 1] = np.float32(-3e38)
    rows.append(("-3e38", x))
    # NaN around a finite maximum: NaN never wins, and never hides a value that does
    c = at(STRIDE + 9)
    x = noise(); x[0:4] = NAN; x[max(c - 1, 0)] = NAN; x[at(c + 1)] = NAN; x[c] = TOP
    rows.append(("nan-around-max", x))
    x = noise(); x[rng.random(vocab) < 0.1] = NAN; x[max(vocab - 2, 0)] = NAN; x[vocab - 1] = TOP
    rows.append(("nan-10pct-max-last", x))
    x = np.full(vocab, NAN, np.float32); x[at(vocab // 2 | 2)] = np.float32(-7.0)
    rows.append(("one-finite-in-nan", x))
    x = np.full(vocab, NAN, np.float32); x[vocab - 1] = np.float32(-1.0)
    rows.append(("nan-but-last", x))
    return rows


# ------------------------------------------------------------------------------------------------ argmax
def _run_argmax(x_pad, ld, vocab, active=None):
    """rr_op_argmax over host rows x_pad [rows][ld] with out_val and pos_inc; tok / val / pos start at -7 / NaN / 1000 + r
    and carry GUARD more entries.  Returns (tok, val, pos), each of rows + GUARD entries."""
    rows = x_pad.shape[0]
    d_x = torch.from_numpy(np.ascontiguousarray(x_pad)).cuda()
    tok = torch.full((rows + GUARD,), -7, dtype=torch.int32, device="cuda")
    val = torch.full((rows + GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    pos = (torch.arange(rows + GUARD, dtype=torch.int32) + 1000).cuda()
    d_act = torch.from_numpy(active).cuda() if active is not None else None
    rc = _lib().rr_op_argmax(_ptr(d_x), ld, rows, vocab, _ptr(tok), _ptr(val), _ptr(d_act), _ptr(pos), None)
    assert rc == 0
    torch.cuda.synchronize()
    return tok.cpu().numpy(), val.cpu().numpy(), pos.cpu().numpy()


def _check(x, tok, val, pos, active, names):
    """tok / val / pos of _run_argmax against ref_pick on the active rows; everything else as it was."""
    rows = x.shape[0]
    want_tok, want_val = ref_pick(x)
    on = np.ones(rows, bool) if active is None else active >= 0
    got_bits, want_bits = _bits(val[:rows]), _bits(want_val)
    bad = [(names[r], int(tok[r]), int(want_tok[r]), float(val[r]), float(want_val[r])) for r in np.flatnonzero(on)
           if tok[r] != want_tok[r] or got_bits[r] != want_bits[r]]
    assert not bad, bad                                                              # (row, got, want, got val, want val)
    assert (tok[:rows][~on] == -7).all() and np.isnan(val[:rows][~on]).all()        # inactive rows keep tok (and val)
    assert (pos[:rows] == 1000 + np.arange(rows) + on).all()                         # + 1 exactly once, active rows only
    assert (tok[rows:] == -7).all() and np.isnan(val[rows:]).all()                   # nothing past rows
    assert (pos[rows:] == 1000 + rows + np.arange(GUARD)).all()


def _pad(x, ld):
    """[rows][ld] with the pad columns holding +inf, NaN and 3e38: any of them read would win or poison a compare."""
    rows, vocab = x.shape
    out = np.empty((rows, ld), np.float32)
    out[:, :vocab] = x
    fill = np.array([INF, NAN, np.float32(3e38)], np.float32)
    out[:, vocab:] = fill[np.arange(ld - vocab) % 3]
    return out


@pytest.mark.parametrize("vocab", [1024, 4096, 32000, 32064, 128256])
@pytest.mark.parametrize("rows", [1, 2, 17, 64, 129, 256])
def test_argmax_at_engine_shapes(vocab, rows):
    """ld = vocab, as the engine's logits buffer.  Even rows run through the special rows (all of them from 129 rows on),
    odd rows are noise with a maximum planted at a random column; every ninth row is inactive (row_active -1, as the slot
    of a free decode row)."""
    rng = np.random.default_rng(vocab * 1000 + rows)
    special = special_rows(vocab, rng)
    x = np.empty((rows, vocab), np.float32)
    names = []
    for r in range(rows):
        if r % 2 == 0:
            n, row = special[(r // 2 + rows) % len(special)]
            x[r] = row
        else:
            x[r] = rng.standard_normal(vocab, dtype=np.float32)
            n = int(rng.integers(0, vocab))
            x[r, n] = TOP
            n = f"noise-max@{n}"
        names.append(n)
    active = np.where(np.arange(rows) % 9 == 4, -1, np.arange(rows)).astype(np.int32)
    tok, val, pos = _run_argmax(x, vocab, vocab, active)
    _check(x, tok, val, pos, active, names)
    # without row_active / pos_inc / out_val, as rr_op_logprobs' callers use it: the same tokens on every row
    d_x = torch.from_numpy(x).cuda()
    t2 = torch.full((rows,), -7, dtype=torch.int32, device="cuda")
    assert _lib().rr_op_argmax(_ptr(d_x), vocab, rows, vocab, _ptr(t2), None, None, None, None) == 0
    assert np.array_equal(t2.cpu().numpy(), ref_pick(x)[0])


@pytest.mark.parametrize("vocab,ld", [(128256, 128256), (32064, 32064), (32000, 32000), (4096, 4096), (1024, 1024),
                                      (32001, 32008), (32002, 32008), (32003, 32004), (1025, 1032), (1026, 1028),
                                      (1027, 1036), (128257, 128264), (5, 8), (4, 4), (1, 4), (3, 4)])
def test_argmax_special_rows(vocab, ld):
    """Every special row of the vocabulary in one launch, all active; with ld > vocab the pad columns hold values that would
    win (+inf, 3e38) or poison a compare (NaN) if they were read."""
    rng = np.random.default_rng(vocab)
    special = special_rows(vocab, rng)
    names = [n for n, _ in special]
    x = np.stack([r for _, r in special])
    tok, val, pos = _run_argmax(_pad(x, ld), ld, vocab)
    _check(x, tok, val, pos, None, names)
    assert ((tok[:len(x)] >= 0) & (tok[:len(x)] < vocab)).all()


def test_argmax_rows_without_a_value_above_ninf_pick_token_0():
    """The hand-off's safety: a row of -inf and NaN only (NaN logits from a checkpoint with non-finite weights, for
    example) picks token 0 with value -inf, as torch.argmax does for an all -inf row, never an id past the vocabulary."""
    vocab = 128256
    x = np.full((6, vocab), -INF, np.float32)
    x[1] = NAN
    x[2, ::2] = NAN
    x[3, vocab // 2:] = NAN
    x[4, 0] = NAN
    x[5, vocab - 1] = NAN
    tok, val, pos = _run_argmax(x, vocab, vocab)
    assert (tok[:6] == 0).all(), tok
    assert (val[:6] == -INF).all() and (pos[:6] == 1001 + np.arange(6)).all()
    want = torch.from_numpy(np.where(np.isnan(x), -INF, x)).argmax(-1).numpy()
    assert (want == 0).all()                                             # torch.argmax agrees on the all -inf rows


# ------------------------------------------------------------------------------------------------ sampler
def _sample(x, ld, vocab, T, P, S, Q, prefill):
    rows = len(T)
    d_x = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_t = torch.tensor(T, dtype=torch.float32, device="cuda")
    d_p = torch.tensor(P, dtype=torch.float32, device="cuda")
    d_s = torch.tensor(np.asarray(S, dtype=np.uint64).view(np.int64), device="cuda")
    d_q = torch.tensor(Q, dtype=torch.int32, device="cuda")
    out = torch.tensor(prefill, dtype=torch.int32, device="cuda")
    rc = _lib().rr_op_sample(_ptr(d_x), ld, rows, vocab, _ptr(d_t), _ptr(d_p), _ptr(d_s), _ptr(d_q), _ptr(out), None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("vocab,ld", [(128256, 128256), (32064, 32064), (1003, 1004)])
def test_sample_without_a_candidate_keeps_the_token(vocab, ld):
    """Rows of -inf and NaN only have no token to draw, at top_p 1 and 0.9: the token already in out_tok (in the engine the
    greedy pick, token 0) stays.  A zero row (the draw is the largest Philox word, known exactly) and a noise row whose
    draw is clear of every rounding margin (sampling_oracle.sample) in the same launch get the oracle's token."""
    rng = np.random.default_rng(vocab + 1)
    empty = []
    for fill in ("ninf", "nan", "mixed"):
        x = np.full(vocab, -INF, np.float32)
        if fill == "nan":
            x[:] = NAN
        elif fill == "mixed":
            x[1::3] = NAN
        empty.append(x)
    rows, T, P = [], [], []
    for x in empty:
        for p in (1.0, 0.9):
            rows.append(x); T.append(1.0); P.append(p)
    n_empty = len(rows)
    rows.append(np.zeros(vocab, np.float32)); T.append(1.0); P.append(1.0)
    noise = rng.standard_normal(vocab, dtype=np.float32) * np.float32(2.0)
    rows.append(noise); T.append(0.8); P.append(0.9)
    S = [(0x9E3779B97F4A7C15 * (r + 3)) % 2**64 for r in range(len(rows))]
    Q = [17 + 5 * r for r in range(len(rows))]
    prefill = [4000 + r if r % 2 else 0 for r in range(len(rows))]
    x = _pad(np.stack(rows), ld)
    got = _sample(x, ld, vocab, T, P, S, Q, prefill)
    assert list(got[:n_empty]) == prefill[:n_empty], got
    z = n_empty
    assert got[z] == int(np.argmax(O.random_words(S[z], Q[z], vocab) >> np.uint64(9)))
    d = O.sample(noise, T[z + 1], P[z + 1], S[z + 1], Q[z + 1], mass_slack=2e-5)
    assert d.stable_nucleus and d.score_gap > d.score_bound              # a clear draw: the kernel must give it
    assert got[z + 1] == d.token


# ------------------------------------------------------------------------------------------------ embed
@pytest.mark.parametrize("hidden", [384, 512, 768, 1024, 3072, 4096, 5120, 8192])
def test_embed_bit_exact_at_max_batch(hidden):
    """256 rows (the engine's largest max_batch): x[r] = table[ids[r]].float() bit for bit, ids 0, vocab - 1 and repeats;
    inactive rows and the row past `rows` keep every bit of what was there."""
    vocab, rows = 32064, 256
    g = torch.Generator(device="cuda").manual_seed(hidden)
    table = torch.randn(vocab, hidden, device="cuda", generator=g).to(torch.bfloat16)
    table[vocab - 1, : hidden // 2] = float("-inf")                 # non-finite and signed-zero entries copy exactly
    table[vocab - 1, hidden // 2:] = -0.0
    ids = torch.randint(0, vocab, (rows,), device="cuda", generator=g, dtype=torch.int32)
    ids[0], ids[1], ids[2:6] = 0, vocab - 1, 77
    ids[200:256:5] = vocab - 1
    active = torch.arange(rows, device="cuda", dtype=torch.int32)
    active[3::11] = -1
    x = torch.randn(rows + 1, hidden, device="cuda", generator=g)
    before = x.clone()
    assert _lib().rr_op_embed(_ptr(ids), _ptr(table), _ptr(x), rows, hidden, _ptr(active), None) == 0
    torch.cuda.synchronize()
    on = active >= 0
    want = table[ids.long()].float()
    assert torch.equal(x[:rows][on].view(torch.int32), want[on].view(torch.int32))
    assert torch.equal(x[:rows][~on].view(torch.int32), before[:rows][~on].view(torch.int32))
    assert torch.equal(x[rows].view(torch.int32), before[rows].view(torch.int32))
    # without row_active every row is gathered
    assert _lib().rr_op_embed(_ptr(ids), _ptr(table), _ptr(x), rows, hidden, None, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(x[:rows].view(torch.int32), want.view(torch.int32))


def test_embed_row_offset_past_2_31_elements():
    """vocab 262160 x hidden 8192 (a 4.3 GB table): id * hidden >= 2^31 from id 262144 on, so the row offset must be
    computed in 64 bits."""
    vocab, hidden = 262160, 8192
    if torch.cuda.mem_get_info()[0] < 8 * 2**30:
        pytest.skip("needs 8 GB of free device memory")
    table = torch.zeros(vocab, hidden, dtype=torch.bfloat16, device="cuda")
    ids = torch.tensor([vocab - 1, 262144, 262143, 0, 131072, vocab - 1, 262150, 1], dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    uniq = ids.long().unique()
    table[uniq] = torch.randn(len(uniq), hidden, device="cuda", generator=g).to(torch.bfloat16)
    rows = len(ids)
    x = torch.full((rows, hidden), float("nan"), device="cuda")
    try:
        assert _lib().rr_op_embed(_ptr(ids), _ptr(table), _ptr(x), rows, hidden, None, None) == 0
        torch.cuda.synchronize()
        assert torch.equal(x.view(torch.int32), table[ids.long()].float().view(torch.int32))
        assert (x.abs().sum(-1) > 0).all()                          # every row read a planted (nonzero) table row
    finally:
        del table
        torch.cuda.empty_cache()
