"""Decode and prefill attention deep in a 65536-token context, over a scattered page pool, against exact references.

At depth the rounding model of test_decode_attn_gpu.py grows with the tiles per split until it no longer tells a wrong
key set from the right one: dropping one key tile of 57345 random keys moves the answer by less than the bound.  So
addressing and masking are checked on operands whose correct answer the kernels compute exactly.

Selection operands.  Every key is a 2-hot code A (e_a + e_b), A = 64, {a, b} an unordered pair of dims below the head dim;
every (row, head) queries one code the same way.  Keys with that code score 2 A^2 = 8192, a power of two, so that the
row maximum, the scale and log2(e) leave them bit-identical and their p is exactly 1; every other key scores A^2 or less,
at least 500 below the maximum in log2 units, and its p is exactly 0 in exp2f and in ex2.approx.ftz.  V is 0 or 1 in
every element.  So l is the number of selected keys and o a count, both exact in fp32, and the output is bf16 of S / n
(S the sum of the selected keys' V, n their number) up to the fp32 roundings of 1 / l and o (1 / l): it must be the bf16
rounding of a value within 2^-21 |S / n| of S / n, and exactly 0 where S / n is 0.

The selection.  With H query heads, period M = 64 (H - 1) + 1: key j of a kv head carries the code of its residue j mod M
(M distinct codes per kv head), and head h of the row at position p queries the code of residue p - d_h with
d_h = 64 ((h + p) mod H).  So it selects keys p - d_h, p - d_h - M, ... >= 0 (key 0 alone where p < d_h): the head with
d = 0 its own position, the one with d = M - 1 the keys p + 1 - M, ... so that key p + 1 carries a code the row selects,
and between them every 64 consecutive keys below p hold a selected key: every key tile of every row is covered.  A
head selects about 65536 / M keys: 33 at H = 32, 68 at H = 16, 146 at H = 8 (1024 tiles over 8 heads cannot stay below
128).  Up to 127 keys, one key more or fewer moves S / n by more than one bf16 spacing wherever S_d > 0.

Decode rows also select position 0, the last key of a deep page and the first key of the next, and their own position
plus one (the same head as their own position), by giving those keys the code a head of the row queries.  Decode rotates q
and the new key itself from the QKV planes with the engine's table: the planes hold the inverse rotation of the targets.
The new key's code is a pair of rotation partners (i, i + head_dim / 2), whose fp32 rotation lands within 1e-5 of A on
both and exactly 0 elsewhere, so the appended key is the code exactly; q codes of other pairs keep residues below 1e-4 in
the partner dims, far too small to change which keys score 2 A^2.

Every case also computes the references of wrong neighbours of the kernel and asserts that each fails the check in at
least one element: one selected key dropped, a deep tile read from the previous tile's page, the last tile dropped, the
prefix before pos0 ignored (prefill) and the causal bound at own position - 1 and + 1.

Decode also runs N(0, 1) operands through check_case's fp64 bound at up to 1024 tiles per split (rounding over 65536 keys
and the appends at deep positions; not addressing), and whole last tiles (RR_ATTN_NO_TRIM=1) against 16-row boxes, bit
for bit.  Engine level: a ~32000-token prompt at kv_splits 1 (512-entry tile table) against the reference model."""
import ctypes as C
import math

import pytest
import torch

from test_decode_attn_gpu import (KV_SPLITS, SHAPES, check_appends, check_output, default_path, kv_splits_rule,  # noqa: F401
                                  rope_table, rounding_check, rows_for)

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAGE = 64
A = 64.0
EXACT = 2.0 ** -21                    # relative slack of the fp32 roundings of 1 / l and o (1 / l)
POISON = 3e3


# ------------------------------------------------------------------------------------------------ selection operands
def period(H):
    return 64 * (H - 1) + 1


def code_table(hd):
    """[n, 2] dim pairs {a, b} of the codes of head dim hd; ids below hd / 2 are the rotation partners (i, i + hd / 2)."""
    half = hd // 2
    a, b = torch.triu_indices(hd, hd, 1)
    keep = b != a + half
    partner = torch.stack([torch.arange(half), torch.arange(half) + half], 1)
    return torch.cat([partner, torch.stack([a[keep], b[keep]], 1)])


def residue_codes(n_kv, H, hd, g, partner_at=None):
    """[n_kv, M] code ids of the residues mod M, distinct within a kv head and drawn from the non-partner pairs; residue
    partner_at gets a partner pair in every kv head."""
    half, n = hd // 2, len(code_table(hd))
    ids = torch.stack([half + torch.randperm(n - half, generator=g)[:period(H)] for _ in range(n_kv)])
    if partner_at is not None:
        ids[:, partner_at] = torch.randint(0, half, (n_kv,), generator=g)
    return ids


def starts(p, H):
    """[len(p), H]: the largest key each (row at position p, head) selects; the rest follow at steps of M."""
    d = 64 * ((torch.arange(H, device=p.device)[None, :] + p[:, None]) % H)
    s = p[:, None] - d
    return torch.where(s >= 0, s, torch.zeros_like(s))


def key_ids(res, n):
    """[n_kv, n] code id of every key: that of its residue."""
    return res[:, torch.arange(n, device=res.device) % res.shape[1]]


def query_ids(res, st, G):
    """[.., H] code id each (row, head) queries, from starts st [.., H]."""
    v = torch.arange(st.shape[-1], device=st.device) // G
    return res[v.expand_as(st), st % res.shape[1]]


def two_hot(ids, hd, table):
    """[.., 128] bf16 rows A (e_a + e_b) of the code ids."""
    x = torch.zeros(*ids.shape, 128, dtype=torch.bfloat16, device=ids.device)
    return x.scatter_(-1, table.to(ids.device)[ids], A)


def values(n_kv, n, hd, g):
    """[n_kv, n, 128] bf16 V of 0 / 1 in the true head dims, 0 in the padding."""
    v = torch.randint(0, 2, (n_kv, n, 128), generator=g, device=g.device).bfloat16()
    v[..., hd:] = 0
    return v


def progression_means(V, st, H, G):
    """S / n [rows, H, hd] of every (row, head) with starts st [rows, H], from the running sums of V [n_kv, n, hd] along
    steps of M (the selected keys of a start, without scanning the context)."""
    M = period(H)
    kv, n, hd = V.shape
    nb = -(-n // M)
    c = torch.zeros(kv, nb * M, hd, dtype=torch.float32, device=V.device)
    c[:, :n] = V.float()
    c = c.view(kv, nb, M, hd).cumsum(1).view(kv, nb * M, hd)
    v = (torch.arange(H, device=st.device) // G).expand_as(st)
    return c[v, st].double() / (st // M + 1)[..., None].double()


def masked_means(ids, V, q_ids, lo, hi, G):
    """(S / n [H, hd], n [H]) over keys lo..hi of one row, whatever their codes: ids [n_kv, n] code id of every key,
    V [n_kv, n, hd], q_ids [H]."""
    kv = ids.shape[0]
    mask = (ids[:, None, lo:hi + 1] == q_ids.view(kv, G)[:, :, None]).double()
    s = mask @ V[:, lo:hi + 1].double()
    cnt = mask.sum(-1)
    return (s / cnt[..., None]).reshape(kv * G, -1), cnt.flatten()


def exact_ok(out, ref):
    """Elementwise: out (bf16) is the bf16 rounding of a value within 2^-21 |ref| of ref, and exactly 0 where ref is."""
    ok = rounding_check(out, ref, EXACT * ref.abs())[0]
    return torch.where(ref == 0, out.double() == 0, ok)


def neighbours(ids, V, q_ids, p, G, pos0=0, tile=300):
    """{what: S / n [H, hd]} of the row at position p under the wrong neighbours of the kernel (keys 0..p, codes ids
    [n_kv, >= p + 2 or p + 1] and V of the row's context)."""
    n_have = ids.shape[1]
    out = {}
    ref, cnt = masked_means(ids, V, q_ids, 0, p, G)
    h = int(cnt.argmax())                                    # a head with a key to spare
    sel = (ids[h // G, :p + 1] == q_ids[h]).nonzero().flatten()
    ids2 = ids.clone()
    ids2[h // G, int(sel[len(sel) // 2])] = -1
    out["one selected key dropped"] = masked_means(ids2, V, q_ids, 0, p, G)[0]
    t = min(tile, p // PAGE - 1)
    ids2, V2 = ids.clone(), V.clone()
    ids2[:, t * PAGE:(t + 1) * PAGE] = ids[:, (t - 1) * PAGE:t * PAGE]
    V2[:, t * PAGE:(t + 1) * PAGE] = V[:, (t - 1) * PAGE:t * PAGE]
    out[f"tile {t} read from tile {t - 1}'s page"] = masked_means(ids2, V2, q_ids, 0, p, G)[0]
    out["last tile dropped"] = masked_means(ids, V, q_ids, 0, p // PAGE * PAGE - 1, G)[0]
    if pos0 > 0:
        out["prefix before pos0 ignored"] = masked_means(ids, V, q_ids, pos0, p, G)[0]
    out["causal bound at p - 1"] = masked_means(ids, V, q_ids, 0, p - 1, G)[0]
    if p + 1 < n_have:
        out["causal bound at p + 1"] = masked_means(ids, V, q_ids, 0, p + 1, G)[0]
    return ref, out


def assert_neighbours_fail(neigh_rows):
    """Every wrong neighbour fails the exact check on at least one element of at least one of the rows given as
    [(out [H, hd], {what: S / n})]."""
    whats = set().union(*(n.keys() for _, n in neigh_rows))
    for what in whats:
        assert any(not bool(exact_ok(o, n[what]).all()) for o, n in neigh_rows if what in n), \
            f"the check accepts the neighbour '{what}'"


# ------------------------------------------------------------------------------------------------ pool helpers
def make_pool(n_kv, ctx, pages_needed, extra, g):
    """Pool as test_paged_kv_gpu.Pool (pages by a random permutation, the sentinel elsewhere)."""
    from test_paged_kv_gpu import Pool
    return Pool(1, n_kv, ctx, pages_needed, extra, g)


def put_rows(pool_t, table, s, x):
    """Contiguous rows x [n_kv, n, 128] (n a multiple of 64) -> the first pages of slot s."""
    n_p = x.shape[1] // PAGE
    pages = table[s, :n_p].long().to(DEV)
    pool_t[0, pages] = x.view(x.shape[0], n_p, PAGE, 128).transpose(0, 1)


def slot_rows(pool_t, table, s, n):
    """The first n rows of slot s, [n_kv, n, 128]."""
    n_p = -(-n // PAGE)
    x = pool_t[0, table[s, :n_p].long().to(DEV)]
    return x.transpose(0, 1).reshape(x.shape[1], n_p * PAGE, 128)[:, :n]


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ decode
DEC_POS = (8191, 8192, 16383, 32767, 32768, 40037, 65471, 65472, 65534, 65535)
DEC_SHAPES = ("llama3-8b", "phi3-mini", "g8")
DEC_CASES = [pytest.param(n, 65536, ks, id=f"{n}-ctx65536-ks{ks}") for n in DEC_SHAPES for ks in KV_SPLITS]
DEC_CASES.append(pytest.param("llama3-8b", 8256, 1, id="llama3-8b-ctx8256-ks1"))     # 129 tiles: one past DEC_TBL


def decode_case(name, ctx, ks, family, seed):
    """Planes, pool, slots and positions of one decode case; family 'select' or 'normal'."""
    nh, nkv, hd, theta, _ = SHAPES[name]
    G = nh // nkv
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = rows_for(ks, nkv, sms)
    if rows is None:
        pytest.skip(f"kv_splits {ks} unreachable for {nkv} kv heads on {sms} SMs")
    assert kv_splits_rule(rows, nkv, sms) == ks
    g = torch.Generator().manual_seed(seed)
    gd = torch.Generator(device=DEV).manual_seed(seed)
    n_slots = rows + 3
    perm = torch.randperm(n_slots, generator=g).tolist()
    for r in range(n_slots):                                         # no row keeps its own index as slot
        if perm[r] == r:
            j = (r + 1) % n_slots
            perm[r], perm[j] = perm[j], perm[r]
    slot = perm[:rows]
    active = [r for r in range(rows) if r % 6 != 4]
    for r in range(rows):
        if r % 6 == 4:
            slot[r] = -1
    plist = sorted({p for p in DEC_POS if p < ctx} | {ctx - 2, ctx - 1})
    pos = [0] * rows
    for j, r in enumerate(active):
        if len(active) >= len(plist):
            pos[r] = plist[j % len(plist)]
        else:                                                        # few rows: spread over the list, both ends included
            pos[r] = plist[round(j * (len(plist) - 1) / max(len(active) - 1, 1))]
    need = [0] * n_slots
    for r in active:
        need[slot[r]] = -(-min(pos[r] + 2, ctx) // PAGE)                  # key pos + 1 too, where the context has it
    pool = make_pool(nkv, ctx, need, 7, g)
    nqkv = (nh + 2 * nkv) * hd
    ld = nqkv + 6
    n_splits = (1, 2, 3, 5)[KV_SPLITS.index(ks)]
    planes = torch.full((n_splits, rows + 1, ld), float("nan"), device=DEV)
    planes[:, :rows, :nqkv] = torch.randn(n_splits, rows, nqkv, device=DEV, generator=gd) / math.sqrt(n_splits)
    table = code_table(hd)
    sel = {}
    for r in active:
        s, p = slot[r], pos[r]
        m = need[s] * PAGE
        if family == "normal":
            def rows_of():
                x = torch.randn(nkv, m, 128, device=DEV, generator=gd)
                sign = torch.randint(0, 2, (nkv, m, 128), device=DEV, generator=gd).float() * 2 - 1
                poison = sign * (1e3 + 9e3 * torch.rand(nkv, m, 128, device=DEV, generator=gd))
                x[:, p:] = poison[:, p:]
                x[..., hd:] = poison[..., hd:]
                return x.bfloat16()
            put_rows(pool.k, pool.table, s, rows_of())
            put_rows(pool.v, pool.table, s, rows_of())
            continue
        res = residue_codes(nkv, nh, hd, g, partner_at=p % period(nh)).to(DEV)
        ids = key_ids(res, m)
        q_ids = query_ids(res, starts(torch.tensor([p], device=DEV), nh), G)[0]
        own = int(((torch.arange(nh) + p) % nh == 0).nonzero())
        # edge keys: position 0, the last key of a deep page and the first of the next, and pos + 1 with the own head
        t = max(1, p // PAGE // 2)
        for key, h in ((0, (own + 3) % nh), (t * PAGE - 1, (own + 5) % nh), (t * PAGE, (own + 5) % nh), (p + 1, own)):
            if key < m:
                ids[h // G, key] = q_ids[h]
        K = two_hot(ids, hd, table)
        V = values(nkv, m, hd, gd)
        kt, vt = K[:, p].clone(), V[:, p].clone()                          # what the call must append
        K[:, p] = POISON
        V[:, p] = POISON
        put_rows(pool.k, pool.table, s, K)
        put_rows(pool.v, pool.table, s, V)
        # planes: the inverse rotation of q and the new key at p, and the new v, split evenly over the planes
        c, sn = rope_table(torch.tensor([p], device=DEV), theta, hd)
        c, sn = c[0], sn[0]

        def unrotate(y):
            lo, hi = y[..., :hd // 2].double(), y[..., hd // 2:hd].double()
            return torch.cat([lo * c + hi * sn, hi * c - lo * sn], -1)
        x = torch.cat([unrotate(two_hot(q_ids, hd, table)).flatten(), unrotate(kt).flatten(), vt[:, :hd].double().flatten()])
        planes[:, r, :nqkv] = (x / n_splits).float()
        sel[r] = dict(ids=ids, q_ids=q_ids, kt=kt, vt=vt)
    cs = dict(shape=(nh, nkv, hd, theta, ctx), rows=rows, n_splits=n_splits, ld=ld, planes=planes, n_slots=n_slots,
              slot=torch.tensor(slot, device=DEV, dtype=torch.int32), pos=torch.tensor(pos, device=DEV, dtype=torch.int32),
              active=active, out_len=rows * nh * hd, slack=nh * hd + 64, pool=pool, sel=sel)
    return cs


def run_decode(cs, k, v):
    """One call of rr_op_decode_attn_qkv_paged on pool tensors k / v (modified in place); returns (out_flat, kv_splits)."""
    from rr_b200 import _lib
    nh, nkv, hd, theta, ctx = cs["shape"]
    pool = cs["pool"]
    out = torch.full((cs["out_len"] + cs["slack"],), float("nan"), device=DEV, dtype=torch.bfloat16)
    ks = C.c_int32(-1)
    p = cs["planes"]
    P = lambda t: C.c_void_p(t.data_ptr())                                       # noqa: E731
    _lib.check(_lib.lib.rr_op_decode_attn_qkv_paged(
        P(p), cs["n_splits"], p.stride(0), cs["ld"], P(k), P(v), P(out), P(cs["slot"]), P(cs["pos"]), cs["rows"], nh, nkv, hd,
        ctx, cs["n_slots"], theta, C.byref(ks), P(pool.dtable), pool.pps, pool.n_pages, None), "decode_attn_qkv_paged")
    torch.cuda.synchronize()
    return out, ks.value


def appended(cs, t):
    """[active rows, n_kv, head_dim] the rows at each active row's pos in pool tensor t, and their (page, in-page) index."""
    hd = cs["shape"][2]
    tab = cs["pool"].table
    at = [(int(tab[int(cs["slot"][r]), int(cs["pos"][r]) // PAGE]), int(cs["pos"][r]) % PAGE) for r in cs["active"]]
    pg = torch.tensor([a for a, _ in at], device=DEV)
    ro = torch.tensor([b for _, b in at], device=DEV)
    return t[0, pg, :, ro, :hd], (pg, ro)


def check_untouched(cs, before, after, what):
    """after differs from before at most in the appended rows (restored in after and put back once compared)."""
    hd = cs["shape"][2]
    new, (pg, ro) = appended(cs, after)
    new = new.clone()
    after[0, pg, :, ro, :hd] = before[0, pg, :, ro, :hd]
    assert torch.equal(_bits(after), _bits(before)), f"{what} pool written outside row pos"
    after[0, pg, :, ro, :hd] = new


@pytest.mark.parametrize("name,ctx,ks", DEC_CASES)
def test_decode_selection_deep_is_exact(name, ctx, ks, default_path):
    cs = decode_case(name, ctx, ks, "select", seed=7 * ctx + 31 * ks + len(name))
    nh, nkv, hd, _, _ = cs["shape"]
    G = nh // nkv
    pool = cs["pool"]
    k0, v0 = pool.k.clone(), pool.v.clone()
    out, ks_got = run_decode(cs, pool.k, pool.v)
    assert ks_got == ks
    act = cs["active"]
    k_new, _ = appended(cs, pool.k)
    v_new, _ = appended(cs, pool.v)
    # by value: the rotation may leave -0 where the code is 0
    assert torch.equal(k_new.float(), torch.stack([cs["sel"][r]["kt"][:, :hd] for r in act]).float()), "appended k != code"
    assert torch.equal(_bits(v_new), _bits(torch.stack([cs["sel"][r]["vt"][:, :hd] for r in act]))), "appended v differs"
    check_appends(cs, k_new, v_new)
    check_untouched(cs, k0, pool.k, "k")
    check_untouched(cs, v0, pool.v, "v")
    o = out[:cs["out_len"]].view(cs["rows"], nh, hd)
    inactive = [r for r in range(cs["rows"]) if r not in set(act)]
    assert torch.isnan(o[inactive]).all() and torch.isnan(out[cs["out_len"]:]).all()
    deepest = max(act, key=lambda r: int(cs["pos"][r]))
    checked = []
    for r in act:
        s, p, sl = int(cs["slot"][r]), int(cs["pos"][r]), cs["sel"][r]
        m = sl["ids"].shape[1]
        V = slot_rows(pool.v, pool.table, s, m)[..., :hd]
        ref, cnt = masked_means(sl["ids"], V, sl["q_ids"], 0, p, G)
        assert 1 <= cnt.min() and cnt.max() <= 127, (r, p, cnt.tolist())
        ok = exact_ok(o[r], ref)
        assert ok.all(), f"row {r} (pos {p}): {int((~ok).sum())} elements off, first (head, dim) {(~ok).nonzero()[0].tolist()}"
        if r == deepest or p in (ctx - 2, 8192, 40037):
            checked.append((o[r], neighbours(sl["ids"], V, sl["q_ids"], p, G)[1]))
    assert_neighbours_fail(checked)
    # whole last tiles against 16-row boxes: the same bits, in the output and the pool
    default_path.setenv("RR_ATTN_NO_TRIM", "1")
    out2, _ = run_decode(cs, k0, v0)
    assert torch.equal(_bits(out2), _bits(out)), "RR_ATTN_NO_TRIM=1 changes the output"
    assert torch.equal(_bits(k0), _bits(pool.k)) and torch.equal(_bits(v0), _bits(pool.v)), "RR_ATTN_NO_TRIM=1 changes the pool"


@pytest.mark.parametrize("name,ctx,ks", DEC_CASES)
def test_decode_normal_operands_deep_within_the_fp64_bound(name, ctx, ks, default_path):
    """check_case's appends and fp64 bound on N(0, 1) operands, up to 1024 tiles per split and pos 65535."""
    cs = decode_case(name, ctx, ks, "normal", seed=11 * ctx + 17 * ks + len(name))
    hd = cs["shape"][2]
    pool = cs["pool"]
    k0, v0 = pool.k.clone(), pool.v.clone()
    out, ks_got = run_decode(cs, pool.k, pool.v)
    assert ks_got == ks
    k_new, _ = appended(cs, pool.k)
    v_new, _ = appended(cs, pool.v)
    check_appends(cs, k_new, v_new)
    check_untouched(cs, k0, pool.k, "k")
    check_untouched(cs, v0, pool.v, "v")
    del k0, v0
    check_output(cs, ks, out, lambda s, n: (slot_rows(pool.k, pool.table, s, n)[..., :hd],
                                            slot_rows(pool.v, pool.table, s, n)[..., :hd]))


# ------------------------------------------------------------------------------------------------ prefill
# (pos0, len): a piece from 0, a partial last query tile, a prefix-cache offset that is not tile-aligned, a piece ending
# at 65535 and one row at 65535
PF_SEQS = [(0, 8192), (8192, 8155), (24576, 8192), (40037, 8192), (57344, 8192), (65535, 1)]


def prefill_sequence(H, KV, n_keys, g, gd):
    """Selection operands of one prefill sequence: residue codes, K and V [KV, n_keys, 128] (g a CPU generator, gd one
    on the device the operands go to)."""
    res = residue_codes(KV, H, 128, g).to(gd.device)
    K = two_hot(key_ids(res, n_keys), 128, code_table(128))
    return res, K, values(KV, n_keys, 128, gd)


def prefill_queries(res, p, H, G):
    """q rows [len(p), H * 128] of the rows at positions p."""
    return two_hot(query_ids(res, starts(p, H), G), 128, code_table(128)).view(len(p), H * 128)


def check_prefill_rows(out, res, V, p, H, G):
    """Every row at positions p (out [len(p), H * 128]) against its exact S / n."""
    ref = progression_means(V, starts(p, H), H, G)
    ok = exact_ok(out.view(len(p), H, 128), ref)
    bad = (~ok).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} elements off, first (row, head, dim) {bad[0].tolist()}"


@pytest.mark.parametrize("H,KV", [(32, 8), (16, 2), (8, 8)])
def test_prefill_selection_deep_is_exact(H, KV):
    from rr_b200 import _lib
    G, ctx = H // KV, 65536
    gd = torch.Generator(device=DEV).manual_seed(100 * H + KV)
    g = torch.Generator().manual_seed(100 * H + KV)
    n = len(PF_SEQS)
    keys = [min(p0 + ln + 1, ctx) for p0, ln in PF_SEQS]                  # key pos + 1 of the last row too
    need = [-(-m // PAGE) for m in keys]
    slots = torch.randperm(n, generator=g).tolist()                      # sequence i -> slot slots[i]
    pool = make_pool(KV, ctx, [need[slots.index(s)] for s in range(n)], 9, g)
    seqs, qs = [], []
    for i, (p0, ln) in enumerate(PF_SEQS):
        m = need[i] * PAGE
        res, K, V = prefill_sequence(H, KV, m, g, gd)
        put_rows(pool.k, pool.table, slots[i], K)
        put_rows(pool.v, pool.table, slots[i], V)
        p = torch.arange(p0, p0 + ln, device=DEV)
        qs.append(prefill_queries(res, p, H, G))
        seqs.append((res, V, p))
        del K
    q = torch.cat(qs)
    del qs
    lens = [ln for _, ln in PF_SEQS]
    start = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), device=DEV, dtype=torch.int32)
    sl = torch.tensor(slots, device=DEV, dtype=torch.int32)
    dp0 = torch.tensor([p0 for p0, _ in PF_SEQS], device=DEV, dtype=torch.int32)
    out = torch.full_like(q, float("nan"))
    P = lambda t: C.c_void_p(t.data_ptr())                                       # noqa: E731
    _lib.check(_lib.lib.rr_op_prefill_attn_cached_paged(P(q), P(pool.k), P(pool.v), P(out), P(start), P(sl), P(dp0), n,
                                                        max(lens), H, KV, ctx, 1 / math.sqrt(128), P(pool.dtable), pool.pps,
                                                        pool.n_pages, None), "prefill_attn_cached_paged")
    torch.cuda.synchronize()
    st = start.tolist()
    checked = []
    for i, ((p0, ln), (res, V, p)) in enumerate(zip(PF_SEQS, seqs)):
        got = out[st[i]:st[i + 1]]
        check_prefill_rows(got, res, V, p, H, G)
        ids = key_ids(res, V.shape[1])
        for r in {ln - 1, ln - 2, ln // 2} - {-1}:                        # neighbours: deep rows of every sequence
            if p0 + r < 2 * PAGE:
                continue
            q_ids = query_ids(res, starts(p[r:r + 1], H), G)[0]
            ref, neigh = neighbours(ids, V, q_ids, p0 + r, G, pos0=p0)
            assert torch.equal(ref, progression_means(V, starts(p[r:r + 1], H), H, G)[0]), "progression != codes"
            checked.append((got[r].view(H, 128), neigh))
    assert_neighbours_fail(checked)


# ------------------------------------------------------------------------------------------------ engine
def test_engine_long_prompt_at_kv_splits_1_matches_the_oracle():
    """The smallest batch the split rule runs at kv_splits 1 on this device (132 rows on 132 SMs): every decode CTA
    covers a whole row, 512 tiles at ctx_max 32768, so the decode kernel's tile table is four times DEC_TBL."""
    from oracle import llama_ref
    from rr_b200 import SPECS, make_weights
    from rr_b200.engine import Engine
    import numpy as np
    spec = SPECS["tiny"]
    w = make_weights(spec, seed=13, sigma=0.05, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = rows_for(1, spec.n_kv_heads, sms)
    assert kv_splits_rule(rows, spec.n_kv_heads, sms) == 1
    eng = Engine(w, max_batch=rows, ctx_max=32768, max_prefill_tokens=8192, kv_cache_tokens=32768 + 4096,
                 use_cuda_graph=True)
    rng = np.random.RandomState(21)
    try:
        p = rng.randint(3, spec.vocab, size=32000).tolist()
        shorts = [rng.randint(3, spec.vocab, size=n).tolist() for n in (40, 300, 700)]
        tk = [eng.submit(p, 3)] + [eng.submit(s, 4) for s in shorts]
        recs = [eng.wait(t, timeout=600) for t in tk]
        assert all(r.status == 0 for r in recs)
    finally:
        eng.close()
    seq = list(p)
    with torch.no_grad():
        for t in recs[0].tokens[:2]:                      # the second comes from a decode step over 32001 keys
            assert t == int(llama_ref.forward_logits(w, seq)[-1].argmax())        # fp32 on the GPU
            seq.append(t)
            torch.cuda.empty_cache()
