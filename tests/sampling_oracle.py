"""CPU restatement of the sampling contract (rr_op_sample, include/rr_b200.h), in numpy: Philox4x32-10 in integer
arithmetic, the top-p nucleus and the Gumbel noise in fp64.  Used by tests/test_sampling_cpu.py and
tests/test_sampling_gpu.py; nothing here runs on the product path.

For fp32 logits x of one row, temperature T > 0, top_p and a 64-bit seed, the token at `position` is

    tau = the largest logit value v with  sum_{x_j >= v} exp((x_j - m) / T)  >=  top_p * sum_j exp((x_j - m) / T)
          (top_p >= 1: every token),
    token = argmax over {i : x_i >= tau} of x_i / T + G_i   (ties to the lowest id),
    G_i = -log(-log u_i),  u_i = (2 (r_i >> 9) + 1) / 2^24,
    r_i = word 0 of Philox4x32-10(counter = (i, position, 0, 0), key = (seed mod 2^32, seed >> 32)).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(c0, c1, c2, c3, k0: int, k1: int):
    """Philox4x32-10 (Salmon et al., SC'11) on arrays of 32-bit counters -> the four output words (uint64 arrays)."""
    c = [np.asarray(v, dtype=np.uint64) & _MASK for v in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c = [v.copy() for v in c]
    k0, k1 = k0 & _MASK, k1 & _MASK
    for _ in range(10):
        p0 = c[0] * np.uint64(_M0)
        p1 = c[2] * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return c


def random_words(seed: int, position: int, n: int) -> np.ndarray:
    """r_i for token ids 0..n-1 (uint64 holding 32-bit words)."""
    seed %= 2**64
    ids = np.arange(n, dtype=np.uint64)
    return philox4x32_10(ids, position, 0, 0, seed & _MASK, seed >> 32)[0]


def uniforms(seed: int, position: int, n: int) -> np.ndarray:
    """u_i, exact in fp64 (and in fp32): odd multiples of 2^-24."""
    r = random_words(seed, position, n)
    return ((r >> np.uint64(9)) * np.uint64(2) + np.uint64(1)).astype(np.float64) / 2.0**24


def gumbel(seed: int, position: int, n: int) -> np.ndarray:
    return -np.log(-np.log(uniforms(seed, position, n)))


def mass_profile(x: np.ndarray, T: float):
    """Distinct logit values in descending order and F(v) / Z at each: the share of softmax(x / T) on {x >= v}."""
    x = np.asarray(x, dtype=np.float64)
    w = np.exp((x - x.max()) / T)
    vals, inv = np.unique(x, return_inverse=True)
    mass = np.bincount(inv, weights=w)[::-1]
    return vals[::-1], np.cumsum(mass) / w.sum()


def threshold(x: np.ndarray, T: float, top_p: float, slack: float = 0.0) -> float:
    """tau of the contract, computed as if every nucleus mass were `slack` lower (slack < 0: higher).  -inf for
    top_p >= 1."""
    if top_p >= 1.0:
        return -np.inf
    vals, frac = mass_profile(x, T)
    k = int(np.searchsorted(frac - slack, np.float64(np.float32(top_p)), side="left"))
    return float(vals[min(k, len(vals) - 1)])


@dataclass
class Draw:
    token: int
    tau: float
    nucleus_size: int
    scores: np.ndarray          # x / T + G over the vocabulary, -inf outside the nucleus
    stable_nucleus: bool        # the winner is the same for every tau a mass error of `mass_slack` could give
    score_gap: float            # best minus second-best score over the largest such nucleus (inf: one token)
    score_bound: float          # fp32 error bound on a score difference (see tests/test_sampling_gpu.py)


def sample(x: np.ndarray, T: float, top_p: float, seed: int, position: int, mass_slack: float = 0.0) -> Draw:
    """The contract's token for one row, with what a test needs to tell a clear draw from a near tie."""
    x = np.asarray(x, dtype=np.float32)
    x64 = x.astype(np.float64)
    T = float(np.float32(T))
    tau = threshold(x, T, top_p)
    g = gumbel(seed, position, len(x))
    s_all = x64 / T + g
    scores = np.where(x64 >= tau, s_all, -np.inf)
    token = int(np.argmax(scores))
    # the GPU's tau lies between the oracle's under masses moved by -slack and +slack
    tau_lo, tau_hi = threshold(x, T, top_p, -mass_slack), threshold(x, T, top_p, mass_slack)
    wide = np.where(x64 >= min(tau_lo, tau_hi), s_all, -np.inf)
    w_tok = int(np.argmax(wide))
    stable = x64[w_tok] >= max(tau_lo, tau_hi) and w_tok == token
    order = np.argsort(-wide, kind="stable")
    gap = np.inf if not np.isfinite(wide[order[1]]) else float(wide[order[0]] - wide[order[1]])
    err = lambda i: 2.0**-22 * (1.0 + abs(g[i]) + abs(x64[i] / T) + abs(s_all[i]))
    bound = err(order[0]) + err(order[1])
    return Draw(token, tau, int((x64 >= tau).sum()), scores, bool(stable), gap, float(bound))
