"""numpy float32 oracle of the penalties / logit-bias contract (rr_op_logit_penalties, include/rr_b200.h §3).

Per row, with c_j the number of times token j occurs in the row's history (its generated tokens) and b_j its bias:
    x'_j = (x_j + b_j) - (c_j * frequency_penalty + [c_j > 0] * presence_penalty)
every operation one float32 round-to-nearest op.  A token without a bias entry skips the addition, one with c_j = 0 the
subtraction; a row with both penalties 0 and no bias entries is left as it is.  numpy's float32 scalar arithmetic rounds
each operation on its own (no FMA contraction), so this reproduces the kernel bit for bit.
"""
from typing import Mapping, Optional, Sequence

import numpy as np


def apply_row(x: np.ndarray, history: Sequence[int] = (), frequency_penalty: float = 0.0, presence_penalty: float = 0.0,
              bias: Optional[Mapping[int, float]] = None) -> np.ndarray:
    """One row of float32 logits -> the processed row (a copy)."""
    y = np.array(x, dtype=np.float32, copy=True)
    af, ap = np.float32(frequency_penalty), np.float32(presence_penalty)
    bias = bias or {}
    if af == 0 and ap == 0 and not bias:
        return y
    for j, b in bias.items():
        y[j] = np.float32(y[j] + np.float32(b))
    if af == 0 and ap == 0:
        return y
    h = np.asarray(history, dtype=np.int64)
    h = h[(h >= 0) & (h < len(y))]
    ids, cnt = np.unique(h, return_counts=True)
    # vectorised, still one float32 rounding per op: c * af, then + ap, then x - that
    pen = (cnt.astype(np.float32) * af).astype(np.float32)
    pen = (pen + ap).astype(np.float32)
    y[ids] = (y[ids] - pen).astype(np.float32)
    return y


def apply(logits: np.ndarray, histories, frequency_penalty, presence_penalty, biases) -> np.ndarray:
    """[rows][vocab] float32 -> processed copy; per-row lists of histories, penalties and bias maps."""
    out = np.array(logits, dtype=np.float32, copy=True)
    for r in range(out.shape[0]):
        out[r] = apply_row(out[r], histories[r], frequency_penalty[r], presence_penalty[r], biases[r])
    return out
