"""Pure-Python statement of the stop-sequence contract (rr_op_stop_match, rr_gen_params.n_stop), for the tests.

The reply text of a token list is what `detokenize` makes of it before decoding: a token t >= 3 is the byte (t - 3) % 256,
a token < 3 is no text.  Stop sequences are byte strings matched on that text."""
from typing import List, Sequence, Tuple


def _text(tokens: Sequence[int]) -> Tuple[bytes, List[int]]:
    """(the text, the index of the token each byte came from)."""
    idx = [i for i, t in enumerate(tokens) if t >= 3]
    return bytes((tokens[i] - 3) % 256 for i in idx), idx


def stop_state(tokens: Sequence[int], stops: Sequence[bytes]) -> Tuple[int, int]:
    """(cut, hold) once the last of `tokens` has been generated.

    cut: -1, or, when the last token has a byte and the text now ends in a stop sequence, the index of the first token of
    the longest such sequence: the tokens before it are kept, byteless ones included.
    hold: 0 on a hit; else the number of newest tokens counted from the first token of the longest suffix of the text that
    is a proper prefix of a stop sequence (0 when there is none).  They may turn out to belong to a stop sequence."""
    text, idx = _text(tokens)
    if tokens and tokens[-1] >= 3:
        hits = [len(s) for s in stops if s and text.endswith(s)]
        if hits:
            return idx[len(text) - max(hits)], 0
    part = max((k for s in stops for k in range(1, min(len(s) - 1, len(text)) + 1) if text[len(text) - k:] == s[:k]),
               default=0)
    return -1, (len(tokens) - idx[len(text) - part] if part else 0)


def stop_scan(tokens: Sequence[int], stops: Sequence[bytes]) -> List[Tuple[int, int]]:
    """stop_state after each token.  Every entry is a function of the tokens up to it alone: the scan does not end at the
    first hit (a choice does; see stop_cut)."""
    return [stop_state(tokens[: i + 1], stops) for i in range(len(tokens))]


def stop_cut(tokens: Sequence[int], stops: Sequence[bytes]) -> Tuple[int, bool]:
    """(tokens kept, finished by a stop sequence) of a reply that would be `tokens` without stop sequences."""
    for i in range(len(tokens)):
        cut, _ = stop_state(tokens[: i + 1], stops)
        if cut >= 0:
            return cut, True
    return len(tokens), False


def visible(tokens: Sequence[int], stops: Sequence[bytes]) -> List[int]:
    """Tokens a streaming reader may have been shown after each token of a running choice: those generated less hold."""
    return [i + 1 - h for i, (_, h) in enumerate(stop_scan(tokens, stops))]
