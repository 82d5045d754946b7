"""The JSON-mode contract (response_format json_object) in plain Python: the byte automaton that rr_op_json_mask /
rr_op_json_advance run on the GPU, written out independently of the kernel.

A state accepts exactly the prefixes of JSON texts (RFC 8259) whose top-level value is an object, with strict UTF-8 in
strings (no overlongs, no UTF-8-encoded surrogates, nothing above U+10FFFF), no raw bytes < 0x20 in strings, at most
MAX_DEPTH open containers and whitespace runs of at most MAX_WS bytes.  After the closing '}' only whitespace follows.

    initial() -> state;  allowed(state) -> set of bytes;  advance(state, byte) -> state (ValueError if not allowed);
    done(state) -> the top-level object is closed;  completion(state) -> bytes that finish the text.

Token t >= 3 of the byte tokenizer is the byte (t - 3) % 256; tokens 0..2 are never allowed (mask_row)."""
from __future__ import annotations

from typing import NamedTuple, Optional, Set

MAX_DEPTH = 64
MAX_WS = 64
WS = frozenset(b" \t\n\r")
DIGITS = frozenset(b"0123456789")
HEX = frozenset(b"0123456789abcdefABCDEF")
ESCAPES = frozenset(b'"\\/bfnrt')
LITERALS = (b"true", b"false", b"null")


class State(NamedTuple):
    node: str                  # see advance()
    stack: tuple = ()          # open containers, outermost first: "{" or "["
    ws: int = 0                # current run of insignificant whitespace
    key: bool = False          # the string being read is an object key
    lit: bytes = b""           # literal bytes still due
    hex: int = 0               # \u hex digits still due
    utf8: tuple = ()           # (bytes due, lo, hi) of a multi-byte character


def initial() -> State:
    return State("start")


def done(s: State) -> bool:
    return s.node == "done"


def _value_start(s: State, c: int) -> Optional[State]:
    if c in b"{[":
        if len(s.stack) >= MAX_DEPTH:
            return None
        return s._replace(node="obj_first" if c == ord("{") else "arr_first", stack=s.stack + (chr(c),), ws=0)
    if c == ord('"'):
        return s._replace(node="str", key=False, ws=0)
    if c == ord("-"):
        return s._replace(node="minus", ws=0)
    if c == ord("0"):
        return s._replace(node="zero", ws=0)
    if c in DIGITS:
        return s._replace(node="int", ws=0)
    for lit in LITERALS:
        if c == lit[0]:
            return s._replace(node="lit", lit=lit[1:], ws=0)
    return None


def _close(s: State) -> State:
    stack = s.stack[:-1]
    return s._replace(node="after" if stack else "done", stack=stack, ws=0)


def _structural(s: State, c: int) -> Optional[State]:
    if c in WS:
        return s._replace(ws=s.ws + 1) if s.ws < MAX_WS else None
    top = s.stack[-1] if s.stack else None
    n = s.node
    if n == "start":
        return s._replace(node="obj_first", stack=("{",), ws=0) if c == ord("{") else None
    if n in ("obj_first", "obj_key"):
        if c == ord('"'):
            return s._replace(node="str", key=True, ws=0)
        if c == ord("}") and n == "obj_first":
            return _close(s)
        return None
    if n == "colon":
        return s._replace(node="value", ws=0) if c == ord(":") else None
    if n == "after":
        if c == ord(","):
            return s._replace(node="value" if top == "[" else "obj_key", ws=0)
        if (c == ord("}") and top == "{") or (c == ord("]") and top == "["):
            return _close(s)
        return None
    if n == "arr_first" and c == ord("]"):
        return _close(s)
    return _value_start(s, c)          # value, arr_first


def step(s: State, c: int) -> Optional[State]:
    """The state after byte c, or None when c is not allowed."""
    n = s.node
    if n == "done":
        return s if c in WS else None
    if n == "minus":
        return s._replace(node="zero" if c == ord("0") else "int") if c in DIGITS else None
    if n in ("zero", "int", "frac", "exp_dig"):
        if c in DIGITS and n != "zero":
            return s
        if c == ord(".") and n in ("zero", "int"):
            return s._replace(node="dot")
        if c in b"eE" and n in ("zero", "int", "frac"):
            return s._replace(node="exp")
        return _structural(s._replace(node="after"), c)     # the byte ends the number
    if n == "dot":
        return s._replace(node="frac") if c in DIGITS else None
    if n == "exp":
        if c in b"+-":
            return s._replace(node="exp_sign")
        return s._replace(node="exp_dig") if c in DIGITS else None
    if n == "exp_sign":
        return s._replace(node="exp_dig") if c in DIGITS else None
    if n == "str":
        if c == ord('"'):
            return s._replace(node="colon" if s.key else "after", key=False)
        if c == ord("\\"):
            return s._replace(node="esc")
        if 0x20 <= c < 0x80:
            return s
        if 0xC2 <= c <= 0xDF:
            return s._replace(node="utf8", utf8=(1, 0x80, 0xBF))
        if 0xE0 <= c <= 0xEF:
            lo, hi = (0xA0 if c == 0xE0 else 0x80), (0x9F if c == 0xED else 0xBF)
            return s._replace(node="utf8", utf8=(2, lo, hi))
        if 0xF0 <= c <= 0xF4:
            lo, hi = (0x90 if c == 0xF0 else 0x80), (0x8F if c == 0xF4 else 0xBF)
            return s._replace(node="utf8", utf8=(3, lo, hi))
        return None
    if n == "utf8":
        due, lo, hi = s.utf8
        if not lo <= c <= hi:
            return None
        return s._replace(node="str", utf8=()) if due == 1 else s._replace(utf8=(due - 1, 0x80, 0xBF))
    if n == "esc":
        if c in ESCAPES:
            return s._replace(node="str")
        return s._replace(node="hex", hex=4) if c == ord("u") else None
    if n == "hex":
        if c not in HEX:
            return None
        return s._replace(node="str", hex=0) if s.hex == 1 else s._replace(hex=s.hex - 1)
    if n == "lit":
        if c != s.lit[0]:
            return None
        return s._replace(node="after", lit=b"") if len(s.lit) == 1 else s._replace(lit=s.lit[1:])
    return _structural(s, c)


def allowed(s: State) -> Set[int]:
    return {c for c in range(256) if step(s, c) is not None}


def advance(s: State, c: int) -> State:
    t = step(s, c)
    if t is None:
        raise ValueError(f"byte {c:#04x} is not allowed in state {s}")
    return t


def accepts(data: bytes, s: Optional[State] = None):
    """-> (state after the longest accepted prefix, its length)."""
    s = initial() if s is None else s
    for i, c in enumerate(data):
        t = step(s, c)
        if t is None:
            return s, i
        s = t
    return s, len(data)


_PREFER = b'"}]:0{'


def completion(s: State) -> bytes:
    """Bytes that take s to done: at every step the first allowed byte of '"', '}', ']', ':', '0', '{', then the lowest
    allowed byte.  Each choice closes a string, a number, a literal or a container, or opens nothing new, so it ends."""
    out = bytearray()
    while not done(s):
        c = next((b for b in _PREFER if step(s, b) is not None), None)
        if c is None:
            a = allowed(s)
            c = min(a - WS) if a - WS else min(a)
        out.append(c)
        s = advance(s, c)
    return bytes(out)


def _rand_str(rng):
    pool = ["a", "Z", " ", "\"", "\\", "/", "\n", "\t", "\x00", "\x1f", "\x7f", "é", "ß", "ࠀ", "￿", "中",
            "\U0001f600", "\U0010ffff", " ", "{", "]", ":", ","]
    return "".join(rng.choice(pool) for _ in range(rng.randint(0, 8)))


def _rand_value(rng, depth):
    k = rng.randint(0, 9 if depth < 5 else 6)
    if k == 0:
        return rng.randint(-10**12, 10**12)
    if k == 1:
        return rng.choice([0.0, -0.0, 1.5, -2.25e-7, 3e+21, 1e300, 123456.789])
    if k == 2:
        return rng.choice([True, False, None])
    if k in (3, 4, 5, 6):
        return _rand_str(rng)
    if k in (7, 8):
        return [_rand_value(rng, depth + 1) for _ in range(rng.randint(0, 4))]
    return _rand_obj(rng, depth + 1)


def _rand_obj(rng, depth=0):
    return {_rand_str(rng): _rand_value(rng, depth) for _ in range(rng.randint(0, 4))}


def random_docs(n: int, seed: int):
    """n seeded json.dumps texts of random nested objects (escapes, exponents, non-ASCII, astral characters), cycling
    through ensure_ascii on / off, indent 2 / tab (whitespace runs well inside MAX_WS) and compact separators."""
    import json
    import random
    rng = random.Random(seed)
    out = []
    for i in range(n):
        kw = [{}, {"ensure_ascii": False}, {"indent": 2}, {"indent": "\t", "ensure_ascii": False},
              {"separators": (",", ":")}][i % 5]
        out.append(json.dumps(_rand_obj(rng), allow_nan=False, **kw).encode("utf-8"))
    return out


def token_byte(t: int) -> Optional[int]:
    return (t - 3) % 256 if t >= 3 else None


def mask_columns(s: State, vocab: int):
    """The columns rr_op_json_mask sets to -inf for a row in state s: a boolean list of length vocab (True: masked)."""
    a = allowed(s)
    return [c < 3 or ((c - 3) % 256) not in a for c in range(vocab)]
