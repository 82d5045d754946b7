"""Host-side mirror of the reference's router interface.

`Router(model_list=..., routing_strategy=..., enable_pre_call_checks=..., allowed_fails=...,
cooldown_time=..., fallbacks=...)` takes the same arguments the reference's gateway builds
`litellm.Router` from (reference config/config.yaml:35-108, launched by bin/start-gateway.sh:54);
`Router.completion(model=, messages=, timeout=)` / `client.chat.completions.create(...)` is the call
the demos make (reference src/demo_load_balancing.py:106-110, src/demo_fallback.py:143-147,
src/demo_quota_isolation.py:52-56), the result exposes `.model` the way they read it (:116), and a
rate-limited request raises `RateLimitError` (HTTP 429; src/demo_quota_isolation.py:80).

All routing state and decisions live in the CUDA library (K1, rr_router.cu), and the whole request lifecycle in its
native gateway (rr_gateway.cu): admission, hand-off to the per-GPU engines or to mock replicas, DONE / FAIL reports and
the fallback walk.  This file validates requests, submits them to the gateway and shapes its results as OpenAI
responses.  There is no Python/CPU implementation of the routing logic or the request lifecycle on this path
(`Router.process` hands event records to K1 directly, for benchmarks and parity tests).
"""
from __future__ import annotations

import base64
import codecs
import ctypes as C
import math
import re
import secrets
import threading
import time
import uuid
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .config import RouterConfig, build_config, load_config
from .models import ring_pages


# ---------------------------------------------------------------- errors (OpenAI-SDK names)
class APIError(Exception):
    status_code = 500

    def __init__(self, message: str, status_code: Optional[int] = None):
        super().__init__(message)
        self.message = message
        if status_code is not None:
            self.status_code = status_code


class RateLimitError(APIError):
    status_code = 429


class BadRequestError(APIError):
    status_code = 400


class APITimeoutError(APIError):
    status_code = 408


class ServiceUnavailableError(APIError):
    status_code = 503


# ---------------------------------------------------------------- response objects
@dataclass
class Message:
    role: str
    content: str


@dataclass
class Choice:
    index: int
    message: Message
    finish_reason: str = "length"
    logprobs: Optional[dict] = None      # OpenAI ChoiceLogprobs {"content": [...], "refusal": None}; only when requested


@dataclass
class Usage:
    prompt_tokens: int
    completion_tokens: int
    total_tokens: int
    # {"cached_tokens": n}: responses of deployments with litellm_params.prefix_cache only (OpenAI's usage shape)
    prompt_tokens_details: Optional[dict] = None


@dataclass
class ModelResponse:
    id: str
    model: str
    choices: List[Choice]
    usage: Usage
    created: int = 0
    object: str = "chat.completion"
    # extras (underscore = not part of the OpenAI shape)
    _token_ids: List[int] = field(default_factory=list)
    _deployment: int = -1
    _model_group: str = ""
    _fell_back: bool = False
    _ttft_s: float = 0.0
    _latency_s: float = 0.0
    _choice_token_ids: List[List[int]] = field(default_factory=list)     # every choice's tokens, choices[i] <-> [i]

    def model_dump(self) -> dict:
        return {"id": self.id, "object": self.object, "created": self.created, "model": self.model,
                "choices": [dict({"index": c.index, "finish_reason": c.finish_reason,
                                  "message": {"role": c.message.role, "content": c.message.content}},
                                 **({} if c.logprobs is None else {"logprobs": c.logprobs}))
                            for c in self.choices],
                "usage": dict({"prompt_tokens": self.usage.prompt_tokens,
                               "completion_tokens": self.usage.completion_tokens,
                               "total_tokens": self.usage.total_tokens},
                              **({} if self.usage.prompt_tokens_details is None
                                 else {"prompt_tokens_details": self.usage.prompt_tokens_details}))}


# ---------------------------------------------------------------- tokenizer (byte level, CUDA kernel K2 in the library)
def tokenize_batch(texts: Sequence[str], vocab: int):
    """Token ids and counts of a batch of messages in ONE launch of the tokenizer kernel (csrc/rr_tokenizer.cu).
    -> (list of int32 arrays, counts int32[n])."""
    raw = [t.encode("utf-8") for t in texts]
    n = len(raw)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(b) for b in raw], out=off[1:])
    blob = b"".join(raw)
    counts = np.zeros(n, dtype=np.int32)
    ids = np.zeros(int(off[-1]) + n, dtype=np.int32)
    ids_off = np.zeros(n + 1, dtype=np.int64)
    _lib.check(_lib.lib.rr_tokenize_batch(blob, off.ctypes.data_as(C.POINTER(C.c_int64)), n, vocab,
                                          counts.ctypes.data_as(C.POINTER(C.c_int32)), ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                          len(ids), ids_off.ctypes.data_as(C.POINTER(C.c_int64))), "rr_tokenize_batch")
    return [ids[ids_off[i]: ids_off[i + 1]] for i in range(n)], counts


def tokenize(text: str, vocab: int) -> np.ndarray:
    return tokenize_batch([text], vocab)[0][0]


def count_tokens(text: str) -> int:
    return int(tokenize_batch([text], 259)[1][0])


def tokenize_host(text: str, vocab: int) -> np.ndarray:
    """Host form of the same tokenizer (rr_tokenize): what the device kernel is checked against."""
    b = text.encode("utf-8")
    ids = np.zeros(len(b) + 1, dtype=np.int32)
    n = C.c_int32()
    _lib.check(_lib.lib.rr_tokenize(b, len(b), vocab, ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                    len(ids), C.byref(n)), "rr_tokenize")
    return ids[: n.value]


def detokenize(ids: Sequence[int]) -> str:
    return bytes(((int(t) - 3) % 256) for t in ids if int(t) >= 3).decode("utf-8", errors="replace")


MAX_TOP_LOGPROBS = 20        # OpenAI's limit


def check_logprobs(logprobs: Any, top_logprobs: Any) -> Optional[int]:
    """OpenAI's rules for the `logprobs` / `top_logprobs` request fields -> None (off) or the number of alternatives per
    token, 0..20.  Raises BadRequestError (HTTP 400) for anything else."""
    if logprobs is not None and not isinstance(logprobs, bool):
        raise BadRequestError("`logprobs` must be a boolean")
    if top_logprobs is not None:
        if not logprobs:
            raise BadRequestError("`top_logprobs` requires `logprobs` to be true")
        if isinstance(top_logprobs, bool) or not isinstance(top_logprobs, int) or not 0 <= top_logprobs <= MAX_TOP_LOGPROBS:
            raise BadRequestError(f"`top_logprobs` must be an integer from 0 to {MAX_TOP_LOGPROBS}")
    if not logprobs:
        return None
    return 0 if top_logprobs is None else top_logprobs


MAX_TEMPERATURE = 2.0        # OpenAI's range for `temperature`


def _is_number(v: Any) -> bool:
    return isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v)


def check_sampling(temperature: Any = None, top_p: Any = None, seed: Any = None) -> Optional[Tuple[float, float, Optional[int]]]:
    """OpenAI's rules for the `temperature` / `top_p` / `seed` request fields -> None (greedy: temperature absent or 0)
    or (temperature, top_p, seed modulo 2^64 or None).  Raises BadRequestError (HTTP 400) for anything else.

    Unlike OpenAI, whose default temperature is 1, an absent temperature means greedy decoding here, so that requests
    without these fields generate exactly what they did before sampling existed."""
    if temperature is not None and (not _is_number(temperature) or not 0 <= temperature <= MAX_TEMPERATURE):
        raise BadRequestError(f"`temperature` must be a number from 0 to {MAX_TEMPERATURE:g}")
    if top_p is not None and (not _is_number(top_p) or not 0 <= top_p <= 1):
        raise BadRequestError("`top_p` must be a number from 0 to 1")
    if seed is not None and (isinstance(seed, bool) or not isinstance(seed, int) or not -2**63 <= seed < 2**64):
        raise BadRequestError("`seed` must be an integer from -2^63 to 2^64 - 1")
    if temperature is None or temperature == 0:
        return None
    return float(temperature), 1.0 if top_p is None else float(top_p), None if seed is None else seed % 2**64


MAX_PENALTY = 2.0            # OpenAI's range for `frequency_penalty` / `presence_penalty`: [-2, 2]
MAX_LOGIT_BIAS = 100.0       # OpenAI's range for a `logit_bias` value: [-100, 100]
MAX_LOGIT_BIAS_ENTRIES = 300  # this project's cap on the `logit_bias` map (PEN_MAX_BIAS of the engine)


def check_penalties(frequency_penalty: Any = None, presence_penalty: Any = None, logit_bias: Any = None,
                    vocab: Optional[int] = None) -> Optional[Tuple[float, float, List[int], List[float]]]:
    """OpenAI's rules for the `frequency_penalty` / `presence_penalty` / `logit_bias` request fields -> None (nothing to
    apply: both penalties absent or 0 and no bias entries) or (frequency_penalty, presence_penalty, bias ids, bias values).
    `logit_bias` maps token ids, as decimal strings of integers, to numbers; ids must be distinct and, with `vocab`, below
    it.  Raises BadRequestError (HTTP 400) for anything else."""
    for name, v in (("frequency_penalty", frequency_penalty), ("presence_penalty", presence_penalty)):
        if v is not None and (not _is_number(v) or not -MAX_PENALTY <= v <= MAX_PENALTY):
            raise BadRequestError(f"`{name}` must be a number from {-MAX_PENALTY:g} to {MAX_PENALTY:g}")
    ids: List[int] = []
    vals: List[float] = []
    if logit_bias is not None:
        if not isinstance(logit_bias, dict):
            raise BadRequestError("`logit_bias` must be an object mapping token ids to numbers")
        if len(logit_bias) > MAX_LOGIT_BIAS_ENTRIES:
            raise BadRequestError(f"`logit_bias` may hold at most {MAX_LOGIT_BIAS_ENTRIES} entries")
        for k, v in logit_bias.items():
            if isinstance(k, bool) or not (isinstance(k, int) or (isinstance(k, str) and re.fullmatch(r"[+-]?[0-9]+", k))):
                raise BadRequestError(f"`logit_bias` key {k!r} is not an integer token id")
            t = int(k)
            if t < 0 or (vocab is not None and t >= vocab):
                raise BadRequestError(f"`logit_bias` token id {t} is out of range"
                                      + ("" if vocab is None else f" [0, {vocab})"))
            if not _is_number(v) or not -MAX_LOGIT_BIAS <= v <= MAX_LOGIT_BIAS:
                raise BadRequestError(f"`logit_bias` values must be numbers from {-MAX_LOGIT_BIAS:g} to {MAX_LOGIT_BIAS:g}")
            ids.append(t)
            vals.append(float(v))
        if len(set(ids)) != len(ids):
            raise BadRequestError("`logit_bias` names the same token id twice")
    fp = 0.0 if frequency_penalty is None else float(frequency_penalty)
    pp = 0.0 if presence_penalty is None else float(presence_penalty)
    if fp == 0 and pp == 0 and not ids:
        return None
    return fp, pp, ids, vals


MAX_N = 128                  # OpenAI's range for `n`: 1..128


def check_n(n: Any) -> int:
    """OpenAI's rule for the `n` request field (the number of choices) -> 1 when absent, else the integer in 1..128.
    Raises BadRequestError (HTTP 400) for anything else, bools and floats included."""
    if n is None:
        return 1
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= MAX_N:
        raise BadRequestError(f"`n` must be an integer from 1 to {MAX_N}")
    return n


MAX_STOP = 4                 # OpenAI's limit on the number of `stop` sequences (STOP_MAX_SEQS of the engine)
MAX_STOP_BYTES = 64          # this project's cap on one stop sequence, in bytes of UTF-8 (STOP_MAX_LEN of the engine)
FINISH_REASONS = ("length", "stop")      # by the native finish code (rr_engine_wait)
JSON_MIN_VOCAB = 259         # JSON mode needs a token for every byte (3 + 256; JSON_MIN_VOCAB of the engine)


def check_stop(stop: Any) -> List[bytes]:
    """OpenAI's rules for the `stop` request field -> the stop sequences as UTF-8 bytes: none for None or [], one for a
    string, else a list of 1..4 strings, each 1..64 bytes long.  They are matched on the bytes of the reply.  Raises
    BadRequestError (HTTP 400) for anything else."""
    if stop is None:
        return []
    seqs = [stop] if isinstance(stop, str) else stop
    if not isinstance(seqs, (list, tuple)) or any(not isinstance(s, str) for s in seqs):
        raise BadRequestError("`stop` must be a string or an array of strings")
    if len(seqs) > MAX_STOP:
        raise BadRequestError(f"`stop` may hold at most {MAX_STOP} sequences")
    out = [s.encode("utf-8") for s in seqs]
    if any(len(b) == 0 for b in out):
        raise BadRequestError("`stop` sequences must not be empty: each is 1 to "
                              f"{MAX_STOP_BYTES} bytes of UTF-8")
    if any(len(b) > MAX_STOP_BYTES for b in out):
        raise BadRequestError(f"a `stop` sequence may be at most {MAX_STOP_BYTES} bytes of UTF-8")
    return out


def check_response_format(value: Any) -> bool:
    """OpenAI's `response_format` request field -> True for JSON mode ({"type": "json_object"}), False for None and
    {"type": "text"}.  Raises BadRequestError (HTTP 400) for `json_schema`, which is not supported, and anything else."""
    if value is None:
        return False
    typ = value.get("type") if isinstance(value, dict) else None
    if typ == "text":
        return False
    if typ == "json_object":
        return True
    if typ == "json_schema":
        raise BadRequestError("`response_format` type `json_schema` is not supported: use {\"type\": \"json_object\"}")
    raise BadRequestError("`response_format` must be {\"type\": \"text\"} or {\"type\": \"json_object\"}")


class GenArgs(NamedTuple):
    """A request's generation parameters in the form the native submit calls take them (gen_args)."""
    params: _lib.GenParams  # rr_gen_params, passed by reference to rr_engine_submit / rr_gateway_submit
    top: Optional[int]     # top_logprobs; None: no logprobs
    width: int             # (logprob, id) pairs per generated token; 0 without logprobs


class StreamItem(tuple):
    """An item of Router.completion_stream; the closing one carries the choice's finish reason."""
    finish_reason: Optional[str] = None


def gen_args(top_logprobs: Optional[int] = None, temperature: Optional[float] = None, top_p: Optional[float] = None,
             seed: Optional[int] = None, frequency_penalty: Optional[float] = None,
             presence_penalty: Optional[float] = None, bias_ids: Sequence[int] = (),
             bias_vals: Sequence[float] = (), stop: Sequence[bytes] = (), json_object: bool = False, n: int = 1) -> GenArgs:
    """None and absent fields take the defaults of a plain greedy request.  A sampled request (temperature > 0) without
    a seed gets a random one here, once, so that a fallback re-admission draws the same tokens; the seed is taken modulo
    2^64.  Without bias entries or stop sequences their arrays are null pointers; otherwise the struct holds the arrays
    (ctypes keeps what a pointer field is assigned).  `stop`: the stop sequences as bytes (check_stop).  json_object:
    JSON mode (check_response_format).  n: the number of choices.  Ranges are checked by the native call (check_* raise
    HTTP 400 first on the router's path)."""
    k = -1 if top_logprobs is None else int(top_logprobs)
    temp = float(temperature or 0.0)
    seed = (secrets.randbits(64) if seed is None else int(seed) % 2**64) if temp else 0
    p = _lib.GenParams(n_choices=n, top_logprobs=k, temperature=temp, top_p=1.0 if top_p is None else float(top_p),
                       seed=seed, frequency_penalty=float(frequency_penalty or 0.0),
                       presence_penalty=float(presence_penalty or 0.0), n_bias=len(bias_ids), n_stop=len(stop),
                       response_format=1 if json_object else 0)
    if len(bias_ids):
        p.bias_ids = np.ctypeslib.as_ctypes(np.ascontiguousarray(bias_ids, dtype=np.int32))
        p.bias_vals = np.ctypeslib.as_ctypes(np.ascontiguousarray(bias_vals, dtype=np.float32))
    if len(stop):
        blob = b"".join(stop)
        off = np.zeros(len(stop) + 1, dtype=np.int32)
        np.cumsum([len(b) for b in stop], out=off[1:])
        p.stop_bytes = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        p.stop_off = np.ctypeslib.as_ctypes(off)
    return GenArgs(p, None if k < 0 else k, (max(1, k) + (1 if temp else 0)) if k >= 0 else 0)


def _token_entry(tok: int, logprob: float) -> dict:
    """One token of the byte tokenizer in OpenAI's logprob shape (`token` is detokenize([tok]), `bytes` its byte)."""
    return {"token": detokenize([tok]), "logprob": logprob, "bytes": [(tok - 3) % 256] if tok >= 3 else []}


def logprobs_content(tokens: Sequence[int], pairs: Sequence[Sequence[Tuple[int, float]]], top: int) -> List[dict]:
    """`choices[0].logprobs.content` for the generated tokens: pairs[i] = the engine's (id, logprob) list of token i, best
    first (a sampled request adds the token's own pair after them); `top` alternatives each.  Alternatives of logprob -inf
    (tokens JSON mode masked out, when fewer than `top` are allowed) are left out: JSON cannot encode -inf."""
    out = []
    for tok, p in zip(tokens, pairs):
        lp = next((v for i, v in p if i == tok), p[0][1])
        e = _token_entry(int(tok), lp)
        e["top_logprobs"] = [_token_entry(i, v) for i, v in p[:top] if v != -math.inf]
        out.append(e)
    return out


def logprob_pairs(lp: np.ndarray, ids: np.ndarray, a: int, b: int) -> List[List[Tuple[int, float]]]:
    """Rows a..b of the library's [tokens][K] logprob / id buffers -> per token [(token id, logprob)], best first."""
    return [[(int(i), float(v)) for i, v in zip(ids[t], lp[t])] for t in range(a, b)]


MAX_COMPLETION_LOGPROBS = 5  # OpenAI's limit for `logprobs` on /v1/completions


def check_text_completion(prompt: Any, max_tokens: Any = None, echo: Any = None, logprobs: Any = None,
                          stream: Any = None, best_of: Any = None, suffix: Any = None):
    """OpenAI's rules for the fields of a /v1/completions request -> (prompts, logprobs).  `prompt` takes OpenAI's four
    forms: a string, an array of strings, an array of token ids or an array of arrays of ids; each element of `prompts` is a
    string or a list of ids (their range is the caller's to check against the vocabulary).  logprobs: None (off) or 0..5.
    Raises BadRequestError (HTTP 400) naming the field for anything else, and for what this server does not serve: `echo`
    with `stream`, `best_of` other than 1, `suffix`, and `max_tokens` 0 (a prefill-only request)."""
    def is_id(v):
        return isinstance(v, int) and not isinstance(v, bool)
    if isinstance(prompt, str):
        prompts: List[Any] = [prompt]
    elif isinstance(prompt, list) and prompt and all(isinstance(p, str) for p in prompt):
        prompts = list(prompt)
    elif isinstance(prompt, list) and prompt and all(is_id(t) for t in prompt):
        prompts = [list(prompt)]
    elif isinstance(prompt, list) and prompt and all(isinstance(p, list) and p and all(is_id(t) for t in p) for p in prompt):
        prompts = [list(p) for p in prompt]
    else:
        raise BadRequestError("`prompt` must be a string, an array of strings, an array of token ids or an array of "
                              "arrays of token ids, none of them empty")
    if max_tokens is not None and (not isinstance(max_tokens, int) or isinstance(max_tokens, bool) or max_tokens < 1):
        raise BadRequestError("`max_tokens` must be an integer of at least 1: prefill-only requests are not served")
    if echo is not None and not isinstance(echo, bool):
        raise BadRequestError("`echo` must be a boolean")
    if stream is not None and not isinstance(stream, bool):
        raise BadRequestError("`stream` must be a boolean")
    if echo and stream:
        raise BadRequestError("`echo` is not available with `stream`: send the request without `stream`")
    if best_of is not None and (isinstance(best_of, bool) or best_of != 1):
        raise BadRequestError("`best_of` other than 1 is not supported: use `n`")
    if suffix is not None:
        raise BadRequestError("`suffix` is not supported")
    if logprobs is not None and (isinstance(logprobs, bool) or not isinstance(logprobs, int)
                                 or not 0 <= logprobs <= MAX_COMPLETION_LOGPROBS):
        raise BadRequestError(f"`logprobs` must be an integer from 0 to {MAX_COMPLETION_LOGPROBS}")
    return prompts, logprobs


MAX_EMBEDDING_INPUTS = 2048  # OpenAI's limit on the inputs of one /v1/embeddings request
ENCODING_FORMATS = ("float", "base64")


def check_embedding(input: Any, encoding_format: Any = None, dimensions: Any = None) -> Tuple[List[Any], str]:
    """OpenAI's rules for the fields of a /v1/embeddings request -> (inputs, encoding format).  `input` takes OpenAI's
    four forms: a string, an array of strings, an array of token ids or an array of arrays of ids; each element of
    `inputs` is a non-empty string or a non-empty list of ids (their range is the caller's to check against the
    vocabulary), at most 2048 of them.  encoding_format: "float" (None) or "base64".  dimensions: None or a positive
    integer (the caller checks it against the model's hidden size).  Raises BadRequestError (HTTP 400) naming the field for
    anything else."""
    def is_id(v):
        return isinstance(v, int) and not isinstance(v, bool)
    if isinstance(input, str) and input:
        inputs: List[Any] = [input]
    elif isinstance(input, list) and input and all(isinstance(p, str) and p for p in input):
        inputs = list(input)
    elif isinstance(input, list) and input and all(is_id(t) for t in input):
        inputs = [list(input)]
    elif isinstance(input, list) and input and all(isinstance(p, list) and p and all(is_id(t) for t in p) for p in input):
        inputs = [list(p) for p in input]
    else:
        raise BadRequestError("`input` must be a string, an array of strings, an array of token ids or an array of "
                              "arrays of token ids, none of them empty")
    if len(inputs) > MAX_EMBEDDING_INPUTS:
        raise BadRequestError(f"`input` holds {len(inputs)} inputs: at most {MAX_EMBEDDING_INPUTS} are allowed")
    fmt = "float" if encoding_format is None else encoding_format
    if fmt not in ENCODING_FORMATS:
        raise BadRequestError("`encoding_format` must be \"float\" or \"base64\"")
    if dimensions is not None and (not is_id(dimensions) or dimensions < 1):
        raise BadRequestError("`dimensions` must be a positive integer")
    return inputs, fmt


def encode_embedding(v: np.ndarray, encoding_format: str):
    """One `data[i].embedding` of /v1/embeddings: a list of floats (each the exact value of its fp32 component), or with
    "base64" the little-endian fp32 bytes, base64-encoded (what the OpenAI SDK asks for by default and decodes itself)."""
    v = np.asarray(v, dtype=np.float32)
    if encoding_format == "base64":
        return base64.b64encode(v.astype("<f4").tobytes()).decode("ascii")
    return [float(x) for x in v]


@dataclass
class EmbeddingResponse:
    """A /v1/embeddings response (OpenAI `CreateEmbeddingResponse`)."""
    model: str
    data: List[Any]                      # per input, in order: its embedding (list of floats or a base64 string)
    prompt_tokens: int
    object: str = "list"

    def model_dump(self) -> dict:
        return {"object": self.object,
                "data": [{"object": "embedding", "index": i, "embedding": e} for i, e in enumerate(self.data)],
                "model": self.model,
                "usage": {"prompt_tokens": self.prompt_tokens, "total_tokens": self.prompt_tokens}}


_invalid_spans = threading.local()


def _note_invalid(exc: UnicodeDecodeError):
    _invalid_spans.v.append((exc.start, exc.end))
    return "\ufffd", exc.end


codecs.register_error("rr_b200_note_invalid", _note_invalid)


def text_offsets(tokens: Sequence[int]) -> Tuple[str, List[int]]:
    """(detokenize(tokens), each token's `text_offset`): the character offset in that text where the token's first byte
    starts.  A continuation byte of a multi-byte character gets its character's offset, and every byte of an invalid
    sequence the offset of the U+FFFD that replaces it; a token without a byte (id < 3) gets the offset of the text after
    the tokens before it."""
    raw = bytes(((int(t) - 3) % 256) for t in tokens if int(t) >= 3)
    _invalid_spans.v = []
    text = raw.decode("utf-8", errors="rr_b200_note_invalid")
    spans = dict(_invalid_spans.v)
    char_of = [0] * (len(raw) + 1)
    i = c = 0
    while i < len(raw):
        b = raw[i]
        end = spans.get(i, i + (1 if b < 0x80 else 2 if b < 0xE0 else 3 if b < 0xF0 else 4))
        for j in range(i, end):
            char_of[j] = c
        i, c = end, c + 1
    char_of[len(raw)] = c
    offs, pos = [], 0
    for t in tokens:
        offs.append(char_of[pos])
        pos += 1 if int(t) >= 3 else 0
    return text, offs


def top_logprobs_dict(tok: int, tok_lp: float, alts: Sequence[Tuple[int, float]]) -> dict:
    """One entry of /v1/completions `logprobs.top_logprobs`: token string -> logprob over the alternatives and the token
    itself (up to k + 1 entries).  The byte tokenizer maps many ids to one string (every id >= 259 folds onto a byte, and
    a lone byte of a multi-byte character is U+FFFD), so a string holds the largest logprob among the listed ids that have
    it.  -inf (a token JSON mode masked out) is left out: JSON cannot encode it."""
    out: Dict[str, float] = {}
    for i, v in list(alts) + [(tok, tok_lp)]:
        s = detokenize([i])
        if v != -math.inf and (s not in out or v > out[s]):
            out[s] = float(v)
    return out


def completion_logprobs(tokens: Sequence[int], token_lps: Sequence[Optional[float]],
                        alts: Sequence[Optional[Sequence[Tuple[int, float]]]]) -> dict:
    """`choices[i].logprobs` of /v1/completions over `tokens` (with `echo` the prompt's, then the generated ones):
    token_lps[t] = the token's logprob and alts[t] its k alternatives as (id, logprob), both None for the first prompt
    token, which has no context."""
    _, offs = text_offsets(tokens)
    return {"tokens": [detokenize([t]) for t in tokens],
            "token_logprobs": [None if v is None else float(v) for v in token_lps],
            "top_logprobs": [None if a is None else top_logprobs_dict(t, v, a) for t, v, a in zip(tokens, token_lps, alts)],
            "text_offset": offs}


@dataclass
class TextChoice:
    index: int
    text: str
    finish_reason: str = "length"
    logprobs: Optional[dict] = None      # {tokens, token_logprobs, top_logprobs, text_offset}; only when requested


@dataclass
class TextCompletionResponse:
    """A /v1/completions response (OpenAI `Completion`)."""
    id: str
    model: str
    choices: List[TextChoice]
    usage: Usage
    created: int = 0
    object: str = "text_completion"

    def model_dump(self) -> dict:
        u = {"prompt_tokens": self.usage.prompt_tokens, "completion_tokens": self.usage.completion_tokens,
             "total_tokens": self.usage.total_tokens}
        if self.usage.prompt_tokens_details is not None:
            u["prompt_tokens_details"] = self.usage.prompt_tokens_details
        return {"id": self.id, "object": self.object, "created": self.created, "model": self.model,
                "choices": [{"index": c.index, "text": c.text, "logprobs": c.logprobs, "finish_reason": c.finish_reason}
                            for c in self.choices], "usage": u}


def messages_to_text(messages: Sequence[dict]) -> str:
    return "\n".join(f"{m.get('role', 'user')}: {m.get('content', '')}" for m in messages)


# ---------------------------------------------------------------- backends
@dataclass
class StubBackend:
    """Mock-completion replica (BASELINE.json configs[0]: plumbing only), served inside the gateway (rr_stub_desc): a
    fixed reply of `reply_tokens` token ids; with fail_every = n, every n-th request handed to it fails."""
    vocab: int = 128256
    reply_tokens: int = 8
    fail_every: int = 0


class EngineBackend:
    """A model replica: the gateway hands its admitted requests to `engine`."""

    def __init__(self, engine):
        self.engine = engine
        self.vocab = engine.spec.vocab


# ---------------------------------------------------------------- the router
def _kv_refusal(backends, n_prompt: int, max_new: int, n: int) -> Optional[int]:
    """The KV cache (tokens) of an attached engine replica that could never hold `n` choices of n_prompt + max_new tokens,
    else None.  As in the gateway, a choice reserves its reach in 64-token pages, at most the ring of a replica whose
    model has a sliding window."""
    pages = -(-(n_prompt + max_new) // 64)
    for b in backends.values():
        if isinstance(b, EngineBackend):
            e = b.engine
            ring = ring_pages(getattr(e.spec, "sliding_window", 0), e.max_prefill_tokens)
            if n * (min(pages, ring) if ring else pages) * 64 > e.kv_cache_tokens:
                return e.kv_cache_tokens
    return None


class Router:
    def __init__(self, model_list: Optional[List[dict]] = None, *, routing_strategy: str = "simple-shuffle",
                 enable_pre_call_checks: bool = False, allowed_fails: Optional[int] = None,
                 cooldown_time: Optional[float] = None, fallbacks: Optional[List[dict]] = None,
                 routing_strategy_args: Optional[dict] = None,
                 config: Optional[RouterConfig] = None, backends: Optional[Dict[int, Any]] = None,
                 seed: int = 0, device: int = 0, clock: Optional[Callable[[], float]] = None,
                 default_max_tokens: int = 128):
        if config is None:
            rs = {"routing_strategy": routing_strategy, "enable_pre_call_checks": enable_pre_call_checks,
                  "fallbacks": fallbacks or [], "routing_strategy_args": routing_strategy_args}
            if allowed_fails is not None:
                rs["allowed_fails"] = allowed_fails
            if cooldown_time is not None:
                rs["cooldown_time"] = cooldown_time
            config = build_config(model_list or [], rs)
        self.cfg = config
        self.backends: Dict[int, Any] = dict(backends or {})
        self._custom_clock = clock is not None
        self.clock = clock or time.time
        self._gw = None                 # rr_gateway handle (native per-request path), created on first use
        self._gw_sig = None
        self._gw_lock = threading.Lock()
        self.record_trace = 0           # > 0: the gateway keeps the last N (event, decision) pairs (gateway_trace())
        self.default_max_tokens = default_max_tokens
        deps = config.deployments
        if not deps:
            raise ValueError("model_list is empty")
        arr = (_lib.DeploymentDesc * len(deps))()
        for i, d in enumerate(deps):
            arr[i] = _lib.DeploymentDesc(d.group, d.rpm, d.tpm, d.weight, d.gpu, 0)
        ng = len(config.groups)
        offs, flat = [0], []
        for g in range(ng):
            flat += config.fallbacks.get(g, [])
            offs.append(len(flat))
        st = _lib.RouterSettings(config.strategy_id, int(config.enable_pre_call_checks), config.allowed_fails,
                                 int(round(config.cooldown_time * 1000)), 0, config.latency_list_size,
                                 config.latency_buffer_ppm, config.latency_ttl_ms)
        self._h = C.c_void_p()
        _lib.check(_lib.lib.rr_router_create(arr, len(deps), ng, (C.c_int32 * len(offs))(*offs),
                                             (C.c_int32 * max(1, len(flat)))(*flat), C.byref(st), seed, device,
                                             C.byref(self._h)), "rr_router_create")

    @classmethod
    def from_config(cls, path: str, **kw) -> "Router":
        return cls(config=load_config(path), **kw)

    def close(self):
        if getattr(self, "_gw", None):
            _lib.lib.rr_gateway_destroy(self._gw)
            self._gw = None
        if getattr(self, "_h", None):
            _lib.lib.rr_router_destroy(self._h)
            self._h = None

    # ---- native per-request path (rr_gateway.cu) ------------------------------------------------------
    def _gateway(self):
        """rr_gateway over this router and its replicas (the engine of an EngineBackend; a StubBackend is a mock replica
        the gateway serves itself), built on first use and again when the backends change."""
        if not self.backends:
            raise ServiceUnavailableError("no backend attached to this router")
        sig = tuple(sorted((k, id(b.engine if isinstance(b, EngineBackend) else b)) for k, b in self.backends.items()))
        with self._gw_lock:
            if self._gw is not None and self._gw_sig == sig:
                return self._gw
            if self._gw is not None:
                _lib.lib.rr_gateway_destroy(self._gw)
                self._gw = None
            keys = sorted(self.backends)
            engs = (C.c_void_p * len(keys))()                # NULL: a mock replica, described in stubs
            stubs = (_lib.StubDesc * len(keys))()
            for i, k in enumerate(keys):
                b = self.backends[k]
                if isinstance(b, StubBackend):
                    stubs[i] = _lib.StubDesc(b.reply_tokens, b.fail_every, b.vocab, 0)
                else:
                    engs[i] = b.engine._h
            reps = (C.c_int32 * len(keys))(*keys)
            opts = _lib.GatewayOpts(1 if self._custom_clock else 0, int(self.record_trace), 0)
            h = C.c_void_p()
            _lib.check(_lib.lib.rr_gateway_create(self._h, engs, reps, len(keys), stubs, C.byref(opts), C.byref(h)),
                       "rr_gateway_create")
            self._gw, self._gw_sig = h, sig
            return h

    def gateway_stats(self) -> dict:
        s = _lib.GatewayStats()
        _lib.check(_lib.lib.rr_gateway_get_stats(self._gateway(), C.byref(s)), "rr_gateway_get_stats")
        return {k: getattr(s, k) for k, _ in s._fields_}

    def gateway_trace(self) -> List[Tuple[Tuple[int, int, int, int, int], Tuple[int, int, int, int]]]:
        """[(event, decision)] recorded by the gateway (record_trace > 0), oldest first: the serialised trace K1 processed.
        Like the snapshots, it waits for the DONE / FAIL reports of finished requests, so it matches the state read after it."""
        gw = self._gateway()
        self._quiesce()
        n = C.c_int32()
        if _lib.lib.rr_gateway_trace(gw, None, None, 0, C.byref(n)) not in (0, 4) or n.value == 0:
            return []
        ev, dec = (_lib.Event * n.value)(), (_lib.Decision * n.value)()
        _lib.check(_lib.lib.rr_gateway_trace(gw, ev, dec, n.value, C.byref(n)), "rr_gateway_trace")
        return [((e.type, e.target, e.tokens, e.chain_start, e.now_ms), (d.status, d.deployment, d.served_group, d.chain_pos))
                for e, d in zip(ev[: n.value], dec[: n.value])]

    def _usage(self, dep: int, n_prompt: int, n_gen: int, n_cached: int = 0) -> Usage:
        """prompt_tokens counts the whole prompt, cached or not (as litellm does; so does the tpm debit)."""
        details = {"cached_tokens": int(n_cached)} if self.cfg.deployments[dep].prefix_cache else None
        return Usage(n_prompt, n_gen, n_prompt + n_gen, details)

    def _gw_response(self, res, toks, n_prompt, t_start, detok=True, logprobs=None, n_tokens=None,
                     finish=None) -> ModelResponse:
        """toks [n choices][max_new] (or one row), logprobs: one `logprobs` object per choice (or None).  n_tokens /
        finish: each choice's token count and finish code (None: res.n_generated and length, as for a plain request)."""
        d = self.cfg.deployments[res.deployment]
        toks = np.atleast_2d(toks)
        n_tokens = [res.n_generated] * len(toks) if n_tokens is None else n_tokens
        finish = [0] * len(toks) if finish is None else finish
        rows = [[int(t) for t in row[:k]] for row, k in zip(toks, n_tokens)]
        lps = logprobs if isinstance(logprobs, list) else [logprobs] * len(rows)
        return ModelResponse(
            id="chatcmpl-" + uuid.uuid4().hex[:24], model=d.response_model,
            choices=[Choice(i, Message("assistant", detokenize(t) if detok else ""), FINISH_REASONS[f], logprobs=lp)
                     for i, (t, lp, f) in enumerate(zip(rows, lps, finish))],
            usage=self._usage(res.deployment, n_prompt, sum(len(t) for t in rows), res.n_cached), created=int(time.time()),
            _token_ids=rows[0], _deployment=res.deployment, _model_group=self.cfg.groups[res.served_group],
            _fell_back=res.chain_pos > 0, _ttft_s=res.t_first_token_s - res.t_submit_s,
            _latency_s=time.perf_counter() - t_start, _choice_token_ids=rows)

    def _limits(self) -> Tuple[int, int, int]:
        """(context window, decode rows, KV cache tokens) of the smallest engine replica attached; a mock replica sets
        none."""
        engs = [b.engine for b in self.backends.values() if isinstance(b, EngineBackend)]
        big = 2**31 - 1
        return (min((e.ctx_max for e in engs), default=big), min((e.max_batch for e in engs), default=big),
                min((e.kv_cache_tokens for e in engs), default=big))

    def _invalid(self, n_prompt: int = 0, max_new: int = 0, n: int = 1) -> BadRequestError:
        """The HTTP 400 of a request the gateway refused with RR_INVALID_ARGUMENT, naming the limit it broke."""
        ctx, rows, _ = self._limits()
        kv = _kv_refusal(self.backends, n_prompt, max_new, n)
        if n > rows:
            return BadRequestError(f"`n` = {n} exceeds the {rows} decode rows of the smallest replica")
        if n_prompt + max_new > ctx:
            return BadRequestError(f"prompt ({n_prompt} tokens) + max_tokens ({max_new}) exceed the context window "
                                   f"({ctx} tokens) of the deployment")
        if kv is not None:
            return BadRequestError(f"`n` ({n}) x (prompt ({n_prompt} tokens) + max_tokens ({max_new})), in 64-token pages, "
                                   f"exceed the KV cache ({kv} tokens) of the deployment")
        return BadRequestError("a token id is outside the vocabulary of the deployment, or a generation parameter is out "
                               "of range")

    def _gw_error(self, status: int, model: str, res=None, timeout=None) -> APIError:
        if status == 1:
            return RateLimitError(f"No deployments available for selected model, passed model={model} (rate limited)")
        if status == 2:
            return BadRequestError(f"Invalid model name passed in model={model}")
        if status == 4:
            return self._invalid() if res is None else self._invalid(res.n_prompt, 0)
        if status == 6:
            return APITimeoutError(f"Request timed out after {timeout}s")
        if status == 7:
            dep = res.deployment if res is not None else -1
            return APIError(f"backend failure on deployment {dep} and no fallback available for model={model}")
        return APIError(f"{_lib.lib.rr_strerror(status).decode()} (model={model})")

    def _gw_submit(self, gw, g: int, prompt_ids, max_new: int, model: str, gen: GenArgs,
                   prompt_top: Optional[int] = None) -> int:
        """prompt_top: also score the prompt (rr_gateway_submit_scored) with that many pairs per position."""
        ids = np.ascontiguousarray(np.asarray(prompt_ids, dtype=np.int32))
        if self._custom_clock:
            _lib.lib.rr_gateway_set_now(gw, self.now_ms())
        t = C.c_uint64()
        if prompt_top is None:
            rc = _lib.lib.rr_gateway_submit(gw, g, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), max_new,
                                            C.byref(gen.params), C.byref(t))
        else:
            rc = _lib.lib.rr_gateway_submit_scored(gw, g, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), max_new,
                                                   C.byref(gen.params), int(prompt_top), C.byref(t))
        if rc == 4:
            raise self._invalid(len(ids), max_new, gen.params.n_choices)
        if rc != 0:
            raise self._gw_error(rc, model)
        return t.value

    @staticmethod
    def _lp_bufs(gen: GenArgs, max_new: int, n: int = 1):
        """[max_new][gen.width] pair buffers of a logprobs request ([n][max_new][gen.width] for n choices)."""
        if gen.top is None:
            return None, None, None, None
        shape = (max_new, gen.width) if n == 1 else (n, max_new, gen.width)
        lp = np.zeros(shape, dtype=np.float32)
        ids = np.zeros(shape, dtype=np.int32)
        return lp, ids, lp.ctypes.data_as(C.POINTER(C.c_float)), ids.ctypes.data_as(C.POINTER(C.c_int32))

    def _completion_gw(self, gw, model, g, prompt_ids, max_new, timeout, gen: GenArgs):
        t_start = time.perf_counter()
        ticket = self._gw_submit(gw, g, prompt_ids, max_new, model, gen)
        n = gen.params.n_choices
        res = _lib.GatewayResult()
        toks = np.zeros(max_new if n == 1 else (n, max_new), dtype=np.int32)
        lp, ids, lp_p, ids_p = self._lp_bufs(gen, max_new, n)
        n_tok, fin = (C.c_int32 * n)(), (C.c_int32 * n)()
        rc = _lib.lib.rr_gateway_wait(gw, ticket, float(timeout or 0.0), C.byref(res),
                                      toks.ctypes.data_as(C.POINTER(C.c_int32)), max_new, lp_p, ids_p, n_tok, fin)
        if rc == 6:                      # client-side timeout: give the rows back, count a failure against the deployment
            _lib.lib.rr_gateway_cancel(gw, ticket, 1)
            raise self._gw_error(6, model, res, timeout)
        if rc != 0:
            raise self._gw_error(rc, model, res, timeout)
        content = None
        n_tok = [min(k, max_new) for k in n_tok]
        if gen.top is not None:
            content = [{"content": logprobs_content(t[:k].tolist(), logprob_pairs(a, b, 0, k), gen.top), "refusal": None}
                       for t, a, b, k in zip(np.atleast_2d(toks), lp.reshape(-1, max_new, gen.width),
                                             ids.reshape(-1, max_new, gen.width), n_tok)]
            content = content[0] if n == 1 else content
        return self._gw_response(res, toks, len(prompt_ids), t_start, logprobs=content, n_tokens=n_tok, finish=list(fin))

    def _stream_gw(self, gw, model, g, prompt_ids, max_new, timeout, gen: GenArgs):
        ticket = self._gw_submit(gw, g, prompt_ids, max_new, model, gen)
        top = gen.top
        deadline = None if not timeout else time.perf_counter() + timeout
        res = _lib.GatewayResult()
        toks = np.zeros(max_new, dtype=np.int32)
        lp, ids, lp_p, ids_p = self._lp_bufs(gen, max_new)
        n, done = C.c_int32(), C.c_int32()
        sent, finished = 0, False

        def item(label, a, b, ttft):
            """(label, tokens a..b, done=False, ttft) + with logprobs: the OpenAI content entries of those tokens."""
            new = [int(t) for t in toks[a: b]]
            if top is None:
                return label, new, False, ttft
            return label, new, False, ttft, logprobs_content(new, logprob_pairs(lp, ids, a, b), top)
        try:
            while True:
                _lib.check(_lib.lib.rr_gateway_peek(gw, ticket, sent, 0.05, toks.ctypes.data_as(C.POINTER(C.c_int32)), max_new,
                                                    C.byref(n), C.byref(done), C.byref(res), lp_p, ids_p), "rr_gateway_peek")
                if done.value:
                    rc = _lib.lib.rr_gateway_wait(gw, ticket, 1.0, C.byref(res), toks.ctypes.data_as(C.POINTER(C.c_int32)),
                                                  max_new, lp_p, ids_p, None, None)
                    finished = True
                    if rc != 0:
                        raise self._gw_error(rc, model, res, timeout)
                    label = self.cfg.deployments[res.deployment].response_model
                    ttft = res.t_first_token_s - res.t_submit_s
                    if res.n_generated > sent:       # the last tokens, with any a pending partial stop match held back
                        yield item(label, sent, res.n_generated, ttft)
                    last = StreamItem((label, [], True, ttft) if top is None else (label, [], True, ttft, []))
                    last.finish_reason = FINISH_REASONS[res.finish]
                    yield last
                    return
                if n.value > sent and res.deployment >= 0:
                    label = self.cfg.deployments[res.deployment].response_model
                    yield item(label, sent, n.value, 0.0)
                    sent = n.value
                if deadline is not None and time.perf_counter() > deadline:
                    _lib.lib.rr_gateway_cancel(gw, ticket, 1)
                    finished = True
                    raise self._gw_error(6, model, res, timeout)
        finally:
            if not finished:             # the consumer went away (SSE client disconnected): free the row, no failure counted
                _lib.lib.rr_gateway_cancel(gw, ticket, 0)

    def _batch_gw(self, gw, model, g, prompts, max_new, timeout):
        t0 = time.perf_counter()
        n = len(prompts)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.int32) for p in prompts]))
        start = np.zeros(n + 1, dtype=np.int32)
        np.cumsum([len(p) for p in prompts], out=start[1:])
        if self._custom_clock:
            _lib.lib.rr_gateway_set_now(gw, self.now_ms())
        tk = (C.c_uint64 * n)()
        rc = _lib.lib.rr_gateway_submit_batch(gw, g, ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                              start.ctypes.data_as(C.POINTER(C.c_int32)), n, max_new,
                                              1 if self.cfg.routing_strategy == "split" else 0, tk)
        if rc == 4:
            raise self._invalid(max(len(p) for p in prompts), max_new)
        if rc != 0:
            raise self._gw_error(rc, model)
        out: List[Any] = [None] * n
        toks = np.zeros(max_new, dtype=np.int32)
        for i in range(n):
            res = _lib.GatewayResult()
            left = None if not timeout else max(0.001, timeout - (time.perf_counter() - t0))
            rc = _lib.lib.rr_gateway_wait(gw, tk[i], float(left or 0.0), C.byref(res),
                                          toks.ctypes.data_as(C.POINTER(C.c_int32)), max_new, None, None, None, None)
            if rc == 6:
                _lib.lib.rr_gateway_cancel(gw, tk[i], 1)
            out[i] = self._gw_response(res, toks, len(prompts[i]), t0, detok=False) if rc == 0 \
                else self._gw_error(rc, model, res, timeout)
        return out

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- K1 calls -------------------------------------------------------------------------------
    def now_ms(self) -> int:
        return int(self.clock() * 1000)

    def process(self, events: Sequence[Tuple[int, int, int, int, int]]) -> List[Tuple[int, int, int, int]]:
        """events: (type, target, tokens, chain_start, now_ms) -> (status, deployment, group, chain_pos)."""
        n = len(events)
        if n == 0:
            return []
        self._quiesce()
        ev = (_lib.Event * n)()
        for i, e in enumerate(events):
            ev[i] = _lib.Event(*e)
        out = (_lib.Decision * n)()
        _lib.check(_lib.lib.rr_router_process(self._h, ev, n, out), "rr_router_process")
        return [(d.status, d.deployment, d.served_group, d.chain_pos) for d in out]

    def _quiesce(self):
        """Let the gateway's dispatcher post what is still queued (DONE / FAIL reports of finished requests)."""
        if self._gw is not None:
            _lib.lib.rr_gateway_quiesce(self._gw, 5.0)

    def snapshot(self) -> List[dict]:
        self._quiesce()
        n = len(self.cfg.deployments)
        s = (_lib.DeploymentState * n)()
        _lib.check(_lib.lib.rr_router_snapshot(self._h, s), "rr_router_snapshot")
        return [{k: getattr(x, k) for k, _ in x._fields_} for x in s]

    def latency_snapshot(self) -> List[Tuple[float, int]]:
        """latency-based-routing: [(mean latency in us per output token, samples held)] per deployment, as stored
        (a group whose ttl ran out is cleared at its next write or pick).  All (0.0, 0) under the other strategies."""
        self._quiesce()
        n = len(self.cfg.deployments)
        mean, cnt = (C.c_double * n)(), (C.c_int32 * n)()
        _lib.check(_lib.lib.rr_router_latency_snapshot(self._h, mean, cnt), "rr_router_latency_snapshot")
        return list(zip(mean, cnt))

    # ---- request path ---------------------------------------------------------------------------
    def _vocab(self) -> int:
        """Token ids must be valid on every replica a request may fall back to: the smallest vocabulary attached."""
        return min((b.vocab for b in self.backends.values()), default=128256)

    def _params(self, logprobs, top_logprobs, temperature, top_p, seed, frequency_penalty, presence_penalty,
                logit_bias, stop=None, response_format=None, n: int = 1) -> GenArgs:
        """The request's validated generation parameters.  Only engine replicas have logits to serve logprobs and to mask
        for JSON mode, and a decode loop that stop sequences can end; bias ids must be valid on every replica the request
        may fall back to, and JSON mode needs a token for every byte there."""
        top = check_logprobs(logprobs, top_logprobs)
        stops = check_stop(stop)
        json_object = check_response_format(response_format)
        mock = any(isinstance(b, StubBackend) for b in self.backends.values())
        if stops and mock:
            raise BadRequestError("`stop` is not available: the backends of this router are not model replicas")
        if top is not None and mock:
            raise BadRequestError("`logprobs` is not available: the backends of this router are not model replicas")
        if json_object and mock:
            raise BadRequestError("`response_format` json_object is not available: the backends of this router are not "
                                  "model replicas")
        if json_object and self._vocab() < JSON_MIN_VOCAB:
            raise BadRequestError(f"`response_format` json_object needs a vocabulary of at least {JSON_MIN_VOCAB} tokens")
        samp = check_sampling(temperature, top_p, seed) or (None, None, None)
        pen = check_penalties(frequency_penalty, presence_penalty, logit_bias, self._vocab()) or (None, None, (), ())
        return gen_args(top, *samp, *pen, stop=stops, json_object=json_object, n=n)

    def completion(self, model: str, messages: Optional[Sequence[dict]] = None, timeout: Optional[float] = None,
                   max_tokens: Optional[int] = None, prompt_ids: Optional[Sequence[int]] = None,
                   logprobs: bool = False, top_logprobs: Optional[int] = None, temperature: Optional[float] = None,
                   top_p: Optional[float] = None, seed: Optional[int] = None, frequency_penalty: Optional[float] = None,
                   presence_penalty: Optional[float] = None, logit_bias: Optional[Dict[str, float]] = None,
                   n: Optional[int] = None, stop: Any = None, response_format: Any = None,
                   **_ignored) -> ModelResponse:
        """logprobs=True: `choices[0].logprobs` carries the logprob of every generated token and its `top_logprobs`
        (0..20) most likely alternatives, as the OpenAI API returns them.  temperature > 0: every token is drawn from
        the top_p nucleus of softmax(logits / temperature) with the request's seed (rr_op_sample); absent or 0 is
        greedy.  frequency_penalty / presence_penalty / logit_bias: applied to the logits before every token is picked
        (rr_op_logit_penalties; the penalties count the tokens generated so far).  Stub backends validate these and keep
        their fixed reply.
        n (1..128, at most the decode rows of the smallest engine replica): n choices of the same prompt, prefilled once
        (rr_gen_params.n_choices).  Choice i of a sampled request is drawn with seed + i (mod 2^64), so it equals the
        n=1 response with that seed; greedy choices are all the greedy response.  usage.completion_tokens sums the
        choices and `_choice_token_ids` holds each choice's tokens (`_token_ids`: choice 0's).
        stop: a string or up to 4 strings of 1..64 bytes of UTF-8 each.  A choice ends where its reply would contain one
        of them: the content stops before it and finish_reason is "stop" (rr_gen_params.n_stop).  They are matched on
        the reply's bytes, so the tokens are a prefix of the same request's without `stop`; each choice ends on its own
        and usage.completion_tokens counts the tokens returned.
        response_format {"type": "json_object"}: JSON mode (rr_gen_params.response_format).  Every token is picked from
        the logits masked to the JSON grammar, so each choice's content is a prefix of a JSON object; the choice whose object
        closes ends there with finish_reason "stop", one that reaches max_tokens first with "length".  {"type": "text"}
        and None change nothing; `json_schema` and anything else raise BadRequestError (check_response_format)."""
        n = check_n(n)
        gen = self._params(logprobs, top_logprobs, temperature, top_p, seed, frequency_penalty, presence_penalty,
                           logit_bias, stop, response_format, n)
        g = self.cfg.group_index(model)
        if g < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        if prompt_ids is None:
            prompt_ids = tokenize(messages_to_text(messages or []), self._vocab())
        max_new = max_tokens or self.default_max_tokens
        if n > self._limits()[1]:
            raise self._invalid(n=n)
        return self._completion_gw(self._gateway(), model, g, prompt_ids, max_new, timeout, gen)

    def completion_stream(self, model: str, messages: Optional[Sequence[dict]] = None, timeout: Optional[float] = None,
                          max_tokens: Optional[int] = None, prompt_ids: Optional[Sequence[int]] = None,
                          logprobs: bool = False, top_logprobs: Optional[int] = None, temperature: Optional[float] = None,
                          top_p: Optional[float] = None, seed: Optional[int] = None,
                          frequency_penalty: Optional[float] = None, presence_penalty: Optional[float] = None,
                          logit_bias: Optional[Dict[str, float]] = None, n: Optional[int] = None, stop: Any = None,
                          response_format: Any = None):
        """Streaming variant (SSE in server.py): admission exactly like completion(); yields
        (model_label, new_token_ids, done, ttft_s) as tokens arrive, with logprobs=True a fifth element: the OpenAI
        `logprobs.content` entries of those tokens.  A backend failure before the first token walks the
        fallback chain; rate limiting raises RateLimitError before anything is yielded.  Sampling, penalties, logit
        bias and response_format as in completion().  n > 1 is not streamed: BadRequestError.  With `stop`, a token is
        yielded only once no stop sequence can take it back; the closing item (a StreamItem) has finish_reason "stop" or
        "length"."""
        if check_n(n) > 1:
            raise BadRequestError("streaming is not available with `n` > 1: send the request without `stream`")
        gen = self._params(logprobs, top_logprobs, temperature, top_p, seed, frequency_penalty, presence_penalty,
                           logit_bias, stop, response_format)
        g = self.cfg.group_index(model)
        if g < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        if prompt_ids is None:
            prompt_ids = tokenize(messages_to_text(messages or []), self._vocab())
        max_new = max_tokens or self.default_max_tokens
        yield from self._stream_gw(self._gateway(), model, g, prompt_ids, max_new, timeout, gen)

    def completion_batch(self, model: str, prompts: Sequence[Sequence[int]], max_tokens: int,
                         timeout: Optional[float] = None) -> List[Any]:
        """Closed burst of requests to one model group (what the demos do with N threads,
        reference src/demo_load_balancing.py:195-203): ONE admission launch over the whole trace,
        dispatch to the per-GPU engines, one DONE launch.  -> ModelResponse or exception per request."""
        g = self.cfg.group_index(model)
        if g < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        return self._batch_gw(self._gateway(), model, g, prompts, max_tokens, timeout)

    def _completion_prompts(self, prompt) -> List[List[int]]:
        """Token ids of check_text_completion's prompts: a string is BOS plus its bytes (no role framing), ids are used as
        they are and must lie in [0, vocab)."""
        vocab = self._vocab()
        out = []
        for p in prompt:
            if isinstance(p, str):
                out.append([int(t) for t in tokenize(p, vocab)])
            elif any(not 0 <= t < vocab for t in p):
                raise BadRequestError(f"`prompt` holds a token id outside the vocabulary [0, {vocab})")
            else:
                out.append(list(p))
        return out

    def text_completion(self, model: str, prompt: Any, max_tokens: Optional[int] = None, echo: bool = False,
                        logprobs: Optional[int] = None, temperature: Optional[float] = None, top_p: Optional[float] = None,
                        seed: Optional[int] = None, n: Optional[int] = None, stop: Any = None,
                        frequency_penalty: Optional[float] = None, presence_penalty: Optional[float] = None,
                        logit_bias: Optional[Dict[str, float]] = None, timeout: Optional[float] = None,
                        best_of: Optional[int] = None, suffix: Any = None, **_ignored) -> TextCompletionResponse:
        """OpenAI's /v1/completions (`client.completions.create`).  prompt: a string, an array of strings, an array of token
        ids or an array of arrays of ids; each prompt is its own request, all submitted together, and choice i * n + c is
        choice c of prompt i.  usage sums over the prompts.
        logprobs = k in 0..5: every generated token's logprob and its k most likely alternatives (the top_logprobs
        machinery of completion()).  echo: `text` starts with the prompt's text, and with logprobs the prompt is scored
        on the GPU (rr_gateway_submit_scored): `logprobs` then covers the prompt's tokens, then the generated ones.  The
        first prompt token has no context: its token_logprobs and top_logprobs entries are None.  top_logprobs[t] maps
        token strings to logprobs over the k alternatives and the token itself (up to k + 1 entries).  The byte
        tokenizer maps many ids to one string, so a string holds the largest logprob among the listed ids that have it.
        text_offset[t] is the character offset in `text` where token t's first byte starts (a continuation byte of a
        multi-byte character gets its character's offset).  A scoring request takes no prefix-cache hit:
        cached_tokens is 0.
        Refused with BadRequestError (check_text_completion): `echo` with streaming, `best_of` other than 1, `suffix`,
        `max_tokens` 0, and `logprobs` on mock replicas.  Sampling, penalties, logit_bias, stop and n as in completion()."""
        prompts, lp = check_text_completion(prompt, max_tokens, echo, logprobs, None, best_of, suffix)
        n = check_n(n)
        gen = self._params(True if lp is not None else None, lp, temperature, top_p, seed, frequency_penalty,
                           presence_penalty, logit_bias, stop, None, n)
        g = self.cfg.group_index(model)
        if g < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        ids = self._completion_prompts(prompts)
        max_new = max_tokens or self.default_max_tokens
        if n > self._limits()[1]:
            raise self._invalid(n=n)
        gw = self._gateway()
        t_start = time.perf_counter()
        score = lp if echo and lp is not None else None
        tickets: List[int] = []
        try:
            for p in ids:
                tickets.append(self._gw_submit(gw, g, p, max_new, model, gen, prompt_top=score))
        except APIError:
            for t in tickets:
                _lib.lib.rr_gateway_cancel(gw, t, 0)
            raise
        choices, usage, label, cached, dep = [], [0, 0], "", 0, 0
        for i, (p, ticket) in enumerate(zip(ids, tickets)):
            try:
                label, plp, waited = self._collect_prompt(gw, model, p, ticket, max_new, timeout, gen, score)
            except APIError:
                for t in tickets[i + 1:]:
                    _lib.lib.rr_gateway_cancel(gw, t, 0)
                raise
            res, toks, pairs, n_tok, fin = waited
            usage[0] += len(p)
            cached, dep = cached + res.n_cached, res.deployment
            for c in range(n):
                gen_toks = toks[c][: n_tok[c]].tolist()
                shown = (list(p) if echo else []) + gen_toks
                text = detokenize(shown)
                lpd = None
                if lp is not None:
                    gp = logprob_pairs(pairs[c][0], pairs[c][1], 0, n_tok[c])
                    g_lps = [next((v for j, v in q if j == t), q[0][1]) for t, q in zip(gen_toks, gp)]
                    g_alts = [q[:lp] for q in gp]
                    if echo:
                        p_lps, p_alts = plp if plp is not None else ([None] * len(p), [None] * len(p))
                        lpd = completion_logprobs(shown, list(p_lps) + g_lps, list(p_alts) + g_alts)
                    else:
                        lpd = completion_logprobs(shown, g_lps, g_alts)
                choices.append(TextChoice(i * n + c, text, FINISH_REASONS[fin[c]], lpd))
                usage[1] += len(gen_toks)
        return TextCompletionResponse("cmpl-" + uuid.uuid4().hex[:24], label, choices, self._usage(dep, *usage, cached),
                                      int(time.time()))

    def _collect_prompt(self, gw, model, p, ticket, max_new, timeout, gen: GenArgs, score: Optional[int]):
        """One prompt of text_completion: its prompt logprobs when score is set (read before the wait consumes the ticket)
        as ([None] + target logprobs, [None] + per position its `score` best (id, logprob) pairs), then its choices
        (_wait_choices).  -> (model label, prompt logprobs or None, _wait_choices' result)."""
        plp = None
        if score is not None:
            m, k = len(p) - 1, max(1, score)
            tgt, alt, alt_id = np.zeros(m, np.float32), np.zeros((m, k), np.float32), np.zeros((m, k), np.int32)
            rc = _lib.lib.rr_gateway_prompt_logprobs(gw, ticket, float(timeout or 0.0),
                                                     tgt.ctypes.data_as(C.POINTER(C.c_float)),
                                                     alt.ctypes.data_as(C.POINTER(C.c_float)),
                                                     alt_id.ctypes.data_as(C.POINTER(C.c_int32)))
            if rc == 0:
                plp = ([None] + tgt.tolist(), [None] + [list(zip(r_id.tolist(), r.tolist()))[:score]
                                                        for r, r_id in zip(alt, alt_id)])
        waited = self._wait_choices(gw, model, ticket, max_new, timeout, gen)
        return self.cfg.deployments[waited[0].deployment].response_model, plp, waited

    def _wait_choices(self, gw, model, ticket, max_new, timeout, gen: GenArgs):
        """rr_gateway_wait for a request of gen.params.n_choices choices -> (result, tokens [n][max_new], per choice
        (logprobs [max_new][width], ids) or None, tokens per choice, finish codes).  Raises the request's APIError."""
        n = gen.params.n_choices
        res = _lib.GatewayResult()
        toks = np.zeros((n, max_new), dtype=np.int32)
        lp, ids, lp_p, ids_p = self._lp_bufs(gen, max_new, n)
        if lp is not None:
            lp, ids = lp.reshape(n, max_new, gen.width), ids.reshape(n, max_new, gen.width)
        n_tok, fin = (C.c_int32 * n)(), (C.c_int32 * n)()
        rc = _lib.lib.rr_gateway_wait(gw, ticket, float(timeout or 0.0), C.byref(res),
                                      toks.ctypes.data_as(C.POINTER(C.c_int32)), max_new, lp_p, ids_p, n_tok, fin)
        if rc == 6:
            _lib.lib.rr_gateway_cancel(gw, ticket, 1)
        if rc != 0:
            raise self._gw_error(rc, model, res, timeout)
        pairs = [(lp[c], ids[c]) for c in range(n)] if lp is not None else None
        return res, toks, pairs, [min(k, max_new) for k in n_tok], list(fin)

    def text_completion_stream(self, model: str, prompt: Any, max_tokens: Optional[int] = None,
                               logprobs: Optional[int] = None, timeout: Optional[float] = None, **kw):
        """/v1/completions with `stream` (no `echo`): one prompt, served by completion_stream on its token ids; yields what
        completion_stream yields (with logprobs, the chat-shaped content entries of the new tokens)."""
        prompts, lp = check_text_completion(prompt, max_tokens, None, logprobs, True, kw.pop("best_of", None),
                                            kw.pop("suffix", None))
        if len(prompts) != 1:
            raise BadRequestError("streaming takes one `prompt`: send several prompts without `stream`")
        if self.cfg.group_index(model) < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        ids = self._completion_prompts(prompts)[0]
        yield from self.completion_stream(model, timeout=timeout, max_tokens=max_tokens, prompt_ids=ids,
                                          logprobs=True if lp is not None else None, top_logprobs=lp, **kw)

    def embedding(self, model: str, input: Any, encoding_format: Optional[str] = None, dimensions: Optional[int] = None,
                  timeout: Optional[float] = None, user: Optional[str] = None, **_ignored) -> EmbeddingResponse:
        """OpenAI's /v1/embeddings (`client.embeddings.create`, litellm's `Router.embedding`): per input the last prompt
        position's final-norm hidden state, L2-normalised, computed on the GPU (rr_gateway_submit_embed), as decoder
        embedding models such as e5-mistral-7b-instruct pool.  input: a string, an array of strings, an array of token
        ids or an array of arrays of ids (check_embedding); a string is BOS plus its bytes (no chat template).  Each input
        is its own gateway request (rpm and tpm count it like a prompt), all submitted together; on the first error the
        rest are cancelled and that error is raised.  encoding_format "float" (default) or "base64" (little-endian fp32).
        dimensions: absent or the model's hidden size (no truncation).  usage counts the inputs' tokens.
        Refused with BadRequestError: anything check_embedding refuses, a token id outside the vocabulary, an input beyond
        the context window or the KV cache, `dimensions` other than the hidden size, and mock replicas (no hidden state)."""
        inputs, fmt = check_embedding(input, encoding_format, dimensions)
        g = self.cfg.group_index(model)
        if g < 0:
            raise BadRequestError(f"Invalid model name passed in model={model}")
        if any(isinstance(b, StubBackend) for b in self.backends.values()):
            raise BadRequestError("embeddings are not available: the backends of this router are not model replicas")
        hidden = {b.engine.spec.hidden for b in self.backends.values() if isinstance(b, EngineBackend)}
        if dimensions is not None and hidden != {dimensions}:
            raise BadRequestError(f"`dimensions` must be the model's hidden size {sorted(hidden)}: embeddings are not "
                                  f"truncated")
        vocab = self._vocab()
        ids = []
        for p in inputs:
            if isinstance(p, str):
                ids.append([int(t) for t in tokenize(p, vocab)])
            elif any(not 0 <= t < vocab for t in p):
                raise BadRequestError(f"`input` holds a token id outside the vocabulary [0, {vocab})")
            else:
                ids.append(list(p))
        ctx = self._limits()[0]
        for i, p in enumerate(ids):
            kv = _kv_refusal(self.backends, len(p), 0, 1)
            if len(p) > ctx or kv is not None:
                raise BadRequestError(f"`input` {i} ({len(p)} tokens) exceeds the context window ({ctx} tokens) or the "
                                      f"KV cache of the deployment")
        gw = self._gateway()
        tickets: List[int] = []
        try:
            for p in ids:
                a = np.ascontiguousarray(np.asarray(p, dtype=np.int32))
                if self._custom_clock:
                    _lib.lib.rr_gateway_set_now(gw, self.now_ms())
                t = C.c_uint64()
                rc = _lib.lib.rr_gateway_submit_embed(gw, g, a.ctypes.data_as(C.POINTER(C.c_int32)), len(a), C.byref(t))
                if rc != 0:
                    raise self._invalid(len(a)) if rc == 4 else self._gw_error(rc, model)
                tickets.append(t.value)
        except APIError:
            for t in tickets:
                _lib.lib.rr_gateway_cancel(gw, t, 0)
            raise
        data, label = [], ""
        for i, t in enumerate(tickets):
            try:
                v, label = self._collect_embedding(gw, model, t, max(hidden, default=1), timeout)
            except APIError:
                for u in tickets[i + 1:]:
                    _lib.lib.rr_gateway_cancel(gw, u, 0)
                raise
            data.append(encode_embedding(v, fmt))
        return EmbeddingResponse(label, data, sum(len(p) for p in ids))

    def _collect_embedding(self, gw, model, ticket, capacity, timeout) -> Tuple[np.ndarray, str]:
        """One input of embedding(): its vector (read before the wait consumes the ticket) and the served model's label.
        Raises the request's APIError; a client-side timeout cancels it as a failure."""
        v = np.zeros(capacity, dtype=np.float32)
        dim = C.c_int32()
        rc = _lib.lib.rr_gateway_embedding(gw, ticket, float(timeout or 0.0), v.ctypes.data_as(C.POINTER(C.c_float)),
                                           capacity, C.byref(dim))
        res = _lib.GatewayResult()
        if rc == 6:
            _lib.lib.rr_gateway_cancel(gw, ticket, 1)
            raise self._gw_error(6, model, res, timeout)
        wrc = _lib.lib.rr_gateway_wait(gw, ticket, 1.0, C.byref(res), None, 0, None, None, None, None)
        if wrc == 6:
            _lib.lib.rr_gateway_cancel(gw, ticket, 1)
        for code in (wrc, rc):
            if code != 0:
                raise self._gw_error(code, model, res, timeout)
        v = v[: dim.value]
        if not np.isfinite(v).all():
            raise APIError(f"the embedding of deployment {res.deployment} holds a non-finite value (model={model})")
        return v, self.cfg.deployments[res.deployment].response_model


# ---------------------------------------------------------------- OpenAI-SDK-shaped facade
class _Completions:
    def __init__(self, router: Router):
        self._r = router

    def create(self, model: str, messages: Sequence[dict], timeout: Optional[float] = None,
               max_tokens: Optional[int] = None, **kw) -> ModelResponse:
        return self._r.completion(model=model, messages=messages, timeout=timeout, max_tokens=max_tokens, **kw)


class _Chat:
    def __init__(self, router: Router):
        self.completions = _Completions(router)


class _TextCompletions:
    def __init__(self, router: Router):
        self._r = router

    def create(self, model: str, prompt: Any, **kw) -> TextCompletionResponse:
        return self._r.text_completion(model=model, prompt=prompt, **kw)


class _Embeddings:
    def __init__(self, router: Router):
        self._r = router

    def create(self, model: str, input: Any, **kw) -> EmbeddingResponse:
        return self._r.embedding(model=model, input=input, **kw)


class OpenAI:
    """In-process stand-in for `openai.OpenAI(api_key=..., base_url=http://0.0.0.0:<port>)`
    (reference src/demo_load_balancing.py:24): same `client.chat.completions.create(...)` call."""

    def __init__(self, router: Router, api_key: str = "demo-key", base_url: Optional[str] = None):
        self.api_key = api_key
        self.base_url = base_url
        self.chat = _Chat(router)
        self.completions = _TextCompletions(router)
        self.embeddings = _Embeddings(router)
