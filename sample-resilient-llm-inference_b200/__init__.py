"""GPU-native (H100) request router + model replicas (drop-in for the litellm.Router hot path of
aws-samples/sample-resilient-llm-inference).  See DESIGN.md.

Importing this package loads librr_b200.so; there is no CPU fallback.
"""
from . import _lib  # noqa: F401  (fails loudly if the CUDA extension is missing)
from ._lib import RRError, lib  # noqa: F401
from .config import RouterConfig, build_config, load_config, strip_provider  # noqa: F401
from .models import SPECS, ModelSpec, Weights, make_weights, resolve_spec, broadcast_weights  # noqa: F401
from .router import (APIError, APITimeoutError, BadRequestError, EngineBackend, ModelResponse,  # noqa: F401
                     OpenAI, RateLimitError, Router, ServiceUnavailableError, StubBackend,
                     count_tokens, detokenize, tokenize)


def __getattr__(name):
    if name == "Engine":           # imports torch.cuda lazily
        from .engine import Engine
        return Engine
    raise AttributeError(name)


__all__ = ["lib", "RRError", "Router", "OpenAI", "RateLimitError", "APIError", "BadRequestError",
           "APITimeoutError", "ServiceUnavailableError", "ModelResponse", "StubBackend", "EngineBackend",
           "Engine", "load_config", "build_config", "RouterConfig", "SPECS", "ModelSpec", "make_weights",
           "resolve_spec", "tokenize", "detokenize", "count_tokens"]
