"""semantic-router_b200: H100-native (sm_90a) signal-extraction hot path of vllm-project/semantic-router.

The product is the C-ABI shared library `lib/libcandle_semantic_router.so` (hand-written sm_90a CUDA behind
the ABI that candle-binding/semantic-router.go links).  This Python package is the host-side mirror used by
the tests and the benchmark: thin ctypes wrappers, no torch types in any signature, NO CPU fallback --
importing works without a GPU (symbol checks), every compute call requires the CUDA library and an sm_90 device.
"""
from .binding import (HOOKS_LIB_PATH, LIB_PATH, Cache, LoraSharedModel, Model, SrError, device_count, hooks, lib, load_library,  # noqa: F401
                      merge_topk, pack)

__all__ = ["Model", "LoraSharedModel", "Cache", "SrError", "lib", "load_library", "device_count", "LIB_PATH", "HOOKS_LIB_PATH", "hooks", "merge_topk", "pack"]
