"""Oracle of exact caches (sr_cache_create_exact; TEST INFRASTRUCTURE ONLY).

Restates src/semantic-router/pkg/cache/inmemory_cache_search.go:14-20 (embeddingDotProduct: sequential f32 sum in index
order) under both ways the Go compiler evaluates `dot += q[i] * c[i]`, through the C restatement cache_exact_scan.c, the
top-k an exact cache must return (descending score, lower index first on ties), and the bound eps of
csrc/cache_scan.cu exact_eps.  PARITY STATUS: restated, not executed against the Go code (no Go toolchain).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libcache_exact_scan.so")


def build_c() -> str:
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    src = os.path.join(_HERE, "cache_exact_scan.c")
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-o", _SO, src, "-lm"])
    return _SO


def scores_go(queries: np.ndarray, entries: np.ndarray, rule: int, threads: int = 0) -> np.ndarray:
    """embeddingDotProduct of every query with every entry, [B, N] float32, under `rule`: 0 rounds each product to f32 and
    then adds (Go on amd64 at GOAMD64=v1), 1 is one fused multiply-add per term (Go on arm64 and amd64 v3+)."""
    assert rule in (0, 1)
    lib = ctypes.CDLL(build_c())
    q = np.ascontiguousarray(queries, dtype=np.float32)
    e = np.ascontiguousarray(entries, dtype=np.float32)
    out = np.empty((q.shape[0], e.shape[0]), dtype=np.float32)
    lib.oracle_scores_go.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_int]
    lib.oracle_scores_go(q.ctypes.data, e.ctypes.data, q.shape[0], e.shape[0], q.shape[1], rule, out.ctypes.data, threads)
    return out


def topk_go(queries: np.ndarray, entries: np.ndarray, k: int, rule: int, valid: Optional[np.ndarray] = None,
            id_offset: int = 0):
    """What an exact cache returns: the Go scores of the valid entries, descending, lower index first on ties, k of them;
    (-1, -inf) past the valid entries.  Returns (idx int32 [B, k], score float32 [B, k])."""
    s = scores_go(queries, entries, rule)
    if valid is not None:
        s[:, ~np.asarray(valid, bool)] = -np.inf
    order = np.argsort(-s, axis=1, kind="stable")[:, :k]
    sc = np.take_along_axis(s, order, axis=1)
    idx = np.where(np.isneginf(sc), -1, order + id_offset).astype(np.int32)
    if idx.shape[1] < k:
        pad = k - idx.shape[1]
        idx = np.pad(idx, ((0, 0), (0, pad)), constant_values=-1)
        sc = np.pad(sc, ((0, 0), (0, pad)), constant_values=-np.inf)
    return idx, sc.astype(np.float32)


def exact_eps(q_norm: float, r_max: float, d: int) -> float:
    """The bound on |fp16-operand score - Go score| of csrc/cache_scan.cu exact_eps (its comment derives it): fp16
    rounding of both operands, the scan's fp32 sum at 8 times the unit roundoff, Go's own sum and underflow."""
    dd, h, u = 2.0 ** -11, 2.0 ** -25, 2.0 ** -24
    S = np.sqrt(float(d))
    g, g8 = d * u / (1 - d * u), d * 8 * u / (1 - d * 8 * u)
    cross = h * (1 + dd) * S * (q_norm + r_max) + d * h * h
    e1 = (2 * dd + dd * dd) * q_norm * r_max + cross
    e2 = g8 * ((1 + dd) * (1 + dd) * q_norm * r_max + cross)
    e3 = g * q_norm * r_max
    e4 = 2.0 * d * 2.0 ** -149
    return (e1 + e2 + e3 + e4) * (1 + 2.0 ** -20)
