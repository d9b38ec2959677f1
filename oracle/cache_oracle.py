"""Semantic-cache lookup oracle (TEST INFRASTRUCTURE ONLY; see encoder_oracle.py header).

Restates, in numpy fp32:
  * embeddingDotProduct + scanLinearForSimilarity + threshold test
    (src/semantic-router/pkg/cache/inmemory_cache_search.go:14-20,65-89,176):
    sequential f32 dot product, best updated on strict `>` (first max wins), nil/expired skipped,
    hit iff best >= threshold.
  * calculate_similarity_batch top-k (candle-binding/src/ffi/embedding.rs:1640-1681):
    cosine = dot/(|q||c|) in f32, STABLE sort descending (ties keep the lower index first), take k
    (k <= 0 or k > n  =>  n).
  * BertSimilarity::find_most_similar (candle-binding/src/core/similarity.rs:278-308): best = -1.0,
    strict `>`.
PARITY STATUS: integer/index semantics restated exactly; the Go toolchain is absent so the Go loop
itself cannot be run here ("parity unpinned" by execution; pinned by the reference's behavioural
tests re-run in tests/test_oracle_pins.py).  cache_scan.c is the same loop in C (CPU baseline).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional, Tuple

import numpy as np


def scan_linear(query: np.ndarray, entries: np.ndarray, valid: Optional[np.ndarray] = None,
                threshold: float = 0.8) -> Tuple[int, float, bool]:
    """scanLinearForSimilarity: returns (bestIndex, bestSimilarity, hit)."""
    q = query.astype(np.float32)
    best_idx, best = -1, np.float32(0.0)
    # vectorised per-row sequential-order dot is too slow in python; f32 matmul then tie rule.
    scores = (entries.astype(np.float32) @ q).astype(np.float32)
    for i, s in enumerate(scores):
        if valid is not None and not valid[i]:
            continue
        if best_idx == -1 or s > best:
            best, best_idx = s, i
    return best_idx, float(best), bool(best_idx >= 0 and best >= np.float32(threshold))


def topk_batch(queries: np.ndarray, entries: np.ndarray, k: int,
               valid: Optional[np.ndarray] = None, normalise: bool = False):
    """Top-k per query with the reference tie rule (stable sort: lower index first).

    queries [B,D], entries [N,D] float32 (values already rounded to whatever the store holds).
    Returns (idx int32 [B,k], score float32 [B,k]); slots beyond the number of valid rows are
    (-1, -inf).  With normalise=True scores are cosine (embedding.rs:1652-1659).
    """
    q = queries.astype(np.float32)
    e = entries.astype(np.float32)
    n = e.shape[0]
    kk = n if (k <= 0 or k > n) else k
    out_i = np.full((q.shape[0], kk), -1, dtype=np.int32)
    out_s = np.full((q.shape[0], kk), -np.inf, dtype=np.float32)
    en = np.linalg.norm(e, axis=1) if normalise else None
    blk = max(1, (1 << 27) // max(n, 1))
    for b0 in range(0, q.shape[0], blk):
        s = (q[b0:b0 + blk] @ e.T).astype(np.float32)
        if normalise:
            qn = np.linalg.norm(q[b0:b0 + blk], axis=1)
            denom = qn[:, None] * en[None, :]
            s = np.where(denom > 0, s / np.where(denom > 0, denom, 1), 0).astype(np.float32)
        if valid is not None:
            s[:, ~valid] = -np.inf
        # stable descending sort == argsort of (-score) with kind='stable'
        order = np.argsort(-s, axis=1, kind="stable")[:, :kk]
        sc = np.take_along_axis(s, order, axis=1)
        order = np.where(np.isneginf(sc), -1, order)
        out_i[b0:b0 + blk] = order.astype(np.int32)
        out_s[b0:b0 + blk] = sc
    return out_i, out_s


def find_most_similar(query: np.ndarray, cands: np.ndarray) -> Tuple[int, float]:
    """core/similarity.rs:278-308: best=-1.0, strict `>` => first max wins; (-1,-1.0) if no candidates."""
    best, idx = np.float32(-1.0), -1
    for i, c in enumerate(cands):
        s = np.float32(np.dot(query.astype(np.float32), c.astype(np.float32)))
        if s > best:
            best, idx = s, i
    return idx, float(best)


def merge_topk(idx_parts, score_parts, k: int):
    """k-way merge of per-shard (score, GLOBAL id) lists (SURVEY 8e): descending score, lower global
    index wins ties.  idx_parts/score_parts: lists of [B,k] arrays."""
    idx = np.concatenate(idx_parts, axis=1).astype(np.int64)
    sc = np.concatenate(score_parts, axis=1).astype(np.float32)
    big = np.iinfo(np.int64).max
    key_idx = np.where(idx < 0, big, idx)
    order = np.lexsort((key_idx, -sc), axis=1)[:, :k]
    return (np.take_along_axis(idx, order, 1).astype(np.int32),
            np.take_along_axis(sc, order, 1))


# ---- C restatement of the Go scalar loop (CPU baseline for the scan) -------------------------
_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libcache_scan.so")


def build_c() -> str:
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    src = os.path.join(_HERE, "cache_scan.c")
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-o", _SO, src])
    return _SO


def scan_linear_c(queries: np.ndarray, entries: np.ndarray, threads: int = 0):
    """Go-equivalent scalar scan for each query (best index + score), optionally OpenMP over queries."""
    lib = ctypes.CDLL(build_c())
    q = np.ascontiguousarray(queries, dtype=np.float32)
    e = np.ascontiguousarray(entries, dtype=np.float32)
    bi = np.empty(q.shape[0], dtype=np.int32)
    bs = np.empty(q.shape[0], dtype=np.float32)
    lib.oracle_scan_linear.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_int]
    lib.oracle_scan_linear(q.ctypes.data, e.ctypes.data, q.shape[0], e.shape[0], e.shape[1],
                           bi.ctypes.data, bs.ctypes.data, threads)
    return bi, bs
