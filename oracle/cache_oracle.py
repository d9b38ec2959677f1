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


# ---- conformance of csrc/cache_scan.cu: exact-score families, stage-1 trace, restated selection -------------------
# Stored rows and queries hold entries m * 2^-4 with |m| <= 16 (exact in fp16) and few non-zeros.  Every product is a
# multiple of 2^-8, and while sum |q| |r| < 2^(24-8) every fp32 partial sum is a multiple of 2^-8 below 2^16, which fp32
# holds exactly: the GEMV's fmaf chains and shuffle tree, and the wgmma accumulation, return the float64 score in any
# order.  On these families the whole expected list (ids and scores) is determined by the tie rule.
SEGMENT = 8192            # stage-1 rows per CTA (kSegment)
WARP_ROWS = 1024          # stage-1 rows per warp, 32 per lane: row = warp base + j * 32 + lane
LIST_CAP = 128            # kListCap: candidates a warp compacts before it falls back to k passes
EXACT_LIMIT = 2.0 ** 16   # sum |q| |r| must stay below this


class Family:
    """rows [N, D], queries [B, D] float32 (fp16-exact), valid [N] bool; `plateaus` = list of (first row, rows, query
    set) for the coverage report; `name` for messages."""

    def __init__(self, name, rows, queries, valid, plateaus=()):
        self.name, self.rows, self.queries, self.valid, self.plateaus = name, rows, queries, valid, list(plateaus)

    def sum_abs_bound(self) -> float:
        """max over pairs of sum |q| |r|: the exactness condition is sum_abs_bound() < 2^16."""
        qa = np.abs(self.queries).astype(np.float64)
        ra = np.abs(self.rows).astype(np.float64)
        return float((qa.max(0) * ra.max(0)).sum()) if len(ra) else 0.0

    def check_exact(self):
        for a in (self.rows, self.queries):
            m = a.astype(np.float64) * 16
            assert np.array_equal(m, np.round(m)) and np.abs(m).max(initial=0) <= 16, self.name
            assert np.array_equal(a.astype(np.float16).astype(np.float32), a), self.name
        assert self.sum_abs_bound() < EXACT_LIMIT, self.name

    def scores64(self):
        return self.queries.astype(np.float64) @ self.rows.astype(np.float64).T


def _sparse(rng, n, d, lo, hi, nnz, mag):
    """n rows over columns [lo, hi) of d: nnz non-zeros each, m * 2^-4 with 1 <= |m| <= mag."""
    out = np.zeros((n, d), np.float32)
    if n == 0 or hi <= lo:
        return out
    cols = lo + rng.integers(0, hi - lo, size=(n, nnz))      # a repeated column leaves fewer non-zeros
    vals = rng.integers(1, mag + 1, size=(n, nnz)) * rng.choice([-1, 1], size=(n, nnz))
    np.put_along_axis(out, cols, (vals / 16.0).astype(np.float32), axis=1)
    return out


def family(kind: str, n: int, d: int, b: int, seed: int, plateaus=(), hot: int = 4, ladders=()):
    """An exact-score family of n rows, dimension d and b queries.

    Columns [0, hot) are "hot channels", the rest background.  Background rows have two non-zeros of magnitude <= 8/16
    among the background columns, queries four of magnitude <= 4/16, so every background score lies in [-1/4, 1/4] and
    falls on a 2^-8 grid: long natural tie runs.  Plateau p (first row, rows) holds copies of one row, 1.0 on hot channel
    p % hot and its own small background part; query i has 1.0 on hot channel i % hot, so the plateaus of that channel
    rank first for it, the lowest-index plateau's rows before the next one's only when their background parts tie.

    kind: "plateau" (the plateaus above), "all_equal" (every row the same), "all_negative" (every score < 0: the queries
    carry -1 on their hot channel and background rows a positive one), "sparse_valid" (plateaus, and only the rows
    listed in `plateaus` valid), "spread" (no hot channels: dense queries against eight non-zeros per row over the
    first 16 columns, so scores spread over hundreds of 2^-8 steps and most warps compact fewer than 128 candidates at
    k <= 32; plateaus are laid over it as given).  The caller invalidates further rows through `valid`.

    ladders: runs (first row, rows) of DISTINCT scores above every plateau and background row, rising with the row:
    the last three columns carry query weights (1, 1, 1/16) and ladder row j holds (1, (j // 16) / 16, (j % 16 - 8) / 16)
    there, for scores 1 + (16 (j // 16) + j % 16 - 8) / 256.  Inside one 1024-row warp window a ladder of 64 rows puts
    two rows on each lane, so the 32nd lane maximum bounds only 32 candidates: the k > 32 rule is what keeps the rest."""
    rng = np.random.default_rng(seed)
    hot = max(1, min(hot, d - 2))
    rows = _sparse(rng, n, d, hot, d, 2, 8)
    q = _sparse(rng, b, d, hot, d, 4, 4)
    q[np.arange(b), np.arange(b) % hot] = 1.0
    valid = np.ones(n, bool)
    pl = []
    if kind == "all_equal":
        rows[:] = rows[0]
    elif kind == "spread":
        w = min(d, 16)
        rows = _sparse(rng, n, d, 0, w, min(8, w), 16)
        q = np.zeros((b, d), np.float32)
        q[:, :w] = rng.integers(-2, 3, size=(b, w)) / 16.0          # scores in [-1, 1], about 37 steps per sigma
    elif kind == "all_negative":
        rows[:, :hot] = rng.integers(12, 17, size=(n, hot)) / 16.0   # background scores -1.25 .. -0.5
        q[np.arange(b), np.arange(b) % hot] = -1.0
    for p, (r0, cnt) in enumerate(plateaus):
        r0, r1 = max(0, r0), min(n, r0 + cnt)
        if r1 <= r0:
            continue
        v = np.zeros(d, np.float32)
        v[p % hot] = 1.0
        v[hot:] = _sparse(rng, 1, d - hot, 0, d - hot, 2, 2)[0]
        if kind == "all_negative":
            v[:hot] = 0.25                                          # plateau scores -0.25 +- 1/16
        rows[r0:r1] = v
        pl.append((r0, r1 - r0, p % hot))
    if ladders:
        assert d >= hot + 5 and kind in ("plateau", "spread", "sparse_valid"), (kind, d)
        rows[:, d - 3:] = 0.0
        q[:, d - 3:] = [1.0, 1.0, 1.0 / 16]
        for r0, cnt in ladders:
            j = np.arange(cnt)
            rows[r0:r0 + cnt] = 0.0
            rows[r0:r0 + cnt, d - 3] = 1.0
            rows[r0:r0 + cnt, d - 2] = (j // 16) / 16.0
            rows[r0:r0 + cnt, d - 1] = (j % 16 - 8) / 16.0
            pl.append((r0, cnt, -1))
    if kind == "sparse_valid":
        valid[:] = False
        for r0, cnt, _ in pl:
            valid[r0:r0 + cnt] = True
    f = Family(kind, rows, q, valid, pl)
    f.check_exact()
    return f


def topk_ref(queries, rows, k, valid=None, block=64, device=None):
    """gemm_oracle.topk of the float64 scores, in query blocks (a [1024, 1.1 M] float64 matrix never exists at once).
    numpy / torch in, (idx int64 [B, k], score float64 [B, k]) numpy out."""
    import torch
    from oracle import gemm_oracle as go
    dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
    r = torch.as_tensor(np.asarray(rows, np.float64), device=dev)
    v = None if valid is None else torch.as_tensor(np.asarray(valid, bool), device=dev)
    qs = np.asarray(queries, np.float64)
    outs_i, outs_s = [], []
    step = max(1, min(block, (1 << 27) // max(1, r.shape[0])))
    for b0 in range(0, qs.shape[0], step):
        s = torch.as_tensor(qs[b0:b0 + step], device=dev) @ r.t()
        i, sc = go.topk(s, k, v)
        outs_i.append(i.cpu().numpy())
        outs_s.append(sc.cpu().numpy())
    return np.concatenate(outs_i), np.concatenate(outs_s)


def _lane_bound(v, k, k32_override=True):
    """v [..., 32 (j), 32 (lane)] of one warp: the stage-1 bound L per warp (the min(k, 32)-th largest lane maximum,
    -inf for k > 32)."""
    lm = v.max(axis=-2)                                    # [..., 32] lane maxima
    L = -np.sort(-lm, axis=-1)[..., min(k, 32) - 1]
    if k > 32 and k32_override:
        L = np.full_like(L, -np.inf)
    return L


def _warp_view(scores, valid, n_pad):
    """scores [B, N] -> [B, warps, 32 (j), 32 (lane)] fp32 with invalid and padding rows at -inf."""
    s = np.asarray(scores, np.float32).copy()
    if valid is not None:
        s[:, ~np.asarray(valid, bool)] = -np.inf
    B, N = s.shape
    full = np.full((B, n_pad), -np.inf, np.float32)
    full[:, :N] = s
    return full.reshape(B, n_pad // WARP_ROWS, 32, 32)


def stage1_trace(scores, valid, k, chunk_rows=None):
    """Restatement of select_stage1's bound and candidate count per (query, warp) of the score chunks: returns
    (count [B, warps], fallback [B, warps] bool), warp w covering local rows of chunk c = w // (chunk_rows / 1024).
    Only proves coverage (which warps take the k-pass fallback); correctness comes from the float64 reference."""
    B, N = np.shape(scores)
    chunk_rows = chunk_rows or max(SEGMENT, -(-N // SEGMENT) * SEGMENT)
    counts, falls = [], []
    for r0 in range(0, N, chunk_rows):
        n = min(chunk_rows, N - r0)
        vv = None if valid is None else np.asarray(valid)[r0:r0 + n]
        w = _warp_view(np.asarray(scores)[:, r0:r0 + n], vv, -(-n // SEGMENT) * SEGMENT)
        L = _lane_bound(w, k)
        cnt = ((w >= L[..., None, None]) & (w != -np.inf)).sum(axis=(-2, -1))
        counts.append(cnt)
        falls.append(cnt > LIST_CAP)
    return np.concatenate(counts, 1), np.concatenate(falls, 1)


def _take(v, i, k, reverse_ties=False):
    """The kernels' k rounds of argmax with better(): descending score, then the lower index (the higher one with
    reverse_ties); index -1 never wins.  v, i [..., m] -> [..., k]."""
    v = np.where(i < 0, -np.inf, v).astype(np.float64)
    key_i = (-i if reverse_ties else i).astype(np.int64)
    none = i < 0                  # sort keys, most significant last: slots with index -1 last, score down, index up

    order = np.lexsort((key_i, -v, none), axis=-1)[..., :k]
    ov = np.take_along_axis(v, order, -1)
    oi = np.take_along_axis(i, order, -1)
    oi = np.where(np.take_along_axis(none, order, -1), -1, oi)
    ov = np.where(oi < 0, -np.inf, ov)
    if ov.shape[-1] < k:
        pad = [(0, 0)] * (ov.ndim - 1) + [(0, k - ov.shape[-1])]
        ov = np.pad(ov, pad, constant_values=-np.inf)
        oi = np.pad(oi, pad, constant_values=-1)
    return ov, oi


def select_two_stage(scores, valid, k, chunk_rows=None, id_offset=0, mutate=()):
    """numpy restatement of the two-pass selection of cache_topk: per score chunk, select_stage1 (per warp the bound L,
    the compacted list or the k-pass fallback, then warp 0's merge of the eight warp lists into the chunk segment's
    entry seg0 + seg), then select_stage2 over all segment entries.  Returns (idx int64 [B, k], score float64 [B, k]).

    mutate: "gt" (candidates v > L instead of >=), "no_k32" (no -inf bound for k > 32), "tie1" / "tie2" (the reversed
    index tie rule in stage 1 / stage 2), "seg0" (every chunk writes its segments from entry 0)."""
    B, N = np.shape(scores)
    chunk_rows = chunk_rows or max(SEGMENT, -(-N // SEGMENT) * SEGMENT)
    segs = -(-N // SEGMENT)
    cand_v = np.full((B, segs, k), -np.inf)
    cand_i = np.full((B, segs, k), -1, np.int64)
    wpseg = SEGMENT // WARP_ROWS
    for r0 in range(0, N, chunk_rows):
        n = min(chunk_rows, N - r0)
        vv = None if valid is None else np.asarray(valid)[r0:r0 + n]
        nseg = -(-n // SEGMENT)
        w = _warp_view(np.asarray(scores)[:, r0:r0 + n], vv, nseg * SEGMENT).astype(np.float64)   # [B, W, 32, 32]
        W = w.shape[1]
        idx = r0 + (np.arange(W)[:, None, None] * WARP_ROWS + np.arange(32)[None, :, None] * 32 +
                    np.arange(32)[None, None, :])
        idx = np.broadcast_to(idx, w.shape)
        L = _lane_bound(w, k, k32_override="no_k32" not in mutate)[..., None, None]
        cand = ((w > L) if "gt" in mutate else (w >= L)) & (w != -np.inf)
        count = cand.sum(axis=(-2, -1))
        flat_v, flat_i, flat_c = w.reshape(B, W, -1), idx.reshape(B, W, -1), cand.reshape(B, W, -1)
        fast_v, fast_i = _take(flat_v, np.where(flat_c, flat_i, -1), k, "tie1" in mutate)
        live = flat_v != -np.inf
        slow_v, slow_i = _take(flat_v, np.where(live, flat_i, -1), k, "tie1" in mutate)
        fb = (count > LIST_CAP)[..., None]
        wv, wi = np.where(fb, slow_v, fast_v), np.where(fb, slow_i, fast_i)          # [B, W, k]
        sv, si = _take(wv.reshape(B, nseg, wpseg * k), wi.reshape(B, nseg, wpseg * k), k, "tie1" in mutate)
        s0 = 0 if "seg0" in mutate else r0 // SEGMENT
        cand_v[:, s0:s0 + nseg], cand_i[:, s0:s0 + nseg] = sv, si
    ov, oi = _take(cand_v.reshape(B, -1), cand_i.reshape(B, -1), k, "tie2" in mutate)
    return np.where(oi >= 0, oi + id_offset, -1), ov


def merge_packed(idx_parts, score_parts, k, mutate=()):
    """numpy restatement of merge_packed_kernel over G lists [G, B, k] of (score, GLOBAL id); mutate "tiepack": the
    reversed index tie rule."""
    ip = np.asarray(idx_parts, np.int64)
    sp = np.asarray(score_parts, np.float64)
    G, B, kk = ip.shape
    ov, oi = _take(sp.transpose(1, 0, 2).reshape(B, G * kk), ip.transpose(1, 0, 2).reshape(B, G * kk), k,
                   "tiepack" in mutate)
    return oi, ov


def gap_rule_check(got_idx, got_score, scores64, bound, valid, k):
    """The rule of test_gemm_conformance_gpu.py::test_cache_scan for inexact scores (torch, on one device): every
    returned id is valid, the list descends, each score lies within `bound` of its float64 score, and ranks whose float64
    gaps to both neighbours exceed twice the largest bound hold exactly the reference's id.  Returns the failures."""
    import torch
    from oracle import gemm_oracle as go
    dev = scores64.device
    n = scores64.shape[1]
    idx_t = torch.as_tensor(np.asarray(got_idx, np.int64), device=dev)
    sc_t = torch.as_tensor(np.asarray(got_score, np.float64), device=dev)
    bad = []
    if not ((idx_t >= 0).all() and (idx_t < n).all() and valid[idx_t.clamp(0, n - 1)].all()):
        return ["invalid or out-of-range id"]
    if not (sc_t[:, 1:] <= sc_t[:, :-1]).all():
        bad.append("scores do not descend")
    if not ((sc_t - scores64.gather(1, idx_t)).abs() <= bound.gather(1, idx_t)).all():
        bad.append("score outside the bound")
    ref_idx, ref_val = go.topk(scores64, k + 1, valid)
    bmax = torch.where(valid[None, :], bound, torch.zeros_like(bound)).max(1).values[:, None]
    gaps = ref_val[:, :-1] - ref_val[:, 1:]
    above = torch.cat([torch.full_like(gaps[:, :1], torch.inf), gaps[:, :k - 1]], 1)
    sure = (above > 2 * bmax) & (gaps[:, :k] > 2 * bmax)
    wrong = sure & (idx_t != ref_idx[:, :k])
    if wrong.any():
        bad.append(f"ids differ where the gaps are sure: {torch.nonzero(wrong)[:4].tolist()}")
    return bad
