"""Conformance of the cache scan's selection and merge (csrc/cache_scan.cu, and the GEMM's fused top-8 epilogue) through
the C ABI (sr_cache_*), against float64.

* Exact-score families (oracle/cache_oracle.py: family): every score is exact in fp32, so ids AND scores must equal the
  float64 reference bitwise, ties resolved lower index first.  Plateaus of identical rows sit inside one 1024-row warp
  window (> 128 of them: stage 1's k-pass fallback), across warp windows, 8192-row segments, 128-row tiles, worker
  ranges and score chunks; ladders of distinct scores inside one warp window need the k > 32 rule.
* Every case asserts the route it covers through sr_test_cache_plan: GEMV + two-stage (B <= 4, B D 4 <= 48 KB), GEMM +
  two-stage, fused top-8 (B > 4, k <= 8), multi-chunk, stage 2 above 48 KB, and the refusals.
* Random unit vectors at the dimension edges keep the score bound and gap rule of test_cache_scan.
* The sharded exchange (sr_cache_topk_packed_dev + sr_cache_merge_packed_dev) on one GPU equals the unsharded scan and
  the host merge.

Run with -s for the cases per route and the stage-1 warps that took the fallback (oracle stage1_trace)."""
import ctypes as C
import math
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import cache_oracle as co
from oracle import gemm_oracle as go

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, W = co.SEGMENT, co.WARP_ROWS
ROUTE_NAMES = {-1: "refused", 0: "empty", 1: "fused", 2: "gemv", 3: "gemm"}
KS = [1, 8, 9, 16, 32, 33, 64]
CASES = Counter()      # cases per route
FALLBACK = Counter()   # stage-1 warps per (route, branch) on the first queries of each two-stage case


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ncache scan cases per route:", dict(CASES))
    print("stage-1 warps per branch (first 8 queries of each two-stage case):", dict(FALLBACK))


@pytest.fixture(scope="module")
def hooks(srlib, cuda):
    return srlib.binding.hooks()


def plan(hooks, b, n, d, k):
    route, chunks, cands = C.c_int(9), C.c_int(0), C.c_int(0)
    rc = hooks.sr_test_cache_plan(b, n, d, k, C.byref(route), C.byref(chunks), C.byref(cands))
    return rc, route.value, chunks.value, cands.value


def expect_route(b, n, d, k):
    if n == 0:
        return 0
    if b > 4 and k <= 8:
        return 1
    return 2 if b <= 4 and b * d * 4 <= 48 * 1024 else 3


def make_cache(srlib, rows, valid=None, id_offset=0, capacity=None):
    c = srlib.Cache(capacity or max(1, len(rows)), rows.shape[1], device=0, id_offset=id_offset)
    if len(rows):
        c.add(rows)
    if valid is not None:
        for r in np.nonzero(~valid)[0]:
            c.invalidate(int(r))
    return c


def _scores(f, m):
    """float64 scores of the first m queries (exact: equal to fp32)"""
    q = torch.from_numpy(f.queries[:m].astype(np.float64)).cuda()
    return (q @ torch.from_numpy(f.rows.astype(np.float64)).cuda().t()).cpu().numpy()


def trace(route, f, k, chunk_rows):
    cnt, fb = co.stage1_trace(_scores(f, 8), f.valid, k, chunk_rows)
    FALLBACK[(ROUTE_NAMES[route], "k>32" if k > 32 else "k<=32", "fallback")] += int(fb.sum())
    FALLBACK[(ROUTE_NAMES[route], "k>32" if k > 32 else "k<=32", "list")] += int((~fb).sum())


def check_exact(hooks, cache, f, k, b=None, tag=""):
    """ids and scores of the ABI bitwise equal to float64 on an exact family; asserts and counts the route."""
    q = f.queries if b is None else f.queries[:b]
    n, d = f.rows.shape
    rc, route, chunks, _ = plan(hooks, q.shape[0], n, d, k)
    assert rc == 0 and route == expect_route(q.shape[0], n, d, k), (tag, rc, route)
    idx, sc = cache.topk(q, k)
    ri, rv = co.topk_ref(q, f.rows, k, f.valid)
    bad = (idx != ri) | (sc.astype(np.float64) != rv)
    if bad.any():
        i, r = [int(x) for x in np.argwhere(bad)[0]]
        raise AssertionError(f"{tag} {f.name} B={q.shape[0]} k={k} route={ROUTE_NAMES[route]}: {int(bad.sum())} "
                             f"entries differ; first query {i} rank {r}: got ({idx[i, r]}, {sc[i, r]!r}), float64 "
                             f"({ri[i, r]}, {rv[i, r]!r}); got ids {idx[i, max(0, r - 3):r + 4].tolist()} want "
                             f"{ri[i, max(0, r - 3):r + 4].tolist()}")
    CASES[ROUTE_NAMES[route]] += 1
    if route in (2, 3):
        trace(route, f, k, None)
    return route, chunks


def edge_plateaus(n, hot):
    """Plateaus of 9..600 rows: > 128 inside one warp window, and across a warp window, a segment, 128-row tiles."""
    pl = [(3 * W + 10, 129), (6 * W, 600), (10 * W - 70, 140), (S - 300, 600), (128 * 50 - 5, 9),
          (128 * 77 - 100, 250), (S + 128 * 9 - 20, 40), (2 * S - 4, 300)]
    if n < 4096:
        pl = [(60, 9), (128 * 3 - 4, 9), (128 * 2 - 60, 129), (128 * 5 - 100, 300)]
    return [(a, c) for a, c in pl if a + c <= n][:max(hot, 8)]


# ---------------------------------------------------------------------------------------------------------------------
# routes x k on exact families
# ---------------------------------------------------------------------------------------------------------------------
ROUTE_CASES = {   # name: (B values, N, D)
    "gemv": ((1, 2, 3, 4), 20000, 64),
    "fused_one_block": ((5, 128), 20000, 64),
    "fused_grouped": ((300,), 20000, 64),
    "fused_few_tiles": ((300,), 1000, 64),
}


@pytest.mark.parametrize("case", list(ROUTE_CASES))
def test_routes_by_k(srlib, hooks, case):
    bs, n, d = ROUTE_CASES[case]
    fams = [co.family("plateau", n, d, max(bs), 11 + n, plateaus=edge_plateaus(n, 8), hot=8),
            co.family("spread", n, d, max(bs), 12 + n, ladders=[(5 * W + 64, 64)] if n > 6 * W else [(0, 64)],
                      plateaus=[(3000, 200)] if n > 4000 else [])]
    for f in fams:
        cache = make_cache(srlib, f.rows, f.valid)
        try:
            for b in bs:
                for k in KS:
                    check_exact(hooks, cache, f, k, b, case)
        finally:
            cache.close()


@pytest.mark.parametrize("b,d", [(3, 4096), (3, 4104), (4, 4096)])
def test_score_memory_edge_of_the_gemv(srlib, hooks, b, d):
    """B D 4 = 48 KB exactly stays on the GEMV; just above it the GEMM scores B <= 4 queries."""
    n = 9000
    assert plan(hooks, b, n, d, 9)[1] == (2 if b * d * 4 <= 48 * 1024 else 3)
    f = co.family("plateau", n, d, b, d + b, plateaus=edge_plateaus(n, 8), hot=8)
    cache = make_cache(srlib, f.rows, f.valid)
    try:
        for k in KS:
            check_exact(hooks, cache, f, k, None, f"D{d}")
    finally:
        cache.close()


FAMILY_CASES = [(2, 20000), (7, 20000), (300, 20000)]


@pytest.mark.parametrize("b,n", FAMILY_CASES)
def test_tie_families(srlib, hooks, b, n):
    """Cut ties, an all-equal store, all-negative scores, fewer valid rows than k spread over warps and segments, and the
    lowest-index members of plateaus invalidated, on the GEMV, GEMM and fused routes."""
    pl = edge_plateaus(n, 8)
    fams = [co.family("plateau", n, 64, b, 21, plateaus=[(100 + 50 * p, 8) for p in range(8)], hot=8),
            co.family("all_equal", n, 64, b, 22),
            co.family("all_negative", n, 64, b, 23, plateaus=pl[:4], hot=8),
            co.family("sparse_valid", 12000, 64, b, 24, plateaus=[(7, 1), (W + 3, 2), (S + 1, 1), (11999, 1)], hot=8)]
    inv = co.family("plateau", n, 64, b, 25, plateaus=pl, hot=8)
    for a, c in pl:
        inv.valid[a:a + min(c - 1, 37)] = False
    inv.name = "invalidated"
    fams.append(inv)
    for f in fams:
        cache = make_cache(srlib, f.rows, f.valid)
        try:
            for k in KS:
                check_exact(hooks, cache, f, k)
        finally:
            cache.close()


@pytest.mark.parametrize("d", [8, 4096, 4104])
def test_random_unit_vectors_at_dimension_edges(srlib, hooks, d):
    """Inexact scores: each within the bound of test_cache_scan, ids exact wherever the float64 gaps are sure."""
    n = 9001 if d > 8 else 60000
    rng = np.random.default_rng(d)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    valid = np.ones(n, bool)
    valid[rng.choice(n, 200, replace=False)] = False
    cache = make_cache(srlib, rows, valid)
    try:
        r64 = torch.from_numpy(rows.astype(np.float16).astype(np.float64)).cuda()
        vmask = torch.from_numpy(valid).cuda()
        for b in (1, 3, 4, 7, 300):
            q = rng.standard_normal((b, d)).astype(np.float32)
            q /= np.linalg.norm(q, axis=1, keepdims=True)
            q64 = torch.from_numpy(q.astype(np.float16).astype(np.float64)).cuda()
            sc64 = q64 @ r64.t()
            for k in (1, 8, 9, 33, 64):
                route = plan(hooks, b, n, d, k)[1]
                tau = max(go.TAU, (8 * math.ceil(d / 256) + 6) * go.U32) if route == 2 else go.TAU
                bound = tau * (q64.abs() @ r64.abs().t())
                idx, sc = cache.topk(q, k)
                bad = co.gap_rule_check(idx, sc, sc64, bound, vmask, k)
                assert not bad, (d, b, k, ROUTE_NAMES[route], bad)
                CASES[ROUTE_NAMES[route] + "-random"] += 1
    finally:
        cache.close()


# ---------------------------------------------------------------------------------------------------------------------
# multi-chunk, large stage 2, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_multi_chunk(srlib, hooks):
    """B = 1024 at k = 9: the 1 GiB score buffer holds 262144 rows, so N = 300000 runs as two chunks whose stage-1
    candidates land at segments 0.. and 32..; plateaus straddle row 262144."""
    b, n, d, k = 1024, 300000, 64, 9
    rc, route, chunks, cands = plan(hooks, b, n, d, k)
    assert (rc, route, chunks, cands) == (0, 3, 2, 37 * k)
    edge = 262144
    pl = [(edge - 70, 140), (edge - 5, 9), (edge - 300, 600), (edge + 3 * W - 64, 129)] + edge_plateaus(n, 8)[:4]
    f = co.family("plateau", n, d, b, 31, plateaus=pl, hot=8)
    f.valid[edge - 70:edge - 66] = False
    cache = make_cache(srlib, f.rows, f.valid)
    try:
        check_exact(hooks, cache, f, k, None, "multi-chunk")
        cnt, fb = co.stage1_trace(_scores(f, 8), f.valid, k, edge)
        assert fb[:, edge // W].any()          # the plateau right after the chunk edge took the fallback
    finally:
        cache.close()


@pytest.mark.parametrize("n", [786432, 800000])
@pytest.mark.parametrize("b", [1, 5])
def test_stage2_above_48k(srlib, hooks, b, n):
    """k = 64 over 800000 rows: 98 segments x 64 candidates = 50176 bytes of stage-2 shared memory; over 786432 rows
    exactly 48 KB, which with stage 2's static shared memory is also more than a launch gets without opting in."""
    d, k = 8, 64
    rc, route, chunks, cands = plan(hooks, b, n, d, k)
    assert rc == 0 and route == (2 if b == 1 else 3) and cands * 8 >= 48 * 1024
    f = co.family("spread", n, d, b, 41 + b, ladders=[(S * 50 + 3 * W, 64)], plateaus=[(S * 97 + 10, 129)], hot=2)
    cache = make_cache(srlib, f.rows, f.valid)
    try:
        for kk in (33, 64):
            check_exact(hooks, cache, f, kk, None, "stage2>48K")
    finally:
        cache.close()


def _refused(srlib, cache, q, k):
    idx = np.full((q.shape[0], k), 0x5A5A5A5A, np.int32)
    sc = np.full((q.shape[0], k), np.nan, np.float32)
    sc.view(np.int32)[:] = 0x7FC0DEAD
    i0, s0 = idx.copy(), sc.copy()
    rc = srlib.lib().sr_cache_topk(cache.handle, q.ctypes.data, q.shape[0], k, idx.ctypes.data, sc.ctypes.data)
    assert rc == -1 and np.array_equal(idx, i0) and np.array_equal(sc.view(np.int32), s0.view(np.int32))


def test_stage2_limit_and_refusals(srlib, hooks):
    """ceil(N / 8192) k = 25600 (200 KB) is accepted at B = 1, D = 8; one row more is refused, as is k = 65; a refusal
    returns -1 and leaves the caller's outputs alone."""
    n, d = 3276800, 8
    assert plan(hooks, 1, n, d, 64)[:2] == (0, 2) and plan(hooks, 1, n, d, 64)[3] == 25600
    assert plan(hooks, 1, n + 1, d, 64)[:2] == (-1, -1)
    assert plan(hooks, 300, n + 1, d, 8)[:2] == (0, 1)       # the fused route has no candidate limit
    assert plan(hooks, 1, 100, d, 65)[0] == -1 and plan(hooks, 0, 100, d, 1)[0] == -1
    f = co.family("plateau", n, d, 1, 51, plateaus=[(n - S - 75, 150)], hot=2)   # across the last segment edge
    cache = make_cache(srlib, f.rows, None, capacity=n + 1)
    try:
        check_exact(hooks, cache, f, 64, None, "200K")
        cache.add(f.rows[-1:])
        q = np.ascontiguousarray(f.queries)
        _refused(srlib, cache, q, 64)
        _refused(srlib, cache, q, 65)
        CASES["refused"] += 2
    finally:
        cache.close()


# ---------------------------------------------------------------------------------------------------------------------
# the fused top-8 epilogue: ties across tiles and workers, and the contiguous schedule in a child process
# ---------------------------------------------------------------------------------------------------------------------
def _fused_family(n):
    pl = [(128 * t - 4, 9) for t in (3, 40, 77)] + [(128 * 11 - 60, 600), (128 * 90 - 200, 300), (128 * 120 + 1, 20),
                                                    (128 * 140 - 64, 129), (128 * 150 - 8, 16)]
    return co.family("plateau", n, 64, 300, 61, plateaus=[(a, c) for a, c in pl if a + c <= n], hot=8)


def test_fused_epilogue_ties(srlib, hooks):
    f = _fused_family(20000)
    cache = make_cache(srlib, f.rows, f.valid)
    try:
        for b in (5, 64, 128, 300):
            for k in (1, 2, 7, 8):
                check_exact(hooks, cache, f, k, b, "fused")
    finally:
        cache.close()


_CHILD = r'''
import os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "tests")]
import numpy as np
import semantic_router_b200 as pkg
import test_cache_topk_conformance_gpu as t
f = t._fused_family(20000)
c = t.make_cache(pkg, f.rows, f.valid)
res = {}
for b in (128, 300):
    res[f"i{b}"], res[f"s{b}"] = c.topk(f.queries[:b], 8)
c.close()
np.savez(sys.argv[2], **res)
'''


def test_fused_contiguous_schedule_bitwise(srlib, cuda, tmp_path):
    base = {k: v for k, v in os.environ.items() if not k.startswith("SRB_TOPK_GROUPED")}
    outs = {}
    for name, extra in (("default", {}), ("contiguous", {"SRB_TOPK_GROUPED": "0"})):
        path = tmp_path / f"{name}.npz"
        r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, str(path)], env=dict(base, **extra), cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, f"{name}: {r.stdout[-2000:]}\n{r.stderr[-4000:]}"
        outs[name] = np.load(path)
    f = _fused_family(20000)
    for key in outs["default"].files:
        assert outs["default"][key].tobytes() == outs["contiguous"][key].tobytes(), key
    for b in (128, 300):
        ri, rv = co.topk_ref(f.queries[:b], f.rows, 8, f.valid)
        assert np.array_equal(outs["contiguous"][f"i{b}"], ri) and np.array_equal(outs["contiguous"][f"s{b}"], rv)


# ---------------------------------------------------------------------------------------------------------------------
# the sharded exchange on one GPU
# ---------------------------------------------------------------------------------------------------------------------
def _shard_bounds(n, g):
    """g contiguous shards of [0, n): for g >= 3 one is empty and one holds 3 rows."""
    if g == 1:
        return [(0, n)]
    cuts = sorted({int(x) for x in np.linspace(0, n, g + 1)[1:-1]})
    if g >= 3:
        cuts[0] = cuts[1]                          # empty shard
        cuts[-1] = n - 3                           # a shard of 3 rows: fewer valid rows than k
    edges = [0] + cuts + [n]
    return list(zip(edges[:-1], edges[1:]))


@pytest.mark.parametrize("g", [1, 2, 3, 8])
def test_packed_shard_exchange(srlib, hooks, g):
    n, b = 20000, 8
    f = co.family("plateau", n, 64, b, 71, plateaus=[(a - 100, 200) for a in range(2500, n, 2500)], hot=8)
    bounds = _shard_bounds(n, g)
    order = list(np.random.default_rng(g).permutation(g))           # slot s holds shard order[s]
    lib = srlib.lib()
    whole = make_cache(srlib, f.rows, f.valid)
    shards = [make_cache(srlib, f.rows[a:e], f.valid[a:e], id_offset=a, capacity=max(1, e - a)) for a, e in bounds]
    stream = torch.cuda.Stream()
    q16 = torch.from_numpy(f.queries).cuda().half()
    torch.cuda.synchronize()
    try:
        for k in (1, 8, 33, 64):
            pairs = torch.full((g, b, k, 2), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
            oi = torch.empty(b, k, dtype=torch.int32, device="cuda")
            os_ = torch.empty(b, k, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            for slot, s in enumerate(order):
                assert lib.sr_cache_topk_packed_dev(shards[s].handle, C.c_void_p(q16.data_ptr()), b, k,
                                                    C.c_void_p(pairs[slot].data_ptr()), C.c_void_p(stream.cuda_stream)) == 0
            assert lib.sr_cache_merge_packed_dev(0, C.c_void_p(pairs.data_ptr()), g, b, k, C.c_void_p(oi.data_ptr()),
                                                 C.c_void_p(os_.data_ptr()), C.c_void_p(stream.cuda_stream)) == 0
            stream.synchronize()
            mi, ms = oi.cpu().numpy(), os_.cpu().numpy()
            ui, us = whole.topk(f.queries, k)
            ri, rv = co.topk_ref(f.queries, f.rows, k, f.valid)
            parts = [shards[s].topk(f.queries, k) for s in order]
            hi, hs = srlib.binding.merge_topk([p[0] for p in parts], [p[1] for p in parts])
            for name, (xi, xs) in (("unsharded", (ui, us)), ("host merge", (hi, hs)), ("float64", (ri, rv))):
                assert np.array_equal(mi, xi) and np.array_equal(ms.astype(np.float64), np.asarray(xs, np.float64)), \
                    (g, k, name)
            pk = pairs.cpu().numpy()
            for slot, s in enumerate(order):                  # the packed lists are the shard's own results
                assert np.array_equal(pk[slot, ..., 1], parts[slot][0]) and \
                    np.array_equal(pk[slot, ..., 0], parts[slot][1].view(np.int32)), (g, k, slot)
            CASES["packed-merge"] += 1
    finally:
        whole.close()
        for c in shards:
            c.close()


@pytest.mark.parametrize("g,k,ok", [(96, 64, True), (1536, 4, True), (767, 8, True), (1229, 5, False), (97, 64, False)])
def test_packed_merge_limit(srlib, cuda, g, k, ok):
    """g k = 6144 entries per query fill the merge's 48 KB (with its static shared memory more than a launch gets
    without opting in, as from g k = 6137 on); one more is refused with the outputs untouched."""
    b = 3
    rng = np.random.default_rng(g * k)
    ids = rng.permutation(g * k * b).reshape(g, b, k).astype(np.int32)
    sc = (rng.integers(-4, 5, size=(g, b, k)) / 8.0).astype(np.float32)     # many exact ties across lists
    ids[:, :, -1:] = -1
    sc[:, :, -1:] = -np.inf
    pairs = torch.from_numpy(np.stack([sc.view(np.int32), ids], -1)).cuda()
    oi = torch.full((b, k), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    os_ = torch.full((b, k), 0x7FC0DEAD, dtype=torch.int32, device="cuda")
    rc = srlib.lib().sr_cache_merge_packed_dev(0, C.c_void_p(pairs.data_ptr()), g, b, k, C.c_void_p(oi.data_ptr()),
                                               C.c_void_p(os_.data_ptr()), None)
    torch.cuda.synchronize()
    if not ok:
        assert rc == -1 and (oi == 0x5A5A5A5A).all() and (os_ == 0x7FC0DEAD).all()
        return
    assert rc == 0
    ri, rv = co.merge_packed(ids, sc, k)
    assert np.array_equal(oi.cpu().numpy(), ri) and np.array_equal(os_.cpu().numpy().view(np.float32), rv.astype(np.float32))


# ---------------------------------------------------------------------------------------------------------------------
# bitwise invariants
# ---------------------------------------------------------------------------------------------------------------------
def test_batch_stream_and_repeat_invariants(srlib, hooks):
    """A query's list does not depend on the batch around it (same route), on the stream the scan runs on, or on the
    call: random unit vectors, so the scores themselves are inexact."""
    n, d = 20000, 200
    rng = np.random.default_rng(81)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    rows[100:400] = rows[7]                                   # a plateau of inexact, identical scores
    q = rng.standard_normal((300, d)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    cache = make_cache(srlib, rows)
    lib = srlib.lib()
    try:
        for k in (8, 9, 64):
            big = cache.topk(q, k)
            small = cache.topk(q[:5], k)
            assert plan(hooks, 5, n, d, k)[1] == plan(hooks, 300, n, d, k)[1]
            assert big[0][:5].tobytes() == small[0].tobytes() and big[1][:5].tobytes() == small[1].tobytes(), k
            again = cache.topk(q, k)
            assert big[0].tobytes() == again[0].tobytes() and big[1].tobytes() == again[1].tobytes(), k
            stream = torch.cuda.Stream()
            q16 = torch.from_numpy(q).cuda().half()
            pairs = torch.empty(300, k, 2, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            assert lib.sr_cache_topk_packed_dev(cache.handle, C.c_void_p(q16.data_ptr()), 300, k,
                                                C.c_void_p(pairs.data_ptr()), C.c_void_p(stream.cuda_stream)) == 0
            stream.synchronize()
            pk = pairs.cpu().numpy()
            assert np.array_equal(pk[..., 1], big[0]) and np.array_equal(pk[..., 0], big[1].view(np.int32)), k
    finally:
        cache.close()
    # alone (the GEMV) and inside a batch of 300 (fused top-8 / GEMM): the same list where the scores are exact
    f = co.family("plateau", n, 64, 300, 82, plateaus=edge_plateaus(n, 8), hot=8)
    cache = make_cache(srlib, f.rows, f.valid)
    try:
        for k in (8, 9, 64):
            big = cache.topk(f.queries, k)
            for i in (0, 1, 299):
                alone = cache.topk(f.queries[i:i + 1], k)
                assert alone[0].tobytes() == big[0][i:i + 1].tobytes() and alone[1].tobytes() == big[1][i:i + 1].tobytes()
    finally:
        cache.close()
