"""Device-resident fp32 queries (sr_cache_topk_f32_dev, sr_cache_topk_packed_f32_dev): on exact caches ids and scores
bitwise those of the host entry sr_cache_topk and of the reference's fp32 linear scan (oracle/cache_exact_oracle.py) under
both sum rules, on both candidate-scan routes, with fallbacks mixed into batches, out-of-range queries refused on the
device, inside a captured CUDA graph, and sharded (one device, and NCCL across GPUs); on default caches bitwise
sr_cache_topk."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch

from oracle import cache_exact_oracle as co
from oracle import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = (0, 1)
ROUTE_GEMV, ROUTE_GEMM = 2, 3          # CacheRoute of csrc/kernels.h


def _clustered(rng, n, d, centres=64, spread=0.03):
    c = synth.make_cache(rng, centres, d)
    rows = c[rng.integers(0, centres, n)] + spread * rng.standard_normal((n, d)).astype(np.float32)
    return (rows / np.linalg.norm(rows, axis=1, keepdims=True)).astype(np.float32)


def _queries(rng, rows, b):
    src = rows[rng.integers(0, len(rows), b)]
    q = src + 0.02 * rng.standard_normal(src.shape).astype(np.float32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)


def _exact(srlib, rows, rule, id_offset=0):
    c = srlib.Cache(max(1, len(rows)), rows.shape[1], id_offset=id_offset, exact=True, sum_rule=rule)
    if len(rows):
        c.add(rows)
    return c


class _Dev:
    """A device buffer of the cache as a torch tensor (no copy), through the CUDA array interface."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": typestr,
                                        "strides": None, "version": 2}


def _views(srlib, c, b, k):
    L = srlib.lib()
    idx = torch.as_tensor(_Dev(L.sr_cache_dev_idx(c.handle), (b, k), "<i4"), device="cuda")
    sc = torch.as_tensor(_Dev(L.sr_cache_dev_score(c.handle), (b, k), "<f4"), device="cuda")
    return idx, sc


def _f32_dev(srlib, c, dq, k, stream=None):
    """sr_cache_topk_f32_dev on a CUDA fp32 tensor; the results copied to the host after the stream is done."""
    b = dq.shape[0]
    s = stream.cuda_stream if stream is not None else None
    assert srlib.lib().sr_cache_topk_f32_dev(c.handle, C.c_void_p(dq.data_ptr()), b, k, s) == 0
    (stream or torch.cuda.current_stream()).synchronize()
    if stream is None:
        torch.cuda.synchronize()
    idx, sc = _views(srlib, c, b, k)
    return idx.cpu().numpy(), sc.cpu().numpy()


def _same(got, want, what=""):
    gi, gs = got
    wi, ws = want
    assert np.array_equal(gi, wi), (what, np.argwhere(gi != wi)[:4])
    assert np.array_equal(np.asarray(gs, np.float32).view(np.uint32), np.asarray(ws, np.float32).view(np.uint32)), what


def _oracle(scores, k, id_offset=0):
    order = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    s = np.take_along_axis(scores, order, 1)
    return np.where(np.isneginf(s), -1, order + id_offset).astype(np.int32), s.astype(np.float32)


def _plan_route(srlib, b, n, d, kc):
    route = C.c_int(-9)
    assert srlib.hooks().sr_test_cache_plan(b, n, d, kc, C.byref(route), None, None) == 0
    return route.value


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("d", [64, 768, 1024])
@pytest.mark.parametrize("n", [8191, 8192, 8193, 65537])
def test_f32_entry_matches_host_entry(srlib, cuda, n, d, rule):
    """Every (b, k): the f32 entry = the host entry = the Go scan, bitwise; b <= 4 on the GEMV candidate scan, b >= 5 on
    the GEMM one.  Over 65 537 rows the Go scan is computed for the first 5 queries of each batch."""
    rng = np.random.default_rng(n * 3 + d + rule)
    rows = _clustered(rng, n, d)
    q = _queries(rng, rows, 256)
    no = 256 if n <= 8193 else 5
    s = co.scores_go(q[:no], rows, rule)
    c = _exact(srlib, rows, rule)
    dq = torch.from_numpy(q).cuda()
    for b in (1, 4, 5, 256):
        for k in (1, 8, 9, 33, 64):
            got = _f32_dev(srlib, c, dq[:b].contiguous(), k)
            kc = c.exact_stats(b)[3]
            assert _plan_route(srlib, b, n, d, kc) == (ROUTE_GEMV if b <= 4 else ROUTE_GEMM)
            _same(got, c.topk(q[:b], k), ("host", b, k))
            m = min(b, no)
            _same((got[0][:m], got[1][:m]), _oracle(s[:m], k), ("go", b, k))
    c.close()


def _plateau_store(rng, d=128, n=20000):
    """test_cache_exact_gpu's fallback case: 100 identical top rows among 0.5-scaled unit rows."""
    rows = 0.5 * synth.make_cache(rng, n, d)
    top = synth.make_cache(rng, 1, d)[0]
    at = rng.choice(n, 100, replace=False)
    rows[at] = top
    return rows.astype(np.float32), top, np.sort(at)


def _fresh(rng, top, b):
    """b unit queries pointing away from the plateau row: the 100 plateau rows (twice the others' norm) score below zero
    and stay out of their candidate lists, so their bands are certified."""
    q = synth.make_cache(rng, b, len(top))
    return np.where((q @ top)[:, None] > 0, -q, q).astype(np.float32)


@pytest.mark.parametrize("rule", RULES)
def test_mixed_batches(srlib, cuda, rule):
    """Plateau queries among fresh ones take the fallback (hook path 1), the others stay certified (path 0); a batch of
    300 plateau queries (more than the fallback's fixed grids hold at once) and a batch without any."""
    rng = np.random.default_rng(101 + rule)
    rows, top, at = _plateau_store(rng)
    fresh = _fresh(rng, top, 300)
    mixed = fresh[:9].copy()
    plateau_at = [1, 4, 5, 8]
    mixed[plateau_at] = top
    batches = {"mixed": mixed, "all": np.repeat(top[None], 300, 0), "none": fresh}
    c = _exact(srlib, rows, rule)
    for name, q in batches.items():
        s = co.scores_go(q, rows, rule)
        dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
        b = len(q)
        want_path = np.zeros(b, np.int32)
        if name == "mixed":
            want_path[plateau_at] = 1
        elif name == "all":
            want_path[:] = 1
        for k in (1, 8, 33, 64):
            got = _f32_dev(srlib, c, dq, k)
            _same(got, _oracle(s, k), (name, k, "go"))
            _same(got, c.topk(q, k), (name, k, "host"))
            got = _f32_dev(srlib, c, dq, k)                   # the hook's record of the device entry's scan
            path, band, eps, kc, nf = c.exact_stats(b)
            if k < kc:
                assert np.array_equal(path, want_path), (name, k, path)
                assert nf == int(want_path.sum())
            else:                                             # k = k' = 64: no candidate below the band, all fall back
                assert (path == 1).all() and nf == b
            for i in np.flatnonzero(want_path):
                assert np.array_equal(got[0][i], at[:k]), (name, k, i)
    c.close()


def test_default_cache_f32_entry(srlib, cuda):
    """A default cache fed fp32 queries on the device: bitwise sr_cache_topk on the same queries, on the GEMV, fused and
    two-stage GEMM routes."""
    rng = np.random.default_rng(111)
    n, d = 20000, 768
    rows = synth.make_cache(rng, n, d)
    q, _ = synth.make_queries(rng, rows, 256)
    q = q.astype(np.float32)
    c = srlib.Cache(n, d)
    c.add(rows)
    dq = torch.from_numpy(q).cuda()
    for b in (1, 4, 5, 256):
        for k in (1, 8, 9, 64):
            _same(_f32_dev(srlib, c, dq[:b].contiguous(), k), c.topk(q[:b], k), (b, k))
    c.close()


@pytest.mark.parametrize("rule", RULES)
def test_graph_capture(srlib, cuda, rule):
    """The exact scan plus a copy of its results captured once and replayed with new query contents: no fallback,
    fallbacks, after set_valid, after move -- each replay equal to the host entry on the same store and to the Go scan."""
    rng = np.random.default_rng(121 + rule)
    rows, top, at = _plateau_store(rng)
    b, k, d = 8, 8, rows.shape[1]
    L = srlib.lib()
    c = _exact(srlib, rows, rule)
    fresh = _fresh(rng, top, 4 * b)
    dq = torch.from_numpy(fresh[:b]).cuda()
    _f32_dev(srlib, c, dq, k)                                 # eager: the scratch is grown before the capture
    src_i, src_s = _views(srlib, c, b, k)
    oi = torch.empty((b, k), dtype=torch.int32, device="cuda")
    os_ = torch.empty((b, k), dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=stream):
        assert L.sr_cache_topk_f32_dev(c.handle, C.c_void_p(dq.data_ptr()), b, k,
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        oi.copy_(src_i)
        os_.copy_(src_s)
    store = rows.copy()
    valid = np.ones(len(rows), bool)
    with_fallback = fresh[b:2 * b].copy()
    with_fallback[[0, 3]] = top
    steps = [("no fallback", fresh[2 * b:3 * b], None), ("fallback", with_fallback, None),
             ("set_valid", with_fallback, "set_valid"), ("move", with_fallback, "move")]
    for name, q, op in steps:
        if op == "set_valid":                                 # the two lowest plateau rows leave the scan
            for r in at[:2]:
                c.set_valid(int(r), False)
                valid[r] = False
        elif op == "move":                                    # a plateau row over a row below every other plateau row
            dst = int(at[0]) - 1 if at[0] > 0 else int(at[0]) + 1
            c.move(dst, int(at[5]))
            store[dst] = store[at[5]]
            valid[dst] = valid[at[5]]
        dq.copy_(torch.from_numpy(np.ascontiguousarray(q)))
        g.replay()
        torch.cuda.synchronize()
        got = (oi.cpu().numpy(), os_.cpu().numpy())
        _same(got, c.topk(q, k), (name, "host"))
        _same(got, co.topk_go(q, store, k, rule, valid), (name, "go"))
        path = c.exact_stats(b)[0]
        assert (path[[0, 3]] == 1).all() if name != "no fallback" else (path == 0).all(), (name, path)
    del g
    c.close()


@pytest.mark.parametrize("rule", RULES)
def test_stream_and_repeat(srlib, cuda, rule):
    """A caller's stream = the cache's own stream (null); a repeated call is bitwise the same."""
    rng = np.random.default_rng(131 + rule)
    rows, top, _ = _plateau_store(rng)
    q = synth.make_cache(rng, 6, rows.shape[1])
    q[2] = top
    c = _exact(srlib, rows, rule)
    dq = torch.from_numpy(q).cuda()
    s = torch.cuda.Stream()
    for k in (1, 9, 64):
        own = _f32_dev(srlib, c, dq, k)
        _same(_f32_dev(srlib, c, dq, k, stream=s), own, ("stream", k))
        _same(_f32_dev(srlib, c, dq, k), own, ("repeat", k))
        _same(own, c.topk(q, k), ("host", k))
    c.close()


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 70000.0])
def test_out_of_range_query_on_device(srlib, cuda, bad, rule):
    """One query of 6 with a component the bound does not cover: (-1, -inf) and hook path 2 for it, in the plain and the
    packed result; the other five (one of them a fallback) exact; the cache serves on."""
    rng = np.random.default_rng(141 + rule)
    rows, top, _ = _plateau_store(rng)
    q = synth.make_cache(rng, 6, rows.shape[1])
    q[4] = top
    q[2, 17] = bad
    good = [0, 1, 3, 4, 5]
    c = _exact(srlib, rows, rule)
    dq = torch.from_numpy(q).cuda()
    for k in (1, 8, 64):
        gi, gs = _f32_dev(srlib, c, dq, k)
        assert (gi[2] == -1).all() and np.isneginf(gs[2]).all()
        path = c.exact_stats(6)[0]
        assert path[2] == 2 and path[4] == 1
        _same((gi[good], gs[good]), co.topk_go(q[good], rows, k, rule), ("go", k))
        pairs = torch.full((6, k, 2), 7, dtype=torch.int32, device="cuda")
        assert srlib.lib().sr_cache_topk_packed_f32_dev(c.handle, C.c_void_p(dq.data_ptr()), 6, k,
                                                        C.c_void_p(pairs.data_ptr()), None) == 0
        torch.cuda.synchronize()
        pk = pairs.cpu().numpy()
        assert (pk[2, :, 1] == -1).all() and np.isneginf(pk[2, :, 0].view(np.float32)).all()
        assert np.array_equal(pk[..., 1], gi) and np.array_equal(pk[..., 0], gs.view(np.int32))
    qs = np.delete(q, 2, 0)
    _same(c.topk(qs, 8), co.topk_go(qs, rows, 8, rule), "after")
    _same(_f32_dev(srlib, c, torch.from_numpy(qs).cuda(), 8), co.topk_go(qs, rows, 8, rule), "after, device")
    c.close()


# shard edges of [0, 20000): g 3 has an empty shard, g 8 an empty one and one of 3 rows (fewer than k); every g > 1 cuts
# at 10 000, through the tie plateau [9990, 10010), and keeps the fallback plateau [2000, 2100) inside its first shard
SHARD_CUTS = {1: [], 2: [10000], 3: [10000, 10000], 8: [3000, 3000, 10000, 12000, 15000, 18000, 19997]}


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("g", [1, 2, 3, 8])
def test_shards_on_one_device(srlib, cuda, g, rule):
    """sr_cache_topk_packed_f32_dev per shard (shards in scrambled slot order) + sr_cache_merge_packed_dev = the unsharded
    exact cache = the Go scan."""
    n, d = 20000, 128
    rng = np.random.default_rng(151 + g + rule)
    rows = _clustered(rng, n, d)
    fb_row, tie_row = synth.make_cache(rng, 2, d)
    rows[2000:2100] = fb_row
    rows[9990:10010] = tie_row
    q = _queries(rng, rows, 7)
    q[2] = fb_row
    q[5] = tie_row
    edges = [0] + SHARD_CUTS[g] + [n]
    bounds = list(zip(edges[:-1], edges[1:]))
    order = list(np.random.default_rng(g).permutation(g))        # slot s holds shard order[s]
    L = srlib.lib()
    whole = _exact(srlib, rows, rule)
    shards = [_exact(srlib, rows[a:e], rule, id_offset=a) for a, e in bounds]
    dq = torch.from_numpy(q).cuda()
    b = len(q)
    for k in (1, 8, 33):
        pairs = torch.full((g, b, k, 2), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        oi = torch.empty(b, k, dtype=torch.int32, device="cuda")
        os_ = torch.empty(b, k, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        for slot, s in enumerate(order):
            assert L.sr_cache_topk_packed_f32_dev(shards[s].handle, C.c_void_p(dq.data_ptr()), b, k,
                                                  C.c_void_p(pairs[slot].data_ptr()), None) == 0
        torch.cuda.synchronize()
        assert L.sr_cache_merge_packed_dev(0, C.c_void_p(pairs.data_ptr()), g, b, k, C.c_void_p(oi.data_ptr()),
                                           C.c_void_p(os_.data_ptr()), None) == 0
        torch.cuda.synchronize()
        got = (oi.cpu().numpy(), os_.cpu().numpy())
        _same(got, whole.topk(q, k), (g, k, "unsharded"))
        _same(got, co.topk_go(q, rows, k, rule), (g, k, "go"))
        assert np.array_equal(got[0][5, :min(k, 20)], np.arange(9990, 9990 + min(k, 20)))   # lower global id first
        assert np.array_equal(got[0][2, :k], np.arange(2000, 2000 + k))
    for s in shards + [whole]:
        s.close()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, rule, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import importlib
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import semantic_router_b200 as pkg
        sh = importlib.import_module("semantic-router_b200.sharding")
        rng = np.random.default_rng(161 + rule)                 # the same data on every rank
        n, d, b = 30001, 256, 33
        rows = _clustered(rng, n, d)
        rows[3000:3100] = rows[7]                               # a fallback plateau inside rank 0's shard
        lo, hi = sh.shard_range(n, world - 1, world)
        rows[lo - 5:lo + 5] = rows[11]                          # a tie plateau across the last shard's lower edge
        queries = _queries(rng, rows, b)
        queries[0] = rows[7]
        queries[1] = rows[11]
        lo, hi = sh.shard_range(n, rank, world)
        cache = pkg.Cache(hi - lo, d, device=rank, id_offset=lo, exact=True, sum_rule=rule)
        cache.add(rows[lo:hi])
        ok = True
        for k in (1, 8, 33):
            oi, os_ = sh.sharded_topk_dev(cache, torch.from_numpy(queries).cuda(), k)
            ri, rs = co.topk_go(queries, rows, k, rule)
            ok = ok and np.array_equal(oi.cpu().numpy(), ri) and \
                np.array_equal(os_.cpu().numpy().view(np.uint32), rs.view(np.uint32))
        cache.close()
        q.put((rank, ok))
    except Exception as e:                                      # reported, not hung on
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("rule", RULES)
def test_nccl_sharded_exact(cuda, rule):
    """world = min(4, GPUs) processes, each holding its shard of an exact cache on its own GPU: sharding.sharded_topk_dev
    with fp32 queries returns the Go scan's result, bitwise, on every rank."""
    import torch.multiprocessing as mp
    world = min(4, torch.cuda.device_count())
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, port, rule, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=600) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert sorted(r for r, _ in res) == list(range(world))
    assert all(ok is True for _, ok in res), res
