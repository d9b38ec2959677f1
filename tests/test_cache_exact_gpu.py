"""Exact caches (sr_cache_create_exact): ids and scores bitwise those of the reference's fp32 linear scan
(pkg/cache/inmemory_cache_search.go:14-20, restated in oracle/cache_exact_scan.c) under both sum rules, on every route of the
candidate scan, across the certified band, the exhaustive fallback, ties, lifecycle calls, shards and the embed-and-scan
entry; and the refusals."""
import numpy as np
import pytest

from oracle import cache_exact_oracle as co
from oracle import synth

pytestmark = pytest.mark.gpu

RULES = (0, 1)


def _clustered(rng, n, d, centres=64, spread=0.03):
    """n unit rows around a few centres: many rows within the fp16 error of each other at the top of a query's list."""
    c = synth.make_cache(rng, centres, d)
    rows = c[rng.integers(0, centres, n)] + spread * rng.standard_normal((n, d)).astype(np.float32)
    return (rows / np.linalg.norm(rows, axis=1, keepdims=True)).astype(np.float32)


def _queries(rng, rows, b):
    src = rows[rng.integers(0, len(rows), b)]
    q = src + 0.02 * rng.standard_normal(src.shape).astype(np.float32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)


def _exact(srlib, rows, rule, valid=None, id_offset=0, capacity=None):
    c = srlib.Cache(capacity or max(1, len(rows)), rows.shape[1], id_offset=id_offset, exact=True, sum_rule=rule)
    if len(rows):
        c.add(rows)
    if valid is not None:
        for i in np.flatnonzero(~valid):
            c.set_valid(int(i), False)
    return c


def _check(c, rows, q, k, rule, valid=None, id_offset=0, scores=None):
    idx, sc = c.topk(q, k)
    if scores is None:
        ref_i, ref_s = co.topk_go(q, rows, k, rule, valid, id_offset)
    else:                                                     # precomputed Go scores [B, N]
        s = scores.copy()
        if valid is not None:
            s[:, ~valid] = -np.inf
        order = np.argsort(-s, axis=1, kind="stable")[:, :k]
        ref_s = np.take_along_axis(s, order, 1)
        ref_i = np.where(np.isneginf(ref_s), -1, order + id_offset).astype(np.int32)
    assert np.array_equal(idx, ref_i), np.argwhere(idx != ref_i)[:4]
    assert np.array_equal(sc.view(np.uint32), ref_s.astype(np.float32).view(np.uint32))
    return idx, sc


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("n,d", [(n, d) for d in (64, 384, 768, 1024) for n in (8191, 8192, 8193, 65537)]
                         + [(8191, 12288), (8192, 12288)])   # 48 KB of fp32 query: the band kernel opts in above 48 KB
def test_exact_topk_matches_go_scan(srlib, cuda, n, d, rule):
    rng = np.random.default_rng(n * 7 + d + rule)
    rows = _clustered(rng, n, d)
    bmax = 256 if n <= 8193 else 5
    q = _queries(rng, rows, bmax)
    s = co.scores_go(q, rows, rule)
    c = _exact(srlib, rows, rule)
    for b in (1, 4, 5, 256):
        if b > bmax:
            continue
        for k in (1, 8, 9, 33, 64):
            _check(c, rows, q[:b], k, rule, scores=s[:b])
    c.close()


@pytest.mark.parametrize("rule", RULES)
def test_fp16_twins_and_one_ulp(srlib, cuda, rule):
    """Rows that round to one fp16 row but differ in fp32, and rows whose Go scores are 1 ulp apart."""
    rng = np.random.default_rng(5 + rule)
    d = 256
    base = synth.make_cache(rng, 1, d)[0]
    twins = np.repeat(base[None], 40, 0)
    for j in range(40):                                       # nudges of a few fp32 ulps: far below the fp16 spacing
        while True:
            t = base.copy()
            i = rng.integers(0, d, 3)
            t[i] *= (1 + rng.integers(-60, 61, 3) * 2.0 ** -23).astype(np.float32)
            if (t.astype(np.float16) == base.astype(np.float16)).all():   # not across an fp16 rounding boundary
                twins[j] = t
                break
    assert (twins.astype(np.float16) == base.astype(np.float16)).all()
    rows = np.concatenate([synth.make_cache(rng, 3000, d), twins, synth.make_cache(rng, 3000, d)]).astype(np.float32)
    q = np.stack([base, twins[7], twins[8]]).astype(np.float32)
    s = np.sort(co.scores_go(q[:1], twins, rule)[0])
    assert (np.diff(s.view(np.int32)) == 1).any()             # some Go scores of the twins are 1 ulp apart
    c = _exact(srlib, rows, rule)
    for k in (1, 8, 33, 64):
        _check(c, rows, q, k, rule)
    c.close()


def _rule_split_pair(rng, d):
    """A query and two rows whose order differs between the two sum rules (searched on random near-duplicates)."""
    for _ in range(2000):
        q = rng.standard_normal(d).astype(np.float32)
        r = (q + 0.5 * rng.standard_normal(d)).astype(np.float32)   # q . r ~ |q|^2: far above the 0.1-scaled filler
        r2 = r.copy()
        r2[rng.integers(0, d)] *= np.float32(1 + 2 ** -20)
        s = [co.scores_go(q[None], np.stack([r, r2]), rule)[0] for rule in RULES]
        o0 = int(s[0][0] > s[0][1]) - int(s[0][0] < s[0][1])
        o1 = int(s[1][0] > s[1][1]) - int(s[1][0] < s[1][1])
        if o0 != o1:
            return q, np.stack([r, r2])
    raise AssertionError("no pair found")


def test_rules_order_rows_differently(srlib, cuda):
    rng = np.random.default_rng(11)
    d = 64
    q, pair = _rule_split_pair(rng, d)
    rows = np.concatenate([0.1 * synth.make_cache(rng, 5000, d), pair]).astype(np.float32)
    i0, _ = co.topk_go(q[None], rows, 2, 0)
    i1, _ = co.topk_go(q[None], rows, 2, 1)
    assert not np.array_equal(i0, i1)                         # the two oracles disagree on this case
    for rule in RULES:
        c = _exact(srlib, rows, rule)
        _check(c, rows, q[None], 2, rule)
        _check(c, rows, np.stack([q, q, q, q, q, q]), 2, rule)   # b > 4: the GEMM candidate scan
        c.close()


@pytest.mark.parametrize("rule", RULES)
def test_ties_beyond_64_and_fallback(srlib, cuda, rule):
    """100 identical top rows: the band is wider than k' (at most 64), the hook reports the fallback, and the lower index
    wins.  At 800 000 rows and k 64 the fallback's stage 2 holds 98 segments x 64 candidates x 8 B = 50 KB of shared
    memory, and the 205 MB of fp32 rows go up in several pieces."""
    rng = np.random.default_rng(21 + rule)
    for n, d, ks in ((20000, 128, (1, 8, 64)), (800000, 64, (64,))):
        rows = 0.5 * synth.make_cache(rng, n, d)
        top = synth.make_cache(rng, 1, d)[0]
        at = rng.choice(n, 100, replace=False)
        rows[at] = top
        q = np.stack([top, synth.make_cache(rng, 1, d)[0]] * 3).astype(np.float32)
        c = _exact(srlib, rows, rule)
        for b in (1, 6):
            for k in ks:
                idx, _ = _check(c, rows, q[:b], k, rule)
                assert np.array_equal(idx[0], np.sort(at)[:k])
                path, band, eps, kc, nf = c.exact_stats(b)
                assert path[0] == 1 and band[0] == kc == (32 if k <= 32 else 64) and nf >= 1
        c.close()


def test_lifecycle_replay(srlib, cuda):
    rng = np.random.default_rng(31)
    d, cap = 96, 12000
    for rule in RULES:
        c = srlib.Cache(cap, d, exact=True, sum_rule=rule)
        store = np.zeros((0, d), np.float32)
        valid = np.zeros(0, bool)
        for step in range(30):
            op = step % 5
            if op == 0:
                new = _clustered(rng, int(rng.integers(200, 900)), d, centres=8)
                c.add(new)
                store = np.concatenate([store, new]); valid = np.concatenate([valid, np.ones(len(new), bool)])
            elif op == 1 and len(store):
                for i in rng.integers(0, len(store), 20):
                    v = bool(rng.random() < 0.5)
                    c.set_valid(int(i), v); valid[i] = v
            elif op == 2 and len(store) > 1:
                for _ in range(10):
                    dst, src = (int(x) for x in rng.integers(0, len(store), 2))
                    c.move(dst, src); store[dst] = store[src]; valid[dst] = valid[src]
            elif op == 3 and len(store):
                n = int(rng.integers(len(store) // 2, len(store) + 1))
                c.truncate(n); store, valid = store[:n], valid[:n]
            elif op == 4 and len(store):
                keep = rng.random(len(store)) < 0.7
                assert c.compact(keep) == int(keep.sum())
                store, valid = store[keep], valid[keep]
            q = _queries(rng, store, 6) if len(store) else synth.make_cache(rng, 6, d)
            for k in (1, 9):
                _check(c, store, q, k, rule, valid)
        c.close()


@pytest.mark.parametrize("rule", RULES)
def test_norms_and_zero_query(srlib, cuda, rule):
    rng = np.random.default_rng(41 + rule)
    d = 384
    rows = synth.make_cache(rng, 9000, d) * rng.uniform(1e-3, 300, (9000, 1)).astype(np.float32)
    rows[:50] *= np.float32(2.0 ** -14)                       # fp16 subnormal components
    q = _queries(rng, rows / np.linalg.norm(rows, axis=1, keepdims=True), 5) * np.float32(7.5)
    q[1] = 0.0
    c = _exact(srlib, rows.astype(np.float32), rule)
    for k in (1, 8, 64):
        _check(c, rows, q, k, rule)
        path, band, eps, kc, nf = c.exact_stats(5)
        want = [co.exact_eps(float(np.linalg.norm(x.astype(np.float64))), float(np.linalg.norm(rows.astype(np.float64), axis=1).max()), d)
                for x in q]
        np.testing.assert_allclose(eps, want, rtol=1e-9)
    c.close()


@pytest.mark.parametrize("rule", RULES)
def test_shards_merge_equals_unsharded(srlib, cuda, rule):
    rng = np.random.default_rng(51 + rule)
    d, n = 256, 40000
    rows = _clustered(rng, n, d)
    q = _queries(rng, rows, 7)
    whole = _exact(srlib, rows, rule)
    cuts = [0, 9000, 20001, 31000, n]
    shards = [_exact(srlib, rows[a:b], rule, id_offset=a) for a, b in zip(cuts, cuts[1:])]
    for k in (1, 8, 33):
        wi, ws = _check(whole, rows, q, k, rule)
        parts = [s.topk(q, k) for s in shards]
        mi, ms = srlib.merge_topk([p[0] for p in parts], [p[1] for p in parts])
        assert np.array_equal(mi, wi) and np.array_equal(ms.view(np.uint32), ws.view(np.uint32))
    for s in shards + [whole]:
        s.close()


def test_lookup_ids_uses_fp32_embedding(srlib, cuda):
    import tempfile
    from oracle import encoder_oracle as eo
    cfg = eo.ModernBertConfig(vocab_size=700, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=0)
    w = synth.make_modernbert_weights(cfg, 2, seed=61)
    rng = np.random.default_rng(61)
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_model_dir(tmp, cfg, w, {0: "a", 1: "b"})
        m = srlib.Model(tmp, device=0)
        stored = synth.make_ids(rng, rng.integers(8, 120, 200).tolist(), cfg.vocab_size)
        emb = m.embed_ids(stored, target_layer=3, target_dim=256)
        rows = np.concatenate([synth.make_cache(rng, 3000, 256), emb]).astype(np.float32)
        for rule in RULES:
            c = _exact(srlib, rows, rule)
            for nq in (1, 6):
                qs = [stored[i] for i in rng.choice(200, nq, replace=False)]
                idx, sc = c.lookup_ids(m, qs, 8, target_layer=3)
                e = m.embed_ids(qs, target_layer=3, target_dim=256)   # the fp32 embedding the lookup scans with
                ri, rs = co.topk_go(e, rows, 8, rule)
                assert np.array_equal(idx, ri)
                assert np.array_equal(sc.view(np.uint32), rs.view(np.uint32))
            c.close()
        m.close()


def test_refusals(srlib, cuda):
    import ctypes as C
    import torch
    L = srlib.lib()
    h = C.c_void_p()
    assert L.sr_cache_create_exact(0, 16, 64, 0, 2, C.byref(h)) != 0
    assert L.sr_cache_create_exact(0, 16, 64, 0, -1, C.byref(h)) != 0
    rng = np.random.default_rng(71)
    rows = synth.make_cache(rng, 100, 64)
    c = _exact(srlib, rows, 0, capacity=200)
    for bad in (np.nan, np.inf, -np.inf, 70000.0):
        r = synth.make_cache(rng, 2, 64)
        r[1, 5] = bad
        with pytest.raises(srlib.SrError):
            c.add(r)
        assert len(c) == 100
        q = synth.make_cache(rng, 2, 64)
        q[0, 3] = bad
        idx = np.full((2, 4), 7, np.int32)
        sc = np.full((2, 4), 7, np.float32)
        assert L.sr_cache_topk(c.handle, q.ctypes.data, 2, 4, idx.ctypes.data, sc.ctypes.data) != 0
        assert (idx == 7).all() and (sc == 7).all()
    q16 = torch.zeros((2, 64), dtype=torch.float16, device="cuda")
    pairs = torch.full((2, 4, 2), 7, dtype=torch.int32, device="cuda")
    assert L.sr_cache_topk_dev(c.handle, q16.data_ptr(), 2, 4, None) != 0
    assert L.sr_cache_topk_packed_dev(c.handle, q16.data_ptr(), 2, 4, pairs.data_ptr(), None) != 0
    torch.cuda.synchronize()
    assert (pairs == 7).all()
    _check(c, rows, synth.make_cache(rng, 3, 64), 4, 0)     # the cache still serves
    c.close()


def test_cfg4_style_fallback_report(srlib, cuda):
    """BASELINE cfg 4 inputs (unit rows, perturbed copies and fresh queries) at reduced N: every query exact, and the
    number that fell back reported."""
    rng = np.random.default_rng(81)
    n, d = 65536, 768
    rows = synth.make_cache(rng, n, d)
    q, _ = synth.make_queries(rng, rows, 64)
    q = q.astype(np.float32)
    for rule in RULES:
        c = _exact(srlib, rows, rule)
        for b in (1, 64):
            _check(c, rows, q[:b], 8, rule)
            path, band, eps, kc, nf = c.exact_stats(b)
            print(f"rule {rule} b {b}: k' {kc}, fallback {nf} of {b}, band max {band.max()}, eps max {eps.max():.3e}")
        c.close()
