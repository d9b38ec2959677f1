"""The cache-scan oracle of oracle/cache_oracle.py, without a GPU: the exact-score families are exact, the numpy
restatement of the two-stage selection (select_stage1 -> select_stage2 of csrc/cache_scan.cu) and of the packed merge
equals the float64 reference, stage1_trace shows which warps each family drives into the k-pass fallback, and each
mutation of the selection logic that tests/test_cache_topk_conformance_gpu.py must catch changes at least one id on
these families."""
import numpy as np
import pytest

from oracle import cache_oracle as co

KS = [1, 7, 8, 9, 31, 32, 33, 63, 64]
N = 40000
CHUNK = 16384          # restated chunk size: two chunk edges inside N, as 262144 rows are for B = 1024
S, W = co.SEGMENT, co.WARP_ROWS


def _families():
    """Small versions of the GPU file's families: plateaus of 129..600 rows inside one warp window, and plateaus across
    a warp window, a segment, a chunk and a 128-row tile; cut ties, an all-equal store, all-negative scores, fewer valid
    rows than k, invalidated low members of a plateau, and a ladder for the k > 32 rule."""
    pl = [(3 * W + 10, 129), (6 * W, 600), (S - 300, 600), (CHUNK - 77, 160), (S + 128 * 40 - 9, 20), (2 * S + 5, 9)]
    out = {
        "plateau": co.family("plateau", N, 64, 8, 1, plateaus=pl),
        "cut_tie": co.family("plateau", N, 64, 8, 2, plateaus=[(100 + 50 * p, 8) for p in range(8)]),
        "all_equal": co.family("all_equal", N, 64, 4, 3),
        "all_negative": co.family("all_negative", N, 64, 8, 4, plateaus=[(W - 64, 200), (CHUNK - 3, 40)]),
        "sparse_valid": co.family("sparse_valid", N, 64, 8, 5,
                                  plateaus=[(7, 1), (W + 3, 2), (S + 1, 1), (CHUNK + 2, 3), (N - 1, 1)]),
        "spread_ladder": co.family("spread", N, 64, 8, 6, ladders=[(5 * W, 64)], plateaus=[(3000, 200), (CHUNK - 100, 200)]),
    }
    inv = co.family("plateau", N, 64, 8, 7, plateaus=[(2 * W - 40, 300), (CHUNK - 20, 150)])
    inv.valid[2 * W - 40:2 * W - 40 + 37] = False          # the lowest-index members of the plateaus
    inv.valid[CHUNK - 20:CHUNK - 14] = False
    inv.name = "invalidated"
    out["invalidated"] = inv
    return out


@pytest.fixture(scope="module")
def fams():
    return _families()


@pytest.fixture(scope="module")
def refs(fams):
    return {(name, k): co.topk_ref(f.queries, f.rows, k, f.valid, device="cpu") for name, f in fams.items() for k in KS}


def test_families_are_exact(fams):
    """Every family meets sum |q| |r| < 2^16 on fp16-exact m / 16 entries, so fp32 sums in any order are the float64
    score: two numpy fp32 summation orders equal float64 bitwise."""
    for name, f in fams.items():
        f.check_exact()
        s64 = f.scores64()
        fwd = np.zeros(s64.shape, np.float32)
        for j in range(f.rows.shape[1]):
            fwd += f.queries[:, j:j + 1] * f.rows[None, :, j][0]
        rev = np.zeros(s64.shape, np.float32)
        for j in reversed(range(f.rows.shape[1])):
            rev = (rev + f.queries[:, j:j + 1] * f.rows[None, :, j][0]).astype(np.float32)
        assert np.array_equal(fwd.astype(np.float64), s64) and np.array_equal(rev.astype(np.float64), s64), name


@pytest.mark.parametrize("k", KS)
def test_restated_selection_equals_reference(fams, refs, k):
    for name, f in fams.items():
        ri, rv = refs[(name, k)]
        s = f.scores64()
        for chunk in (None, CHUNK):
            oi, ov = co.select_two_stage(s, f.valid, k, chunk_rows=chunk)
            assert np.array_equal(oi, ri) and np.array_equal(ov, rv), (name, k, chunk)
        ti, ts = co.topk_batch(f.queries, f.rows, k, f.valid)
        assert np.array_equal(ti, ri) and np.array_equal(ts.astype(np.float64), rv), (name, k)


def test_packed_merge_restatement_equals_reference(fams):
    """Shards of the plateau family in a scrambled id order, one of them empty: merging their lists gives the unsharded
    list, as do the host merge oracle and the float64 reference."""
    f = fams["plateau"]
    bounds = [0, 3 * W + 70, 3 * W + 70, 6 * W + 333, S + 1, N]            # the second shard is empty
    for k in (1, 8, 33, 64):
        ri, rv = co.topk_ref(f.queries, f.rows, k, f.valid, device="cpu")
        parts_i, parts_s = [], []
        for a, b in zip(bounds[:-1], bounds[1:]):
            if b > a:
                pi, ps = co.topk_ref(f.queries, f.rows[a:b], k, f.valid[a:b], device="cpu")
                pi = np.where(pi >= 0, pi + a, -1)
            else:
                pi, ps = np.full((f.queries.shape[0], k), -1), np.full((f.queries.shape[0], k), -np.inf)
            parts_i.append(pi)
            parts_s.append(ps)
        order = [3, 0, 4, 1, 2]
        mi, ms = co.merge_packed([parts_i[g] for g in order], [parts_s[g] for g in order], k)
        assert np.array_equal(mi, ri) and np.array_equal(ms, rv), k
        hi, hs = co.merge_topk([parts_i[g] for g in order], [parts_s[g].astype(np.float32) for g in order], k)
        assert np.array_equal(hi, ri), k


def test_stage1_trace_coverage(fams):
    """Plateaus of > 128 rows inside one warp window drive that warp into the fallback at k <= 32 while warps of the
    spread family take the compacted list; at k > 32 every warp with > 128 valid rows falls back."""
    f = fams["plateau"]
    s = f.scores64()
    for k in (1, 8, 9, 32):
        cnt, fb = co.stage1_trace(s, f.valid, k)
        # plateau p is on hot channel p % 4, query i on channel i % 4: 129 rows in warp 3 (plateau 0), 600 rows over
        # warp 6 (plateau 1), 300 + 300 rows in warps 7 and 8, across the first segment edge (plateau 2)
        assert fb[[0, 4], 3].all() and fb[[1, 5], 6].all() and fb[[2, 6]][:, 7:9].all(), k
    sp = fams["spread_ladder"]
    cnt, fb = co.stage1_trace(sp.scores64(), sp.valid, 9)
    assert (~fb).mean() > 0.9
    for name, f in fams.items():
        cnt, fb = co.stage1_trace(f.scores64(), f.valid, 33)
        nvalid = co._warp_view(np.zeros((1, N)), f.valid, -(-N // S) * S)[0] != -np.inf
        many = nvalid.sum(axis=(-2, -1)) > co.LIST_CAP
        assert (fb == many[None, :]).all(), name


MUTATIONS = {   # restatement mutation -> families on which it must change an id
    "gt": ["plateau", "spread_ladder"],
    "no_k32": ["spread_ladder"],
    "tie1": ["plateau", "cut_tie", "all_equal", "invalidated"],
    "tie2": ["plateau", "cut_tie", "all_equal"],
    "seg0": ["plateau", "spread_ladder", "sparse_valid"],
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_families_catch_each_mutation(fams, refs, mutation):
    for name in MUTATIONS[mutation]:
        f = fams[name]
        s = f.scores64()
        changed = 0
        for k in KS:
            oi, _ = co.select_two_stage(s, f.valid, k, chunk_rows=CHUNK, mutate=(mutation,))
            changed += int((oi != refs[(name, k)][0]).sum())
        assert changed > 0, (mutation, name)


def test_reversed_tie_rule_of_the_packed_merge_is_caught(fams):
    f = fams["all_equal"]
    k = 8
    parts = [co.topk_ref(f.queries, f.rows[a:a + 100], k, None, device="cpu") for a in (0, 100)]
    ids = [np.where(p[0] >= 0, p[0] + a, -1) for p, a in zip(parts, (0, 100))]
    good, _ = co.merge_packed(ids, [p[1] for p in parts], k)
    bad, _ = co.merge_packed(ids, [p[1] for p in parts], k, mutate=("tiepack",))
    assert (good == np.arange(k)).all() and (bad != good).any()
