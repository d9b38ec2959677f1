"""CPU checks of oracle/attn_oracle.py: its value against torch softmax attention and the masks of encoder_oracle in
float64, its bound against a float32 restatement of the wgmma attention kernel's order of operations on every input
family of tests/test_attention_conformance_gpu.py, and that on those inputs a window or key length off by one, a
skipped 64-key block and a missing alpha rescale each move the output by more than 10x the bound."""
import numpy as np
import pytest
import torch

from oracle import attn_oracle as ao
from oracle import encoder_oracle as eo

f32, f16 = np.float32, np.float16
C = f32(f32(0.125) * f32(1.4426950408889634))


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


def _split(qkv, nH):
    x = qkv.float().view(-1, 3, nH, 64)
    return x[:, 0], x[:, 1], x[:, 2]


# ---- value ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [0, 1, 5, 40])
def test_value_is_softmax_attention(window):
    lens, nH = [1, 7, 64, 65, 130], 3
    cu = _cu(lens)
    qkv = ao.make_qkv("random", cu, nH, seed=1)
    ref = ao.attention(qkv, cu, nH, window)
    q, k, v = (t.double() for t in _split(qkv, nH))
    for b, L in enumerate(lens):
        s = slice(cu[b], cu[b + 1])
        att = torch.einsum("ihd,jhd->hij", q[s], k[s]) * 0.125
        if window > 0:
            i = torch.arange(L)
            att = att.masked_fill((i[None, :] - i[:, None]).abs()[None] > window, -torch.inf)
        want = torch.einsum("hij,jhd->ihd", torch.softmax(att, -1), v[s]).reshape(L, nH * 64)
        torch.testing.assert_close(ref.value[s], want, rtol=1e-12, atol=1e-13)


def test_window_is_the_local_mask_of_modernbert():
    """window = local_attention // 2 reproduces the encoder oracle's local + global mask (modernbert.rs:376-393)"""
    L, nH, local_attention = 300, 2, 128
    cu = [0, L]
    qkv = ao.make_qkv("random", cu, nH, seed=2)
    ref = ao.attention(qkv, cu, nH, local_attention // 2)
    q, k, v = (t.double() for t in _split(qkv, nH))
    att = torch.einsum("ihd,jhd->hij", q, k) * 0.125 + eo.local_mask(L, local_attention // 2).double()[None]
    want = torch.einsum("hij,jhd->ihd", torch.softmax(att, -1), v).reshape(L, nH * 64)
    torch.testing.assert_close(ref.value, want, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("kv", [1, 20, 63, 64, 65, 99, 100])
def test_kv_lens_is_the_bert_key_mask(kv):
    """kv_lens: keys >= kv are masked for every row and the pads stay queries, as the additive mask of bert_forward"""
    L, nH = 100, 2
    cu = [0, L]
    qkv = ao.make_qkv("random", cu, nH, seed=3)
    ref = ao.attention(qkv, cu, nH, 0, kv_lens=[kv])
    q, k, v = (t.double() for t in _split(qkv, nH))
    mask = torch.zeros(1, L, dtype=torch.long)
    mask[0, :kv] = 1
    att = torch.einsum("ihd,jhd->hij", q, k) * 0.125 + eo.global_mask_4d(mask).double()[0]
    want = torch.einsum("hij,jhd->ihd", torch.softmax(att, -1), v).reshape(L, nH * 64)
    torch.testing.assert_close(ref.value, want, rtol=1e-12, atol=1e-13)


def test_sampled_rows_and_chunks_equal_the_full_reference():
    lens, nH = [700, 300], 2
    cu = _cu(lens)
    qkv = ao.make_qkv("random", cu, nH, seed=4)
    full = ao.attention(qkv, cu, nH, 0)
    sel = torch.tensor([0, 63, 64, 350, 699, 700, 701, 999])
    part = ao.attention(qkv, cu, nH, 0, sel=sel)
    for a, b in ((part.value, full.value[sel]), (part.coef, full.coef[sel]), (part.eps, full.eps[sel])):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=0)


# ---- a float32 restatement of the kernel ---------------------------------------------------------------------------
def emulate(q, k, v, window, klen, drop_block=None, alpha_o=True, alpha_l=True):
    """attn_wgmma_kernel for one (sequence, head): q, k, v fp16 [L, 64] -> fp16 [L, 64].  The tensor-core products are
    exact sums rounded to fp32 (within TAU of the accumulation model); everything else is the kernel's fp32 order:
    online max, alpha, exp2 in fp32, fp16 P, l as 4 per-thread chains of pair-sums, 2 shuffle levels, 1 / l.
    drop_block skips one key block; alpha_o / alpha_l = False drop the rescale of o / l."""
    L = len(q)
    qd, kd, vd = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    out = np.empty((L, 64), f16)
    for q0 in range(0, L, 64):
        rows = np.arange(q0, min(q0 + 64, L))
        lo, hi = ao.blocks(L, window, torch.tensor([q0]))
        m = np.full(len(rows), -np.inf, f32)
        l = np.zeros((len(rows), 4), f32)
        o = np.zeros((len(rows), 64), f32)
        for kb in range(int(lo), int(hi) + 1):
            if kb == drop_block:
                continue
            keys = kb * 64 + np.arange(64)
            kin = keys < L
            kz = np.where(kin[:, None], kd[np.minimum(keys, L - 1)], 0.0)
            vz = np.where(kin[:, None], vd[np.minimum(keys, L - 1)], 0.0)
            s = (qd[rows] @ kz.T).astype(f32)
            ok = (keys[None, :] < klen) & np.ones((len(rows), 1), bool)
            if window > 0:
                ok &= np.abs(keys[None, :] - rows[:, None]) <= window
            s = np.where(ok, s, f32(-np.inf)).astype(f32)
            m_new = np.maximum(m, s.max(1))
            m_use = np.where(m_new == -np.inf, f32(0), m_new).astype(f32)
            with np.errstate(invalid="ignore"):
                alpha = np.exp2((m - m_use) * C).astype(f32)
            m = m_new
            if alpha_l:
                l = (l * alpha[:, None]).astype(f32)
            p = np.exp2((s - m_use[:, None]) * C).astype(f32)
            pairs = (p[:, 0::2] + p[:, 1::2]).astype(f32)              # pair 4j + t: keys 8j + 2t, 8j + 2t + 1
            for j in range(8):
                l = (l + pairs[:, 4 * j:4 * j + 4]).astype(f32)
            if alpha_o:
                o = (o * alpha[:, None]).astype(f32)
            o = (o + (p.astype(f16).astype(np.float64) @ vz).astype(f32)).astype(f32)
        tot = ((l[:, 0] + l[:, 1]).astype(f32) + (l[:, 2] + l[:, 3]).astype(f32)).astype(f32)
        inv = (f32(1) / tot).astype(f32)
        out[rows] = (o * inv[:, None]).astype(f32).astype(f16)
    return out


def emulate_pack(qkv, cu, nH, window, kv_lens=None, **kw):
    x = qkv.numpy().reshape(-1, 3, nH, 64)
    out = np.zeros((int(cu[-1]), nH * 64), f16)
    for b in range(len(cu) - 1):
        s0, s1 = int(cu[b]), int(cu[b + 1])
        klen = min(s1 - s0, int(kv_lens[b])) if kv_lens is not None else s1 - s0
        for h in range(nH):
            out[s0:s1, h * 64:(h + 1) * 64] = emulate(x[s0:s1, 0, h], x[s0:s1, 1, h], x[s0:s1, 2, h], window, klen, **kw)
    return torch.from_numpy(out)


def _ratio(got, ref):
    err = (got.double() - ref.value).abs()
    return float((err / ref.bound()).max())


# the CPU-sized cases of the GPU test: packs around the 64-row edges, a long single sequence, key lengths
PACK = [5, 1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 3]
CASES = [(PACK, w, None) for w in (0, 1, 17, 64, 65, 128, 192)] + [([1100], 0, None), ([1100], 64, None),
                                                                   ([128] * 6, 0, [1, 63, 64, 65, 127, 128])]


@pytest.mark.parametrize("family", ao.FAMILIES)
@pytest.mark.parametrize("lens,window,kv", CASES, ids=[f"{len(c[0])}x{max(c[0])}-w{c[1]}-kv{c[2] is not None}" for c in CASES])
def test_bound_holds_for_the_emulated_kernel(family, lens, window, kv):
    cu = _cu(lens)
    qkv = ao.make_qkv(family, cu, 2, window, kv, seed=len(lens) + window)
    ref = ao.attention(qkv, cu, 2, window, kv)
    got = emulate_pack(qkv, cu, 2, window, kv)
    r = _ratio(got, ref)
    assert r <= 1.0, f"{family}: |err| / bound = {r:.3g}"


# ---- sensitivity: each kernel defect moves the output by > 10x the bound on the test's inputs -----------------------
def _moved(ref, other):
    """largest |other - ref| / bound"""
    return float(((other.double() - ref.value).abs() / ref.bound()).max())


@pytest.mark.parametrize("family", ["needle", "random", "uniform", "position"])
@pytest.mark.parametrize("window", [1, 17, 63, 64, 65, 127, 128])
def test_window_off_by_one_is_seen(family, window):
    cu = _cu(PACK)
    qkv = ao.make_qkv(family, cu, 2, window, seed=window)
    ref = ao.attention(qkv, cu, 2, window)
    for w2 in (window - 1, window + 1):
        if w2 >= 1:
            assert _moved(ref, ao.attention(qkv, cu, 2, w2).value) > 10, (family, window, w2)


@pytest.mark.parametrize("family", ["needle", "random"])
@pytest.mark.parametrize("L", [32, 128, 256, 512])
def test_kv_len_off_by_one_is_seen(family, L):
    kvs = sorted({min(x, L) for x in (1, 63, 64, 65, L - 1, L)})
    cu = _cu([L] * len(kvs))
    qkv = ao.make_qkv(family, cu, 2, 0, kvs, seed=L)
    ref = ao.attention(qkv, cu, 2, 0, kvs)
    for d in (-1, 1):
        kv2 = [min(max(x + d, 1), L) for x in kvs]
        got = ao.attention(qkv, cu, 2, 0, kv2).value
        for b, (x, y) in enumerate(zip(kvs, kv2)):
            if x != y:
                s = slice(cu[b], cu[b + 1])
                r = float(((got[s] - ref.value[s]).abs() / ref.bound()[s]).max())
                assert r > 10, (family, L, x, y, r)


@pytest.mark.parametrize("family", ["position", "random", "uniform"])
@pytest.mark.parametrize("L,window", [(1100, 0), (1100, 64), (300, 0)])
def test_skipped_block_is_seen(family, L, window):
    cu = [0, L]
    qkv = ao.make_qkv(family, cu, 1, window, seed=L)
    ref = ao.attention(qkv, cu, 1, window)
    for blk in sorted({0, 1, (L - 1) // 128, (L - 1) // 64}):
        assert _moved(ref, emulate_pack(qkv, cu, 1, window, drop_block=blk)) > 10, (family, blk)


@pytest.mark.parametrize("family", ["late", "random"])
@pytest.mark.parametrize("L,window", [(1100, 0), (1100, 64), (300, 0)])
@pytest.mark.parametrize("which", ["o", "l"])
def test_missing_alpha_is_seen(family, L, window, which):
    cu = [0, L]
    qkv = ao.make_qkv(family, cu, 1, window, seed=L + 1)
    ref = ao.attention(qkv, cu, 1, window)
    got = emulate_pack(qkv, cu, 1, window, alpha_o=which != "o", alpha_l=which != "l")
    assert _moved(ref, got) > 10


def test_needle_dominates_at_the_mask_edge():
    """the needle family's hidden key would carry most of its row's weight if it were visible"""
    L, w = 300, 17
    qkv = ao.make_qkv("needle", [0, L], 1, w, seed=0)
    q, k, _ = (t.double()[:, 0] for t in _split(qkv, 1))
    s = 0.125 * q @ k.t()
    i = torch.arange(20, L - 20)
    t = i + torch.where(i % 2 == 0, w + 1, -(w + 1))
    inside = i + torch.where(i % 2 == 0, w, -w)
    hidden_p = torch.softmax(s[i], -1)[torch.arange(len(i)), t]
    assert float(hidden_p.min()) > 0.5
    visible = s[i].masked_fill((torch.arange(L)[None] - i[:, None]).abs() > w, -torch.inf)
    assert torch.equal(visible.argmax(-1), inside)          # the best visible key is the edge key
