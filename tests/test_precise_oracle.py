"""CPU checks of oracle/precise_oracle.py and of gemm_oracle.gemm(split=True): every reference equals a plain torch float64
computation, the float32 restatement of each precise-path kernel stays inside its bound with a margin >= 2 on every input
family of tests/test_precise_kernels_gpu.py, and each wrong kernel of precise_oracle.MUTATIONS leaves the bound by more
than 10x on those inputs.  The attention kernel with one fp32 chain over all keys (the accumulation before per-tile sums)
leaves the tiled kernel's bound on constant V columns at 32 768 keys."""
import math

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, gemm_oracle as go, precise_oracle as po

PACK = [1, 63, 64, 65, 127, 128, 129, 5]
WIDTHS = [384, 320, 1088]


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


def _ratio(got, ref_value, bound):
    r = (torch.as_tensor(np.asarray(got)).double() - ref_value).abs() / bound
    return float(torch.nan_to_num(r, nan=torch.inf).max())                 # a NaN output is outside every bound


def _rows(T, H, seed, family):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, H, generator=g) * torch.exp(torch.randn(T, 1, generator=g))
    if family == "specials":
        x[0, :8] = torch.tensor([65504.0, -65504.0, 2.0 ** -14, 0.75 * 2.0 ** -14, 1e-40, 0.0, -0.0, 2.0 ** -24])
        x[1] = 2.0 ** -10 * torch.randn(H, generator=g)
    elif family == "tiny":
        x[0] = 1000.0 + 1e-3 * torch.randn(H, generator=g)
        x[1] = 7.0
        x[1, ::7] = 7.0 + 2.0 ** -21
    return x


def _gamma(H):
    g = torch.Generator().manual_seed(H)
    return torch.exp(torch.empty(H).uniform_(math.log(0.05), math.log(8.0), generator=g))


# ---- values --------------------------------------------------------------------------------------------------------
def test_split_halves_are_fp16_rn():
    x = _rows(9, 384, 1, "specials")
    hi, lo = po.split_halves(x.numpy())
    th = x.half()
    assert np.array_equal(hi.view(np.int16), th.numpy().view(np.int16))
    assert np.array_equal(lo.view(np.int16), (x - th.float()).half().numpy().view(np.int16))
    gh, gl = go.split_pair(x)
    assert np.array_equal(gh.numpy().view(np.int16), hi.view(np.int16))
    assert np.array_equal(gl.numpy().view(np.int16), lo.view(np.int16))


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_split_ln_value_is_layer_norm(eps):
    x, g = _rows(7, 320, 2, "random"), _gamma(320)
    want = torch.nn.functional.layer_norm(x.double(), (320,), g.double(), None, eps)
    torch.testing.assert_close(po.split_ln(x, g, eps).value, want, rtol=1e-12, atol=1e-13)


def test_rope_value_is_rotate_half():
    heads, T = 3, 40
    x = torch.randn(T, 3 * heads * 64)
    pos = torch.arange(T) * 7
    cos_t, sin_t = eo.rope_tables(64, 160000.0, 300)
    ref = po.rope(x, pos, heads, cos_t, sin_t)
    c, s = cos_t.double()[pos].repeat(1, 2)[:, None], sin_t.double()[pos].repeat(1, 2)[:, None]
    for third in (0, 1):
        blk = x.double()[:, third * heads * 64:(third + 1) * heads * 64].view(T, heads, 64)
        rot = torch.cat([-blk[..., 32:], blk[..., :32]], -1)
        want = (blk * c + rot * s).reshape(T, -1)
        torch.testing.assert_close(ref.value[:, third * heads * 64:(third + 1) * heads * 64], want, rtol=1e-12, atol=1e-13)
    assert torch.equal(ref.value[:, 2 * heads * 64:], x.double()[:, 2 * heads * 64:])


def test_geglu_value_is_gelu_erf_times_b():
    ab = torch.randn(5, 2 * 320) * 3
    torch.testing.assert_close(po.geglu(ab, 320).value, eo.gelu_erf(ab.double()[:, :320]) * ab.double()[:, 320:],
                               rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("window", [0, 1, 33])
def test_attention_value_is_softmax_attention(window):
    lens, nH = [1, 7, 64, 65, 130], 2
    cu = _cu(lens)
    qkv = po.make_qkv("random", cu, nH, seed=1)
    ref = po.attention(qkv, cu, nH, window)
    x = qkv.double().view(-1, 3, nH, 64)
    for b, L in enumerate(lens):
        s = slice(cu[b], cu[b + 1])
        att = torch.einsum("ihd,jhd->hij", x[s, 0], x[s, 1]) * 0.125
        if window > 0:
            i = torch.arange(L)
            att = att.masked_fill((i[None, :] - i[:, None]).abs()[None] > window, -torch.inf)
        want = torch.einsum("hij,jhd->ihd", torch.softmax(att, -1), x[s, 2]).reshape(L, nH * 64)
        torch.testing.assert_close(ref.value[s], want, rtol=1e-12, atol=1e-13)


def test_attention_sampled_rows_equal_all_rows():
    cu = _cu([300, 200])
    qkv = po.make_qkv("sink", cu, 2, seed=4)
    full = po.attention(qkv, cu, 2, 0)
    sel = torch.tensor([0, 31, 32, 299, 300, 499])
    part = po.attention(qkv, cu, 2, 0, sel=sel)
    torch.testing.assert_close(part.value, full.value[sel], rtol=1e-12, atol=0)
    torch.testing.assert_close(part.bound, full.bound[sel], rtol=1e-12, atol=0)


def test_gemm_split_value_is_the_unsplit_product():
    g = torch.Generator().manual_seed(5)
    a, w = torch.randn(33, 96, generator=g), 0.02 * torch.randn(40, 96, generator=g)
    r = torch.randn(33, 40, generator=g)
    ref = go.gemm(go.EPI_RESID, a, w, 40, resid=r, split=True)
    torch.testing.assert_close(ref.value, r.double() + a.double() @ w.double().t(), rtol=1e-12, atol=1e-13)
    a3, w3 = go.split3(a, w)
    assert a3.shape == (33, 288) and w3.shape == (40, 288)
    hi, lo = po.split_halves(a.numpy())
    assert np.array_equal(a3[:, :96].numpy().view(np.int16), hi.view(np.int16))
    assert np.array_equal(a3[:, 96:192].numpy().view(np.int16), lo.view(np.int16))
    assert np.array_equal(a3[:, 192:].numpy().view(np.int16), hi.view(np.int16))


# ---- restatements inside the bounds, mutations outside -------------------------------------------------------------
@pytest.mark.parametrize("family", ["random", "specials", "tiny"])
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_split_ln_restatement_and_mutations(family, H, eps):
    x, g = _rows(9, H, H + len(family), family), _gamma(H)
    ref = po.split_ln(x, g, eps)
    hi, lo, v = po.restate_split(x.numpy(), g.numpy(), eps)
    assert _ratio(v, ref.value, ref.bound - ref.split) <= 0.5           # the LayerNorm's arithmetic, with a margin of 2
    assert _ratio(hi.astype(np.float64) + lo.astype(np.float64), ref.value, ref.bound) <= 1.0
    if family == "random":
        for mut in ("split_no_lo", "ln_no_gamma"):
            mh, ml, _ = po.restate_split(x.numpy(), g.numpy(), eps, mut=mut)
            assert _ratio(mh.astype(np.float64) + ml.astype(np.float64), ref.value, ref.bound) > 10, mut


@pytest.mark.parametrize("heads", [1, 12])
def test_rope_restatement_and_mutations(heads):
    lens = [1, 63, 300, 129]
    cu = _cu(lens)
    T = cu[-1]
    pos = torch.cat([torch.arange(n) for n in lens])
    x = 3 * torch.randn(T, 3 * heads * 64, generator=torch.Generator().manual_seed(heads))
    cos_g, sin_g = eo.rope_tables(64, 160000.0, 400)
    cos_l, sin_l = eo.rope_tables(64, 10000.0, 400)
    ref = po.rope(x, pos, heads, cos_g, sin_g)
    bound = ref.bound + 2.0 ** -140
    got = po.restate_rope(x.numpy(), pos.numpy(), heads, cos_g.numpy(), sin_g.numpy())
    assert _ratio(got, ref.value, bound) <= 0.5
    for mut in ("rope_swapped_halves", "rope_local_table"):
        bad = po.restate_rope(x.numpy(), pos.numpy(), heads, cos_g.numpy(), sin_g.numpy(), mut=mut,
                              cos_other=cos_l.numpy(), sin_other=sin_l.numpy())
        assert _ratio(bad, ref.value, bound) > 10, mut


@pytest.mark.parametrize("I", [320, 1088])
def test_geglu_restatement_and_mutation(I):
    T = 7
    a = torch.linspace(-10.0, 10.0, T * I).view(T, I)
    b = 2 * torch.randn(T, I, generator=torch.Generator().manual_seed(I))
    ab = torch.cat([a, b], 1)
    ref = po.geglu(ab, I)
    assert _ratio(po.restate_geglu(ab.numpy(), I), ref.value, ref.bound) <= 0.5
    assert _ratio(po.restate_geglu(ab.numpy(), I, mut="gelu_tanh"), ref.value, ref.bound) > 10
    tail = (a < -4).numpy()                                   # the cancelling tail: an element-relative check fails there
    tail &= ref.value.numpy() != 0
    rel = np.abs(po.restate_geglu(ab.numpy(), I).astype(np.float64) - ref.value.numpy())[tail] / ref.value.abs().numpy()[tail]
    assert rel.max() > 1e-3


@pytest.mark.parametrize("family", po.FAMILIES)
@pytest.mark.parametrize("window", [0, 1, 31, 33, 64])
def test_attention_restatement_within_bound(family, window):
    cu = _cu(PACK)
    qkv = po.make_qkv(family, cu, 2, window, seed=window + 3)
    ref = po.attention(qkv, cu, 2, window)
    got = po.restate_attention(qkv.numpy(), cu, 2, window)
    r = _ratio(got, ref.value, ref.bound)
    assert r <= 0.5, r


@pytest.mark.parametrize("mut,window", [("window_minus_one", 33), ("window_minus_one", 1), ("short_tile", 0),
                                        ("short_tile", 31), ("no_alpha", 0), ("scale_twice", 0)])
def test_attention_mutations_leave_the_bound(mut, window):
    cu = _cu(PACK)
    family = "late" if mut == "no_alpha" else "random"
    qkv = po.make_qkv(family, cu, 2, window, seed=7)
    ref = po.attention(qkv, cu, 2, window)
    bad = po.restate_attention(qkv.numpy(), cu, 2, window, mut=mut)
    assert _ratio(bad, ref.value, ref.bound) > 10, mut


def test_one_chain_leaves_the_tiled_bound_at_32768_constant_keys():
    """constant V under uniform scores: the tiled kernel stays inside its bound, one chain over every key does not"""
    L = 32768
    cu = [0, L]
    qkv = po.make_qkv("constant", cu, 1, seed=1)
    sel = np.array([0, L // 2, L - 1])
    ref = po.attention(qkv, cu, 1, 0, sel=torch.from_numpy(sel))
    tiled = po.restate_attention(qkv.numpy(), cu, 1, 0, sel=sel)
    one = po.restate_attention(qkv.numpy(), cu, 1, 0, sel=sel, chain="one")
    assert _ratio(tiled, ref.value, ref.bound) <= 0.5
    assert _ratio(one, ref.value, ref.bound) > 2
