"""CPU checks of oracle/row_oracle.py: its values against torch / encoder_oracle in float64, its bounds against a
float32 restatement of the kernels' summation order, the tie rules, and that the inputs of tests/test_row_kernels_gpu.py
make every parameter move the output by at least 10x the bound."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import encoder_oracle as eo
from oracle import row_oracle as ro

f32 = np.float32


def _rows(T, H, g, mean=0.5, small_every=3):
    """the row recipe of the GPU test: every `small_every`-th row has a variance of ~1e-4"""
    x = torch.randn(T, H, generator=g)
    x[::small_every] *= 1e-2
    return x + mean * torch.randn(T, 1, generator=g)


def _head_inputs(B, H, g):
    x = (1.0 + 2.0 * torch.rand(B, H, generator=g)) * torch.sign(torch.randn(B, H, generator=g))
    x[1::2] = 2.0 + 0.005 * torch.randn(x[1::2].shape, generator=g)
    return x


def _min_ratio(a, b):
    """smallest |a - b| / (bound_a + bound_b) over rows, each row's largest element"""
    r = (a.value - b.value).abs() / (a.eps + b.eps)
    return float(r.amax(-1).min())


# ---- values against torch and encoder_oracle --------------------------------------------------------------------
@pytest.mark.parametrize("bias", [False, True])
def test_layer_norm_value(bias):
    g = torch.Generator().manual_seed(1)
    x = _rows(50, 384, g).double()
    w, b = torch.randn(384, generator=g).double(), (torch.randn(384, generator=g).double() if bias else None)
    ref = ro.layer_norm(x, w, b, 1e-5, ro.warp_ln_depth(384))
    torch.testing.assert_close(ref.value, F.layer_norm(x, (384,), w, b, 1e-5), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("erf", [False, True])
def test_gelu_value(erf):
    x = torch.linspace(-8, 8, 4001, dtype=torch.float64)
    ref = ro.gelu(x, erf)
    torch.testing.assert_close(ref.value, F.gelu(x, approximate="none" if erf else "tanh"), rtol=1e-13, atol=1e-15)


def test_softmax_value():
    g = torch.Generator().manual_seed(2)
    l = torch.randn(20, 33, generator=g, dtype=torch.float64) * 5
    p = ro.softmax(ro.Ref(l, torch.zeros_like(l), torch.zeros_like(l)))
    torch.testing.assert_close(p.value, torch.softmax(l, -1), rtol=1e-14, atol=0)


@pytest.mark.parametrize("ln", [False, True])
def test_pool_value(ln):
    g = torch.Generator().manual_seed(3)
    lens = [5, 1, 57, 12]
    S, H = max(lens), 384
    hidden = torch.randn(len(lens), S, H, generator=g, dtype=torch.float64)
    mask = torch.zeros(len(lens), S, dtype=torch.long)
    for i, L in enumerate(lens):
        mask[i, :L] = 1
    w = torch.randn(H, generator=g, dtype=torch.float64) if ln else None
    rows = torch.cat([hidden[i, :L] for i, L in enumerate(lens)])
    cu = np.concatenate([[0], np.cumsum(lens)])
    got = ro.pool_rows(rows, cu, 0, w, None, 1e-5)
    want = eo.masked_mean_pool(eo.layer_norm(hidden, w, None, 1e-5) if ln else hidden, mask)
    torch.testing.assert_close(got.value, want, rtol=1e-12, atol=1e-12)
    cls = ro.pool_rows(rows, cu, 1, w, None, 1e-5)
    torch.testing.assert_close(cls.value, (eo.layer_norm(hidden, w, None, 1e-5) if ln else hidden)[:, 0])
    div = ro.pool_rows(rows, cu, 0, None, None, 0.0, div_lens=[2, 1, 50, 12])
    torch.testing.assert_close(div.value[2], hidden[2, :57].sum(0) / 50)


@pytest.mark.parametrize("hf", [False, True])
def test_seq_head_value(hf):
    g = torch.Generator().manual_seed(4)
    H = 384
    wts = {"head.dense.weight": torch.randn(H, H, generator=g, dtype=torch.float64) / H ** 0.5,
           "head.norm.weight": torch.randn(H, generator=g, dtype=torch.float64)}
    x = torch.randn(6, H, generator=g, dtype=torch.float64)
    hid = ro.seq_head_hidden(x, 1, wts["head.dense.weight"], None, wts["head.norm.weight"], gelu_erf=hf,
                             head_eps=1e-5 if hf else 1e-12)
    want = eo.modernbert_head_hf(wts, x, 1e-5) if hf else eo.modernbert_head(wts, x)
    torch.testing.assert_close(hid.value, want, rtol=1e-10, atol=1e-10)
    p = torch.randn(H, H, generator=g, dtype=torch.float64)
    b = torch.randn(H, generator=g, dtype=torch.float64)
    torch.testing.assert_close(ro.seq_head_hidden(x, 2, p, b).value, torch.tanh(x @ p.t() + b))
    torch.testing.assert_close(ro.seq_head_hidden(x, 3, p, b).value, torch.tanh(x @ p + b))


# ---- bounds against a float32 restatement of the kernels --------------------------------------------------------------
def _warp_sum(lanes):
    """xor butterfly over a [..., 32] array in float32"""
    v = lanes.astype(f32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., np.arange(32) ^ o]).astype(f32)
    return v[..., 0]


def _warp_ln_f32(x, w, b, eps):
    """row_layernorm: lane l holds float4 #(i * 32 + l) for i < NV, (x + y) + (z + w) per float4, NV partials in
    order, 5 shuffle levels, times 1/H; the same for the centred squares"""
    T, H = x.shape
    NV = H // 128
    v = x.astype(f32).reshape(T, NV, 32, 4)
    inv_h = f32(1.0) / f32(H)

    def lane_sums(a):
        s = np.zeros((T, 32), f32)
        for i in range(NV):
            s = (s + ((a[:, i, :, 0] + a[:, i, :, 1]) + (a[:, i, :, 2] + a[:, i, :, 3]))).astype(f32)
        return s
    mean = (_warp_sum(lane_sums(v)) * inv_h).astype(f32)
    d = (v - mean[:, None, None, None]).astype(f32)
    q = _warp_sum(lane_sums((d * d).astype(f32)))
    rstd = (f32(1.0) / np.sqrt((q * inv_h + f32(eps)).astype(f32))).astype(f32)
    y = (d * rstd[:, None, None, None]).astype(f32).reshape(T, H) * w.astype(f32)
    if b is not None:
        y = (y.astype(f32) + b.astype(f32)).astype(f32)
    return y.astype(f32)


@pytest.mark.parametrize("H", [384, 768, 1024])
@pytest.mark.parametrize("eps", [1e-5, 1e-12])
def test_layer_norm_bound_f32(H, eps):
    g = torch.Generator().manual_seed(H)
    x = (_rows(300, H, g) * 3).float()
    x[1::7] += 40.0   # rows whose mean dwarfs their spread
    w, b = torch.randn(H, generator=g), torch.randn(H, generator=g)
    ref = ro.layer_norm(x, w, b, eps, ro.warp_ln_depth(H))
    y = torch.from_numpy(_warp_ln_f32(x.numpy(), w.numpy(), b.numpy(), eps)).double()
    ratio = float(((y - ref.value).abs() / ref.eps).max())
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("Cn", [1, 2, 9, 33, 100, 256])
def test_softmax_bound_f32(Cn):
    """token_head's softmax: exact max, per-lane sums over the 8 slots, 5 shuffle levels, one division"""
    g = torch.Generator().manual_seed(Cn)
    l = (torch.randn(200, Cn, generator=g) * torch.tensor([0.1, 3.0, 30.0]).repeat(67)[:200, None]).float()
    ref = ro.softmax(ro.Ref(l.double(), torch.zeros(l.shape, dtype=torch.float64), torch.zeros(l.shape, dtype=torch.float64)))
    ln = l.numpy()
    lanes = np.full((200, 8 * 32), -np.inf, f32)
    lanes[:, :Cn] = ln
    mx = ln.max(1)
    e = np.exp((lanes - mx[:, None]).astype(f32)).astype(f32).reshape(200, 8, 32)
    se = np.zeros((200, 32), f32)
    for k in range(8):
        se = (se + e[:, k]).astype(f32)
    p = (e.reshape(200, 256)[:, :Cn] / _warp_sum(se)[:, None]).astype(f32)
    ratio = float(((torch.from_numpy(p).double() - ref.value).abs() / ref.eps).max())
    assert ratio <= 1.0, ratio


# ---- tie rules ---------------------------------------------------------------------------------------------------------
def test_tie_rules():
    p = np.array([0.1, 0.4, 0.1, 0.4], f32)
    assert ro.seq_class(p, 0) == 1 and ro.seq_class(p, 1) == 3
    assert ro.seq_class(np.array([0.5, 0.5], f32), 0) == 0 and ro.seq_class(np.array([0.5, 0.5], f32), 1) == 1
    l = np.array([-3.0, -1.0, -2.0, -1.0, -5.0], f32)   # negative logits: the token argmax does not start from 0.0
    assert ro.token_pred(l, 0) == 1 and ro.token_pred(l, 1) == 3
    assert ro.token_pred(np.array([2.0], f32), 0) == 0 == ro.token_pred(np.array([2.0], f32), 1)
    assert eo.argmax_max_by(p) == ro.seq_class(p, 1)


# ---- every parameter is visible at the test inputs ---------------------------------------------------------------
def test_knobs_exceed_bounds():
    g = torch.Generator().manual_seed(7)
    H = 768
    sel = lambda r, s: ro.Ref(r.value[s], r.coef[s], r.eps[s])   # noqa: E731
    # LayerNorm eps on the small-variance rows
    x = _rows(30, H, g)
    w = 1.0 + 0.5 * torch.randn(H, generator=g)
    a, b = (ro.layer_norm(x, w, None, e, ro.warp_ln_depth(H)) for e in (1e-5, 1e-12))
    assert _min_ratio(sel(a, slice(0, None, 3)), sel(b, slice(0, None, 3))) > 10
    # head GELU flavour and head eps (sequence head, ModernBERT mode)
    pooled = _head_inputs(8, H, g)
    dw = torch.eye(H) + 0.002 * torch.randn(H, H, generator=g) / H ** 0.5
    nw = 0.5 + torch.rand(H, generator=g)
    hid = {(erf, e): ro.seq_head_hidden(pooled, 1, dw, None, nw, gelu_erf=erf, head_eps=e)
           for erf in (False, True) for e in (1e-5, 1e-12)}
    assert _min_ratio(sel(hid[(False, 1e-12)], slice(0, None, 2)), sel(hid[(True, 1e-12)], slice(0, None, 2))) > 10
    assert _min_ratio(sel(hid[(True, 1e-5)], slice(1, None, 2)), sel(hid[(True, 1e-12)], slice(1, None, 2))) > 10
    # BERT type row and bias
    word = _rows(40, H, g)
    pos_emb, type0 = 0.5 * torch.randn(16, H, generator=g), 0.5 * torch.randn(H, generator=g)
    lw, lb = 1.0 + 0.5 * torch.randn(H, generator=g), 0.5 * torch.randn(H, generator=g)
    ids, pos = torch.arange(40), torch.arange(40) % 16
    with_t = ro.embed_ln_bert(ids, pos, word, pos_emb, type0, lw, lb, 1e-12, 16)
    no_t = ro.embed_ln_bert(ids, pos, word, pos_emb, torch.zeros(H), lw, lb, 1e-12, 16)
    assert _min_ratio(with_t, no_t) > 10
    # L2 norm_eps and its position at the smallest row scale of the GPU test
    p = torch.randn(4, H, generator=g) * 1e-12 / 8.0
    for dim in (1, 64, H):
        a, b = ro.l2_normalize(p, dim, 1e-12), ro.l2_normalize(p, dim, 0.0)
        assert _min_ratio(a, b) > 10
        inside = p.double()[:, :dim] / torch.sqrt((p.double()[:, :dim] ** 2).sum(1, keepdim=True) + 1e-12)
        assert float(((inside - a.value).abs() / a.eps).amax(-1).min()) > 10
