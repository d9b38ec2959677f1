"""The float64 GEMM reference (oracle/gemm_oracle.py) against independent formulations of each epilogue (CPU only)."""
import math

import pytest
import torch

from oracle import gemm_oracle as go


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _f16(shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).half()


def _interleave(wi):
    """GeGLU weight layout of the device: rows regrouped in 32-row (a | b) pairs."""
    i = wi.shape[0] // 2
    perm = torch.empty_like(wi)
    for j in range(i // 32):
        perm[64 * j:64 * j + 32] = wi[32 * j:32 * j + 32]
        perm[64 * j + 32:64 * j + 64] = wi[i + 32 * j:i + 32 * j + 32]
    return perm


def test_tau_cap():
    # one missing k-term of average size at K <= 4096 is >= 2^-12 S: at least 16x the accumulation bound
    assert 0 < go.TAU <= 2.0 ** -16


def test_ulp16():
    y = torch.tensor([1.0, 1.5, 2.0, 1000.0, -3.0, 2.0 ** -14, 2.0 ** -20, 0.0], dtype=torch.float64)
    want = torch.tensor([2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 0.5, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24],
                        dtype=torch.float64)
    assert torch.equal(go.ulp16(y), want)
    # fp16 rounding of an fp32 value moves it by at most half an ulp
    x = (torch.randn(10000, generator=_gen(0), dtype=torch.float64) * 10).float().double()
    assert ((x.half().double() - x).abs() <= 0.5 * go.ulp16(x)).all()


def test_geglu_interleave():
    g = _gen(1)
    M, K, I = 37, 72, 192
    a, wi = _f16((M, K), g), _f16((2 * I, K), g, 0.1)
    r = go.gemm(go.EPI_GEGLU, a, _interleave(wi), 2 * I)
    full = a.double() @ wi.double().t()
    want = torch.nn.functional.gelu(full[:, :I]) * full[:, I:]
    torch.testing.assert_close(r.value, want, rtol=1e-12, atol=1e-12)
    assert (r.coef > 0).all() and (r.eps > 0).all()


def test_rope_is_complex_multiplication():
    g = _gen(2)
    M, K, N, rope_cols = 29, 64, 320, 192
    a, w = _f16((M, K), g), _f16((N, K), g, 0.1)
    pos = torch.randint(0, 50, (M,), generator=g, dtype=torch.int32)
    theta = torch.rand(50, 32, generator=g, dtype=torch.float64) * 6.3
    cos, sin = torch.cos(theta).float(), torch.sin(theta).float()
    r = go.gemm(go.EPI_ROPE, a, w, rope_cols=rope_cols, pos=pos, rope_cos=cos, rope_sin=sin)
    full = a.double() @ w.double().t()
    rot = torch.complex(cos.double()[pos.long()], sin.double()[pos.long()])
    for h0 in range(0, N, 64):
        z = torch.complex(full[:, h0:h0 + 32], full[:, h0 + 32:h0 + 64])
        if h0 < rope_cols:
            z = z * rot
        torch.testing.assert_close(r.value[:, h0:h0 + 32], z.real, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(r.value[:, h0 + 32:h0 + 64], z.imag, rtol=1e-12, atol=1e-12)
    # the accumulation term of a rotated column: |cos| S1 + |sin| S2
    s = a.double().abs() @ w.double().abs().t()
    c, sn = cos.double()[pos.long()], sin.double()[pos.long()]
    torch.testing.assert_close(r.coef[:, :32], c.abs() * s[:, :32] + sn.abs() * s[:, 32:64])


@pytest.mark.parametrize("epi", [go.EPI_ROPE, go.EPI_GEGLU])
def test_fold_is_layernorm_then_matmul(epi):
    g = _gen(3)
    M, H, N = 45, 256, 256
    x = _f16((M, H), g, 2.0).double() + 0.5
    gamma = 1 + 0.2 * torch.randn(H, generator=g, dtype=torch.float64)
    w = torch.randn(N, H, generator=g, dtype=torch.float64) * 0.05
    wf = w * gamma[None, :]
    wf = wf - wf.mean(1, keepdim=True)     # zero-sum rows: the mean subtraction lives in the weights
    st = torch.stack([x.view(M, H // 128, 128).sum(2), (x * x).view(M, H // 128, 128).sum(2)], -1).transpose(0, 1)
    ln = torch.nn.functional.layer_norm(x, (H,), gamma, None, 1e-5)
    if epi == go.EPI_ROPE:
        r = go.gemm(epi, x, wf, fold_stats=st.float(), fold_eps=1e-5, fold_h=H)
        want = ln @ w.t()
    else:
        r = go.gemm(epi, x, _interleave(wf), fold_stats=st.float(), fold_eps=1e-5, fold_h=H)
        f = ln @ w.t()
        want = torch.nn.functional.gelu(f[:, :N // 2]) * f[:, N // 2:]
    # the statistics went through fp32: relative 1e-6
    torch.testing.assert_close(r.value, want, rtol=1e-6, atol=1e-6)
    rstd, rel = go.fold_rstd(st.float(), M, 1e-5, H)
    torch.testing.assert_close(rstd, 1.0 / torch.sqrt(x.var(1, unbiased=False) + 1e-5), rtol=1e-6, atol=0)
    assert (rel < 1e-5).all()


def test_grouped_weights():
    g = _gen(5)
    rows, G, K, N = 128, 3, 64, 128
    a, w = _f16((G * rows - 7, K), g), _f16((G * N, K), g, 0.1)
    r = go.gemm(go.EPI_RESID, a, w, N, w_groups=G, w_group_rows=rows)
    for i in range(G):
        sl = slice(i * rows, (i + 1) * rows)
        torch.testing.assert_close(r.value[sl], a[sl].double() @ w[i * N:(i + 1) * N].double().t(), rtol=1e-14, atol=0)


@pytest.mark.parametrize("epi", [go.EPI_F16, go.EPI_GELU, go.EPI_RESID])
def test_grouped_weights_with_a_bias_per_group(epi):
    """bias_per_group: rows of group g are group g's GEMM with group g's bias (the last group partly empty), and one
    bias for every group -- a group's rows adding group 0's vector -- is far outside the bound"""
    g = _gen(7)
    rows, G, K, N = 128, 3, 64, 128
    M = G * rows - 7
    a, w = _f16((M, K), g), _f16((G * N, K), g, 0.1)
    bias = torch.randn(G * N, generator=g)
    resid = torch.randn(M, N, generator=g) if epi == go.EPI_RESID else None
    r = go.gemm(epi, a, w, N, bias=bias, resid=resid, w_groups=G, w_group_rows=rows, bias_per_group=True)
    for i in range(G):
        sl = slice(i * rows, min((i + 1) * rows, M))
        one = go.gemm(epi, a[sl], w[i * N:(i + 1) * N], N, bias=bias[i * N:(i + 1) * N],
                      resid=None if resid is None else resid[sl])
        for x, y in ((r.value, one.value), (r.coef, one.coef), (r.eps, one.eps)):
            torch.testing.assert_close(x[sl], y, rtol=0, atol=0)
    shared = go.gemm(epi, a, w, N, bias=bias, resid=resid, w_groups=G, w_group_rows=rows)
    assert torch.equal(shared.value[:rows], r.value[:rows])
    assert ((shared.value[rows:] - r.value[rows:]).abs() > r.bound()[rows:]).any()


def test_gelu_derivative_and_bound_covers_rounding():
    x = torch.linspace(-8, 8, 2001, dtype=torch.float64)
    h = 1e-6
    torch.testing.assert_close(go.gelu_deriv(x), (go.gelu(x + h) - go.gelu(x - h)) / (2 * h), rtol=1e-6, atol=1e-8)
    # an exact accumulator rounded to fp16 output passes with TAU = 0
    g = _gen(6)
    a, w = _f16((20, 72), g), _f16((64, 72), g, 0.1)
    bias = torch.randn(64, generator=g)
    for epi in (go.EPI_F16, go.EPI_GELU):
        r = go.gemm(epi, a, w, bias=bias)
        assert r.tau_needed(r.value.half()) == 0.0
    r = go.gemm(go.EPI_F16, a, w, bias=bias)
    # a bias on the neighbouring column pair is far outside the bound
    bad = a.double() @ w.double().t() + bias.view(-1, 2).flip(1).reshape(-1).double()
    assert ((bad - r.value).abs() > r.bound()).any()


def test_topk_ties_lower_index_first():
    s = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0, -1.0], [0.5, 0.5, 0.5, 0.5, 0.5, 0.5]], dtype=torch.float64)
    idx, val = go.topk(s, 4)
    assert idx.tolist() == [[1, 2, 4, 3], [0, 1, 2, 3]]
    valid = torch.tensor([1, 1, 0, 1, 1, 1], dtype=torch.uint8)
    idx, val = go.topk(s, 4, valid)
    assert idx.tolist() == [[1, 4, 3, 0], [0, 1, 3, 4]]
    idx, val = go.topk(s, 8, valid)
    assert idx[0, 5:].tolist() == [-1, -1, -1] and math.isinf(float(val[0, 7]))
