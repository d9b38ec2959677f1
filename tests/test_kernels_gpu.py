"""Unit parity of the CUDA kernels through the C ABI (sr_test_* hooks) against fp32 torch math on the
same fp16-rounded operands.  Tolerances: fp32 outputs 1e-4 relative (accumulation order only), fp16 outputs
one fp16 ulp (2^-10 relative) plus the same."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_F16, EPI_ROPE, EPI_RESID, EPI_GEGLU, EPI_GELU = range(5)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _gemm(lib, a, w, out, epi, bias=None, resid=None, pos=None, cos=None, sin=None, rope_cols=0):
    M, K = a.shape
    N = w.shape[0]
    rc = lib.sr_test_gemm(_ptr(a), _ptr(w), _ptr(out), M, N, K, epi, out.shape[1], _ptr(bias), _ptr(resid),
                          _ptr(pos), _ptr(cos), _ptr(sin), rope_cols)
    torch.cuda.synchronize()
    assert rc == 0


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 768, 768), (300, 2304, 768), (1000, 768, 1152),
                                   (77, 384, 384), (4096, 768, 768), (1, 256, 768), (129, 1152, 384),
                                   (2177, 2304, 768), (2048, 256, 64), (5000, 768, 1152)])  # M >= 2048: many row blocks per worker
def test_gemm_f16_store(srlib, cuda, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = (torch.randn(N, K, device=cuda, generator=g) * 0.05).half()
    bias = torch.randn(N, device=cuda, generator=g)
    out = torch.full((M, N), float("nan"), device=cuda, dtype=torch.float16)
    _gemm(srlib.lib(), a, w, out, EPI_F16, bias=bias)
    ref = a.float() @ w.float().t() + bias
    torch.testing.assert_close(out.float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("M,N,K", [(128, 768, 768), (515, 768, 1152), (200, 384, 1536), (2500, 768, 1152),
                                   (4224, 768, 768)])
def test_gemm_resid_f32(srlib, cuda, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = (torch.randn(N, K, device=cuda, generator=g) * 0.05).half()
    resid = torch.randn(M, N, device=cuda, generator=g)
    bias = torch.randn(N, device=cuda, generator=g)
    x = resid.clone()
    _gemm(srlib.lib(), a, w, x, EPI_RESID, resid=x, bias=bias)          # in place
    ref = a.float() @ w.float().t() + bias + resid
    torch.testing.assert_close(x, ref, rtol=1e-4, atol=1e-4)
    out = torch.zeros(M, N, device=cuda)
    _gemm(srlib.lib(), a, w, out, EPI_RESID)                             # plain fp32 store
    torch.testing.assert_close(out, a.float() @ w.float().t(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("M", [260, 2300])
def test_gemm_geglu(srlib, cuda, M):
    H, I = 768, 1152
    g = torch.Generator(device="cuda").manual_seed(9)
    a = torch.randn(M, H, device=cuda, generator=g).half()
    wi = (torch.randn(2 * I, H, device=cuda, generator=g) * 0.05).half()
    perm = torch.empty_like(wi)
    for j in range(I // 32):
        perm[64 * j:64 * j + 32] = wi[32 * j:32 * j + 32]
        perm[64 * j + 32:64 * j + 64] = wi[I + 32 * j:I + 32 * j + 32]
    out = torch.zeros(M, I, device=cuda, dtype=torch.float16)
    _gemm(srlib.lib(), a, perm.contiguous(), out, EPI_GEGLU)
    full = a.float() @ wi.float().t()
    ref = torch.nn.functional.gelu(full[:, :I]) * full[:, I:]
    torch.testing.assert_close(out.float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("M", [140, 2100])
def test_gemm_gelu_bias(srlib, cuda, M):
    N, K = 3072, 768
    g = torch.Generator(device="cuda").manual_seed(10)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = (torch.randn(N, K, device=cuda, generator=g) * 0.05).half()
    bias = torch.randn(N, device=cuda, generator=g)
    out = torch.zeros(M, N, device=cuda, dtype=torch.float16)
    _gemm(srlib.lib(), a, w, out, EPI_GELU, bias=bias)
    ref = torch.nn.functional.gelu(a.float() @ w.float().t() + bias)
    torch.testing.assert_close(out.float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("M", [333, 2333])
def test_gemm_rope(srlib, cuda, M):
    from oracle import encoder_oracle as eo
    H, nH = 768, 12
    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randn(M, H, device=cuda, generator=g).half()
    w = (torch.randn(3 * H, H, device=cuda, generator=g) * 0.05).half()
    pos = torch.randint(0, 700, (M,), device=cuda, generator=g, dtype=torch.int32)
    cos, sin = eo.rope_tables(64, 160000.0, 1024)
    cos, sin = cos.to(cuda).contiguous(), sin.to(cuda).contiguous()
    out = torch.zeros(M, 3 * H, device=cuda, dtype=torch.float16)
    _gemm(srlib.lib(), a, w, out, EPI_ROPE, pos=pos, cos=cos, sin=sin, rope_cols=2 * H)
    full = (a.float() @ w.float().t()).reshape(M, 3, nH, 64)
    c, s = cos[pos.long()][:, None, :], sin[pos.long()][:, None, :]
    ref = full.clone()
    for t in range(2):
        x1, x2 = full[:, t, :, :32], full[:, t, :, 32:]
        ref[:, t, :, :32] = x1 * c - x2 * s
        ref[:, t, :, 32:] = x1 * s + x2 * c
    torch.testing.assert_close(out.float(), ref.reshape(M, 3 * H), rtol=2e-3, atol=2e-3)


def _attn_ref(qkv, cu, nH, window):
    T = qkv.shape[0]
    H = nH * 64
    out = torch.zeros(T, H, device=qkv.device)
    q, k, v = qkv.float().reshape(T, 3, nH, 64).unbind(1)
    for b in range(len(cu) - 1):
        s, e = cu[b], cu[b + 1]
        qs, ks, vs = (t[s:e].transpose(0, 1) for t in (q, k, v))      # [nH, L, 64]
        att = (qs * 0.125) @ ks.transpose(-2, -1)
        if window > 0:
            idx = torch.arange(e - s, device=qkv.device)
            att = att.masked_fill((idx[None, :] - idx[:, None]).abs()[None] > window, float("-inf"))
        p = torch.softmax(att, -1)
        out[s:e] = (p @ vs).transpose(0, 1).reshape(e - s, H)
    return out


@pytest.mark.parametrize("impl", ["tcgen05", "mma_sync", "tcgen05_window"])
@pytest.mark.parametrize("window", [0, 64, 17])
@pytest.mark.parametrize("lens", [[512], [1, 2, 63, 64, 65], [129, 130, 700, 31], [2048], [128, 256, 127, 257, 5]])
def test_attention(srlib, cuda, lens, window, impl):
    nH = 12
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    T = int(cu[-1])
    g = torch.Generator(device="cuda").manual_seed(T + window)
    qkv = torch.randn(T, 3 * nH * 64, device=cuda, generator=g).half()
    out = torch.full((T, nH * 64), float("nan"), device=cuda, dtype=torch.float16)
    cu_d = torch.from_numpy(cu).to(cuda)
    if impl == "tcgen05_window" and window == 0:
        pytest.skip("the one-shot window kernel needs a window")
    if impl == "tcgen05_window":
        rc = srlib.lib().sr_test_attention_win(qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), len(lens), T, max(lens), nH, window)
    elif impl == "tcgen05":
        rc = srlib.lib().sr_test_attention_tc(qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), len(lens), T, max(lens), nH, window)
    else:
        rc = srlib.lib().sr_test_attention(qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), len(lens), max(lens), nH, window)
    torch.cuda.synchronize()
    assert rc == 0
    ref = _attn_ref(qkv, cu.tolist(), nH, window)
    torch.testing.assert_close(out.float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("H", [384, 768, 1024])
def test_layernorm(srlib, cuda, H):
    T = 1037
    g = torch.Generator(device="cuda").manual_seed(H)
    x = torch.randn(T, H, device=cuda, generator=g) * 3 + 0.5
    w = torch.randn(H, device=cuda, generator=g)
    b = torch.randn(H, device=cuda, generator=g)
    y32 = torch.zeros_like(x)
    y16 = torch.zeros(T, H, device=cuda, dtype=torch.float16)
    rc = srlib.lib().sr_test_layernorm(x.data_ptr(), T, H, w.data_ptr(), b.data_ptr(), 1e-5, y32.data_ptr(), y16.data_ptr())
    torch.cuda.synchronize()
    assert rc == 0
    ref = torch.nn.functional.layer_norm(x, (H,), w, b, 1e-5)
    torch.testing.assert_close(y32, ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(y16.float(), ref, rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("M", [300, 2500])
def test_gemm_layernorm_fold(srlib, cuda, M):
    """LayerNorm folded into the GEMMs around it: the residual GEMM emits fp16(x) and per-row (sum, sum of squares);
    the consuming projections multiply the raw rows with W diag(gamma) re-centred to zero-sum rows (the mean subtraction
    moves into the weights) and scale by the row's rstd in the epilogue.
    Checked against torch LayerNorm + plain matmuls, for the RoPE and the GeGLU consumer."""
    from oracle import encoder_oracle as eo
    lib = srlib.lib()
    H, I, nH = 768, 1152, 12
    g = torch.Generator(device="cuda").manual_seed(M)
    # ---- producer: x += a @ w^T, fp16 copy, row statistics
    a = torch.randn(M, H, device=cuda, generator=g).half()
    w = (torch.randn(H, H, device=cuda, generator=g) * 0.05).half()
    x0 = torch.randn(M, H, device=cuda, generator=g) * 2 + 0.3
    x = x0.clone()
    stats = torch.full((H // 128, M, 2), float("nan"), device=cuda)   # per-128-column partials, each written once
    raw = torch.full((M, H), float("nan"), device=cuda, dtype=torch.float16)
    rc = lib.sr_test_gemm_fold(_ptr(a), _ptr(w), _ptr(x), M, H, H, EPI_RESID, H, None, _ptr(x), None, None, None, 0,
                               _ptr(stats), _ptr(raw), None, 0.0, 0, None, None, None)
    torch.cuda.synchronize()
    assert rc == 0
    ref_x = a.float() @ w.float().t() + x0
    torch.testing.assert_close(x, ref_x, rtol=1e-4, atol=2e-4)
    torch.testing.assert_close(raw.float(), ref_x, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(stats[..., 0].sum(0), ref_x.sum(1), rtol=1e-4, atol=2e-2)
    torch.testing.assert_close(stats[..., 1].sum(0), (ref_x * ref_x).sum(1), rtol=1e-4, atol=1e-1)
    torch.testing.assert_close(stats[2, :, 0], ref_x[:, 256:384].sum(1), rtol=1e-4, atol=1e-2)
    gamma = 1 + 0.2 * torch.randn(H, device=cuda, generator=g)
    ln = torch.nn.functional.layer_norm(ref_x, (H,), gamma, None, 1e-5)
    # ---- consumer 1: Wqkv + RoPE over the raw rows
    wq = (torch.randn(3 * H, H, device=cuda, generator=g) * 0.05)
    wq_f = wq * gamma[None, :]
    wq_f = (wq_f - wq_f.mean(1, keepdim=True)).half()          # zero-sum rows: the mean subtraction lives in the weights
    pos = torch.randint(0, 700, (M,), device=cuda, generator=g, dtype=torch.int32)
    cos, sin = eo.rope_tables(64, 160000.0, 1024)
    cos, sin = cos.to(cuda).contiguous(), sin.to(cuda).contiguous()
    out = torch.zeros(M, 3 * H, device=cuda, dtype=torch.float16)
    rc = lib.sr_test_gemm_fold(_ptr(raw), _ptr(wq_f), _ptr(out), M, 3 * H, H, EPI_ROPE, 3 * H, None, None, _ptr(pos), _ptr(cos),
                               _ptr(sin), 2 * H, None, None, _ptr(stats), 1e-5, H, None, None, None)
    torch.cuda.synchronize()
    assert rc == 0
    full = (ln @ wq.t()).reshape(M, 3, nH, 64)
    c, s = cos[pos.long()][:, None, :], sin[pos.long()][:, None, :]
    ref = full.clone()
    for t in range(2):
        x1, x2 = full[:, t, :, :32], full[:, t, :, 32:]
        ref[:, t, :, :32] = x1 * c - x2 * s
        ref[:, t, :, 32:] = x1 * s + x2 * c
    torch.testing.assert_close(out.float(), ref.reshape(M, 3 * H), rtol=3e-3, atol=3e-3)
    # ---- consumer 2: Wi + GeGLU
    wi = torch.randn(2 * I, H, device=cuda, generator=g) * 0.05
    wi_f = wi * gamma[None, :]
    wi_f = (wi_f - wi_f.mean(1, keepdim=True)).half()
    perm = torch.empty_like(wi_f)
    for j in range(I // 32):
        perm[64 * j:64 * j + 32] = wi_f[32 * j:32 * j + 32]
        perm[64 * j + 32:64 * j + 64] = wi_f[I + 32 * j:I + 32 * j + 32]
    perm = perm.contiguous()
    mid = torch.zeros(M, I, device=cuda, dtype=torch.float16)
    rc = lib.sr_test_gemm_fold(_ptr(raw), _ptr(perm), _ptr(mid), M, 2 * I, H, EPI_GEGLU, I, None, None, None, None, None, 0,
                               None, None, _ptr(stats), 1e-5, H, None, None, None)
    torch.cuda.synchronize()
    assert rc == 0
    fi = ln @ wi.t()
    # products of two projections (|values| up to ~10): the bound is relative to that scale
    torch.testing.assert_close(mid.float(), torch.nn.functional.gelu(fi[:, :I]) * fi[:, I:], rtol=4e-3, atol=8e-3)


def test_gemm_layernorm_fold_pivot(srlib, cuda):
    """Rows whose common offset dwarfs their spread (mean 300, std 1): fp16(x) alone would lose x - mean; the fold takes
    its fp16 copy and statistics of x - pivot, the pivot being the row mean after the previous residual GEMM."""
    lib = srlib.lib()
    M, H = 700, 768
    g = torch.Generator(device="cuda").manual_seed(77)
    a = torch.randn(M, H, device=cuda, generator=g).half()
    w = (torch.randn(H, H, device=cuda, generator=g) * 0.02).half()
    x0 = torch.randn(M, H, device=cuda, generator=g) + 300.0 + 20.0 * torch.randn(M, 1, device=cuda, generator=g)
    x = x0.clone()
    parts = H // 128
    recs = [torch.full((parts * M * 2 + M,), float("nan"), device=cuda) for _ in range(2)]
    raw = torch.zeros(M, H, device=cuda, dtype=torch.float16)
    def producer(k):
        dst, prev = recs[k & 1], recs[(k - 1) & 1]
        piv_out = dst[parts * M * 2:]
        rc = lib.sr_test_gemm_fold(_ptr(a), _ptr(w), _ptr(x), M, H, H, EPI_RESID, H, None, _ptr(x), None, None, None, 0,
                                   _ptr(dst), _ptr(raw), None, 0.0, 0, piv_out.data_ptr(),
                                   prev[parts * M * 2:].data_ptr() if k else None, _ptr(prev) if k else None)
        torch.cuda.synchronize()
        assert rc == 0
    ref_x = x0.clone()
    for k in range(2):     # the second GEMM has a pivot (the first one's row means)
        producer(k)
        ref_x = a.float() @ w.float().t() + ref_x
    torch.testing.assert_close(x, ref_x, rtol=1e-5, atol=1e-3)
    piv = recs[1][parts * M * 2:]
    assert (piv - (ref_x - a.float() @ w.float().t()).mean(1)).abs().max() < 1e-2      # = mean after the first GEMM
    # consumer on the pivoted copy: LN(x) Wq^T with zero-sum-row weights
    gamma = 1 + 0.2 * torch.randn(H, device=cuda, generator=g)
    wq = torch.randn(256, H, device=cuda, generator=g) * 0.05
    wq_f = wq * gamma[None, :]
    wq_f = (wq_f - wq_f.mean(1, keepdim=True)).half()
    out = torch.zeros(M, 256, device=cuda, dtype=torch.float16)
    pos = torch.zeros(M, device=cuda, dtype=torch.int32)
    cos = torch.ones(4, 32, device=cuda); sin = torch.zeros(4, 32, device=cuda)
    rc = lib.sr_test_gemm_fold(_ptr(raw), _ptr(wq_f), _ptr(out), M, 256, H, EPI_ROPE, 256, None, None, _ptr(pos), _ptr(cos), _ptr(sin),
                               0, None, None, _ptr(recs[1]), 1e-5, H, None, None, None)
    torch.cuda.synchronize()
    assert rc == 0
    ref = torch.nn.functional.layer_norm(ref_x, (H,), gamma, None, 1e-5) @ wq.t()
    torch.testing.assert_close(out.float(), ref, rtol=3e-3, atol=3e-3)


@pytest.mark.parametrize("M,K", [(300, 768), (700, 1152), (2500, 768), (4224, 1152)])   # M >= 2048: many row blocks per worker
def test_gemm_resid_fp16_pair(srlib, cuda, M, K):
    """EPI_RESID_HL: the residual stream as an fp16 pair, in place -- x - pivot = hi + lo.  Three chained GEMMs on rows with a
    large common offset: after each one hi + lo + pivot_out must equal the fp32 reference to ~2^-22 of the row spread, hi must
    be fp16(x - pivot) (the A operand of the next projection), the statistics those of x - pivot, and the pivot the row mean
    after the previous GEMM."""
    lib = srlib.hooks()
    H = 768
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = (torch.randn(H, K, device=cuda, generator=g) * 0.02).half()
    bias = torch.randn(H, device=cuda, generator=g) * 0.1
    x0 = torch.randn(M, H, device=cuda, generator=g) + 30.0 + 5.0 * torch.randn(M, 1, device=cuda, generator=g)
    hi = x0.half()
    lo = (x0 - hi.float()).half()
    parts = H // 128
    recs = [torch.full((parts * M * 2 + M,), float("nan"), device=cuda) for _ in range(2)]
    ref = hi.float() + lo.float()                  # what the pair holds (x0 to 2^-22)
    prev_pair = ref.clone()
    for k in range(3):
        dst, prev = recs[k & 1], recs[(k - 1) & 1]
        rc = lib.sr_test_gemm_resid_hl(_ptr(a), _ptr(w), _ptr(hi), _ptr(lo), M, H, K, _ptr(bias) if k == 1 else None, _ptr(dst),
                                       dst[parts * M * 2:].data_ptr(), prev[parts * M * 2:].data_ptr() if k else None,
                                       _ptr(prev) if k else None)
        torch.cuda.synchronize()
        assert rc == 0
        ref = ref + a.float() @ w.float().t() + (bias if k == 1 else 0.0)
        piv = dst[parts * M * 2:]
        st = dst[:parts * M * 2].view(parts, M, 2)
        pair = hi.float() + lo.float()
        x = torch.empty(M, H, device=cuda)
        assert lib.sr_test_hl_to_f32(_ptr(hi), _ptr(lo), piv.data_ptr(), M, H, _ptr(x)) == 0
        torch.cuda.synchronize()
        torch.testing.assert_close(x, ref, rtol=0, atol=2e-4)                      # accumulation order + 2^-22 of the spread
        torch.testing.assert_close(x, pair + piv[:, None], rtol=0, atol=1e-5)
        # the pivot: 0 for the first GEMM, then the row mean of the previous state
        want_piv = torch.zeros(M, device=cuda) if k == 0 else prev_x.mean(1)
        assert (piv - want_piv).abs().max() < 1e-3
        # hi = fp16(x - pivot), lo the rounding rest: at most half an ulp of hi (2^-11 relative; an exact tie may round either way)
        assert (lo.float().abs() <= hi.float().abs() * 2.0 ** -11 * 1.001 + 1e-7).all()
        assert (hi != pair.half()).float().mean() < 1e-3
        torch.testing.assert_close(st[..., 0].sum(0), pair.sum(1), rtol=1e-4, atol=2e-2)
        torch.testing.assert_close(st[..., 1].sum(0), (pair * pair).sum(1), rtol=1e-4, atol=1e-1)
        torch.testing.assert_close(st[2, :, 0], pair[:, 256:384].sum(1), rtol=1e-4, atol=1e-2)
        prev_x = x.clone()
