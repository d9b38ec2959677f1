"""Thread-block clusters of the GEMM (gemm_wgmma.cu): the cluster size the library picks per GEMM, and the fp16-pair
residual GEMM at shapes whose column tiles do not pair up (N / 128 odd), with enough rows that every worker of the
persistent grid walks several tiles."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_ROPE, EPI_GEGLU, EPI_TOPK, EPI_RESID_HL = 1, 3, 5, 6


def _cluster(lib, epi, n, k):
    f = lib.sr_test_gemm_cluster
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    cn, workers = C.c_int(0), C.c_int(0)
    assert f(epi, n, k, C.byref(cn), C.byref(workers)) == 0
    return cn.value, workers.value


def test_cluster_choice(srlib, cuda):
    lib = srlib.hooks()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # ModernBERT-base: Wqkv and Wi share A in pairs; the residual GEMMs and the cache scan run without clusters
    assert _cluster(lib, EPI_ROPE, 2304, 768)[0] == 2
    assert _cluster(lib, EPI_GEGLU, 2304, 768)[0] == 2
    assert _cluster(lib, EPI_RESID_HL, 768, 1152) == (1, sms)
    assert _cluster(lib, EPI_RESID_HL, 768, 768) == (1, sms)
    assert _cluster(lib, EPI_TOPK, 1024, 768) == (1, sms)
    for epi, n, k in [(EPI_ROPE, 1152, 384), (EPI_ROPE, 1920, 640), (EPI_GEGLU, 1536, 384), (EPI_RESID_HL, 384, 1152),
                      (EPI_RESID_HL, 640, 1152), (EPI_ROPE, 3072, 1024)]:
        cn, workers = _cluster(lib, epi, n, k)
        assert ((n + 127) // 128) % cn == 0, (epi, n, k, cn)   # no cluster carries a tile wholly past N
        assert 0 < workers * cn <= sms


@pytest.mark.parametrize("M,N,K", [(20000, 384, 1152), (9000, 640, 1152), (20000, 1024, 1152)])
def test_gemm_resid_pair_odd_column_tiles(srlib, cuda, M, N, K):
    """Two chained EPI_RESID_HL GEMMs (the second with pivots in): hi + lo + pivot_out must equal the fp32 reference."""
    lib = srlib.hooks()
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = (torch.randn(N, K, device=cuda, generator=g) * 0.02).half()
    x0 = torch.randn(M, N, device=cuda, generator=g) + 3.0
    hi = x0.half()
    lo = (x0 - hi.float()).half()
    ref = hi.float() + lo.float()
    parts = N // 128
    recs = [torch.full((parts * M * 2 + M,), float("nan"), device=cuda) for _ in range(2)]
    for step in range(2):
        dst, prev = recs[step & 1], recs[(step - 1) & 1]
        rc = lib.sr_test_gemm_resid_hl(a.data_ptr(), w.data_ptr(), hi.data_ptr(), lo.data_ptr(), M, N, K, None, dst.data_ptr(),
                                       dst[parts * M * 2:].data_ptr(), prev[parts * M * 2:].data_ptr() if step else None,
                                       prev.data_ptr() if step else None)
        torch.cuda.synchronize()
        assert rc == 0
        ref = ref + a.float() @ w.float().t()
        x = torch.empty(M, N, device=cuda)
        assert lib.sr_test_hl_to_f32(hi.data_ptr(), lo.data_ptr(), dst[parts * M * 2:].data_ptr(), M, N, x.data_ptr()) == 0
        torch.cuda.synchronize()
        torch.testing.assert_close(x, ref, rtol=0, atol=2e-4)
        st = dst[:parts * M * 2].view(parts, M, 2)
        pair = hi.float() + lo.float()
        torch.testing.assert_close(st[..., 0].sum(0), pair.sum(1), rtol=1e-4, atol=2e-2)
