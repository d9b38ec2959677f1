"""The thread-block cluster rule of the LayerNorm-fold projections (gemm_cluster_size), host side only: a pair of CTAs
shares A only where N's column-tile count is even both in 128-wide and in 192-wide tiles.  The even count at 192 keeps
every cluster free of a tile wholly past N; the even count at 128 keeps the schedule the clustered kernel was measured
with.  Every other epilogue runs unclustered."""
import ctypes as C

import pytest

EPI_F16, EPI_ROPE, EPI_RESID, EPI_GEGLU, EPI_GELU, EPI_TOPK, EPI_RESID_HL = range(7)


@pytest.fixture(scope="module")
def cluster_size(srlib):
    f = srlib.hooks().sr_test_gemm_cluster
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def size(epi, n, k=768):
        cn = C.c_int(0)
        assert f(epi, n, k, C.byref(cn), None) == 0
        return cn.value
    return size


def test_pairs_only_where_both_widths_pair(cluster_size):
    for epi in (EPI_ROPE, EPI_GEGLU):
        for n in range(64, 6145, 64):
            even = ((n + 127) // 128) % 2 == 0 and ((n + 191) // 192) % 2 == 0
            assert cluster_size(epi, n) == (2 if even else 1), (epi, n)
    # ModernBERT-base Wqkv / Wi pair; a 1152-wide projection (9 tiles of 128) and 1280 (7 tiles of 192) do not
    assert cluster_size(EPI_ROPE, 2304) == cluster_size(EPI_GEGLU, 2304) == 2
    assert cluster_size(EPI_ROPE, 1152) == cluster_size(EPI_ROPE, 1280) == 1


def test_other_epilogues_unclustered(cluster_size):
    for epi in (EPI_F16, EPI_RESID, EPI_GELU, EPI_TOPK, EPI_RESID_HL):
        for n in (256, 768, 1152, 2304, 3072):
            assert cluster_size(epi, n) == 1, (epi, n)
