"""The LayerNorm-fold projections (EPI_ROPE, EPI_GEGLU) run on 128 x 192 tiles with two MMA warpgroups and epilogues
from registers (gemm_wide_kernel).  Per element the accumulation over K and the epilogue expressions are those of the
128 x 128 kernel, so the outputs must be bitwise equal: the 128 x 128 kernel runs in a child process with
SRB_GEMM_WIDE=0 (the switch is read once per process), the wide kernel here, on the same seeded inputs.  Shapes cover
partial last tiles (N % 192 != 0), odd row counts, clustered and unclustered launches, grouped weights, and NaN rows
behind M in A that must not leak into the output (rows past M are never written)."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPI_ROPE, EPI_GEGLU = 1, 3
K = 768
MS = [1, 40, 65, 127, 2333, 16897, 20000]
NS_ROPE = [192, 320, 640, 1152, 2304]
NS_GEGLU = [640, 1152, 2304]   # EPI_GEGLU needs N % 128 == 0


def _cases():
    cases = []
    for epi, ns in ((EPI_ROPE, NS_ROPE), (EPI_GEGLU, NS_GEGLU)):
        for n in ns:
            for m in MS:
                for fold in (False, True):
                    cases.append(dict(epi=epi, m=m, n=n, fold=fold, groups=0, grp_rows=0))
        for n in (1152, 2304):   # unclustered and 1 x 2 clusters (the shared-LoRA serving shape)
            for grp_rows in (128, 256):
                for fold in (False, True):
                    cases.append(dict(epi=epi, m=3 * grp_rows, n=n, fold=fold, groups=3, grp_rows=grp_rows))
    return cases


def _run_all():
    """Every case on the kernel this process selects; returns the full output buffers (rows past M included)."""
    sys.path.insert(0, ROOT)
    import semantic_router_b200 as pkg
    dev = "cuda"
    outs = []
    for i, c in enumerate(_cases()):
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        m, n, epi = c["m"], c["n"], c["epi"]
        pad = 64
        a = torch.randn(m + pad, K, device=dev, generator=g).half()
        a[m:] = float("nan")   # stale rows behind M
        ws = max(c["groups"], 1)
        w = (torch.randn(ws * n, K, device=dev, generator=g) * 0.05).half()
        n_out = n // 2 if epi == EPI_GEGLU else n
        out = torch.full((m + pad, n_out), -7.0, device=dev, dtype=torch.float16)
        f = {}
        if c["fold"]:
            f = dict(fold_stats=torch.rand(K // 128, m, 2, device=dev, generator=g) + 0.5, fold_eps=1e-5, fold_h=K)
        if epi == EPI_ROPE:
            f.update(pos=torch.randint(0, 1024, (m,), device=dev, dtype=torch.int32, generator=g),
                     rope_cos=torch.rand(1024, 32, device=dev, generator=g) * 2 - 1,
                     rope_sin=torch.rand(1024, 32, device=dev, generator=g) * 2 - 1,
                     rope_cols=(2 * n // 3) // 64 * 64)
        if c["groups"]:
            f.update(w_groups=c["groups"], w_group_rows=c["grp_rows"])
        rc, _ = pkg.binding.run_gemm(m=m, n=n, k=K, a=a, a_rows=m + pad, w=w, out=out, ldo=n_out, epi=epi, **f)
        assert rc == 0, c
        torch.cuda.synchronize()
        outs.append(out.cpu())
    return outs


def test_wide_kernel_bitwise_equals_128x128(cuda, tmp_path):
    if os.environ.get("SRB_GEMM_WIDE", "1")[:1] == "0":
        pytest.skip("SRB_GEMM_WIDE=0: this process runs the 128 x 128 kernel too")
    ref_path = tmp_path / "narrow.pt"
    env = dict(os.environ, SRB_GEMM_WIDE="0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(ref_path)], env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    ref = torch.load(ref_path)
    got = _run_all()
    cases = _cases()
    assert len(ref) == len(got) == len(cases)
    bad = []
    for c, x, y in zip(cases, got, ref):
        m = c["m"]
        assert (x[m:] == -7.0).all(), ("rows past M written", c)
        if not torch.equal(x.view(torch.int16), y.view(torch.int16)):
            d = (x.float() - y.float()).abs()
            bad.append((c, int((x.view(torch.int16) != y.view(torch.int16)).sum()), float(d[d == d].max())))
    assert not bad, bad[:5]


def test_wide_cluster_workers(srlib, cuda):
    """The pair count of the kernel each clustered shape launches fits the device."""
    lib = srlib.hooks()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    f = lib.sr_test_gemm_cluster
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    for epi in (EPI_ROPE, EPI_GEGLU):
        for n in (512, 1152, 1280, 1536, 2304, 3072):
            cn, workers = C.c_int(0), C.c_int(0)
            assert f(epi, n, K, C.byref(cn), C.byref(workers)) == 0
            assert 0 < workers.value * cn.value <= sms, (epi, n)


if __name__ == "__main__":
    torch.save(_run_all(), sys.argv[1])
