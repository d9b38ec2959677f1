"""The fp16-pair residual GEMM (EPI_RESID_HL) at the encoder's shapes over many tiles per worker.

The epilogue warps keep a ring of (hi, lo) box pairs that they load ahead, update in place and store from, and carry
the row pivots from one row block to the next.  At M = 20000 and N = 768 there are 157 x 6 tiles, about 7 per worker
on the H100, in the interleaved schedule and in contiguous ranges alike, where the other parity cases give each worker
one or two: a wrong barrier phase, a load into a box before its store has been read out, or stale pivot state corrupts
the pair or the row statistics here.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gemm_conformance_gpu as conf
from oracle.gemm_oracle import EPI_RESID_HL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, N = 20000, 768


@pytest.mark.parametrize("K", [768, 1152])
def test_pair_many_tiles(srlib, cuda, K):
    """float64 parity of hi + lo, and the row statistics of the 128-column slices against the float64 sums of the
    result (they are taken of the fp32 x before it is split, which hi + lo holds to 2^-22 relative)."""
    p = conf.problem(EPI_RESID_HL, M, N, K, seed=K, bias=True)
    conf.check_parity(p, tag="resid_hl-20000")
    x = p.result().view(M, N // 128, 128)
    st = p.desc["row_stats"].double()
    s1, s2 = x.sum(-1).t(), (x * x).sum(-1).t()
    scale = x.abs().sum(-1).t()
    assert ((st[..., 0] - s1).abs() <= 1e-5 * scale + 1e-6).all()
    assert ((st[..., 1] - s2).abs() <= 1e-5 * (x * x).sum(-1).t() + 1e-6).all()
    assert (p.desc["pivot_out"] == 0).all()   # no pivot in: the pivot stays 0


_CHILD = r'''
import os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "tests")]
import numpy as np
import torch
import test_gemm_conformance_gpu as t
res = {}
# three chained fp16-pair residual GEMMs with pivots, queued back to back as the encoder issues them (the PDL chain)
M, N = 20000, 768
p = t.problem(t.EPI_RESID_HL, M, N, 1152, seed=7, bias=True)
part = N // 128 * M * 2
recs = [torch.zeros(part + M, device="cuda") for _ in range(2)]
for step in range(3):
    dst, prev = recs[step & 1], recs[(step - 1) & 1]
    ds = dict(p.desc, row_stats=dst, pivot_out=dst[part:])
    if step:
        ds.update(pivot_in=prev[part:], pivot_in_stats=prev)
    assert t.run(sync=False, **ds)[0] == 0
torch.cuda.synchronize()
res["hl_hi"], res["hl_lo"] = p.out.cpu().numpy(), p.lo.cpu().numpy()
res["hl_stats"] = torch.cat(recs).cpu().numpy()
np.savez(sys.argv[2], **res)
'''


def test_pair_schedules_bitwise(cuda, tmp_path):
    """Interleaved tiles (the default) against contiguous ranges (SRB_RESID_INTERLEAVE=0), with and without PDL: the
    worker and order change, the pair and its statistics do not, bit for bit."""
    base_env = {k: v for k, v in os.environ.items() if not k.startswith(("SRB_RESID_INTERLEAVE", "SRB_PDL"))}
    settings = {"default": {}, "a": {"SRB_RESID_INTERLEAVE": "0", "SRB_PDL": "1"},
                "b": {"SRB_RESID_INTERLEAVE": "0", "SRB_PDL": "0"}, "c": {"SRB_RESID_INTERLEAVE": "1", "SRB_PDL": "0"}}
    outs = {}
    for name, extra in settings.items():
        path = tmp_path / f"{name}.npz"
        r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, str(path)], env=dict(base_env, **extra), cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, f"{name}: {r.stdout[-2000:]}\n{r.stderr[-4000:]}"
        outs[name] = np.load(path)
    base = outs.pop("default")
    for name, o in outs.items():
        for k in base.files:
            a, b = base[k], o[k]
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (name, settings[name], k)
