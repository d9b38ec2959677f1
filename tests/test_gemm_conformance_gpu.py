"""Conformance of the wgmma GEMM (csrc/gemm_wgmma.cu) over everything the engine asks of it, through the full
descriptor (sr_test_gemm_desc).

* Float64 parity: every epilogue at the shape edges (M around the 64-row cluster slices and the 128-row blocks, N with a
  half-empty last column tile, K with a partial last k-block), the LayerNorm fold, grouped weights and the cache scan,
  each element within the bound of oracle/gemm_oracle.py.  Every A has stale NaN / inf rows past M, as behind the engine's a_rows = cap_tokens, and every output has sentinel rows past M
  and sentinel columns [n_out, ldo) that must survive.
* Bitwise invariants: clusters against the unclustered halves, grouped weights against per-group GEMMs, stale rows against a_rows = M, and the launch schedules chosen by environment
  variables (child processes) against the default.
* Refusals: shapes gemm_f16 rejects return non-zero and leave the output alone.

Run with -s to see the largest |err| / S per epilogue (what TAU in oracle/gemm_oracle.py is set from)."""
import ctypes as C
import math
import os
import subprocess
import sys
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle import gemm_oracle as go
from oracle.gemm_oracle import EPI_F16, EPI_GEGLU, EPI_GELU, EPI_RESID, EPI_RESID_HL, EPI_ROPE

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S16 = 0x7E5A          # sentinel bits: fp16 NaN with a payload
S32 = 0x7FC0DEAD      # fp32 NaN with a payload
DEV = "cuda"


@pytest.fixture(scope="module")
def lib(srlib, cuda):
    return srlib.hooks()


_TAU_SEEN = {}


@pytest.fixture(scope="module", autouse=True)
def _tau_report():
    yield
    if _TAU_SEEN:
        print("\nlargest |err| / S beyond the epilogue's own error, per epilogue (oracle TAU = 2^%.1f):"
              % math.log2(go.TAU))
        for k in sorted(_TAU_SEEN):
            v = _TAU_SEEN[k]
            print(f"  {k:10s} {v:.3e}" + (f"  (2^{math.log2(v):.2f})" if v > 0 else ""))


def run(sync=True, **kw):
    import semantic_router_b200 as pkg
    rc, lists = pkg.binding.run_gemm(**kw)
    if sync:
        torch.cuda.synchronize()
    return rc, lists


def _cluster(lib, epi, n, k):
    cn, workers = C.c_int(0), C.c_int(0)
    assert lib.sr_test_gemm_cluster(epi, n, k, C.byref(cn), C.byref(workers)) == 0
    return cn.value


def test_wide_cluster_workers(lib):
    """The pair count of the kernel each clustered shape launches fits the device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    f = lib.sr_test_gemm_cluster
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    for epi in (EPI_ROPE, EPI_GEGLU):
        for n in (512, 1152, 1280, 1536, 2304, 3072):
            cn, workers = C.c_int(0), C.c_int(0)
            assert f(epi, n, 768, C.byref(cn), C.byref(workers)) == 0
            assert 0 < workers.value * cn.value <= sms, (epi, n)


def _up(x, a):
    return (x + a - 1) // a * a


def _stale(t, m):
    """rows [m, end) of t: fp16 NaN, +inf, -inf in turn"""
    n = t[m:].numel()
    if n:
        pat = torch.tensor([float("nan"), float("inf"), float("-inf")], device=t.device).half()
        t[m:] = pat.repeat(n // 3 + 1)[:n].view_as(t[m:])


def _fold_stats(m, h, g):
    """[h/128][m][2] slice partials of rows with mean ~0.05 and variances log-uniform in [1e-5, 4]: some rows have a
    variance comparable to the LayerNorm epsilon, where rstd depends on it."""
    dev = torch.device(DEV)
    parts = h // 128
    mu = 0.05 * torch.randn(m, generator=g, device=dev, dtype=torch.float64)
    var = torch.exp(math.log(1e-5) + torch.rand(m, generator=g, device=dev, dtype=torch.float64) * math.log(4e5))
    wt = torch.rand(parts, m, generator=g, device=dev, dtype=torch.float64) + 0.5
    wt = wt / wt.sum(0)
    return torch.stack([h * mu * wt, h * (var + mu * mu) * wt], -1).float().contiguous()


def _rope_tables():
    from oracle import encoder_oracle as eo
    cos, sin = eo.rope_tables(64, 160000.0, 1024)
    return cos.to(DEV).contiguous(), sin.to(DEV).contiguous()


@dataclass
class Problem:
    epi: int
    M: int
    n_out: int
    desc: dict
    oracle: dict = field(default_factory=dict)
    lo: torch.Tensor = None

    @property
    def out(self):
        return self.desc["out"]

    def result(self):
        if self.epi == EPI_RESID_HL:
            return self.out[:self.M].double() + self.lo[:self.M].double()
        return self.out[:self.M, :self.n_out].double()

    def reference(self):
        d = self.desc
        return go.gemm(self.epi, d["a"][:self.M], d["w"], d["n"], **self.oracle)

    def check_sentinels(self):
        bufs = [self.out] + ([self.lo] if self.lo is not None else [])
        for b in bufs:
            bits = b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int16)
            s = S32 if b.dtype == torch.float32 else S16
            assert (bits[self.M:] == s).all(), "rows past M were written"
            assert (bits[:, self.n_out:] == s).all(), "columns [n_out, ldo) were written"


def problem(epi, M, N, K, seed, *, bias=False, resid=True, fold=False, rope_cols=0, w_groups=0, w_group_rows=0,
            stale=True, w_scale=0.05, bias_per_group=False):
    dev = torch.device(DEV)
    g = torch.Generator(device=dev).manual_seed(seed)
    a_rows = _up(M, 128) + 64 if stale else M
    A = torch.randn(a_rows, K, generator=g, device=dev).half()
    W = (torch.randn(N * max(w_groups, 1), K, generator=g, device=dev) * w_scale).half()
    d = dict(m=M, n=N, k=K, a=A, a_rows=a_rows, w=W, epi=epi)
    o = {}
    _stale(A, M)
    if bias:                                   # bias_per_group: one vector per stacked matrix
        b = torch.randn(N * (w_groups if bias_per_group else 1), generator=g, device=dev)
        d["bias"] = o["bias"] = b
        if bias_per_group:
            d["bias_per_group"], o["bias_per_group"] = 1, True
    if epi == EPI_ROPE:
        cos, sin = _rope_tables()
        pos = torch.randint(0, 1024, (M,), generator=g, device=dev, dtype=torch.int32)
        d.update(pos=pos, rope_cos=cos, rope_sin=sin, rope_cols=rope_cols)
        o.update(pos=pos, rope_cos=cos, rope_sin=sin, rope_cols=rope_cols)
    if fold:
        st = _fold_stats(M, 768, g)
        d.update(fold_stats=st, fold_eps=1e-5, fold_h=768)
        o.update(fold_stats=st, fold_eps=1e-5, fold_h=768)
    if w_groups:
        d.update(w_groups=w_groups, w_group_rows=w_group_rows)
        o.update(w_groups=w_groups, w_group_rows=w_group_rows)
    n_out = N // 2 if epi == EPI_GEGLU else N
    p = Problem(epi, M, n_out, d, o)
    if epi == EPI_RESID_HL:
        x0 = torch.randn(M + 3, N, generator=g, device=dev) + 3.0
        hi = x0.half()
        lo = (x0 - hi.float()).half()
        hi[M:].view(torch.int16).fill_(S16)
        lo[M:].view(torch.int16).fill_(S16)
        o["resid"] = hi[:M].double() + lo[:M].double()
        d.update(out=hi, ldo=N, lo16=lo, row_stats=torch.zeros(N // 128, M, 2, device=dev),
                 pivot_out=torch.zeros(M, device=dev))
        p.lo = lo
    elif epi == EPI_RESID:
        ldo = N + 8
        out = torch.empty(M + 3, ldo, device=dev)
        out.view(torch.int32).fill_(S32)
        d.update(out=out, ldo=ldo)
        if resid:
            r0 = torch.randn(M, N, generator=g, device=dev)
            out[:M, :N] = r0
            d.update(resid=out, ldr=ldo)
            o["resid"] = r0
    else:
        ldo = n_out + 64
        out = torch.empty(M + 3, ldo, device=dev, dtype=torch.float16)
        out.view(torch.int16).fill_(S16)
        d.update(out=out, ldo=ldo)
    return p


def check_parity(p, tag=None):
    rc, _ = run(**p.desc)
    assert rc == 0
    p.check_sentinels()
    got = p.result()
    assert torch.isfinite(got).all(), "non-finite output (stale rows leaked in?)"
    ref = p.reference()
    name = tag or go.EPI_NAMES[p.epi]
    _TAU_SEEN[name] = max(_TAU_SEEN.get(name, 0.0), ref.tau_needed(got))
    err = (got - ref.value).abs()
    bound = ref.bound()
    bad = err > bound
    if bad.any():
        r, c = [int(x) for x in torch.nonzero(bad)[0]]
        raise AssertionError(f"{int(bad.sum())} elements outside the bound; first at ({r}, {c}): got {float(got[r, c])!r}, "
                             f"float64 {float(ref.value[r, c])!r}, |err| {float(err[r, c]):.3e} > bound "
                             f"{float(bound[r, c]):.3e} (S-term {float(ref.coef[r, c]):.3e}, epilogue {float(ref.eps[r, c]):.3e})")


# ---------------------------------------------------------------------------------------------------------------------
# float64 parity
# ---------------------------------------------------------------------------------------------------------------------
MS = [1, 40, 64, 65, 127, 129, 2333, 16897]   # 16897 = 132 * 128 + 1: several tiles per worker and one row past a block
NS = [64, 192, 320, 2304]                      # 192: two column tiles (a 2-CTA cluster for RoPE), the second half empty
NS_128 = [128, 640, 2304]                      # GeGLU and the fp16 pair need N % 128 == 0
KS = [8, 72, 200, 768, 1160]                   # all but 768 end in a partial k-block
ROPE_COLS = {64: 64, 192: 128, 320: 192, 1152: 768, 2304: 1536}
EPIS = [EPI_F16, EPI_ROPE, EPI_RESID, EPI_GEGLU, EPI_GELU, EPI_RESID_HL]


def _shape_cases():
    out = []
    for e, epi in enumerate(EPIS):
        ns = NS_128 if epi in (EPI_GEGLU, EPI_RESID_HL) else NS
        for i, m in enumerate(MS):
            out.append((epi, m, ns[(i + e) % len(ns)], KS[(i + e) % len(KS)], i))
    return out


@pytest.mark.parametrize("epi,M,N,K,i", _shape_cases(),
                         ids=[f"{go.EPI_NAMES[c[0]]}-{c[1]}x{c[2]}x{c[3]}" for c in _shape_cases()])
def test_shape_edges(lib, epi, M, N, K, i):
    p = problem(epi, M, N, K, seed=1000 * epi + i, bias=epi in (EPI_F16, EPI_RESID, EPI_GELU, EPI_RESID_HL),
                resid=(i % 2 == 0), rope_cols=ROPE_COLS.get(N, 0))
    check_parity(p)


@pytest.mark.parametrize("epi,N,M", [(EPI_ROPE, 2304, 2333), (EPI_ROPE, 320, 127), (EPI_GEGLU, 2304, 65),
                                     (EPI_GEGLU, 640, 2333), (EPI_ROPE, 1152, 20000), (EPI_GEGLU, 2304, 20000)])
def test_layernorm_fold(lib, epi, N, M):
    """The fold scales the whole accumulator by the row's rstd, which depends on the LayerNorm epsilon for rows of small
    variance.  M = 20000 gives every worker several row blocks, unclustered (N = 1152) and in pairs (N = 2304)."""
    p = problem(epi, M, N, 768, seed=31 * M, fold=True, rope_cols=ROPE_COLS.get(N, 0), w_scale=0.01)
    check_parity(p, tag=go.EPI_NAMES[epi] + "+fold")


# (epi, N, K, fold, a bias per group).  GeGLU N = 640 / 2176 / 5248 (I = 320 / 1088 / 2624): the wide kernel's last
# 192-column tile of a group reaches into the next group's matrix, which must be clipped.  The per-group biases are
# BERT's grouped epilogues: Wqkv (EPI_F16), Wi (EPI_GELU), Wo and Wo2 (EPI_RESID in place).
GROUPED = [(EPI_F16, 384, 200, False, False), (EPI_ROPE, 2304, 768, False, False), (EPI_ROPE, 2304, 768, True, False),
           (EPI_ROPE, 1152, 768, False, False), (EPI_ROPE, 1152, 768, True, False), (EPI_GEGLU, 2304, 768, False, False),
           (EPI_GEGLU, 2304, 768, True, False), (EPI_RESID_HL, 768, 768, False, False),
           (EPI_GEGLU, 640, 384, False, False), (EPI_GEGLU, 640, 384, True, False),
           (EPI_GEGLU, 2176, 768, False, False), (EPI_GEGLU, 2176, 768, True, False),
           (EPI_GEGLU, 5248, 1024, False, False), (EPI_GEGLU, 5248, 1024, True, False),
           (EPI_F16, 2304, 768, False, True), (EPI_GELU, 3072, 768, False, True), (EPI_GELU, 1536, 384, False, True),
           (EPI_RESID, 768, 3072, False, True), (EPI_RESID, 1024, 4096, False, True)]


@pytest.mark.parametrize("rows", [128, 256])
@pytest.mark.parametrize("epi,N,K,fold,gbias", GROUPED,
                         ids=[f"{e}-{n}-{k}" + ("-fold" if f else "") + ("-gbias" if b else "") for e, n, k, f, b in GROUPED])
def test_grouped_weights(lib, epi, N, K, fold, gbias, rows):
    """w_groups = 3 stacked matrices; the last group is partly empty.  Row blocks of 128 never straddle two groups
    when w_group_rows is a multiple of 128, which is what gemm_f16 accepts.  The LayerNorm-fold projections run in
    pairs at N = 2304 and unclustered at N = 1152 (the shared-LoRA serving shapes).  gbias: each group adds its own
    bias (EPI_RESID in place over a residual)."""
    p = problem(epi, 3 * rows - 5, N, K, seed=rows + epi, w_groups=3, w_group_rows=rows, rope_cols=ROPE_COLS.get(N, 0),
                bias=epi == EPI_F16 or gbias, bias_per_group=gbias, fold=fold, w_scale=0.01 if fold else 0.05)
    check_parity(p, tag=go.EPI_NAMES[epi] + ("+grp+fold" if fold else "+grp") + ("+gbias" if gbias else ""))


# ---- the cache scan: GEMV (B <= 4), fused top-8 epilogue (one row block, and the grouped schedule), two-pass (k > 8)
def _cache_rows(n, D, rng):
    rows = rng.standard_normal((n, D)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    # a tie group scored exactly (small dyadic entries): rows 4..15 = v, and 2 v in the next 32-column chunk of the
    # same tile.  The top-8 epilogue meets the ties first and must keep the lowest indices.
    v = np.zeros(D, np.float32)
    v[rng.choice(D, 8, replace=False)] = rng.choice([-0.5, -0.25, 0.25, 0.5], 8)
    rows[4:16] = v
    rows[40] = 2 * v
    return rows, v


@pytest.mark.parametrize("D", [72, 200, 520])
def test_cache_scan(srlib, cuda, D):
    n = 9001                                            # not a multiple of 256; > 66 column tiles: grouped schedule
    rng = np.random.default_rng(D)
    rows, v = _cache_rows(n, D, rng)
    valid = np.ones(n, bool)
    valid[rng.choice(n, 300, replace=False)] = False
    valid[5] = False                                    # one of the tie group
    cache = srlib.Cache(n, D, device=0)
    try:
        cache.add(rows)
        for r in np.nonzero(~valid)[0]:
            cache.invalidate(int(r))
        r64 = torch.from_numpy(rows.astype(np.float16).astype(np.float64)).cuda()
        vmask = torch.from_numpy(valid).cuda()
        for B in (1, 3, 7, 130, 300):
            q = rng.standard_normal((B, D)).astype(np.float32)
            q /= np.linalg.norm(q, axis=1, keepdims=True)
            q[0] = v                                    # exact scores for the tie group
            q64 = torch.from_numpy(q.astype(np.float16).astype(np.float64)).cuda()
            sc64 = q64 @ r64.t()
            S = q64.abs() @ r64.abs().t()
            # the GEMV accumulates each lane's ceil(D / 256) 8-wide chunks with fmaf, then a 5-level shuffle tree
            tau = max(go.TAU, (8 * math.ceil(D / 256) + 6) * go.U32) if B <= 4 else go.TAU
            bound = tau * S
            for k in (1, 8, 16):
                idx, sc = cache.topk(q, k)
                ref_idx, ref_val = go.topk(sc64, k + 1, vmask)
                idx_t = torch.from_numpy(idx.astype(np.int64)).cuda()
                assert (idx_t >= 0).all() and (idx_t < n).all() and vmask[idx_t].all(), (B, k)
                assert (np.diff(sc, axis=1) <= 0).all(), (B, k)
                sc_t = torch.from_numpy(sc.astype(np.float64)).cuda()
                assert ((sc_t - sc64.gather(1, idx_t)).abs() <= bound.gather(1, idx_t)).all(), (B, k)
                bmax = torch.where(vmask[None, :], bound, torch.zeros_like(bound)).max(1).values[:, None]
                gaps = ref_val[:, :-1] - ref_val[:, 1:]               # gap below rank r
                above = torch.cat([torch.full_like(gaps[:, :1], torch.inf), gaps[:, :k - 1]], 1)
                sure = (above > 2 * bmax) & (gaps[:, :k] > 2 * bmax)
                wrong = sure & (idx_t != ref_idx[:, :k])
                assert not wrong.any(), (B, k, torch.nonzero(wrong)[:4].tolist())
                # the tie group is scored exactly: the whole list of query 0 is determined, lower index first
                assert idx[0].tolist() == ref_idx[0, :k].tolist(), (B, k, idx[0].tolist())
    finally:
        cache.close()


# ---------------------------------------------------------------------------------------------------------------------
# bitwise invariants
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


@pytest.mark.parametrize("fold", [False, True])
@pytest.mark.parametrize("epi", [EPI_ROPE, EPI_GEGLU], ids=["rope", "geglu"])
def test_cluster_pair_equals_unclustered_halves(lib, epi, fold):
    """N = 2304 (18 column tiles) runs as 2-CTA clusters sharing A by multicast; as two N = 1152 halves (9 tiles each)
    it runs without clusters.  The tiles, their wgmma sequences and epilogues are the same: bitwise equal outputs."""
    assert _cluster(lib, epi, 2304, 768) == 2 and _cluster(lib, epi, 1152, 768) == 1
    for M in (1, 40, 65, 127, 2333, 20000):
        p = problem(epi, M, 2304, 768, seed=M + fold, fold=fold, rope_cols=1536, w_scale=0.01 if fold else 0.05)
        d = p.desc
        assert run(**d)[0] == 0
        full = p.out[:M].clone()
        p.out.view(torch.int16).fill_(S16)
        half_out = p.n_out // 2
        for h in range(2):
            dh = dict(d, n=1152, w=d["w"][1152 * h:1152 * (h + 1)], out=p.out[:, half_out * h:])
            if epi == EPI_ROPE:
                dh["rope_cols"] = 1152 if h == 0 else 1536 - 1152
            assert run(**dh)[0] == 0
        assert torch.equal(_bits(full), _bits(p.out[:M])), M


@pytest.mark.parametrize("rows", [128, 256])
@pytest.mark.parametrize("epi,gbias", [(EPI_RESID, False), (EPI_F16, False), (EPI_RESID, True), (EPI_F16, True),
                                       (EPI_GELU, True)],
                         ids=["resid", "f16", "resid-gbias", "f16-gbias", "gelu-gbias"])
def test_grouped_weights_are_per_group_gemms(lib, epi, gbias, rows):
    """gbias: each group's GEMM gets its own bias (EPI_RESID over a residual, in place)"""
    M, N, K = 3 * rows, 384, 200
    p = problem(epi, M, N, K, seed=rows, w_groups=3, w_group_rows=rows, resid=gbias, bias=gbias, bias_per_group=gbias)
    d = p.desc
    out0 = p.out.clone()
    assert run(**d)[0] == 0
    grouped = p.out[:M].clone()
    p.out.copy_(out0)
    for g in range(3):
        dg = {k: v for k, v in d.items() if k not in ("w_groups", "w_group_rows", "bias_per_group")}
        dg.update(m=rows, a=d["a"][g * rows:], a_rows=rows, w=d["w"][g * N:(g + 1) * N], out=p.out[g * rows:])
        if gbias:
            dg["bias"] = d["bias"][g * N:(g + 1) * N]
        if "resid" in d:
            dg["resid"] = dg["out"]
        assert run(**dg)[0] == 0
    assert torch.equal(_bits(grouped), _bits(p.out[:M]))


@pytest.mark.parametrize("M", [40, 65])
@pytest.mark.parametrize("epi,N", [(EPI_F16, 320), (EPI_ROPE, 2304), (EPI_RESID, 192), (EPI_GEGLU, 2304),
                                   (EPI_GELU, 192), (EPI_RESID_HL, 640)], ids=lambda x: str(x))
def test_stale_rows(lib, epi, N, M):
    """Rows [M, a_rows) of A hold NaN / inf (the engine's A covers cap_tokens rows).  With a 2-CTA cluster at M = 40
    the second CTA's multicast slice (rows 64..127) lies wholly past M.  Rows < M must equal a run over exactly M rows,
    and nothing past M or past n_out may be written (checked by the sentinels)."""
    p = problem(epi, M, N, 200, seed=M + epi, rope_cols=ROPE_COLS.get(N, 0),
                bias=epi in (EPI_F16, EPI_GELU, EPI_RESID_HL))
    d = p.desc
    out0 = p.out.clone()
    lo0 = p.lo.clone() if p.lo is not None else None
    assert run(**d)[0] == 0
    p.check_sentinels()
    stale = [p.out[:M].clone()] + ([p.lo[:M].clone()] if p.lo is not None else [])
    p.out.copy_(out0)
    if lo0 is not None:
        p.lo.copy_(lo0)
    exact = dict(d, a=d["a"][:M].clone(), a_rows=M)
    assert run(**exact)[0] == 0
    again = [p.out[:M]] + ([p.lo[:M]] if p.lo is not None else [])
    for x, y in zip(stale, again):
        assert torch.equal(_bits(x), _bits(y))


# ---- launch schedules chosen by environment variables (read once per process): a child process per setting
_CHILD = r'''
import os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "tests")]
import numpy as np
import torch
import semantic_router_b200 as pkg
import test_gemm_conformance_gpu as t
res = {}
# fp32 residual GEMMs in place: interleaved by default for K > 768, for every K with SRB_RESID_INTERLEAVE=2;
# N = 704 ends in a half-empty column tile, where the residual prefetch cursor must stop at n_out
for name, (M, N, K) in {"resid_704_1152": (2333, 704, 1152), "resid_768_768": (2333, 768, 768),
                        "resid_704_768": (16897, 704, 768)}.items():
    p = t.problem(t.EPI_RESID, M, N, K, seed=N + K, bias=True)
    assert t.run(**p.desc)[0] == 0
    res[name] = p.out.cpu().numpy()
# three chained fp16-pair residual GEMMs with pivots, queued back to back as the encoder issues them (the PDL chain)
M, N = 2333, 768
p = t.problem(t.EPI_RESID_HL, M, N, 768, seed=5, bias=True)
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
# the cache scan's fused top-8 epilogue: grouped schedule by default, contiguous ranges with SRB_TOPK_GROUPED=0
rng = np.random.default_rng(1)
rows, v = t._cache_rows(9001, 200, rng)
cache = pkg.Cache(9001, 200, device=0)
cache.add(rows)
for B in (130, 300):
    q = rng.standard_normal((B, 200)).astype(np.float32)
    q[0] = v
    res[f"topk_idx_{B}"], res[f"topk_sc_{B}"] = cache.topk(q, 8)
cache.close()
np.savez(sys.argv[2], **res)
'''


def test_schedules_bitwise(cuda, tmp_path):
    """SRB_RESID_INTERLEAVE = 0 / 1 / 2, SRB_TOPK_GROUPED = 0 / 1 and SRB_PDL = 0 / 1 change which worker computes a tile
    and when, never how: outputs are bitwise those of the default process."""
    base_env = {k: v for k, v in os.environ.items() if not k.startswith(("SRB_RESID_INTERLEAVE", "SRB_TOPK_GROUPED",
                                                                           "SRB_PDL"))}
    settings = {"default": {}, "a": {"SRB_RESID_INTERLEAVE": "0", "SRB_TOPK_GROUPED": "0", "SRB_PDL": "1"},
                "b": {"SRB_RESID_INTERLEAVE": "2", "SRB_TOPK_GROUPED": "1", "SRB_PDL": "0"},
                "c": {"SRB_RESID_INTERLEAVE": "1", "SRB_PDL": "1"}}
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


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
REFUSED = {
    "n_mod_64": dict(epi=EPI_F16, N=100, K=64),
    "k_mod_8": dict(epi=EPI_F16, N=128, K=100),
    "geglu_n_mod_128": dict(epi=EPI_GEGLU, N=192, K=64),
    "group_rows_192": dict(epi=EPI_F16, N=128, K=64, groups=192),
    "group_rows_64": dict(epi=EPI_F16, N=128, K=64, groups=64),
    "stats_not_pair": dict(epi=EPI_RESID, N=128, K=64, row_stats=True),
    "pivot_not_pair": dict(epi=EPI_F16, N=128, K=64, pivot_out=True),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_refusals(lib, case):
    c = REFUSED[case]
    M, N, K = 256, c["N"], c["K"]
    dev = torch.device(DEV)
    a = torch.randn(M, K, device=dev).half()
    w = torch.randn(N * 3, K, device=dev).half()
    n_out = N // 2 if c["epi"] == EPI_GEGLU else N
    ldo = (n_out + 7) // 8 * 8
    out = torch.empty(M, ldo, device=dev, dtype=torch.float16)
    out.view(torch.int16).fill_(S16)
    d = dict(m=M, n=N, k=K, a=a, w=w, out=out, ldo=ldo, epi=c["epi"])
    if "groups" in c:
        d.update(w_groups=3, w_group_rows=c["groups"])
    if "row_stats" in c:
        d.update(row_stats=torch.zeros(N // 128, M, 2, device=dev))
    if "pivot_out" in c:
        d.update(pivot_out=torch.zeros(M, device=dev))
    rc, _ = run(**d)
    assert rc != 0
    assert (out.view(torch.int16) == S16).all()
