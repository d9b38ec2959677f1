"""Float64 reference of the wgmma GEMM (csrc/gemm.h) with an explicit per-element error bound.

The fp16 operands are exact in float64, so `value` is the epilogue of gemm.h applied to the exact product.  A kernel
result x is correct when |x - value| <= TAU * coef + eps, where
  * coef carries the accumulation error: TAU * S with S = sum_k |a_k w_k| per accumulator,
    propagated through the epilogue (RoPE: |cos| S1 + |sin| S2; GELU / GeGLU: through the derivative; LayerNorm fold:
    times rstd);
  * eps is the epilogue's own error: fp32 rounding of its adds and products, the polynomial erf of the GELU epilogues,
    the rstd of the fold and the final rounding (one fp16 ulp of the reference for fp16 outputs).

TAU bounds |acc - exact| / S for the fp32 accumulation of the tensor cores.  IEEE sequential fp32 accumulation could
need K * 2^-24; wgmma's accumulation inside one k16 step is not documented to be IEEE, so TAU is measured: over every
GEMM of tests/test_gemm_conformance_gpu.py on an H100 80GB HBM3 at a 700 W power limit, the largest |err| / S beyond
the epilogue's own error was 4.47e-7 = 2^-21.09 (the fp32 residual epilogue, K = 1160; 2^-23.0 to 2^-23.4 where an fp16
output rounds).  TAU = 2^-20 is 2.1x that.  Longer sums reach more: the grouped fp32 residual GEMMs with a bias per
group at K = 3072 and 4096 (BERT's Wo2) reach 7.0e-7 = 2^-20.44, 1.4x under TAU.  It must stay <= 2^-16: then at
K <= 4096 one missing k-term of average size (S / K >= 2^-12 S) is 16x the bound, so a dropped k-column or k-block
cannot pass.

The precise path's GEMMs (gemm(..., split=True)) sum three times as deep, K' = 3K up to 3 x 4096 = 12 288, and there the
error per unit of S' grows with the depth: over tests/test_precise_kernels_gpu.py on an H100 80GB HBM3 at 700 W the
largest (|err| - eps) / S' was 4.7e-7 at K' = 1152, 7.2e-7 - 7.6e-7 at K' = 2304 - 3456, 1.6e-6 at K' = 7872 and
1.8e-6 = 2^-19.1 at K' = 12 288 (M 17 370, N 1024): beyond TAU, close to the sqrt(K) growth of a sum of
roundings of either sign.  So the split form carries TAU depth_scale(K') = 2^-20 sqrt(K' / 1024), 3.3e-6 at K' = 12 288,
1.8x the measured value (1.0e-6 at K' <= 1024, 2.2x the 4.47e-7 above).  One missing k-term of average size is still
S' / K' = 8e-5 S' at K' = 12 288, 25x the bound.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

EPI_F16, EPI_ROPE, EPI_RESID, EPI_GEGLU, EPI_GELU, EPI_TOPK, EPI_RESID_HL = range(7)
EPI_NAMES = {EPI_F16: "f16", EPI_ROPE: "rope", EPI_RESID: "resid", EPI_GEGLU: "geglu", EPI_GELU: "gelu",
             EPI_TOPK: "topk", EPI_RESID_HL: "resid_hl"}

TAU = 2.0 ** -20
U32 = 2.0 ** -24            # unit roundoff of fp32
ERF_GELU = 1e-6             # |erf error| of gelu_erf_fast_f (tests/test_device_math_constants.py)
ERF_GEGLU = 2e-6            # |erf error| of geglu_fold_f (same test)


@dataclass
class Ref:
    value: torch.Tensor     # float64 reference output
    coef: torch.Tensor      # accumulation error per unit of TAU
    eps: torch.Tensor       # epilogue error

    def bound(self, tau: float = TAU) -> torch.Tensor:
        return tau * self.coef + self.eps

    def tau_needed(self, got: torch.Tensor) -> float:
        """Smallest TAU under which `got` would pass: max over elements of (|err| - eps) / coef."""
        err = (got.double() - self.value).abs() - self.eps
        need = torch.where(self.coef > 0, err / self.coef.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
        return float(need.max().clamp_min(0.0)) if need.numel() else 0.0


def ulp16(y: torch.Tensor) -> torch.Tensor:
    """One fp16 ulp at |y| (subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10.0)


def gelu(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def gelu_deriv(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.special.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def fold_rstd(stats: torch.Tensor, m: int, eps: float, h: int):
    """rstd per row from the [h/128][>=m][2] (sum, sum of squares) slice partials, as the consumer epilogue defines it,
    and a bound on the relative error of the kernel's fp32 evaluation (slice sums, mean^2 cancellation, rsqrtf)."""
    st = stats.double()[:, :m]
    parts = st.shape[0]
    s1, s2 = st[..., 0].sum(0), st[..., 1].sum(0)
    mean = s1 / h
    var = (s2 / h - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + eps)
    cancel = (st[..., 1].abs().sum(0) / h + mean * mean) / (var + eps)
    rel = (parts + 4) * U32 * cancel + 4 * U32
    return rstd, rel


def accumulate(a, w, n, w_groups=0, w_group_rows=0):
    """acc = A W^T and S = |A| |W|^T, float64; grouped weights: row r of A multiplies
    matrix r // w_group_rows of the stack W [w_groups * n, K]."""
    a, w = a.double(), w.double()
    m = a.shape[0]
    if w_groups > 1:
        acc = torch.empty(m, n, dtype=torch.float64, device=a.device)
        s = torch.empty_like(acc)
        for g in range(w_groups):
            r0, r1 = g * w_group_rows, min((g + 1) * w_group_rows, m)
            if r0 >= r1:
                break
            wg = w[g * n:(g + 1) * n]
            acc[r0:r1] = a[r0:r1] @ wg.t()
            s[r0:r1] = a[r0:r1].abs() @ wg.abs().t()
    else:
        acc = a @ w[:n].t()
        s = a.abs() @ w[:n].abs().t()
    return acc, s


def depth_scale(k: int) -> float:
    """TAU's growth with the depth of the sum beyond K = 1024: sqrt(K / 1024) (module docstring)"""
    return max(1.0, math.sqrt(k / 1024.0))


def split_pair(x: torch.Tensor):
    """(hi, lo) fp16 of fp32 x: hi = fp16_rn(x), lo = fp16_rn(x - hi), as precise.cu's split_weight and split_rows_kernel"""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def split3(a: torch.Tensor, w: torch.Tensor):
    """the precise path's triple-depth operands of fp32 A [M, K] and W [N, K]: A' = [A_hi | A_lo | A_hi] and
    W' = [W_hi | W_hi | W_lo], fp16 [*, 3K], so that A' W'^T = A_hi W_hi^T + A_lo W_hi^T + A_hi W_lo^T"""
    ah, al = split_pair(a)
    wh, wl = split_pair(w)
    return torch.cat([ah, al, ah], 1).contiguous(), torch.cat([wh, wh, wl], 1).contiguous()


def _split_terms(a, w, n):
    """(A W^T of the unsplit fp32 operands, S' = |A'| |W'|^T, the split's own error) in float64: the dropped A_lo W_lo^T
    and the residuals |x - hi - lo| of both operands (half an fp16 ulp of x - hi: 2^-25 where lo is subnormal)"""
    w = w[:n]
    (ah, al), (wh, wl) = split_pair(a), split_pair(w)
    a64, w64 = a.double(), w.double()
    ra, rw = (a64 - ah.double() - al.double()).abs(), (w64 - wh.double() - wl.double()).abs()
    ah, al, wh, wl = (t.double().abs() for t in (ah, al, wh, wl))
    acc = a64 @ w64.t()
    s = ah @ wh.t() + al @ wh.t() + ah @ wl.t()
    own = al @ wl.t() + ra @ w64.abs().t() + a64.abs() @ rw.t()
    return acc, s, own


def gemm(epi: int, a: torch.Tensor, w: torch.Tensor, n: Optional[int] = None, *, bias=None, resid=None, pos=None,
         rope_cos=None, rope_sin=None, rope_cols: int = 0, fold_stats=None, fold_eps: float = 0.0, fold_h: int = 0,
         w_groups: int = 0, w_group_rows: int = 0, bias_per_group: bool = False, split: bool = False) -> Ref:
    """Reference of gemm_f16 for a = A [M, K] (only the M rows the GEMM computes), w = W [N, K] (grouped: the stack),
    n = N.  EPI_RESID / EPI_RESID_HL: resid = the stream before the GEMM (the fp16 pair as hi + lo), or None.
    EPI_GEGLU: w rows interleaved in 32-row (a | b) groups; the result is [M, N / 2].  bias_per_group (grouped
    weights): bias is w_groups vectors of n stacked like the matrices, and rows of group g add bias[g n:(g + 1) n].
    split (EPI_RESID only): a and w are the fp32 operands of the precise path, which multiplies split3(a, w) at depth 3K;
    the value is the float64 product of the UNSPLIT a and w, coef is S' over the three parts, and eps also carries the
    dropped A_lo W_lo^T and the split residuals."""
    n = w.shape[0] if n is None else n
    m = a.shape[0]
    if split:
        assert epi == EPI_RESID and w_groups <= 1 and bias is None
        acc, s, own = _split_terms(a, w, n)
        r = resid.double()[:m, :n] if resid is not None else torch.zeros_like(acc)
        v = r + acc
        return Ref(v, s * depth_scale(3 * a.shape[1]), 2 * U32 * (r.abs() + v.abs()) + own)
    acc, s = accumulate(a, w, n, w_groups, w_group_rows)
    if bias is None:
        b = torch.zeros(n, dtype=torch.float64, device=acc.device)
    elif bias_per_group and w_groups > 1:
        group = torch.arange(m, device=acc.device) // w_group_rows
        b = bias.double()[:w_groups * n].reshape(w_groups, n)[group]        # [M, N]: each row its group's bias
    else:
        b = bias.double()[:n]
    zero = torch.zeros_like(acc)
    if epi == EPI_F16:
        v = acc + b
        eps = 2 * U32 * (b.abs() + v.abs()) + ulp16(v)
        return Ref(v, s, eps)
    if epi in (EPI_RESID, EPI_RESID_HL):
        r = resid.double()[:m, :n] if resid is not None else zero
        v = r + acc + b
        if epi == EPI_RESID:
            eps = 2 * U32 * (r.abs() + b.abs() + v.abs())
        else:   # hi + lo carries 22 bits of the new value; lo may be an fp16 subnormal (spacing 2^-24)
            eps = 8 * U32 * (r.abs() + b.abs() + v.abs()) + 2.0 ** -25
        return Ref(v, s, eps)
    if epi == EPI_GELU:
        x = acc + b
        v = gelu(x)
        d = gelu_deriv(x).abs()
        eps = d * U32 * (x.abs() + b.abs()) + 0.5 * x.abs() * ERF_GELU + 4 * U32 * v.abs() + ulp16(v)
        return Ref(v, d * s, eps)
    rstd, rel = (None, None)
    if fold_stats is not None:
        rstd, rel = fold_rstd(fold_stats, m, fold_eps, fold_h)
        rstd, rel = rstd[:, None], rel[:, None]
    if epi == EPI_ROPE:
        x = acc * rstd if rstd is not None else acc.clone()
        sx = s * rstd if rstd is not None else s.clone()
        v, coef = x.clone(), sx.clone()
        mag = x.abs()
        if rope_cols > 0:
            p = pos.long()[:m]
            c, sn = rope_cos.double()[p], rope_sin.double()[p]   # [M, 32]
            for h0 in range(0, rope_cols, 64):
                x1, x2 = x[:, h0:h0 + 32], x[:, h0 + 32:h0 + 64]
                s1, s2 = sx[:, h0:h0 + 32], sx[:, h0 + 32:h0 + 64]
                v[:, h0:h0 + 32] = x1 * c - x2 * sn
                v[:, h0 + 32:h0 + 64] = x1 * sn + x2 * c
                coef[:, h0:h0 + 32] = c.abs() * s1 + sn.abs() * s2
                coef[:, h0 + 32:h0 + 64] = sn.abs() * s1 + c.abs() * s2
                mag[:, h0:h0 + 32] = (x1 * c).abs() + (x2 * sn).abs()
                mag[:, h0 + 32:h0 + 64] = (x1 * sn).abs() + (x2 * c).abs()
        eps = 4 * U32 * mag + ulp16(v)
        if rel is not None:
            eps = eps + rel * mag
        return Ref(v, coef, eps)
    if epi == EPI_GEGLU:
        assert n % 128 == 0
        idx = torch.arange(n // 2, device=acc.device)
        ca = (idx // 32) * 64 + idx % 32          # accumulator column of output column j's `a`; `b` is 32 further
        ga, gb, sa, sb = acc[:, ca], acc[:, ca + 32], s[:, ca], s[:, ca + 32]
        rs = rstd if rstd is not None else torch.ones(m, 1, dtype=torch.float64, device=acc.device)
        xa, xb = ga * rs, gb * rs
        v = gelu(xa) * xb
        d = gelu_deriv(xa).abs()
        coef = rs * (d * xb.abs() * sa + gelu(xa).abs() * sb)
        eps = 0.5 * (xa * xb).abs() * ERF_GEGLU + 8 * U32 * (xa * xb).abs() + ulp16(v)
        if rel is not None:   # rstd error enters both factors
            eps = eps + rel * ((xa * d * xb).abs() + v.abs())
        return Ref(v, coef, eps)
    raise ValueError(f"epilogue {epi}")


def topk(scores: torch.Tensor, k: int, valid: Optional[torch.Tensor] = None):
    """Brute-force top-k per row: descending score, the lower index first on ties; invalid columns never appear.
    Returns (idx [B, k] int64, -1 past the valid count; score [B, k] float64, -inf there)."""
    s = scores.double().clone()
    if valid is not None:
        s[:, ~valid.bool()] = -torch.inf
    if s.shape[1] < k:
        s = torch.cat([s, torch.full((s.shape[0], k - s.shape[1]), -torch.inf, dtype=s.dtype, device=s.device)], 1)
    order = torch.sort(-s, dim=1, stable=True).indices[:, :k]
    val = torch.gather(s, 1, order)
    idx = torch.where(torch.isfinite(val), order, torch.full_like(order, -1))
    return idx, val
