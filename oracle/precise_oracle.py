"""Float64 references of the precise path's row kernels (csrc/precise.cu) with per-element error bounds, and float32
restatements of each kernel's order of operations (TEST INFRASTRUCTURE ONLY).

U = 2^-24 is the unit roundoff of fp32 and gamma(n) = n U / (1 - n U) the bound on n successive roundings.  A kernel
output x is correct when |x - value| <= bound, element by element.  The triple-depth GEMM that sits between these kernels
is gemm_oracle.gemm(..., split=True).

  * Split (split_rows_kernel).  Rows are [hi | lo | hi] with hi = fp16_rn(v), lo = fp16_rn(v - hi); v - hi is exact in
    fp32, so for a given v both halves are deterministic and checked bitwise (`split_halves`).  Without the LayerNorm
    v = x.  With it, v is compared with float64 LN(x) = (x - mu) / sqrt(var + eps) gamma through hi + lo (`split_ln`).
    Sources: each lane sums H / 32 terms and the warp butterfly adds 5 levels, so the mean is within
    dm = gamma(H / 32 + 6) sum |x| / H; x - mean rounds once (U |x - mu|, plus dm); the variance sums squares of those
    differences along the same H / 32 + 5 links (gamma(H / 32 + 5) + 3U relative, plus dm^2: sum_i (x_i - mu) = 0 kills
    the cross term), then / H and + eps round once each (2U); rsqrtf is within 2 ulp (4U); (v - mean) * rstd * gamma
    rounds twice.  So |v - LN| <= |gamma| rstd (dm (1 + U) + U |x - mu|) + |LN| (e_r + 2U) with e_r = e_v / 2 + e_v^2 +
    4U the rstd error.  hi + lo misses v by the split residual, at most half an fp16 ulp of |v - hi| <= ulp16(v) / 2:
    2^-25 absolute where lo is an fp16 subnormal, 2^-22 |v| otherwise.
  * RoPE (rope_f32_kernel) on the given fp32 tables: out = a c - b s and b c + a s, two products and one add (or one
    fmaf and one product): |err| <= 2U (|a c| + |b s|).  Three roundings at their worst attain that (the float32
    restatement reaches 0.9995 of it), so the bound is twice it, 4U (|a c| + |b s|), for the margin of 2 the other bounds
    keep; an fp16-rounded operand or table (2^-11) is still 100x outside.  The hook takes the tables, so this checks the
    kernel, not the tables (those are tests/test_encoder_long_context_gpu.py's far-position mutations).
  * GeGLU (geglu_f32_kernel): 0.5 a (1 + erff(a / sqrt 2)) b.  erff is within 2 ulp (2U absolute: |erf| < 1); the
    argument a * fp32(1 / sqrt 2) rounds twice (2U |x| moves erf by at most 2U |x| erf'(x) <= 0.97 U); 1 + erf rounds
    once (U absolute); the two products round once each.  The bound is ABSOLUTE in |a| |b|:
    2U |a| |b| + 3U |out|.  It cannot be relative to the output: for a <~ -4, 1 + erff(a / sqrt 2) cancels, the kernel's
    absolute 2U error on erff becomes most of the tiny output, and an element-relative check would fail a correct kernel.
  * Attention (attention_f32_kernel): one thread per query row; its 64-row CTA visits keys [k_lo, k_hi) (global: the
    sequence) in nt tiles of 32.  Per tile: scores q' . k_j with q' = q * 0.125 (exact) as a 64-link fmaf chain, running
    max m, alpha = expf(m_old - m), p_j = expf(s_j - m), lt = sum of the tile's p_j, l = fmaf(l, alpha, lt), and per
    column acc = sum_j p_j v_jd (32 fmaf) then o = fmaf(o, alpha, acc); at the end out = o * (1 / l).  Softmax is
    shift-invariant, so an error x_j in key j's exponent moves the output by (1 / Z) sum_j P_j (e^{x_j} - 1)(v_j - out),
    at most F sum_j P_j |x_j| D_j with D_j = |v_j - out| and F = exp(2 max |x_j|).  The sources:
      - score: the 64-link fmaf chain, gamma(64) a_j with a_j = 0.125 sum_d |q_d k_jd|;
      - exponent: s_j - m and every alpha argument m_old - m round once each, and those arguments telescope to
        m - s_j: U (m - s_j); expf is within 2 ulp (4U relative) for p_j and for each of at most nt alphas: 4U (nt + 1);
      - sums: every term p_j v_jd passes through at most 32 roundings in its tile and one per later tile in o, and the
        same for l: gamma(32 + nt) (sum_j P_j |v_jd| + |out_d|), times F;
      - out: 1 / l and the product, gamma(2) |out|; weights and partial sums in the fp32 subnormals add at most 2^-149
        per rounding: (32 + nt) n 2^-149 (1 + max |v|).
    The same kernel with ONE chain over the keys (o = o alpha per tile, then o = fmaf(p_j, v_j, o) per key) passes the
    first terms through n + nt roundings.  Its error grows as n U where the terms are correlated: constant V columns
    under uniform scores (family "constant") reach 4.9e-4 relative at 32 768 keys in the float32 restatement (the
    column 1 + 2^-10), 3.9x this bound, where the tiled sums stay at 0.08 of it (tests/test_precise_oracle.py).

The float32 restatements (`restate_*`) follow each kernel's order of operations in numpy.  fmaf is emulated as the
float64 product of two fp32 values (exact) plus the fp32 addend, rounded once to fp32: equal to fmaf except for rare
double rounding.  expf and erff are the float64 functions rounded to fp32 (correctly rounded, where the GPU's are within
2 ulp).  tests/test_precise_oracle.py shows every restatement inside its bound with a margin >= 2 on every input family
of tests/test_precise_kernels_gpu.py, and each of MUTATIONS outside it by > 10x.  The split residual is an exact
rounding that reaches its bound, so there the margin applies to the LayerNorm's arithmetic (v against the bound less the
residual) and hi + lo is checked against the whole bound.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from oracle import attn_oracle as ao

U = 2.0 ** -24
TILE = 32            # keys per tile
ROWS = 64            # query rows per CTA
SUBN = 2.0 ** -149   # fp32 subnormal spacing
f32, f64 = np.float32, np.float64
INV_SQRT2_F32 = f32(0.70710678118654752440)
MUTATIONS = ("split_no_lo", "ln_no_gamma", "rope_swapped_halves", "rope_local_table", "gelu_tanh", "window_minus_one",
             "short_tile", "no_alpha", "scale_twice")
ATTN_SOURCES = ("score", "exponent", "sums", "out")


def gamma(n):
    return n * U / (1.0 - n * U)


def ulp16(y: torch.Tensor) -> torch.Tensor:
    """one fp16 ulp at |y| (subnormal spacing 2^-24 below 2^-14)"""
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10.0)


def split_residual(v: torch.Tensor) -> torch.Tensor:
    """bound on |v - hi - lo|: half an fp16 ulp of |v - hi| <= ulp16(v) / 2"""
    return 0.5 * ulp16(0.5 * ulp16(v.abs() * (1 + 2.0 ** -20)))


# ---- split ---------------------------------------------------------------------------------------------------------
def split_halves(v: np.ndarray):
    """(hi, lo) fp16 of fp32 v: hi = fp16_rn(v), lo = fp16_rn(v - hi) -- bitwise what split_rows_kernel and split_weight
    store (numpy's float32 -> float16 conversion rounds to nearest even)"""
    v = np.asarray(v, dtype=f32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(f32)).astype(np.float16)
    return hi, lo


@dataclass
class RowRef:
    value: torch.Tensor     # float64 reference
    bound: torch.Tensor     # per-element bound on |kernel - value|
    split: Optional[torch.Tensor] = None   # split_ln: the part of the bound that is the split residual |v - hi - lo|


def split_ln(x: torch.Tensor, gamma_: torch.Tensor, eps: float) -> RowRef:
    """the LayerNorm variant: value = float64 LN(x) gamma, bound on |hi + lo - value| (module docstring)"""
    x = x.double()
    g = gamma_.double()
    H = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = d.pow(2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = d * rstd * g
    links = H // 32 + (1 if H % 32 else 0) + 5
    dm = gamma(links + 1) * x.abs().sum(-1, keepdim=True) / H
    e_v = ((gamma(links) + 3 * U) * var + dm * dm + 2 * U * dm * d.abs().mean(-1, keepdim=True)) / (var + eps) + 2 * U
    e_r = e_v / 2 + e_v * e_v + 4 * U
    bound = g.abs() * rstd * (dm * (1 + U) + U * d.abs()) + y.abs() * (e_r + 2 * U)
    res = split_residual(y.abs() + bound)
    return RowRef(y, bound + res, res)


def restate_split(x: np.ndarray, gamma_: Optional[np.ndarray], eps: float, mut: Optional[str] = None):
    """split_rows_kernel in float32: lane-strided sums, the warp butterfly, rsqrt; returns (hi, lo) fp16 [T, H] and the
    fp32 v they split"""
    x = np.asarray(x, dtype=f32)
    T, H = x.shape
    if gamma_ is not None:
        if mut == "ln_no_gamma":
            gamma_ = np.ones(H, dtype=f32)

        def warp_sum(vals):                                     # vals [T, H] -> per-lane partials -> butterfly
            lanes = np.zeros((T, 32), dtype=f32)
            for i in range(H):
                lanes[:, i % 32] = lanes[:, i % 32] + vals[:, i]
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[:, np.arange(32) ^ o]
            return lanes[:, 0]

        mean = warp_sum(x) / f32(H)
        dd = x - mean[:, None]
        var = warp_sum(dd * dd)
        rstd = (f32(1.0) / np.sqrt((var / f32(H) + f32(eps)).astype(f64))).astype(f32)
        v = ((x - mean[:, None]) * rstd[:, None]) * np.asarray(gamma_, dtype=f32)[None, :]
    else:
        v = x
    hi, lo = split_halves(v)
    if mut == "split_no_lo":
        lo = np.zeros_like(lo)
    return hi, lo, v


# ---- RoPE ----------------------------------------------------------------------------------------------------------
def rope(qkv: torch.Tensor, pos: torch.Tensor, heads: int, cos_t: torch.Tensor, sin_t: torch.Tensor) -> RowRef:
    """rotate-half RoPE of the q and k thirds of qkv [T, 3 heads 64] (fp32 values) at rows pos of the [*, 32] tables;
    the v third is unchanged (bound 0)"""
    x = qkv.double().clone()
    T = x.shape[0]
    H = heads * 64
    c, s = cos_t.double()[pos.long()][:, None, :], sin_t.double()[pos.long()][:, None, :]    # [T, 1, 32]
    bound = torch.zeros_like(x)
    for third in (0, 1):
        blk = x[:, third * H:(third + 1) * H].reshape(T, heads, 64)
        a, b = blk[..., :32], blk[..., 32:]
        out = torch.cat([a * c - b * s, b * c + a * s], -1)
        bd = torch.cat([4 * U * ((a * c).abs() + (b * s).abs()), 4 * U * ((b * c).abs() + (a * s).abs())], -1)
        x[:, third * H:(third + 1) * H] = out.reshape(T, H)
        bound[:, third * H:(third + 1) * H] = bd.reshape(T, H)
    return RowRef(x, bound)


def restate_rope(qkv: np.ndarray, pos: np.ndarray, heads: int, cos_t: np.ndarray, sin_t: np.ndarray,
                 mut: Optional[str] = None, cos_other=None, sin_other=None) -> np.ndarray:
    """rope_f32_kernel in float32 (products rounded, then the add).  rope_local_table: the other layer kind's tables"""
    x = np.array(qkv, dtype=f32, copy=True)
    T = x.shape[0]
    H = heads * 64
    if mut == "rope_local_table":
        cos_t, sin_t = cos_other, sin_other
    c = np.asarray(cos_t, dtype=f32)[pos][:, None, :]
    s = np.asarray(sin_t, dtype=f32)[pos][:, None, :]
    for third in (0, 1):
        blk = x[:, third * H:(third + 1) * H].reshape(T, heads, 64)
        a, b = blk[..., :32].copy(), blk[..., 32:].copy()
        if mut == "rope_swapped_halves":
            a, b = b, a
        blk[..., :32] = a * c - b * s
        blk[..., 32:] = b * c + a * s
        x[:, third * H:(third + 1) * H] = blk.reshape(T, H)
    return x


# ---- GeGLU ---------------------------------------------------------------------------------------------------------
def geglu(ab: torch.Tensor, I: int) -> RowRef:
    """gelu_erf(a) * b over ab [T, 2I] (fp32 values); the bound is absolute in |a| |b| (module docstring)"""
    x = ab.double()
    a, b = x[:, :I], x[:, I:2 * I]
    v = 0.5 * a * (1.0 + torch.special.erf(a / math.sqrt(2.0))) * b
    return RowRef(v, 2 * U * (a * b).abs() + 3 * U * v.abs() + 2.0 ** -140)


def restate_geglu(ab: np.ndarray, I: int, mut: Optional[str] = None) -> np.ndarray:
    """geglu_f32_kernel in float32: 0.5f * a * (1 + erff(a * 0.70710678f)) * b"""
    ab = np.asarray(ab, dtype=f32)
    a, b = ab[:, :I], ab[:, I:2 * I]
    if mut == "gelu_tanh":
        a64 = a.astype(f64)
        t = np.tanh(math.sqrt(2.0 / math.pi) * (a64 + 0.044715 * a64 ** 3)).astype(f32)
        return (f32(0.5) * a * (f32(1.0) + t)) * b
    arg = a * INV_SQRT2_F32
    erf = torch.special.erf(torch.from_numpy(arg.astype(f64))).numpy().astype(f32)
    return ((f32(0.5) * a) * (f32(1.0) + erf)) * b


# ---- attention -----------------------------------------------------------------------------------------------------
@dataclass
class AttnRef:
    value: torch.Tensor
    bound: torch.Tensor
    terms: Dict[str, torch.Tensor] = field(default_factory=dict)


def key_range(len_: int, window: int, q0: int):
    """[k_lo, k_hi) of the CTA whose first query row is q0"""
    if window <= 0:
        return 0, len_
    return max(q0 - window, 0), min(q0 + ROWS + window, len_)


def _tiles(len_: int, window: int, rows: torch.Tensor) -> torch.Tensor:
    q0 = (rows // ROWS) * ROWS
    if window <= 0:
        return torch.full_like(rows, (len_ + TILE - 1) // TILE)
    lo = (q0 - window).clamp_min(0)
    hi = (q0 + ROWS + window).clamp_max(len_)
    return (hi - lo + TILE - 1) // TILE


def _rows_chunk(heads: int, keys: int) -> int:
    r = 1024
    while r > 1 and r * keys * heads * 64 > (1 << 27):
        r //= 2
    return r


def _seq(q, k, v, rows, len_, window):
    """one sequence, every head: q, k, v [nH, len, 64] float64 -> value, terms [nH, R, 64]"""
    r0, r1 = int(rows.min()), int(rows.max())
    j0, j1 = (max(0, r0 - window), min(len_, r1 + window + 1)) if window > 0 else (0, len_)
    kk, vv, qq = k[:, j0:j1], v[:, j0:j1], q[:, rows]
    s = 0.125 * (qq @ kk.transpose(1, 2))
    a = 0.125 * (qq.abs() @ kk.abs().transpose(1, 2))
    j = torch.arange(j0, j1, device=q.device)
    vis = torch.ones(len(rows), j1 - j0, dtype=torch.bool, device=q.device)
    if window > 0:
        vis = (j[None, :] - rows[:, None]).abs() <= window
    vis = vis[None].expand_as(s)
    s = torch.where(vis, s, -torch.inf)
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    p = e / e.sum(-1, keepdim=True)
    out = p @ vv
    nt = _tiles(len_, window, rows).double()[None, :, None]                    # [1, R, 1]
    zero = torch.zeros_like(s)
    xs = torch.where(vis, gamma(64) * a, zero)
    rho = torch.where(vis, U * (m - s) + 4 * U * (nt + 1), zero)
    F = torch.exp(2 * (xs + rho).amax(-1, keepdim=True))
    d = (vv[:, None, :, :] - out[:, :, None, :]).abs()                         # [nH, R, Kk, 64]
    score = F * torch.einsum("hrk,hrkd->hrd", p * xs, d)
    expo = F * torch.einsum("hrk,hrkd->hrd", p * rho, d)
    del d
    av = vv.abs()
    n_vis = vis.sum(-1, keepdim=True).double()
    sums = F * gamma(32 + nt) * (p @ av + out.abs())
    outt = gamma(2) * out.abs() + (32 + nt) * n_vis * SUBN * (1 + av.amax(1, keepdim=True))
    return out, {"score": score, "exponent": expo, "sums": sums, "out": outt}


def attention(qkv: torch.Tensor, cu: Sequence[int], heads: int, window: int = 0,
              sel: Optional[torch.Tensor] = None) -> AttnRef:
    """reference of precise_attention for fp32 qkv [>= T, 3 heads 64] packed by `cu`, on output rows `sel` (global
    indices, ascending; default all).  Rows are computed in chunks over only the keys they see."""
    dev = qkv.device
    H = heads * 64
    T = int(cu[-1])
    sel = torch.arange(T, device=dev) if sel is None else sel.to(dev).long()
    val = torch.zeros(sel.numel(), H, dtype=torch.float64, device=dev)
    terms = {k: torch.zeros_like(val) for k in ATTN_SOURCES}
    cu_t = torch.as_tensor(list(cu), device=dev)
    seq_of = torch.searchsorted(cu_t, sel, right=True) - 1
    for b in torch.unique(seq_of).tolist():
        s0, s1 = int(cu[b]), int(cu[b + 1])
        idx = (seq_of == b).nonzero().flatten()
        len_ = s1 - s0
        x = qkv[s0:s1].double().view(len_, 3, heads, 64).permute(1, 2, 0, 3)
        rows_all = sel[idx] - s0
        keys = len_ if window <= 0 else min(len_, 2 * window + 1 + 1024)
        step = _rows_chunk(heads, keys)
        for c0 in range(0, idx.numel(), step):
            ii, rows = idx[c0:c0 + step], rows_all[c0:c0 + step]
            o, tm = _seq(x[0], x[1], x[2], rows, len_, window)
            val[ii] = o.permute(1, 0, 2).reshape(-1, H)
            for kname, t in tm.items():
                terms[kname][ii] = t.permute(1, 0, 2).reshape(-1, H)
    bound = sum(terms.values())
    return AttnRef(val, bound, terms)


def _fma(a, b, c):
    """fmaf emulation: float64 product (exact for fp32 operands) plus the addend, rounded once to fp32"""
    return (a.astype(f64) * b.astype(f64) + c.astype(f64)).astype(f32)


def _expf(x):
    return np.exp(x.astype(f64)).astype(f32)


def restate_attention(qkv: np.ndarray, cu: Sequence[int], heads: int, window: int = 0,
                      sel: Optional[np.ndarray] = None, chain: str = "tile", mut: Optional[str] = None) -> np.ndarray:
    """attention_f32_kernel in float32 on output rows `sel` -> [len(sel), heads 64].  chain "one": the kernel with one
    fmaf chain over all keys (the accumulation before per-tile sums).  mut: window_minus_one, short_tile (k_hi one tile
    short), no_alpha, scale_twice."""
    qkv = np.asarray(qkv, dtype=f32)
    H = heads * 64
    T = int(cu[-1])
    sel = np.arange(T) if sel is None else np.asarray(sel)
    out = np.zeros((len(sel), H), dtype=f32)
    scale = f32(0.125 * 0.125) if mut == "scale_twice" else f32(0.125)
    wv = window - 1 if (mut == "window_minus_one" and window > 0) else window
    cu_a = np.asarray(cu)
    seq_of = np.searchsorted(cu_a, sel, side="right") - 1
    for b in np.unique(seq_of):
        s0, len_ = int(cu[b]), int(cu[b + 1]) - int(cu[b])
        x = qkv[s0:s0 + len_].reshape(len_, 3, heads, 64)
        idx_b = np.nonzero(seq_of == b)[0]
        rows_b = sel[idx_b] - s0
        for q0 in np.unique((rows_b // ROWS) * ROWS):
            ii = idx_b[(rows_b // ROWS) * ROWS == q0]
            rows = sel[ii] - s0
            k_lo, k_hi = key_range(len_, window, int(q0))
            if mut == "short_tile":
                k_hi = max(k_lo, k_hi - TILE)
            for h in range(heads):
                q = x[rows, 0, h] * scale                                   # [R, 64]
                R = len(rows)
                m = np.full(R, -np.inf, dtype=f32)
                l = np.zeros(R, dtype=f32)
                o = np.zeros((R, 64), dtype=f32)
                for k0 in range(k_lo, k_hi, TILE):
                    kj = np.arange(k0, k0 + TILE)
                    ok = kj < len_
                    kt = np.where(ok[:, None], x[np.minimum(kj, len_ - 1), 1, h], f32(0))
                    vt = np.where(ok[:, None], x[np.minimum(kj, len_ - 1), 2, h], f32(0))
                    acc = np.zeros((R, TILE), dtype=f32)
                    for d in range(64):
                        acc = _fma(q[:, d:d + 1], kt[None, :, d], acc)
                    vis = ok[None, :] & np.ones((R, 1), dtype=bool)
                    if window > 0:
                        vis = vis & (np.abs(kj[None, :] - rows[:, None]) <= wv)
                    s = np.where(vis, acc, f32(-np.inf))
                    tm = s.max(1)
                    live = tm != -np.inf
                    mn = np.maximum(m, tm)
                    with np.errstate(invalid="ignore"):
                        alpha = np.where(m == -np.inf, f32(0), _expf(m - mn))
                        if mut == "no_alpha":
                            alpha = np.where(m == -np.inf, f32(0), f32(1))
                        p = np.where(s == -np.inf, f32(0), _expf(s - mn[:, None]))
                    if chain == "one":
                        l2 = l * alpha
                        o2 = o * alpha[:, None]
                        for j in range(TILE):
                            l2 = l2 + p[:, j]
                            o2 = _fma(p[:, j:j + 1], vt[None, j], o2)
                    else:
                        lt = np.zeros(R, dtype=f32)
                        for j in range(TILE):
                            lt = lt + p[:, j]
                        l2 = _fma(l, alpha, lt)
                        a2 = np.zeros((R, 64), dtype=f32)
                        for j in range(TILE):
                            a2 = _fma(p[:, j:j + 1], vt[None, j], a2)
                        o2 = _fma(o, alpha[:, None], a2)
                    l = np.where(live, l2, l)
                    o = np.where(live[:, None], o2, o)
                    m = np.where(live, mn, m)
                with np.errstate(divide="ignore", invalid="ignore"):
                    out[ii, h * 64:(h + 1) * 64] = o * (f32(1.0) / l)[:, None]
    return out


# ---- input families ------------------------------------------------------------------------------------------------
FAMILIES = ao.FAMILIES + ("constant",)


def constant_columns() -> torch.Tensor:
    """the V row of family "constant": column 0 = 1 + 2^-10, column d = fp32(1.3 + d / 64)"""
    c = torch.tensor([1.3 + d / 64.0 for d in range(64)], dtype=torch.float32)
    c[0] = 1.0 + 2.0 ** -10
    return c


def make_qkv(family: str, cu: Sequence[int], heads: int, window: int = 0, seed: int = 0, device="cpu") -> torch.Tensor:
    """fp32 qkv [cu[-1], 3 heads 64] of one family: attn_oracle.make_qkv's families (fp16 values; "random" has full fp32
    mantissas), and "constant": q = 0 (uniform scores), every V row the same constant_columns() -- every output element
    is that column's constant exactly, and the weighted terms of a row's sums are all equal."""
    T = int(cu[-1])
    if family == "random":
        g = torch.Generator(device=device).manual_seed(seed)
        return torch.randn(T, 3 * heads * 64, generator=g, device=device, dtype=torch.float32)
    if family == "constant":
        x = ao.make_qkv("random", cu, heads, window, seed=seed, device=device).float().view(T, 3, heads, 64)
        x[:, 0] = 0.0
        x[:, 2] = constant_columns().to(device)
        return x.reshape(T, 3 * heads * 64).contiguous()
    return ao.make_qkv(family, cu, heads, window, seed=seed, device=device).float()
