"""Float64 reference of the wgmma attention kernel (csrc/attention_wgmma.cu) with an explicit per-element error bound.

value: out_i = sum_j P_ij v_j with P_i = softmax_j(0.125 q_i . k_j) over the visible keys j < min(len, kv_lens[b]) and,
when window > 0, |i - j| <= window; the fp16 operands are exact in float64.  A kernel output x is correct when
|x - value| <= TAU * coef + eps (gemm_oracle.Ref), with u = 2^-24 and gamma(n) = n u / (1 - n u).

The kernel (per row i, per 64-key block b of the nb blocks its 64-row tile visits): S = Q K^T on the tensor cores (fp32
accumulation), m_b = running max, alpha = exp2f((m_{b-1} - m_b) c'), p_j = exp2f((S_j - m_b) c') in fp32 with
c' = fp32(0.125 * fp32(log2 e)), l = l alpha + sum of the fp32 p_j, o = o alpha + fp16(p) V on the tensor cores; at the end
out = fp16(o * (1 / l)).  Softmax is shift-invariant, so an error x_j in the exponent of key j (natural units) moves the
output by exactly sum_j (P'_j - P_j)(v_j - out) = (1 / Z) sum_j P_j (e^{x_j} - 1)(v_j - out), hence by at most
F sum_j P_j |x_j| D_j with D_j = |v_j - out| and F = exp(2 max |x_j|).  The sources:

  * Score accumulation.  wgmma accumulates q . k over K = 64 in fp32 within TAU * a_j, a_j = sum_d |q_d k_jd| (the
    constant of gemm_oracle, measured there for K <= 1160): x_j gets 0.125 TAU a_j -> coef += F 0.125 sum_j P_j a_j D_j.
  * Exponent argument.  c' is within EPS_C = 2^-26.2 of 0.125 log2 e; S_j - m_b and the product with c' round once each,
    and so do m_{b-1} - m_b and its product for every alpha a key's weight passes through.  Those arguments add up to
    c (m - s_j), so x_j gets 0.125 (m - s_j) (EPS_C + 2u).  exp2f is within 2 ulp (4u relative; no --use_fast_math) for p_j
    and for each of at most nb alphas, which multiply o and l alike: x_j gets 4u (nb + 1).  -> eps += F sum_j P_j x_j D_j.
  * fp16 P.  o takes fp16(p_j) while l sums the fp32 p_j, so the weights are not renormalised: each p_j >= 2^-14 is off by
    2^-11 relative, a subnormal or flushed p_j (< 2^-14 in the scale of the running max) by up to 2^-25 absolute.  The
    later alphas are <= 1 and l >= Lf = sum_j exp(0.125 (s_j - m)) >= 1, so the output moves by at most
    2^-11 sum_j P_j |v_j| + 2^-25 sum_{j: P_j Lf < 2^-13} |v_j| / Lf.  The second term is the one that grows with the
    key count: with one dominant key it reaches ~ L 2^-25 max |v| (8e-4 at 32 k keys); it is carried as is.
  * The sum l.  One fp32 chain per thread: per block one alpha product and 8 adds of a pair-sum, then 2 shuffle adds, so
    every p_j passes through at most n = 9 nb + 2 roundings: eps += gamma(9 nb + 2) |out|.
  * PV accumulation.  wgmma accumulates the 64 keys of a block into o (fp32) and o is rescaled by alpha once per block:
    the chain over the row's keys has nb links of 64 keys.  Each link is bounded like a GEMM accumulation of K = 64,
    TAU sum |p v| (the GEMM's TAU covers a whole K <= 1160 chain), and the chains add linearly, the worst case:
    coef += F nb sum_j P_j |v_j|; the alpha products add u nb sum_j P_j |v_j| to eps.
  * Output.  1 / l and the product round once each (2u |out|), then the fp16 store (one fp16 ulp of the reference, as
    gemm_oracle), and a 2^-140 floor for fp32 subnormal p_j.

The two tensor-core accumulations are the only sources without a documented constant, so they carry TAU, measured for
the GEMM.  Over every launch of tests/test_attention_conformance_gpu.py (3.3e8 output elements) on an H100 80GB HBM3 at
a 400 W power limit, no element needed any of it: the largest (|err| - eps) / coef was <= 0, because the fp16 store
(2^-11 relative) hides fp32 accumulation errors of these sizes.  The largest |err| / bound, by the source that dominates
the bound, was 0.73 (fp16 P), 0.69 (output rounding), 0.24 (score accumulation), 0.15 (PV accumulation).  A constant set
from a zero measurement would be zero, so TAU = 2^-20 stays: it is what the tensor cores were measured to need for one
fp32 chain of K <= 1160, and it stays small enough for tests/test_attn_oracle.py: at nb <= 512 blocks the PV term
TAU nb sum P |v| <= 2^-11 sum P |v| is no larger than the fp16-P term, and the score term 0.125 TAU a_j is <= 5e-3 in
the exponent for |q|, |k| ~ 30, while a window or key length off by one, a skipped block or a missing alpha moves the
output by > 10x the whole bound on the test inputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence

import torch

from oracle.gemm_oracle import TAU, Ref, ulp16

U = 2.0 ** -24
TINY = 2.0 ** -140
BQ = BKV = 64                  # query rows per CTA, keys per block
C_LOG2 = 0.125 / math.log(2.0)
C_F32 = float(torch.tensor(0.125, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32))
EPS_C = abs(C_F32 / C_LOG2 - 1.0)
SOURCES = ("score", "exponent", "p16", "l", "pv", "out")


def gamma(n):
    return n * U / (1.0 - n * U)


@dataclass
class AttnRef(Ref):
    terms: Dict[str, torch.Tensor] = field(default_factory=dict)   # bound of each source (at TAU), same shape as value


def blocks(len_: int, window: int, q0):
    """(kb_lo, kb_hi) of the key blocks the CTA of query tile q0 (a tensor of tile starts) visits"""
    if window <= 0:
        return torch.zeros_like(q0), torch.full_like(q0, (len_ - 1) // BKV)
    lo = (q0 - window).clamp_min(0) // BKV
    hi = (q0 + BQ - 1 + window).clamp_max(len_ - 1) // BKV
    return lo, hi


def _rows_chunk(heads: int, keys: int, window: int) -> int:
    """query rows per chunk: the [heads, rows, keys, 64] float64 tensor of |v_j - out| stays below 1 GiB"""
    r = 1024
    while r > 1 and r * ((min(keys, r + 2 * window + 64)) if window > 0 else keys) * heads * 64 > (1 << 27):
        r //= 2
    return r


def _seq(q, k, v, rows, len_, klen, window, tau):
    """one sequence, every head: q [nH, len, 64], rows = local query rows -> (value, coef, eps, terms) [nH, R, 64]"""
    r0, r1 = int(rows.min()), int(rows.max())
    if window > 0:
        j0, j1 = max(0, r0 - window), min(klen, r1 + window + 1)
    else:
        j0, j1 = 0, klen
    kk, vv = k[:, j0:j1], v[:, j0:j1]
    qq = q[:, rows]
    s = qq @ kk.transpose(1, 2)                                          # [nH, R, Kk] unscaled
    a = qq.abs() @ kk.abs().transpose(1, 2)
    j = torch.arange(j0, j1, device=q.device)
    vis = (j[None, :] < klen).expand(len(rows), -1)
    if window > 0:
        vis = vis & ((j[None, :] - rows[:, None]).abs() <= window)
    vis = vis[None].expand_as(s)
    s = torch.where(vis, s, -torch.inf)
    m = s.amax(-1, keepdim=True)
    e = torch.exp(0.125 * (s - m))
    lf = e.sum(-1, keepdim=True)
    p = e / lf
    out = p @ vv
    lo, hi = blocks(len_, window, (rows // BQ) * BQ)
    nb = (hi - lo + 1).double()[None, :, None]                           # [1, R, 1]
    g = torch.where(vis, m - s, torch.zeros_like(s))
    rho = 0.125 * g * (EPS_C + 2 * U) + 4 * U * (nb + 1)
    xs = 0.125 * a
    F = torch.exp(2 * torch.where(vis, tau * xs + rho, torch.zeros_like(s)).amax(-1, keepdim=True))
    d = (vv[:, None, :, :] - out[:, :, None, :]).abs()                   # [nH, R, Kk, 64]
    score = F * torch.einsum("hrk,hrkd->hrd", p * xs, d)
    expo = F * torch.einsum("hrk,hrkd->hrd", p * rho, d)
    del d
    av = vv.abs()
    pv = p @ av
    sub = (vis & (p * lf < 2.0 ** -13)).double()
    p16 = F * (2.0 ** -11 * pv + 2.0 ** -25 * (sub @ av) / lf)
    lterm = gamma(9 * nb + 2) * out.abs()
    pvc = F * nb * pv
    outt = 2 * U * out.abs() + ulp16(out) + TINY
    coef = score + pvc
    eps = expo + p16 + lterm + U * nb * pv + outt
    terms = {"score": tau * score, "exponent": expo, "p16": p16, "l": lterm, "pv": tau * pvc + U * nb * pv, "out": outt}
    return out, coef, eps, terms


def attention(qkv: torch.Tensor, cu: Sequence[int], num_heads: int, window: int = 0,
              kv_lens: Optional[Sequence[int]] = None, sel: Optional[torch.Tensor] = None, tau: float = TAU) -> AttnRef:
    """Reference of attention_wgmma_fwd for qkv [>= T, 3 * num_heads * 64] (fp16, any device) packed by cu_seqlens `cu`,
    on the output rows `sel` (global token indices, ascending; default every row).  Windowed rows are computed over
    their band of keys only, and rows in chunks, so no full L x L matrix is built for long sequences.
    Returns value, coef, eps [len(sel), num_heads * 64] and the bound of each source in `terms`."""
    dev = qkv.device
    H = num_heads * 64
    T = int(cu[-1])
    sel = torch.arange(T, device=dev) if sel is None else sel.to(dev).long()
    n = sel.numel()
    val = torch.zeros(n, H, dtype=torch.float64, device=dev)
    coef, eps = torch.zeros_like(val), torch.zeros_like(val)
    terms = {k: torch.zeros_like(val) for k in SOURCES}
    for b in range(len(cu) - 1):
        s0, s1 = int(cu[b]), int(cu[b + 1])
        if s1 <= s0:
            continue
        idx = ((sel >= s0) & (sel < s1)).nonzero().flatten()
        if idx.numel() == 0:
            continue
        len_ = s1 - s0
        klen = min(len_, int(kv_lens[b])) if kv_lens is not None else len_
        x = qkv[s0:s1].double().view(len_, 3, num_heads, 64).permute(1, 2, 0, 3)   # [3, nH, len, 64]
        q, k, v = x[0], x[1], x[2]
        rows_all = sel[idx] - s0
        step = _rows_chunk(num_heads, klen, window)
        for c0 in range(0, idx.numel(), step):
            ii, rows = idx[c0:c0 + step], rows_all[c0:c0 + step]
            o, cf, ep, tm = _seq(q, k, v, rows, len_, klen, window, tau)
            val[ii] = o.permute(1, 0, 2).reshape(-1, H)
            coef[ii] = cf.permute(1, 0, 2).reshape(-1, H)
            eps[ii] = ep.permute(1, 0, 2).reshape(-1, H)
            for kname, t in tm.items():
                terms[kname][ii] = t.permute(1, 0, 2).reshape(-1, H)
    return AttnRef(val, coef, eps, terms)


# ---- input families of tests/test_attention_conformance_gpu.py (and, at CPU sizes, tests/test_attn_oracle.py) --------
FAMILIES = ("random", "position", "needle", "sink", "late", "tied", "uniform", "large")


def _local(cu, T, dev):
    """local row index of every packed row (rows past cu[-1]: 0) and its sequence"""
    pos = torch.zeros(T, dtype=torch.long, device=dev)
    seq = torch.zeros(T, dtype=torch.long, device=dev)
    for b in range(len(cu) - 1):
        s0, s1 = int(cu[b]), int(cu[b + 1])
        pos[s0:s1] = torch.arange(s1 - s0, device=dev)
        seq[s0:s1] = b
    return pos, seq


NEEDLE_THETA = [1.5 * 0.8 ** f for f in range(32)]      # incommensurate angles: one sharp peak, no alias within 4 k


def make_qkv(family: str, cu: Sequence[int], num_heads: int, window: int = 0, kv_lens: Optional[Sequence[int]] = None,
             seed: int = 0, device="cpu", head_dim_used: int = 64) -> torch.Tensor:
    """qkv [cu[-1], 3 * num_heads * 64] fp16 of one input family; dims >= head_dim_used of q / k / v are zero.
      random   N(0, 1) q, k, v
      position v_jd = 1 where (j // 64) % 64 == d: a skipped or doubled key block moves whole output columns
      needle   q_i . k_j = 16 sum_f cos(theta_f (t_i - j)) peaks at j = t_i, the first key the mask hides: i +- (window
               + 1) (windowed; the sign alternates with i), kv_lens[b] (key lengths), len (otherwise, the next
               sequence's first row); the visible best key sits at the mask edge
      sink     key 0 of every sequence 10-28 (natural units) above the others, which fall into the fp16 subnormal and
               flush range relative to it
      late     scores rise by 0.02 per key: the running max and alpha change in every block
      tied     keys j % 80 == 40 share the top score exactly, 30 above the rest (flushed): P = 1 / (visible peaks)
      uniform  q = 0
      large    q, k ~ 30 N(0, 1): only the argmax keys survive"""
    T = int(cu[-1])
    g = torch.Generator(device=device).manual_seed(seed)
    nH = num_heads

    def rn(*shape):
        return torch.randn(*shape, generator=g, device=device, dtype=torch.float64)

    q, k, v = rn(T, nH, 64), rn(T, nH, 64), rn(T, nH, 64)
    pos, seq = _local(cu, T, device)
    pf = pos.double()[:, None]
    if family == "position":
        v = ((pos // 64) % 64)[:, None, None] == torch.arange(64, device=device)[None, None, :]
        v = v.double().expand(T, nH, 64).clone()
    elif family == "needle":
        lens = torch.tensor([int(cu[b + 1]) - int(cu[b]) for b in range(len(cu) - 1)], device=device)[seq]
        if kv_lens is not None:
            t = torch.tensor([int(x) for x in kv_lens], device=device)[seq].double()
        elif window > 0:
            sign = 1.0 - 2.0 * (pos % 2).double()
            t = pos.double() + sign * (window + 1)
        else:
            t = lens.double()
        th = torch.tensor(NEEDLE_THETA, dtype=torch.float64, device=device)[None, :]
        qa, ka = t[:, None] * th, pf * th
        q = 4.0 * torch.cat([torch.cos(qa), torch.sin(qa)], 1)[:, None, :].expand(T, nH, 64).clone()
        k = 4.0 * torch.cat([torch.cos(ka), torch.sin(ka)], 1)[:, None, :].expand(T, nH, 64).clone()
    elif family in ("sink", "late", "tied"):
        q = 0.1 * q
        k = 0.1 * k
        q[..., 0] = 8.0                                                  # 0.125 q . k = k[0] + O(0.1)
        if family == "sink":
            gap = 10.0 + 18.0 * torch.rand(T, generator=g, device=device, dtype=torch.float64)
            k[..., 0] = torch.where(pos == 0, torch.zeros_like(gap), -gap)[:, None]
        elif family == "late":
            k[..., 0] = (0.02 * pf).expand(T, nH)
        else:
            q[..., 1:] = 0.0
            k[..., 1:] = 0.0
            k[..., 0] = torch.where(pos % 80 == 40, 0.0, -30.0)[:, None].double()
    elif family == "uniform":
        q = torch.zeros_like(q)
    elif family == "large":
        q, k = 30.0 * q, 30.0 * k
    elif family != "random":
        raise ValueError(family)
    if head_dim_used < 64:
        for t in (q, k, v):
            t[..., head_dim_used:] = 0.0
    return torch.stack([q, k, v], 1).reshape(T, 3 * nH * 64).half().contiguous()
