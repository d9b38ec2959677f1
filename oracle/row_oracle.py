"""Float64 reference of the row kernels of csrc/elementwise.cu with an explicit per-element error bound.

Every function takes the exact fp32 (or fp16) inputs of one launcher and returns `gemm_oracle.Ref(value, coef, eps)`
with coef = 0: a kernel output x is correct when |x - value| <= eps.  These kernels run on the CUDA cores without
--use_fast_math, so + - * / and sqrtf round correctly (unit roundoff u = 2^-24), and expf, tanhf and erff are within
2 ulp (CUDA Math API), i.e. within 4u relative.  Each bound below is derived from the kernel's order of operations, to
first order in u, with gamma(n) = n u / (1 - n u) for a chain of n roundings (Higham, Accuracy and Stability, 3.1):

  * Sums.  A sum computed with at most n sequential roundings on the path of every term is within gamma(n) sum |t|.
    The warp LayerNorm (row_layernorm, H = 128 NV) adds each float4 as (x + y) + (z + w), then NV partials per lane,
    then 5 warp-shuffle levels: n = NV + 7.  The block LayerNorm of the sequence head has one element per thread,
    5 shuffle levels, then the 32 warp partials in order: n = 38.  The dense and classifier GEMVs chain four products
    per float4, NV float4s per lane, 5 shuffle levels and the bias: n = NV + 10.  The BERT pooler in P layout is one
    sequential sum per output: n = H + 2.  Pooling adds ceil(L / 64) rows per virtual warp, then 8 warps, then 8 parts:
    n = ceil(L / 64) + 14.  The L2 norm adds ceil(dim / 32) squares per lane and 5 shuffle levels: n = ceil(dim/32) + 6.
  * LayerNorm (two-pass).  The mean is off by e <= gamma(n + 2) mean|x| (the sum, then the scale by 1/H).  The kernel
    centres with its own mean, d = fl(x - mean'), and sum (x - mean')^2 = sum (x - mean)^2 + H e^2 because the exact
    centred values sum to zero: the mean error enters the variance only as e^2.  With the product, the two roundings of
    d, the scale, the + eps, V = var + eps carries a relative error rho_V <= (gamma(n + 6) (var + e^2 + eps) + e^2) / V,
    and rstd = 1 / sqrtf(V) a relative error rho_r <= rho_V / 2 + 2u.  Each output d rstd w (+ b) is then off by at
    most |w| rstd (e + u (|c| + e)) + |w| rstd |c| (rho_r + 2u) + u (|y| + |b| + |c rstd w|), c = x - mean.  An error
    dx already on the inputs adds |w| rstd (dx + mean dx) + |w| rstd |c| rho_in, rho_in = sum |c| (dx + mean dx) / (H V)
    (the first-order change of rstd).
  * GELU.  tanh form: z = k0 (x + k1 x^3) takes 7 roundings (both constants, the cube, the products, the add), tanhf
    4u, 1 + t one rounding, the last product one more; erf form: z = x k takes 2, erff 4u.  The bound is
    0.5 |x| (f'(z) dz + 4u |f(z)| + u |1 + f(z)|) + 2u |g|, plus |g'(x)| dx (+ dx^2 / 2, |g''| < 1) for an input error.
  * Softmax.  The max is exact.  e_j = expf(l_j - max) is within a_j = 4u + u |l_j - max| relative; the sum of
    ceil(C / 32) terms per lane and 5 shuffle levels is within gamma(ceil(C/32) + 5) + sum_j p_j a_j; the division adds
    u.  Logit errors dl move p_c by at most p_c (dl_c + sum_j p_j dl_j) (1 + max dl).  An expf result in the fp32
    subnormal range is off by at most 2^-148 absolute, covered by a 2^-140 floor.
  * L2 normalisation.  The squared norm is within gamma(ceil(dim/32) + 6), sqrtf and + norm_eps add u each, the
    division u: relative error gamma(ceil(dim/32) + 6) / 2 + 3u.
  * fp16 outputs add one fp16 ulp of the reference (gemm_oracle.ulp16): half an ulp of rounding, doubled for a value
    that the fp32 error carries across a binade.

Integer outputs (positions, classes, predictions) and the fp16 pair's low half are exact, and the cast is exact.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import torch

from oracle.encoder_oracle import argmax_first, argmax_last
from oracle.gemm_oracle import Ref, ulp16

U = 2.0 ** -24
K0 = math.sqrt(2.0 / math.pi)
K1 = 0.044715
TINY = 2.0 ** -140
KWARPS_POOL = 64                # 8 CTAs x 8 warps stride over the rows of one sequence


def gamma(n) -> float:
    return n * U / (1.0 - n * U)


def warp_ln_depth(h: int) -> int:
    return h // 128 + 7


BLOCK_LN_DEPTH = 38


def gemv_depth(h: int) -> int:
    return h // 128 + 10


def _ref(v: torch.Tensor, bound: torch.Tensor) -> Ref:
    return Ref(v, torch.zeros_like(v), bound)


# ---- LayerNorm -------------------------------------------------------------------------------------------------------
def layer_norm(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], eps: float, depth: int,
               dx: Optional[torch.Tensor] = None) -> Ref:
    """LayerNorm over the last dim of x (float64 exact inputs), fp32 output; `depth` = roundings of the kernel's sums;
    dx = error bound already on x (or None)."""
    x = x.double()
    h = x.shape[-1]
    w = w.double()
    b = b.double() if b is not None else torch.zeros_like(w)
    mu = x.mean(-1, keepdim=True)
    c = x - mu
    var = (c * c).mean(-1, keepdim=True)
    V = var + eps
    r = V.rsqrt()
    y = c * r * w + b
    e = gamma(depth + 2) * x.abs().mean(-1, keepdim=True)
    rho_v = (gamma(depth + 6) * (var + e * e + eps) + e * e) / V
    rho_r = rho_v / 2 + 2 * U
    aw = w.abs()
    err = aw * r * (e + U * (c.abs() + e)) + aw * r * c.abs() * (rho_r + 2 * U) + U * (y.abs() + b.abs() + (c * r * w).abs())
    if dx is not None:
        dc = dx + dx.mean(-1, keepdim=True)
        rho_in = (c.abs() * dc).sum(-1, keepdim=True) / (h * V)
        err = err + aw * r * dc + aw * r * c.abs() * rho_in
    return _ref(y, err)


def f16_out(ref: Ref) -> Ref:
    """The fp16 copy of an fp32 output."""
    return _ref(ref.value, ref.eps + ulp16(ref.value))


# ---- embeddings -------------------------------------------------------------------------------------------------------
def clamp_ids(ids: torch.Tensor, n: int) -> torch.Tensor:
    return ids.long().clamp(0, n - 1)


def embed_ln_modernbert(ids, table, w, eps) -> Ref:
    """x = LN_nobias(table[clamp(id)]): computed per table row, then gathered."""
    rows = layer_norm(table, w, None, eps, warp_ln_depth(table.shape[1]))
    i = clamp_ids(ids, table.shape[0]).to(table.device)
    return _ref(rows.value[i], rows.eps[i])


def embed_ln_bert(ids, pos, word, pos_emb, type0, w, b, eps, max_pos: int) -> Ref:
    """x = LN(word[clamp(id)] + type0 + pos_emb[min(p, max_pos - 1)]); the two fp32 adds are the input error."""
    i = clamp_ids(ids, word.shape[0]).to(word.device)
    p = pos.long().clamp(max=max_pos - 1).to(word.device)
    wt = word.double()[i] + type0.double()
    v = wt + pos_emb.double()[p]
    dx = U * (wt.abs() + v.abs())
    return layer_norm(v, w, b, eps, warp_ln_depth(word.shape[1]), dx)


def positions(cu: Sequence[int]) -> np.ndarray:
    return np.concatenate([np.arange(cu[i + 1] - cu[i], dtype=np.int32) for i in range(len(cu) - 1)] + [np.zeros(0, np.int32)])


# ---- pooling and L2 normalisation ----------------------------------------------------------------------------------
def pool_rows(x: torch.Tensor, cu: Sequence[int], mode: int, ln_w=None, ln_b=None, eps: float = 0.0,
              div_lens: Optional[Sequence[int]] = None) -> Ref:
    """pooled[b] = sum / n of the (LayerNorm'ed) rows of sequence b (mode 0, n = length or div_lens[b]); mode 1: the
    first row (zero for an empty sequence)."""
    hdim = x.shape[1]
    if ln_w is not None:
        rows = layer_norm(x, ln_w, ln_b, eps, warp_ln_depth(hdim))
        y, ey = rows.value, rows.eps
    else:
        y, ey = x.double(), torch.zeros(x.shape, dtype=torch.float64, device=x.device)
    out = torch.zeros(len(cu) - 1, hdim, dtype=torch.float64, device=x.device)
    err = torch.zeros_like(out)
    for s in range(len(cu) - 1):
        a, e = int(cu[s]), int(cu[s + 1])
        if mode == 1:
            if e > a:
                out[s], err[s] = y[a], ey[a]
            continue
        n = int(div_lens[s]) if div_lens is not None else e - a
        n = n if n > 0 else 1
        if e == a:
            continue
        ya = y[a:e]
        depth = -(-(e - a) // KWARPS_POOL) + 14
        out[s] = ya.sum(0) / n
        err[s] = (gamma(depth) * (ya.abs() + ey[a:e]).sum(0) + ey[a:e].sum(0)) / n + 2 * U * out[s].abs()
    return _ref(out, err)


def l2_normalize(pooled: torch.Tensor, dim: int, norm_eps: float) -> Ref:
    p = pooled.double()[:, :dim]
    v = p / (p.norm(dim=1, keepdim=True) + norm_eps)
    rel = gamma(-(-dim // 32) + 6) / 2 + 3 * U
    return _ref(v, rel * v.abs())


# ---- activations ------------------------------------------------------------------------------------------------------
def gelu(x: torch.Tensor, erf: bool, dx: Optional[torch.Tensor] = None) -> Ref:
    """fp32 gelu_erf_f / gelu_tanh_f of csrc/common.cuh on exact inputs x (+ input error dx)."""
    x = x.double()
    if erf:
        z = x / math.sqrt(2.0)
        f = torch.special.erf(z)
        dz = 2 * U * z.abs()
        fp = 2.0 / math.sqrt(math.pi) * torch.exp(-z * z)
        g = 0.5 * x * (1.0 + f)
        gp = 0.5 * (1.0 + f) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    else:
        z = K0 * (x + K1 * x ** 3)
        f = torch.tanh(z)
        dz = 7 * U * K0 * (x.abs() + K1 * x.abs() ** 3)
        fp = 1.0 - f * f
        g = 0.5 * x * (1.0 + f)
        gp = 0.5 * (1.0 + f) + 0.5 * x * fp * K0 * (1.0 + 3 * K1 * x * x)
    err = 0.5 * x.abs() * (fp * dz + 4 * U * f.abs() + U * (1.0 + f).abs()) + 2 * U * g.abs()
    if dx is not None:
        err = err + gp.abs() * dx + 0.5 * dx * dx
    return _ref(g, err)


def tanh(x: torch.Tensor, dx: torch.Tensor) -> Ref:
    t = torch.tanh(x.double())
    return _ref(t, (1.0 - t * t) * dx + 4 * U * t.abs())


# ---- GEMV and softmax --------------------------------------------------------------------------------------------------
def gemv(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], depth: int, dx: Optional[torch.Tensor] = None,
         transpose: bool = False) -> Ref:
    """y = x W^T + b (transpose: x W + b) with fp32 accumulation of `depth` roundings per term."""
    x, w = x.double(), w.double()
    wt = w if transpose else w.t()
    bb = b.double() if b is not None else torch.zeros(wt.shape[1], dtype=torch.float64, device=x.device)
    v = x @ wt + bb
    err = gamma(depth) * (x.abs() @ wt.abs() + bb.abs())
    if dx is not None:
        err = err + dx @ wt.abs()
    return _ref(v, err)


def softmax(logits: Ref) -> Ref:
    l, dl = logits.value, logits.eps
    C = l.shape[-1]
    m = l.max(-1, keepdim=True).values
    p = torch.softmax(l, -1)
    a = 4 * U + U * (l - m).abs()
    rho = a + gamma(-(-C // 32) + 5) + (p * a).sum(-1, keepdim=True) + U
    prop = (dl + (p * dl).sum(-1, keepdim=True)) * (1.0 + dl.max(-1, keepdim=True).values)
    return _ref(p, p * (rho + prop) + TINY)


# ---- heads -------------------------------------------------------------------------------------------------------------
def seq_head_hidden(pooled: torch.Tensor, dense_mode: int, dense_w=None, dense_b=None, norm_w=None, gelu_erf: bool = False,
                    head_eps: float = 1e-12) -> Ref:
    """The classifier input of seq_head: mode 0 the pooled row, 1 LN(gelu(x W^T)), 2 tanh(x P^T + b), 3 tanh(x P + b)."""
    h = pooled.shape[1]
    if dense_mode == 0:
        x = pooled.double()
        return _ref(x, torch.zeros_like(x))
    if dense_mode == 3:
        pre = gemv(pooled, dense_w, dense_b, h + 2, transpose=True)
    else:
        pre = gemv(pooled, dense_w, dense_b, gemv_depth(h))
    if dense_mode == 1:
        g = gelu(pre.value, gelu_erf, pre.eps)
        return layer_norm(g.value, norm_w, None, head_eps, BLOCK_LN_DEPTH, g.eps)
    return tanh(pre.value, pre.eps)


def seq_head(pooled, cls_w, cls_b, **kw):
    """-> (logits Ref, probs Ref) of seq_head."""
    hid = seq_head_hidden(pooled, **kw)
    logits = gemv(hid.value, cls_w, cls_b, gemv_depth(pooled.shape[1]), hid.eps)
    return logits, softmax(logits)


def token_head_hidden(h: int, hidden32=None, dense16=None, norm_w=None, pre_ln_w=None, pre_ln_eps: float = 0.0,
                      gelu_erf: bool = False, head_eps: float = 1e-12) -> Ref:
    if dense16 is not None:
        g = gelu(dense16.double(), gelu_erf)
        return layer_norm(g.value, norm_w, None, head_eps, warp_ln_depth(h), g.eps)
    if pre_ln_w is not None:
        return layer_norm(hidden32, pre_ln_w, None, pre_ln_eps, warp_ln_depth(h))
    x = hidden32.double()
    return _ref(x, torch.zeros_like(x))


def token_head(cls_w, cls_b, h: int, **kw):
    """-> (logits Ref, probs Ref) of token_head."""
    hid = token_head_hidden(h, **kw)
    logits = gemv(hid.value, cls_w, cls_b, gemv_depth(h), hid.eps)
    return logits, softmax(logits)


# ---- tie rules -------------------------------------------------------------------------------------------------------
def seq_class(probs: np.ndarray, argmax_last_: int) -> int:
    """seq_head's class from its probabilities: first max from 0.0 (classify_internal) or the last max (max_by)."""
    return argmax_last(probs) if argmax_last_ else argmax_first(probs)


def token_pred(logits: np.ndarray, argmax_last_: int) -> int:
    """token_head's prediction: argmax over the logits, the lowest index on ties, or the highest (argmax_last)."""
    return argmax_last(logits) if argmax_last_ else int(np.argmax(logits))
