"""Float64 references, bounds and float32 restatements of the precise path's BERT / MiniLM forms (csrc/precise.cu), next to
oracle/precise_oracle.py (TEST INFRASTRUCTURE ONLY).  Its notation, sources of error and emulation of fmaf / expf / erff
hold here; only what the BERT forms add is stated below.

  * Attention (attention_f32_kernel<D>) over heads of D = 64 or 32: qkv rows [T, 3 heads D], out rows [T, heads D].  The
    kernel scales q by c = fp32(D^-1/2): 0.125 exactly at D = 64; at D = 32 c is itself rounded (U / 2 relative) and so is
    q * c (U), so the score of key j carries the D-link fmaf chain plus 2 roundings, gamma(D + 2) a_j with
    a_j = D^-1/2 sum_d |q_d k_jd| (gamma(64) a_j at D = 64, as in precise_oracle).  Global attention with key lengths:
    keys j >= kv_lens[b] of sequence b are never visited (k_hi = min(len, kv_lens[b])); every row stays a query.  The
    other sources (exponent, sums, out) are precise_oracle's with nt the tiles of the visited keys.  At D = 64 without key
    lengths `attention` and `restate_attention` give bitwise precise_oracle's (tests/test_precise_bert_oracle.py).
  * GELU (gelu_f32_kernel): 0.5 a (1 + erff(a / sqrt 2)), GeGLU's arithmetic without b: 2U |a| + 3U |out|, absolute in
    |a| for the reason precise_oracle gives for GeGLU.
  * The forward (`bert_precise_restated`): encoder_oracle's BERT forward in float32 over projection weights replaced by
    their fp16 split pairs -- the BERT twin of hidden_oracle.modernbert_precise_restated, with the same things left out.
    Its rows are checked against hidden_oracle.row_bound(..., hidden_oracle.precise_u(cfg)); precise_u reads only
    hidden_size and intermediate_size, which a BertConfig has.

BERT_MUTATIONS are wrong kernels tests/test_precise_bert_oracle.py shows > 10x outside these bounds on some family."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle import attn_oracle as ao, encoder_oracle as eo, hidden_oracle as ho
from oracle.precise_oracle import (ATTN_SOURCES, INV_SQRT2_F32, ROWS, SUBN, TILE, U, AttnRef, RowRef, _expf, _fma, _tiles,
                                   constant_columns, f32, f64, gamma)

# 64^-1/2 at D = 32, the key mask ignored, one key past the key length visible, tanh GELU
BERT_MUTATIONS = ("scale_64_at_32", "kv_ignored", "kv_plus_one", "gelu_tanh")


def scale_of(head_dim: int) -> float:
    """the kernel's score scale: fp32(head_dim^-1/2), 0.125 exactly at 64"""
    return float(f32(head_dim ** -0.5))


# ---- GELU ----------------------------------------------------------------------------------------------------------
def gelu(x: torch.Tensor) -> RowRef:
    """gelu_erf(x) over fp32 values; the bound is GeGLU's with b = 1, absolute in |x|"""
    a = x.double()
    v = 0.5 * a * (1.0 + torch.special.erf(a / math.sqrt(2.0)))
    return RowRef(v, 2 * U * a.abs() + 3 * U * v.abs() + 2.0 ** -140)


def restate_gelu(x: np.ndarray, mut: Optional[str] = None) -> np.ndarray:
    """gelu_f32_kernel in float32: 0.5f * a * (1 + erff(a * 0.70710678f)); gelu_tanh: the tanh approximation"""
    a = np.asarray(x, dtype=f32)
    if mut == "gelu_tanh":
        a64 = a.astype(f64)
        t = np.tanh(math.sqrt(2.0 / math.pi) * (a64 + 0.044715 * a64 ** 3)).astype(f32)
        return (f32(0.5) * a) * (f32(1.0) + t)
    erf = torch.special.erf(torch.from_numpy((a * INV_SQRT2_F32).astype(f64))).numpy().astype(f32)
    return (f32(0.5) * a) * (f32(1.0) + erf)


# ---- attention -----------------------------------------------------------------------------------------------------
def key_range(len_: int, window: int, q0: int, klen: int):
    """[k_lo, k_hi) of the CTA whose first query row is q0; global attention visits keys < klen"""
    if window <= 0:
        return 0, min(klen, len_)
    return max(q0 - window, 0), min(q0 + ROWS + window, len_)


def _rows_chunk(heads: int, keys: int, head_dim: int) -> int:
    r = 1024
    while r > 1 and r * keys * heads * head_dim > (1 << 27):
        r //= 2
    return r


def _seq(q, k, v, rows, len_, window, klen):
    """one sequence, every head: q, k, v [nH, len, D] float64 -> value, terms [nH, R, D]; global: keys j < klen"""
    D = q.shape[-1]
    sc, chain = 1.0 / math.sqrt(D), (64 if D == 64 else D + 2)
    r0, r1 = int(rows.min()), int(rows.max())
    keys = min(klen, len_)
    j0, j1 = (max(0, r0 - window), min(len_, r1 + window + 1)) if window > 0 else (0, keys)
    kk, vv, qq = k[:, j0:j1], v[:, j0:j1], q[:, rows]
    s = sc * (qq @ kk.transpose(1, 2))
    a = sc * (qq.abs() @ kk.abs().transpose(1, 2))
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
    nt = _tiles(keys if window <= 0 else len_, window, rows).double()[None, :, None]     # [1, R, 1]
    zero = torch.zeros_like(s)
    xs = torch.where(vis, gamma(chain) * a, zero)
    rho = torch.where(vis, U * (m - s) + 4 * U * (nt + 1), zero)
    F = torch.exp(2 * (xs + rho).amax(-1, keepdim=True))
    d = (vv[:, None, :, :] - out[:, :, None, :]).abs()                                  # [nH, R, Kk, D]
    score = F * torch.einsum("hrk,hrkd->hrd", p * xs, d)
    expo = F * torch.einsum("hrk,hrkd->hrd", p * rho, d)
    del d
    av = vv.abs()
    n_vis = vis.sum(-1, keepdim=True).double()
    sums = F * gamma(32 + nt) * (p @ av + out.abs())
    outt = gamma(2) * out.abs() + (32 + nt) * n_vis * SUBN * (1 + av.amax(1, keepdim=True))
    return out, {"score": score, "exponent": expo, "sums": sums, "out": outt}


def attention(qkv: torch.Tensor, cu: Sequence[int], heads: int, window: int = 0, sel: Optional[torch.Tensor] = None,
              head_dim: int = 64, kv_lens: Optional[Sequence[int]] = None) -> AttnRef:
    """reference of precise_attention for fp32 qkv [>= T, 3 heads D] (D = head_dim) packed by `cu`, on output rows `sel`
    (global indices, ascending; default all); global attention sees keys j < kv_lens[b] of sequence b (default all)"""
    assert kv_lens is None or window <= 0
    dev, D = qkv.device, head_dim
    H = heads * D
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
        klen = len_ if kv_lens is None else int(kv_lens[b])
        x = qkv[s0:s1].double().view(len_, 3, heads, D).permute(1, 2, 0, 3)
        rows_all = sel[idx] - s0
        keys = len_ if window <= 0 else min(len_, 2 * window + 1 + 1024)
        step = _rows_chunk(heads, keys, D)
        for c0 in range(0, idx.numel(), step):
            ii, rows = idx[c0:c0 + step], rows_all[c0:c0 + step]
            o, tm = _seq(x[0], x[1], x[2], rows, len_, window, klen)
            val[ii] = o.permute(1, 0, 2).reshape(-1, H)
            for kname, t in tm.items():
                terms[kname][ii] = t.permute(1, 0, 2).reshape(-1, H)
    return AttnRef(val, sum(terms.values()), terms)


def restate_attention(qkv: np.ndarray, cu: Sequence[int], heads: int, window: int = 0, sel: Optional[np.ndarray] = None,
                      head_dim: int = 64, kv_lens: Optional[Sequence[int]] = None, mut: Optional[str] = None) -> np.ndarray:
    """attention_f32_kernel<D> in float32 (per-tile sums) on output rows `sel` -> [len(sel), heads D].  mut:
    scale_64_at_32 (0.125 whatever D), kv_ignored (every key visible), kv_plus_one (one key past kv_lens visible)."""
    qkv = np.asarray(qkv, dtype=f32)
    D = head_dim
    H = heads * D
    T = int(cu[-1])
    sel = np.arange(T) if sel is None else np.asarray(sel)
    out = np.zeros((len(sel), H), dtype=f32)
    scale = f32(0.125) if mut == "scale_64_at_32" else f32(scale_of(D))
    cu_a = np.asarray(cu)
    seq_of = np.searchsorted(cu_a, sel, side="right") - 1
    for b in np.unique(seq_of):
        s0, len_ = int(cu[b]), int(cu[b + 1]) - int(cu[b])
        x = qkv[s0:s0 + len_].reshape(len_, 3, heads, D)
        klen = len_
        if kv_lens is not None and mut != "kv_ignored":
            klen = min(len_, int(kv_lens[b]) + (1 if mut == "kv_plus_one" else 0))
        idx_b = np.nonzero(seq_of == b)[0]
        rows_b = sel[idx_b] - s0
        for q0 in np.unique((rows_b // ROWS) * ROWS):
            ii = idx_b[(rows_b // ROWS) * ROWS == q0]
            rows = sel[ii] - s0
            k_lo, k_hi = key_range(len_, window, int(q0), klen)
            for h in range(heads):
                q = x[rows, 0, h] * scale                                   # [R, D]
                R = len(rows)
                m = np.full(R, -np.inf, dtype=f32)
                l = np.zeros(R, dtype=f32)
                o = np.zeros((R, D), dtype=f32)
                for k0 in range(k_lo, k_hi, TILE):
                    kj = np.arange(k0, k0 + TILE)
                    ok = kj < klen
                    kt = np.where(ok[:, None], x[np.minimum(kj, len_ - 1), 1, h], f32(0))
                    vt = np.where(ok[:, None], x[np.minimum(kj, len_ - 1), 2, h], f32(0))
                    acc = np.zeros((R, TILE), dtype=f32)
                    for d in range(D):
                        acc = _fma(q[:, d:d + 1], kt[None, :, d], acc)
                    vis = ok[None, :] & np.ones((R, 1), dtype=bool)
                    if window > 0:
                        vis = vis & (np.abs(kj[None, :] - rows[:, None]) <= window)
                    s = np.where(vis, acc, f32(-np.inf))
                    tm = s.max(1)
                    live = tm != -np.inf
                    mn = np.maximum(m, tm)
                    with np.errstate(invalid="ignore"):
                        alpha = np.where(m == -np.inf, f32(0), _expf(m - mn))
                        p = np.where(s == -np.inf, f32(0), _expf(s - mn[:, None]))
                    lt = np.zeros(R, dtype=f32)
                    for j in range(TILE):
                        lt = lt + p[:, j]
                    a2 = np.zeros((R, D), dtype=f32)
                    for j in range(TILE):
                        a2 = _fma(p[:, j:j + 1], vt[None, j], a2)
                    l = np.where(live, _fma(l, alpha, lt), l)
                    o = np.where(live[:, None], _fma(o, alpha[:, None], a2), o)
                    m = np.where(live, mn, m)
                with np.errstate(divide="ignore", invalid="ignore"):
                    out[ii, h * D:(h + 1) * D] = o * (f32(1.0) / l)[:, None]
    return out


def make_qkv(family: str, cu: Sequence[int], heads: int, window: int = 0, seed: int = 0, device="cpu", head_dim: int = 64,
             kv_lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """fp32 qkv [cu[-1], 3 heads D] of one family of precise_oracle.FAMILIES: at D = 32 the first 32 of each head's 64
    dimensions of attn_oracle's families ("random": full fp32 mantissas; "constant": q = 0 and constant_columns()[:D] as
    every V row); needles aim at kv_lens when given"""
    T, D = int(cu[-1]), head_dim
    if family == "random":
        g = torch.Generator(device=device).manual_seed(seed)
        return torch.randn(T, 3 * heads * D, generator=g, device=device, dtype=torch.float32)
    x = ao.make_qkv("random" if family == "constant" else family, cu, heads, window, kv_lens=kv_lens, seed=seed,
                    device=device).float().view(T, 3, heads, 64)[..., :D].clone()
    if family == "constant":
        x[:, 0] = 0.0
        x[:, 2] = constant_columns()[:D].to(device)
    return x.reshape(T, 3 * heads * D).contiguous()


# ---- the forward ---------------------------------------------------------------------------------------------------
def bert_precise_restated(weights: Dict[str, np.ndarray], cfg: eo.BertConfig, ids, real_len: Optional[int] = None,
                          prefix: str = "bert") -> List[torch.Tensor]:
    """encoder_forward_precise's BERT branch on one sequence: [S, H] rows after every layer of encoder_oracle's BERT
    forward in float32 (fp32 biases, post-LN LayerNorm, erf GELU, softmax over the model's own heads with keys >= real_len
    masked) over projection weights replaced by their fp16 split pairs (hidden_oracle.split16)"""
    w32 = {}
    for k, v in weights.items():
        t = torch.from_numpy(np.ascontiguousarray(v))
        is_proj = ".encoder.layer." in "." + k and k.endswith(".weight") and not k.endswith("LayerNorm.weight")
        w32[k] = ho.split16(t).float() if is_proj else t
    t = torch.as_tensor(np.asarray(ids, dtype=np.int64))[None]
    mask = torch.ones_like(t)
    if real_len is not None:
        mask[0, real_len:] = 0
    out: List[torch.Tensor] = []
    eo.bert_forward(w32, cfg, t, mask, prefix=prefix, collect=out)
    return [x[0] for x in out]
