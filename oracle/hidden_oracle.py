"""Per-token hidden rows of the whole encoder against float64 (TEST INFRASTRUCTURE ONLY; see encoder_oracle.py header).

Five things, used by tests/test_hidden_oracle.py (CPU), tests/test_encoder_hidden_conformance_gpu.py and
tests/test_encoder_long_context_gpu.py (GPU):

  * `trained_like_modernbert_weights`: a second synthetic family next to synth.make_modernbert_weights with the statistics
    of trained ModernBERT / mmBERT checkpoints that the LayerNorm fold and the fp16 pair exist for: LayerNorm gains
    log-uniform over [0.05, 8], a few outlier residual channels 34 - 58x the median entry, row means far from zero.
  * `modernbert_hidden64` / `bert_hidden64`: the residual stream after every layer from encoder_oracle's forward, run on
    float64 copies of the fp32 checkpoint values.
  * `modernbert_hidden64_long`: the same forward for sequences up to 32 768 tokens and batches of 131 072 rows.  It takes
    [B, S] ids, runs attention a chunk of queries at a time over only the keys they see (`chunked_attention`: all keys on a
    global layer, the band |i - j| <= local_attention / 2 on a local one), so no [S, S] tensor exists, and keeps float64
    rows only at the depths asked for, with the running sum_j s_j that row_bound needs (`Hidden64`).  Its memory is
    bounded by B and the query chunk (its docstring).
  * `row_bound`: the per-row error bound, stated once, for the production path (fp16 operands) and the precise path
    (fp32 accumulation on the tensor cores).
  * `modernbert_restated` / `bert_restated`: the float64 forward with operands rounded to fp16 exactly where
    csrc/engine.cu's encoder_forward rounds them (the activations entering each GEMM, the stored weights including
    W diag(gamma) of the LayerNorm fold, q / k / v, P, ctx, the GeGLU output, the residual stream as the (hi, lo) pair
    around the pivot with its row statistics in 128-column blocks).  It is the CPU evidence for the bound, and with a
    `mut` it is a wrong engine the bound must reject.

THE BOUND.  A row x_l of the residual stream after layer l (BERT: of the hidden states) is correct when every element is
within

    row_bound = GAIN * u * sum_{j <= l} s_j,     s_j = RMS of the centred row after layer j (float64),

u the unit roundoff of the operands: U16 = 2^-11 on the production path, precise_u(cfg) on the precise path (below).
Derivation, to first order.  A layer adds two updates to the row, each a GEMM over rounded operands.  Between one residual
value and the next the production path rounds twelve times: the raw row entering Wqkv, Wqkv itself, q, k, v, P, ctx, Wo;
then the raw row entering Wi, Wi, the GeGLU output, Wo2.  One rounding moves each term of the update it feeds by at most
u relative, so it moves the update by at most u times the update's own size; an update is no larger than the row it
produces, whose scale is s_j (the scale the next LayerNorm divides by -- an error is worth what it is against THAT, which
is why the centred RMS and not the RMS is used: a common offset is invisible to every consumer).  Twelve roundings in the
worst case add: 12 per layer.  An error made at layer j is carried to layer l by the identity path of the residual
stream unchanged, and through the later layers' LayerNorms in proportion to the row scale: the sum over j.  The fp16 pair
adds 2^-22 per update and the fp32 accumulation 2^-20 (gemm_oracle.TAU); both vanish next to 12 * 2^-11.
What this leaves out is the worst case over ELEMENTS: an element's error is bounded by 12 u s_j only as far as no
element of the update is larger than the row's scale, and a layer that reads the raw embedding rows (layer 0 has no
attn_norm) sees their outlier channels unnormalised.  The restatement below measures what that costs: its largest error
is 0.73 of 12 u sum s_j (H 1024, trained-like family, depth 1; <= 0.14 on the plain family).  GAIN = 24 doubles the count
to cover it with the margin of 2 a bound should keep; nothing else in it is fitted.  So the bound is justified by the
restatement and not by the derivation alone: tests/test_hidden_oracle.py shows that on every family and geometry the restated engine
stays inside it with a margin >= 2 and by how much each wrong engine of MUTATIONS leaves it (> 10x, but for one
dropped statistics block at the geometries where a block is a third or a sixth of the row: 5.7x - 9x).

LONG CONTEXT.  The count above does not depend on the number of keys n: a softmax row is a weighted mean of v, and
rounding each normal weight of P to fp16 moves it by at most 2^-11 of the weighted mean of |v|, whatever n.  Two terms do
grow with n.  Weights below 2^-14 are fp16 subnormals, rounded with an absolute 2^-25 against a denominator >= 1: n 2^-25
in the worst case (2^-10 at 32 768 keys), but the roundings take either sign and add as sqrt(n) 2^-25, 2^-17.5 at 32 768.
The fp32 denominator summed over n / 64 key blocks adds (n / 64) 2^-24 at worst, 2^-15 at 32 768.  Both stay below the
2^-11 of one rounding.  The restatement, with the same chunked attention as the long form, shows it at 4096 tokens
(global layers over all 4096 keys, windows at positions up to 4095): at most 0.31 of the bound on the plain,
trained-like and wide families at H 768 and 384, as at 300 tokens.  A rope row read at fp16(position) or at
position % 2048 leaves the bound by > 70x on the rows past 2048 (wide family, H 768).  Measured on an H100 80GB HBM3 at
700 W, the engine's rows at 2049, 8192 and 32 768 tokens and in the 131 072-row batch reach at most 0.47 of the bound on
the production path and 0.39 on the precise one.  The precise path's attention used to sum all keys of a global row in
one fp32 chain; on the trained-like family its worst row went from 0.14 of the bound at 8192 tokens to 0.37 at 32 768,
the longest position table of the mmBERT checkpoints.  That chain was the cause.  Its rounding grows linearly in n where
the terms are correlated: on constant V columns under uniform scores at 32 768 keys the chained kernel was 4.9e-4
relative off (3.9x the bound of oracle/precise_oracle.py for per-tile sums, 2.4x at 8192 keys; the same numbers as the
float32 restatement), the kernel that sums each 32-key tile first and then adds it to the running sums 1.0e-5 (0.08 of
that bound).  With per-tile sums the trained-like rows are at 0.15 of the bound at 8192 tokens and 0.16 at 32 768 (plain
family 0.045 at both; H100 80GB HBM3, 700 W).

The precise path (csrc/precise.cu) splits every GEMM operand into an fp16 pair and accumulates in fp32 on the tensor
cores; everything between the GEMMs is fp32.  Its u is precise_u(cfg) = TAU_MEASURED * 0.64 sqrt(K), K = max(H, I) the
longest dot product of the model, with the same GAIN (the same places, now each a GEMM):
  * The accumulation error of the tensor cores is proportional to S = sum |a w|, not to the result: gemm_oracle measured
    up to TAU_MEASURED = 4.47e-7 = 2^-21.09 of S over the GEMMs of tests/test_gemm_conformance_gpu.py at K <= 1160
    (the bound there, TAU = 2^-20, is 2.1x that; 7.0e-7 at K = 3072 / 4096, below the sqrt(K) growth assumed here).  For operands of random sign S = (2 / pi) K |a| |w| against a result of sqrt(K) |a| |w|:
    S is 0.64 sqrt(K) results, 18 at K = 768 and 41 at K = 4096.  So u = 2^-16.9 ... 2^-15.7 here, 50 - 100x the fp32
    unit roundoff: the precise path is fp32-ACCUMULATED, not fp32-accurate, per row.
  * The split itself is smaller.  A weight of size 2^-7 (N(0, 0.02^2)) has a high half with ulp 2^-17, so its low half
    is an fp16 subnormal (spacing 2^-24) and the pair is within 2^-25 absolute, 2^-18 relative, not 2^-22.
    `modernbert_precise_restated` (float32 arithmetic over split-pair weights, all a CPU can restate) reaches 0.002 -
    0.03 of the bound; a CPU has no tensor-core adder, so the evidence for the accumulation term is the GEMM
    conformance measurement above and the H100 rows themselves: measured on an H100 80GB HBM3 at 700 W the worst row is
    0.2 - 0.45 of this bound at every geometry from K = 384 to K = 4096, which a u independent of K does not give (under
    a fixed 2^-17 the same rows span 0.2 - 1.06).
"""
from __future__ import annotations

import math
from dataclasses import replace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import encoder_oracle as eo
from .synth import STD, make_modernbert_weights

U16 = 2.0 ** -11
TAU_MEASURED = 4.47e-7          # largest |accumulation error| / sum |a w| of the wgmma GEMMs (gemm_oracle's docstring)
GAIN = 24.0
FP16_SAFE = 3e4                 # trained-like family: |q|, |k|, |v|, |ctx|, |GeGLU| stay below this in float64
OUTLIER_CHANNELS = 4
OUTLIER_ROW_SCALE = 4.0
COMMON_SIGMA = 3.0
Q_CHUNK = 256                   # query rows per attention chunk of the float64 forwards (chunked_attention)


# --------------------------------------------------------------------------------------
# the trained-like family
# --------------------------------------------------------------------------------------
def trained_like_modernbert_weights(cfg: eo.ModernBertConfig, num_classes: int = 0, seed: int = 1234,
                                    layer0_attn_norm: bool = False, drop_attn_norm: Sequence[int] = ()) -> Dict[str, np.ndarray]:
    """make_modernbert_weights with the statistics of a trained checkpoint (seeded, deterministic):
      * every LayerNorm gain log-uniform over [0.05, 8], Wqkv and Wi divided by the RMS of the gain before them;
      * OUTLIER_CHANNELS channels c: the embedding column is a signed constant (+-10 sigma) plus noise and its embedding
        gain is 4, so the stream starts with entries ~50x the typical one there; rows c of every Wo / mlp.Wo are x 4,
        so the updates keep feeding them;
      * every Wo / mlp.Wo gets a rank-one term 1 v^T (|v| ~ 3 sigma): each update moves all channels of a row together,
        so row means random-walk away from zero to several times a typical channel's spread.
    Everything else is N(0, 0.02^2) as in the plain family."""
    w = make_modernbert_weights(cfg, num_classes, seed=seed, with_head=False)
    rng = np.random.default_rng(seed + 7919)
    H = cfg.hidden_size
    chans = rng.choice(H, OUTLIER_CHANNELS, replace=False)
    for k in list(w):
        if k.endswith("norm.weight"):
            w[k] = np.exp(rng.uniform(math.log(0.05), math.log(8.0), H)).astype(np.float32)
    emb = w["model.embeddings.tok_embeddings.weight"]
    for c in chans:
        emb[:, c] = np.float32(STD) * (np.float32(rng.choice([-10.0, 10.0])) + rng.standard_normal(emb.shape[0], dtype=np.float32))
        w["model.embeddings.norm.weight"][c] = 4.0
    for li in range(cfg.num_hidden_layers):
        for name, norm in (("attn.Wqkv", "attn_norm"), ("mlp.Wi", "mlp_norm")):   # pre-activations stay O(1), as training leaves them
            g = w.get(f"model.layers.{li}.{norm}.weight")
            if g is not None:
                w[f"model.layers.{li}.{name}.weight"] /= np.sqrt(np.mean(g.astype(np.float64) ** 2)).astype(np.float32)
        for name in ("attn.Wo", "mlp.Wo"):
            m = w[f"model.layers.{li}.{name}.weight"]
            m[chans, :] *= np.float32(OUTLIER_ROW_SCALE)
            m += (rng.standard_normal(m.shape[1], dtype=np.float32) * np.float32(COMMON_SIGMA * STD))[None, :]
    set_attn_norm_layout(w, cfg, rng, layer0_attn_norm, drop_attn_norm)
    return w


def set_attn_norm_layout(w: Dict[str, np.ndarray], cfg: eo.ModernBertConfig, rng, layer0: bool, drop: Sequence[int]):
    """Give layer 0 an attn_norm (gains as the layer-1 ones, reshuffled) and / or take it from later layers."""
    if layer0:
        w["model.layers.0.attn_norm.weight"] = rng.permutation(w["model.layers.1.attn_norm.weight"]).astype(np.float32)
    for li in drop:
        del w[f"model.layers.{li}.attn_norm.weight"]


# --------------------------------------------------------------------------------------
# float64 hidden rows and the bound
# --------------------------------------------------------------------------------------
def to64(weights: Dict[str, np.ndarray], device="cpu") -> Dict[str, torch.Tensor]:
    """float64 copies of the fp32 checkpoint values"""
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device=device, dtype=torch.float64) for k, v in weights.items()}


def _ids(ids, device):
    return torch.as_tensor(np.asarray(ids, dtype=np.int64), device=device)[None]


def modernbert_hidden64(w64: Dict[str, torch.Tensor], cfg: eo.ModernBertConfig, ids, num_layers: int) -> List[torch.Tensor]:
    """[S, H] float64 residual rows of one sequence after each of the first `num_layers` layers"""
    dev = next(iter(w64.values())).device
    t = _ids(ids, dev)
    out: List[torch.Tensor] = []
    eo.modernbert_forward(w64, cfg, t, torch.ones_like(t), num_layers, collect=out)
    return [x[0] for x in out]


def bert_hidden64(w64: Dict[str, torch.Tensor], cfg: eo.BertConfig, ids, real_len: Optional[int] = None,
                  prefix: str = "bert") -> List[torch.Tensor]:
    """[S, H] float64 hidden rows of one sequence after every layer; positions >= real_len are masked as keys only"""
    dev = next(iter(w64.values())).device
    t = _ids(ids, dev)
    mask = torch.ones_like(t)
    if real_len is not None:
        mask[0, real_len:] = 0
    out: List[torch.Tensor] = []
    eo.bert_forward(w64, cfg, t, mask, prefix=prefix, collect=out)
    return [x[0] for x in out]


class Hidden64:
    """One sequence's float64 rows at some depths (1-based) and, per depth d, the [S] sum_{j <= d} s_j of row_bound"""

    def __init__(self, rows: Dict[int, torch.Tensor], scale_sums: Dict[int, torch.Tensor]):
        self.rows, self.scale_sums = rows, scale_sums


def modernbert_hidden64_long(w64: Dict[str, torch.Tensor], cfg: eo.ModernBertConfig, ids, depths: Sequence[int],
                             q_chunk: int = Q_CHUNK) -> List[Hidden64]:
    """encoder_oracle.modernbert_forward on B sequences of S tokens each (ids [B, S]; unmasked), on the device of w64:
    the float64 rows after each layer in `depths` and their row_bound scale sums, one Hidden64 per sequence.  Attention
    runs per chunk of q_chunk queries over the keys the chunk sees (chunked_attention).  Peak memory is about
    8 B S (7 H + 4 I) bytes for the activations plus 24 B heads q_chunk K bytes for one chunk's scores (K = S on a global
    layer, q_chunk + local_attention on a local one), beside the rows kept: the caller bounds it with B and q_chunk."""
    W = lambda name: eo._w(w64, name, eo.MODERNBERT_PREFIXES)
    dev = next(iter(w64.values())).device
    t = torch.as_tensor(np.asarray(ids, dtype=np.int64), device=dev)
    t = t[None] if t.dim() == 1 else t
    B, S = t.shape
    H, heads, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps
    depths = sorted(set(depths))
    tables = {local: tuple(c.to(dev).double()[None, :, None, :] for c in eo.rope_tables(64, theta, S))
              for local, theta in ((False, cfg.global_rope_theta), (True, cfg.local_rope_theta))}

    def rope(x, cos, sin):
        x = x.reshape(B, S, heads, 64)
        x1, x2 = x[..., :32], x[..., 32:]
        return torch.cat([x1 * cos - x2 * sin, x1 * sin + x2 * cos], -1).reshape(B, S, H)

    x = eo.layer_norm(W("embeddings.tok_embeddings.weight")[t], W("embeddings.norm.weight"), None, eps)
    scale_sum = torch.zeros(B, S, dtype=torch.float64, device=dev)
    rows, sums = {}, {}
    for li in range(depths[-1]):
        local = (li % cfg.global_attn_every_n_layers) != 0
        g_an = W(f"layers.{li}.attn_norm.weight")
        h = x if g_an is None else eo.layer_norm(x, g_an, None, eps)
        qkv = h @ W(f"layers.{li}.attn.Wqkv.weight").t()
        cos, sin = tables[local]
        q, k, v = rope(qkv[..., :H], cos, sin), rope(qkv[..., H:2 * H], cos, sin), qkv[..., 2 * H:]
        del qkv, h
        ctx = chunked_attention(q, k, v, heads, cfg.local_attention // 2 if local else 0, q_chunk=q_chunk)
        del q, k, v
        x = ctx @ W(f"layers.{li}.attn.Wo.weight").t() + x
        del ctx
        a, b = (eo.layer_norm(x, W(f"layers.{li}.mlp_norm.weight"), None, eps) @ W(f"layers.{li}.mlp.Wi.weight").t()).chunk(2, dim=-1)
        x = x + (eo.gelu_erf(a) * b) @ W(f"layers.{li}.mlp.Wo.weight").t()
        del a, b
        scale_sum = scale_sum + centred_rms(x)
        if li + 1 in depths:
            rows[li + 1], sums[li + 1] = x, scale_sum
    return [Hidden64({d: rows[d][i] for d in depths}, {d: sums[d][i] for d in depths}) for i in range(B)]


def precise_u(cfg) -> float:
    """u of the precise path for a ModernBertConfig (module docstring)"""
    return TAU_MEASURED * 0.64 * math.sqrt(max(cfg.hidden_size, cfg.intermediate_size))


def centred_rms(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return (x - x.mean(-1, keepdim=True)).pow(2).mean(-1).sqrt()


def row_bound(hidden64, depth: int, u: float = U16) -> torch.Tensor:
    """Bound [S] on every element of the rows after layer `depth` (1-based), given the float64 rows after layers 1 ...
    depth or a Hidden64 holding that depth (module docstring)."""
    if isinstance(hidden64, Hidden64):
        return GAIN * u * hidden64.scale_sums[depth]
    s = sum(centred_rms(hidden64[j]) for j in range(depth))
    return GAIN * u * s


def worst_over_bound(got, hidden64, depth: int, u: float = U16, rows=slice(None)) -> float:
    """max over `rows` of (largest element error) / bound; inf when `got` holds a NaN or inf.  hidden64: the float64 rows
    after layers 1 ... depth, or a Hidden64 holding that depth."""
    ref = hidden64.rows[depth] if isinstance(hidden64, Hidden64) else hidden64[depth - 1]
    got = torch.as_tensor(got).to(ref.device).double()
    if not bool(torch.isfinite(got).all()):
        return math.inf
    err = (got - ref).abs().amax(-1)
    return float((err / row_bound(hidden64, depth, u))[rows].max())


# --------------------------------------------------------------------------------------
# the engine restated in float64 with fp16 operands
# --------------------------------------------------------------------------------------
MUTATIONS = ("global_every", "rope_tables", "window", "geglu_halves", "fold_gamma", "stale_pivot", "stats_block", "stale_rows")
# wrong engines that differ only at positions past 2048, config-wide: the rope row read at fp16(position), or at position % 2048
FAR_POSITION_MUTATIONS = ("rope_pos_fp16", "rope_wrap_2048")


def r16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16).to(torch.float64)


def _fold(w: torch.Tensor, gamma: torch.Tensor) -> torch.Tensor:
    """engine.cu fold_weights: W diag(gamma), rows re-centred until the ROUNDED row sums to zero, fp16"""
    row = w * gamma[None, :]
    row = row - row.mean(1, keepdim=True)
    for _ in range(3):
        row = row - r16(row).sum(1, keepdim=True) / row.shape[1]
    return r16(row)


def chunked_attention(q, k, v, heads: int, window: int, kv_len: Optional[int] = None, q_chunk: int = Q_CHUNK,
                      p16: bool = False) -> torch.Tensor:
    """softmax(0.125 q k^T) v on rows [B, S, heads * 64], a chunk of q_chunk query rows at a time over only the keys that
    chunk can see: all of them (j < kv_len), or |i - j| <= window when window > 0.  No [S, S] tensor is built: one chunk's
    scores are B * heads * q_chunk * K values, K = min(S, kv_len) or q_chunk + 2 window.  p16: P is rounded to fp16 for
    P V while the denominator sums the unrounded weights, as attention_wgmma does."""
    B, S, W = q.shape
    sp = lambda t: t.reshape(B, S, heads, -1).transpose(1, 2)          # [B, heads, S, 64]
    qh, kh, vh = sp(q), sp(k), sp(v)
    keys = S if kv_len is None else min(S, kv_len)
    out = torch.empty_like(qh)
    for c0 in range(0, S, q_chunk):
        c1 = min(S, c0 + q_chunk)
        k0, k1 = (max(0, c0 - window), min(keys, c1 + window)) if window > 0 else (0, keys)
        s = 0.125 * (qh[:, :, c0:c1] @ kh[:, :, k0:k1].transpose(-1, -2))
        if window > 0:
            i = torch.arange(c0, c1, device=q.device)
            j = torch.arange(k0, k1, device=q.device)
            s = s.masked_fill((j[None, :] - i[:, None]).abs() > window, -math.inf)
        p = torch.exp(s - s.amax(-1, keepdim=True))
        out[:, :, c0:c1] = ((r16(p) if p16 else p) @ vh[:, :, k0:k1]) / p.sum(-1, keepdim=True)
    return out.transpose(1, 2).reshape(B, S, W)


def _attention(q, k, v, heads: int, window: int, kv_len: Optional[int] = None) -> torch.Tensor:
    """attention_wgmma on fp16 q / k / v rows [S, heads * 64]: fp32 scores * 0.125, P rounded to fp16 for P V while the
    denominator sums the unrounded weights, fp16 context"""
    return r16(chunked_attention(q[None], k[None], v[None], heads, window, kv_len, p16=True)[0])


class _Pair:
    """The residual stream of gemm.h EPI_RESID_HL: x - pivot = hi + lo, statistics of x - pivot per 128-column block"""

    def __init__(self, x0: torch.Tensor):
        self.hi = r16(x0)
        self.lo = r16(x0 - self.hi)
        self.pivot = torch.zeros(x0.shape[0], 1, dtype=torch.float64, device=x0.device)
        self.prev_pivot = self.pivot
        self.s1 = self.s2 = None        # [S, H / 128]

    def x(self):
        return self.pivot + self.hi + self.lo

    def update(self, acc: torch.Tensor, stale_pivot: bool = False):
        S, H = acc.shape
        pv = torch.zeros_like(self.pivot) if self.s1 is None else self.s1.sum(1, keepdim=True) / H
        xn = (self.hi + self.lo) + (acc - pv)
        blocks = xn.reshape(S, H // 128, 128)
        self.s1, self.s2 = blocks.sum(-1), blocks.pow(2).sum(-1)
        base = self.prev_pivot if stale_pivot else self.pivot
        self.prev_pivot = self.pivot
        self.pivot = base + pv
        self.hi = r16(xn)
        self.lo = r16(xn - self.hi)

    def rstd(self, eps: float, drop=None):
        """the consumer's rstd; drop = (row, block): that block's partial is left out of that row's sums (block < 0: the
        block with the row's largest sum of squares, where an outlier channel sits)"""
        s1, s2 = self.s1, self.s2
        if drop is not None:
            keep = torch.ones_like(s1)
            keep[drop[0], drop[1] if drop[1] >= 0 else int(s2[drop[0]].argmax())] = 0.0
            s1, s2 = s1 * keep, s2 * keep
        H = 128 * s1.shape[1]
        mean = s1.sum(1, keepdim=True) / H
        var = (s2.sum(1, keepdim=True) / H - mean * mean).clamp_min(0.0)
        return 1.0 / torch.sqrt(var + eps)

    def state(self):
        return (self.hi, self.lo, self.pivot, self.prev_pivot, self.s1, self.s2)

    def keep_rows(self, old, r0: int):
        """rows >= r0 go back to the state `old`"""
        new = []
        for n, o in zip(self.state(), old):
            if o is None:               # no statistics before the first update: those rows read zeros
                o = torch.zeros_like(n)
            n = n.clone()
            n[r0:] = o[r0:]
            new.append(n)
        self.hi, self.lo, self.pivot, self.prev_pivot, self.s1, self.s2 = new


def modernbert_restated(w64: Dict[str, torch.Tensor], cfg: eo.ModernBertConfig, ids, num_layers: int,
                        mut: Optional[str] = None, mut_layer: int = 1, mut_row: int = 0, mut_block: int = 0,
                        probe: Optional[Dict[str, float]] = None) -> List[torch.Tensor]:
    """encoder_forward's ModernBERT branch on one sequence: [S, H] float64 rows (pivot + hi + lo) after each layer.
    mut: one of MUTATIONS, applied at layer `mut_layer` (config-wide for the first three), or one of
    FAR_POSITION_MUTATIONS (config-wide).  `probe` receives the largest
    |value| met at each place the engine stores fp16."""
    if mut == "global_every":
        cfg = replace(cfg, global_attn_every_n_layers=cfg.global_attn_every_n_layers + 1)
    if mut == "rope_tables":
        cfg = replace(cfg, global_rope_theta=cfg.local_rope_theta, local_rope_theta=cfg.global_rope_theta)
    if mut == "window":
        cfg = replace(cfg, local_attention=2 * cfg.local_attention)
    W = lambda name: eo._w(w64, name, eo.MODERNBERT_PREFIXES)
    dev = next(iter(w64.values())).device
    t = torch.as_tensor(np.asarray(ids, dtype=np.int64), device=dev)
    S, H, heads, eps = len(t), cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps

    def see(name, v):
        if probe is not None:
            probe[name] = max(probe.get(name, 0.0), float(v.abs().max()))

    def rope(x, cos, sin):
        x = x.reshape(S, -1, 64)
        x1, x2 = x[..., :32], x[..., 32:]
        return torch.cat([x1 * cos[:, None] - x2 * sin[:, None], x1 * sin[:, None] + x2 * cos[:, None]], -1).reshape(S, -1)

    pos = torch.arange(S)
    if mut == "rope_pos_fp16":          # the table row read at fp16(position): exact only up to 2048
        pos = pos.to(torch.float16).long()
    if mut == "rope_wrap_2048":
        pos = pos % 2048
    tables = {local: tuple(c[pos] for c in eo.rope_tables(64, theta, int(pos.max()) + 1))
              for local, theta in ((False, cfg.global_rope_theta), (True, cfg.local_rope_theta))}
    x0 =eo.layer_norm(W("embeddings.tok_embeddings.weight")[t], W("embeddings.norm.weight"), None, eps)
    st = _Pair(x0)
    out = []
    for li in range(num_layers):
        here = li == mut_layer
        before = st.state()
        local = (li % cfg.global_attn_every_n_layers) != 0
        g_an = W(f"layers.{li}.attn_norm.weight")
        wqkv = W(f"layers.{li}.attn.Wqkv.weight")
        if li > 0 and g_an is not None:      # LayerNorm fold: raw rows times W diag(gamma), rstd in the epilogue
            g = torch.ones_like(g_an) if (mut == "fold_gamma" and here) else g_an
            qkv = st.rstd(eps) * (st.hi @ _fold(wqkv, g).t())
        elif li == 0:
            a = st.hi if g_an is None else r16(eo.layer_norm(x0, g_an, None, eps))
            qkv = a @ r16(wqkv).t()
        else:                                 # a later layer without attn_norm: fp16 of the rebuilt fp32 rows
            qkv = r16(st.x()) @ r16(wqkv).t()
        cos, sin = (c.to(dev).double() for c in tables[local])
        q, k, v = r16(rope(qkv[:, :H], cos, sin)), r16(rope(qkv[:, H:2 * H], cos, sin)), r16(qkv[:, 2 * H:])
        ctx = _attention(q, k, v, heads, cfg.local_attention // 2 if local else 0)
        for n, val in (("q", q), ("k", k), ("v", v), ("ctx", ctx)):
            see(n, val)
        st.update(ctx @ r16(W(f"layers.{li}.attn.Wo.weight")).t(), stale_pivot=(mut == "stale_pivot" and here))
        g_mn = W(f"layers.{li}.mlp_norm.weight")
        drop = (mut_row, mut_block) if (mut == "stats_block" and here) else None
        wi = st.rstd(eps, drop) * (st.hi @ _fold(W(f"layers.{li}.mlp.Wi.weight"), g_mn).t())
        a, b = wi.chunk(2, dim=-1)
        if mut == "geglu_halves" and here:
            a, b = b, a
        act = r16(eo.gelu_erf(a) * b)
        see("geglu", act)
        st.update(act @ r16(W(f"layers.{li}.mlp.Wo.weight")).t())
        if mut == "stale_rows" and here and S % 128:
            st.keep_rows(before, S // 128 * 128)
        out.append(st.x())
    return out


def split16(t: torch.Tensor) -> torch.Tensor:
    """precise.cu's operand: hi + lo with hi = fp16(t), lo = fp16(t - hi); lo falls in the fp16 subnormals (spacing 2^-24)
    once |t| < 2^-3, so the pair is within 2^-25 ABSOLUTE of a checkpoint weight, not 2^-22 relative"""
    hi = r16(t)
    return hi + r16(t.double() - hi)


def modernbert_precise_restated(weights: Dict[str, np.ndarray], cfg: eo.ModernBertConfig, ids, num_layers: int) -> List[torch.Tensor]:
    """encoder_forward_precise on one sequence: encoder_oracle's forward in float32 (fp32 LayerNorm, RoPE, softmax, GeGLU and
    accumulation) over projection weights replaced by their fp16 split pairs.  hi + lo has 22 significant bits and is exact
    in float32.  The activations' pairs (values of O(1): normal low halves, 2^-22) and the dropped A_lo W_lo term are
    below the float32 arithmetic itself and are not modelled."""
    w32 = {}
    for k, v in weights.items():
        t = torch.from_numpy(np.ascontiguousarray(v))
        is_proj = any(k.endswith(n + ".weight") for n in ("attn.Wqkv", "attn.Wo", "mlp.Wi", "mlp.Wo"))
        w32[k] = split16(t).float() if is_proj else t
    t, out = _ids(ids, "cpu"), []
    eo.modernbert_forward(w32, cfg, t, torch.ones_like(t), num_layers, collect=out)
    return [x[0] for x in out]


def bert_restated(w64: Dict[str, torch.Tensor], cfg: eo.BertConfig, ids, real_len: Optional[int] = None,
                  prefix: str = "bert") -> List[torch.Tensor]:
    """encoder_forward's BERT branch on one sequence: the fp32 stream, with fp16 copies entering every GEMM, fp16 q / k / v
    (heads of 32: the query rows carry sqrt(2) for the kernels' 64^-0.5), fp16 P, ctx and GELU output."""
    p = (prefix + ".") if prefix else ""
    dev = next(iter(w64.values())).device
    t = torch.as_tensor(np.asarray(ids, dtype=np.int64), device=dev)
    S, H, heads, eps = len(t), cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps
    D = H // heads
    qs = math.sqrt(2.0) if D == 32 else 1.0
    E = p + "embeddings."
    x = w64[E + "word_embeddings.weight"][t] + w64[E + "token_type_embeddings.weight"][0] + w64[E + "position_embeddings.weight"][:S]
    x = eo.layer_norm(x, w64[E + "LayerNorm.weight"], w64[E + "LayerNorm.bias"], eps)
    pad = lambda m: torch.nn.functional.pad(m.reshape(S, heads, D), (0, 64 - D)).reshape(S, heads * 64)
    out = []
    for li in range(cfg.num_hidden_layers):
        Lp = f"{p}encoder.layer.{li}."
        lin = lambda a, name, sc=1.0: a @ r16(w64[Lp + name + ".weight"] * sc).t() + w64[Lp + name + ".bias"] * sc
        h = r16(x)
        q, k, v = (r16(lin(h, "attention.self." + n, sc)) for n, sc in (("query", qs), ("key", 1.0), ("value", 1.0)))
        ctx = _attention(pad(q), pad(k), pad(v), heads, 0, real_len).reshape(S, heads, 64)[..., :D].reshape(S, H)
        x = eo.layer_norm(x + lin(ctx, "attention.output.dense"), w64[Lp + "attention.output.LayerNorm.weight"],
                          w64[Lp + "attention.output.LayerNorm.bias"], eps)
        inter = r16(eo.gelu_erf(lin(r16(x), "intermediate.dense")))
        x = eo.layer_norm(x + lin(inter, "output.dense"), w64[Lp + "output.LayerNorm.weight"],
                          w64[Lp + "output.LayerNorm.bias"], eps)
        out.append(x)
    return out


# --------------------------------------------------------------------------------------
# the cases both test files run
# --------------------------------------------------------------------------------------
# name -> ModernBertConfig fields (model_load accepts hidden 384 / 768 / 1024, any I % 64 == 0, heads of 64)
GEOMETRIES = {
    "base-768":      dict(hidden_size=768, num_attention_heads=12, intermediate_size=1152),
    "small-384":     dict(hidden_size=384, num_attention_heads=6, intermediate_size=1152),
    "large-1024":    dict(hidden_size=1024, num_attention_heads=16, intermediate_size=2624),
    "i1088-every2":  dict(hidden_size=768, num_attention_heads=12, intermediate_size=1088, global_attn_every_n_layers=2,
                          local_attention=64),
    "i320-global":   dict(hidden_size=384, num_attention_heads=6, intermediate_size=320, global_attn_every_n_layers=1),
    "i4096-every4":  dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, global_attn_every_n_layers=4,
                          local_attention=256, local_rope_theta=500000.0, global_rope_theta=10000.0, layer_norm_eps=1e-6),
}
FAMILIES = ("plain", "trained", "wide")
WIDE_STD = 0.05     # family "wide": the plain family at N(0, (0.05 sqrt(768 / H))^2) -- peaked attention and updates as large
                    # as the rows at every H, so the kind of a layer, its window and its rope table decide the rows


def depth(geometry: str) -> int:
    """Layers both test files run: enough to reach the second global layer (index global_every) wherever global_every > 1
    leaves room, so `li % global_every` differs from `li % (global_every + 1)` and from "only layer 0 is global"."""
    return max(4, GEOMETRIES[geometry].get("global_attn_every_n_layers", 3) + 1)
VOCAB = 600


def modernbert_config(geometry: str, layers: int) -> eo.ModernBertConfig:
    return eo.ModernBertConfig(vocab_size=VOCAB, num_hidden_layers=layers, max_position_embeddings=1024, pad_token_id=0,
                               **GEOMETRIES[geometry])


def modernbert_weights(cfg: eo.ModernBertConfig, family: str, seed: int = 1234, layer0_attn_norm: bool = False,
                       drop_attn_norm: Sequence[int] = ()) -> Dict[str, np.ndarray]:
    if family == "trained":
        return trained_like_modernbert_weights(cfg, 0, seed, layer0_attn_norm, drop_attn_norm)
    w = make_modernbert_weights(cfg, 0, seed=seed, with_head=False, std=WIDE_STD * math.sqrt(768.0 / cfg.hidden_size) if family == "wide" else STD)
    set_attn_norm_layout(w, cfg, np.random.default_rng(seed + 1), layer0_attn_norm, drop_attn_norm)
    return w
