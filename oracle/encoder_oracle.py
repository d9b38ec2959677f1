"""CPU oracle for the signal-extraction hot path (TEST INFRASTRUCTURE ONLY).

This file is a PyTorch-fp32 *restatement* of the reference's CPU algorithm (the
Rust candle-binding path of vllm-project/semantic-router).  It is the checker for
the CUDA path; it is never imported by the product (`semantic-router_b200/`), only by
`tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs.

PARITY STATUS: **parity unpinned by the reference** -- the reference holds no golden
logits/probabilities/embeddings for BERT or ModernBERT (SURVEY.md section 8c), its
Rust/Go toolchain is absent here (no cargo/rustc/go, no network for candle 0.9.2-alpha.1)
so it cannot be run.  What pins this restatement instead:
  * the reference's own behavioural tests re-run against it (RoPE identities, local-mask
    structure, CLS-pool exact copy, L2 norm == 1, determinism): tests/test_oracle_pins.py
  * an independent implementation of the same architectures: HuggingFace transformers 5.5
    `ModernBertModel` / `BertModel` (eager attention) on the same random-init weights:
    tests/golden/gen_golden.py records the max |delta| and tests/test_oracle_pins.py asserts it.
  * the ONE vector the reference holds on this path, candle-binding/test_data/long_prompt_fixtures.json (prompts of ~4 k / ~8 k
    tokens are cut to exactly 512, short ones untouched, the mmBERT-32K classifiers answer: mmbert_classifier.rs:1250-1420,
    semantic-router_test.go:4489-4640), imported by tools/import_reference_fixtures.py into tests/golden/
    reference_long_prompts.json and replayed by tests/test_reference_long_prompts.py (CPU: token counts; GPU: the classifiers).
    It pins the tokenisation / truncation contract, not logits: for the arithmetic the status above stands.

Third-party arithmetic the reference delegates to (not vendored in the reference checkout):
candle-core / candle-nn / candle-transformers 0.9.2-alpha.1 (candle-binding/Cargo.lock:356-453).
`BertModel` below restates candle-transformers `models/bert.rs` semantics (post-LN BERT,
erf-GELU, additive f32::MIN mask).

All citations are relative to candle-binding/src/ unless noted.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

F32_MIN = float(np.finfo(np.float32).min)
MAX_CLASSIFICATION_SEQ_LEN = 512  # model_architectures/traditional/modernbert.rs:20


# --------------------------------------------------------------------------------------
# configs
# --------------------------------------------------------------------------------------
@dataclass
class ModernBertConfig:
    """candle_models/modernbert.rs:21-38 (Config) / mmbert_embedding.rs:82-101 defaults."""
    vocab_size: int = 50368
    hidden_size: int = 768
    num_hidden_layers: int = 22
    num_attention_heads: int = 12
    intermediate_size: int = 1152
    max_position_embeddings: int = 8192
    layer_norm_eps: float = 1e-5
    pad_token_id: int = 50283
    global_attn_every_n_layers: int = 3
    global_rope_theta: float = 160000.0
    local_attention: int = 128
    local_rope_theta: float = 10000.0

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    def to_json(self, id2label: Optional[Dict[int, str]] = None) -> dict:
        d = {
            "architectures": ["ModernBertForSequenceClassification"],
            "model_type": "modernbert",
            "vocab_size": self.vocab_size, "hidden_size": self.hidden_size,
            "num_hidden_layers": self.num_hidden_layers,
            "num_attention_heads": self.num_attention_heads,
            "intermediate_size": self.intermediate_size,
            "max_position_embeddings": self.max_position_embeddings,
            "layer_norm_eps": self.layer_norm_eps, "norm_eps": self.layer_norm_eps,
            "pad_token_id": self.pad_token_id,
            "global_attn_every_n_layers": self.global_attn_every_n_layers,
            "global_rope_theta": self.global_rope_theta,
            "local_attention": self.local_attention,
            "local_rope_theta": self.local_rope_theta,
            "classifier_pooling": "mean",
        }
        if id2label is not None:
            d["id2label"] = {str(k): v for k, v in id2label.items()}
            d["label2id"] = {v: k for k, v in id2label.items()}
        return d


@dataclass
class BertConfig:
    """candle-transformers bert.rs Config (BERT-base defaults; MiniLM: hidden 384, L6/12, I 1536)."""
    vocab_size: int = 30522
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    intermediate_size: int = 3072
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    layer_norm_eps: float = 1e-12
    pad_token_id: int = 0

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    def to_json(self, id2label: Optional[Dict[int, str]] = None) -> dict:
        d = {
            "architectures": ["BertForSequenceClassification"], "model_type": "bert",
            "vocab_size": self.vocab_size, "hidden_size": self.hidden_size,
            "num_hidden_layers": self.num_hidden_layers,
            "num_attention_heads": self.num_attention_heads,
            "intermediate_size": self.intermediate_size, "hidden_act": "gelu",
            "max_position_embeddings": self.max_position_embeddings,
            "type_vocab_size": self.type_vocab_size, "layer_norm_eps": self.layer_norm_eps,
            "pad_token_id": self.pad_token_id, "position_embedding_type": "absolute",
        }
        if id2label is not None:
            d["id2label"] = {str(k): v for k, v in id2label.items()}
            d["label2id"] = {v: k for k, v in id2label.items()}
        return d


# --------------------------------------------------------------------------------------
# shared elementwise pieces
# --------------------------------------------------------------------------------------
def layer_norm(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], eps: float) -> torch.Tensor:
    """candle_nn::LayerNorm (remove_mean=true): (x-mean)/sqrt(var+eps)*w (+b); biased variance."""
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    """Tensor::gelu_erf -- exact erf GELU (candle_models/modernbert.rs:238)."""
    return F.gelu(x, approximate="none")


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    """Tensor::gelu -- candle's `gelu` is the tanh approximation (traditional/modernbert.rs:326)."""
    return F.gelu(x, approximate="tanh")


def rope_tables(head_dim: int, theta: float, max_pos: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """RotaryEmbedding::new (candle_models/modernbert.rs:61-80, mmbert_embedding.rs:183-207).

    inv_freq[i] = 1f32 / (theta.powf(i/dim) as f32)  -- powf in f64, cast to f32, THEN reciprocal in f32.
    freqs = t(f32) @ inv_freq(f32); sin/cos in f32.
    """
    i = np.arange(0, head_dim, 2, dtype=np.float64)
    denom = np.power(np.float64(theta), i / np.float64(head_dim)).astype(np.float32)
    inv_freq = (np.float32(1.0) / denom).astype(np.float32)
    t = np.arange(max_pos, dtype=np.float32)
    freqs = torch.from_numpy(t[:, None] * inv_freq[None, :])  # f32 product of one term: exact as matmul
    return torch.cos(freqs), torch.sin(freqs)


def rope_rotate_half(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """candle_nn::rotary_emb::rope = NON-interleaved (rotate-half) form.

    x: [B, H, S, D]; cos/sin: [S, D/2].  out[..., :D/2] = x1*cos - x2*sin ; out[..., D/2:] = x1*sin + x2*cos.
    """
    d2 = x.shape[-1] // 2
    x1, x2 = x[..., :d2], x[..., d2:]
    return torch.cat([x1 * cos - x2 * sin, x1 * sin + x2 * cos], dim=-1)


def global_mask_4d(mask: torch.Tensor) -> torch.Tensor:
    """prepare_4d_attention_mask (candle_models/modernbert.rs:355-373): (1-mask)*f32::MIN, [B,1,1,S]."""
    return ((1.0 - mask.to(torch.float32)) * F32_MIN)[:, None, None, :]


def local_mask(seq_len: int, max_distance: int) -> torch.Tensor:
    """get_local_attention_mask (candle_models/modernbert.rs:376-393): -inf where |j-i| > max_distance."""
    idx = torch.arange(seq_len)
    dist = (idx[None, :] - idx[:, None]).abs()
    m = torch.zeros(seq_len, seq_len, dtype=torch.float32)
    m[dist > max_distance] = float("-inf")
    return m


# --------------------------------------------------------------------------------------
# ModernBERT / mmBERT encoder
# --------------------------------------------------------------------------------------
def _w(weights: Dict[str, torch.Tensor], name: str, prefixes: Sequence[str]) -> Optional[torch.Tensor]:
    for p in prefixes:
        k = f"{p}.{name}" if p else name
        if k in weights:
            return weights[k]
    return None


MODERNBERT_PREFIXES = ("model", "_orig_mod.model", "", "_orig_mod")


def modernbert_forward(weights: Dict[str, torch.Tensor], cfg: ModernBertConfig,
                       ids: torch.Tensor, mask: torch.Tensor,
                       num_layers: Optional[int] = None,
                       collect: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
    """ModernBert::forward (candle_models/modernbert.rs:460-472) and
    MmBertEncoder::forward_to_layer (mmbert_embedding.rs:500-526) when `num_layers` is given.

    ids, mask: [B, S] integer tensors (mask 1 = real token).  Returns final_norm(hidden) [B,S,H] f32.
    `collect` (optional) receives the residual stream after every layer (for per-layer parity).
    """
    P = MODERNBERT_PREFIXES
    B, S = ids.shape
    nH, D = cfg.num_attention_heads, cfg.head_dim
    L = cfg.num_hidden_layers if num_layers is None else min(num_layers, cfg.num_hidden_layers)
    gmask = global_mask_4d(mask)
    lmask = local_mask(S, cfg.local_attention // 2)
    cos_g, sin_g = rope_tables(D, cfg.global_rope_theta, S)
    cos_l, sin_l = rope_tables(D, cfg.local_rope_theta, S)

    x = F.embedding(ids.long(), _w(weights, "embeddings.tok_embeddings.weight", P))
    x = layer_norm(x, _w(weights, "embeddings.norm.weight", P), None, cfg.layer_norm_eps)
    for li in range(L):
        is_local = (li % cfg.global_attn_every_n_layers) != 0          # :425
        residual = x
        h = x
        w_an = _w(weights, f"layers.{li}.attn_norm.weight", P)           # `.ok()` -> absent on layer 0 (:266-271)
        if w_an is not None:
            h = layer_norm(h, w_an, None, cfg.layer_norm_eps)
        qkv = h @ _w(weights, f"layers.{li}.attn.Wqkv.weight", P).t()    # :123-133
        qkv = qkv.reshape(B, S, 3, nH, D).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        cos, sin = (cos_l, sin_l) if is_local else (cos_g, sin_g)
        q = rope_rotate_half(q, cos, sin)
        k = rope_rotate_half(k, cos, sin)
        q = q * (float(D) ** -0.5)                                       # :141-142 (pre-scaled q)
        att = q @ k.transpose(-2, -1)                                     # :205
        att = att + ((gmask + lmask) if is_local else gmask)             # :206, :295-299
        att = torch.softmax(att, dim=-1)
        ctx = (att @ v).transpose(1, 2).reshape(B, S, nH * D)
        x = ctx @ _w(weights, f"layers.{li}.attn.Wo.weight", P).t() + residual
        h = layer_norm(x, _w(weights, f"layers.{li}.mlp_norm.weight", P), None, cfg.layer_norm_eps)
        wi = h @ _w(weights, f"layers.{li}.mlp.Wi.weight", P).t()        # :234-240
        a, b = wi.chunk(2, dim=-1)
        x = x + (gelu_erf(a) * b) @ _w(weights, f"layers.{li}.mlp.Wo.weight", P).t()
        if collect is not None:
            collect.append(x.clone())
    return layer_norm(x, _w(weights, "final_norm.weight", P), None, cfg.layer_norm_eps)


def masked_mean_pool(hidden: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """traditional/modernbert.rs:1146-1169 and embedding/pooling.rs:57-85: sum(h*mask)/sum(mask)."""
    m = mask.to(torch.float32)[..., None]
    return (hidden * m).sum(1) / m.sum(1)


def modernbert_head(weights: Dict[str, torch.Tensor], pooled: torch.Tensor) -> torch.Tensor:
    """FixedModernBertHead (traditional/modernbert.rs:303-329): dense(no bias) -> gelu(tanh) -> LN(w, 0, 1e-12)."""
    h = pooled @ weights["head.dense.weight"].t()
    h = gelu_tanh(h)
    return layer_norm(h, weights["head.norm.weight"], torch.zeros_like(weights["head.norm.weight"]), 1e-12)


def argmax_first(p: np.ndarray) -> int:
    """classify_internal :1184-1192 -- strict `>` starting from 0.0 => FIRST maximum wins."""
    best, idx = np.float32(0.0), 0
    for i, v in enumerate(p):
        if v > best:
            best, idx = v, i
    return idx


def argmax_last(p: np.ndarray) -> int:
    """Iterator::max_by(partial_cmp) (traditional/bert.rs:248-252) => LAST maximum wins."""
    best, idx = None, 0
    for i, v in enumerate(p):
        if best is None or not (v < best):   # max_by keeps the later element on Equal
            best, idx = v, i
    return idx


def modernbert_classify(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor,
                        num_layers: Optional[int] = None):
    """TraditionalModernBertClassifier::classify_internal (traditional/modernbert.rs:1125-1203).

    Pooling is ALWAYS mean (modernbert.rs:818).  Returns dict(logits, probs, cls, conf) with
    logits/probs [B,C] float32 numpy, cls int64 [B], conf float32 [B].
    """
    hidden = modernbert_forward(weights, cfg, ids, mask, num_layers)
    pooled = masked_mean_pool(hidden, mask)
    h = modernbert_head(weights, pooled) if "head.dense.weight" in weights else pooled
    logits = h @ weights["classifier.weight"].t() + weights["classifier.bias"]
    probs = torch.softmax(logits, dim=-1)
    pn = probs.numpy()
    cls = np.array([argmax_first(r) for r in pn], dtype=np.int64)
    conf = np.array([pn[i, c] if pn[i, c] > 0 else 0.0 for i, c in enumerate(cls)], dtype=np.float32)
    return {"logits": logits.numpy(), "probs": pn, "cls": cls, "conf": conf, "pooled": pooled.numpy()}


def modernbert_classify_tokens(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor):
    """TraditionalModernBertTokenClassifier::classify_tokens (traditional/modernbert.rs:1376-1406):
    head per token, classifier Linear(+bias), softmax; prediction = tensor argmax over LOGITS (first max)."""
    hidden = modernbert_forward(weights, cfg, ids, mask)
    h = modernbert_head(weights, hidden) if "head.dense.weight" in weights else hidden
    logits = h @ weights["classifier.weight"].t() + weights["classifier.bias"]
    probs = torch.softmax(logits, dim=-1)
    pred = torch.argmax(logits, dim=-1)
    return {"logits": logits.numpy(), "probs": probs.numpy(), "pred": pred.numpy()}


# ---- onnx-binding flavour: the exported HF graph + the Rust post-processing around it --------------------
def modernbert_head_hf(weights: Dict[str, torch.Tensor], x: torch.Tensor, eps: float) -> torch.Tensor:
    """HF ModernBertPredictionHead as an ONNX export carries it: dense (no bias) -> erf GELU
    (config.classifier_activation = "gelu") -> LayerNorm(weight, no bias, eps = config.norm_eps).  The candle head
    (modernbert_head above) differs in both the activation (tanh) and eps (1e-12)."""
    h = gelu_erf(x @ weights["head.dense.weight"].t())
    return layer_norm(h, weights["head.norm.weight"], None, eps)


def argmax_max_by(p: np.ndarray) -> int:
    """`iter().enumerate().max_by(|a,b| a.partial_cmp(b).unwrap_or(Less))`
    (onnx-binding/src/model_architectures/classification/mmbert_classifier.rs:809-813): a later element replaces
    the running maximum unless the maximum is strictly greater (so ties and NaNs go to the later index)."""
    best = 0
    for c in range(1, len(p)):
        if not (p[best] > p[c]):
            best = c
    return best


def modernbert_classify_onnx(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor,
                             pooling: str = "cls"):
    """MmBertSequenceClassifier::classify_batch (mmbert_classifier.rs:519-581) over the exported
    ModernBertForSequenceClassification graph: final_norm -> pooling per config.classifier_pooling ("cls": token 0,
    "mean": masked mean) -> head -> classifier; then logits_to_classification_results (:796-830): softmax, max_by."""
    hidden = modernbert_forward(weights, cfg, ids, mask)
    pooled = hidden[:, 0] if pooling == "cls" else masked_mean_pool(hidden, mask)
    h = modernbert_head_hf(weights, pooled, cfg.layer_norm_eps)
    logits = (h @ weights["classifier.weight"].t() + weights["classifier.bias"]).numpy()
    ex = np.exp(logits - logits.max(axis=1, keepdims=True))
    probs = (ex / ex.sum(axis=1, keepdims=True)).astype(np.float32)
    cls = np.array([argmax_max_by(r) for r in probs], dtype=np.int64)
    conf = np.array([probs[i, c] for i, c in enumerate(cls)], dtype=np.float32)
    return {"logits": logits, "probs": probs, "cls": cls, "conf": conf}


def modernbert_classify_tokens_onnx(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor):
    """MmBertTokenClassifier::detect_entities (mmbert_classifier.rs:892-941) up to the per-token softmax/max_by of
    bio_decode_entities (:975-990), over the exported ModernBertForTokenClassification graph."""
    hidden = modernbert_forward(weights, cfg, ids, mask)
    h = modernbert_head_hf(weights, hidden, cfg.layer_norm_eps)
    logits = (h @ weights["classifier.weight"].t() + weights["classifier.bias"]).numpy()
    ex = np.exp(logits - logits.max(axis=-1, keepdims=True))
    probs = (ex / ex.sum(axis=-1, keepdims=True)).astype(np.float32)
    pred = np.array([[argmax_max_by(r) for r in b] for b in probs], dtype=np.int64)
    return {"logits": logits, "probs": probs, "pred": pred}


def bio_decode_onnx(pred: Sequence[int], conf: Sequence[float], offsets: Sequence[Tuple[int, int]],
                    id2label: Dict[int, str], text_len: int):
    """bio_decode_entities (mmbert_classifier.rs:952-1050): B- opens (closing any open entity), an I- of the SAME
    type extends with the running pairwise mean, any other I- is ignored (the entity stays open), everything else
    closes; tokens with offset (0,0) are skipped; entities whose span falls outside the text are dropped."""
    out, cur = [], None

    def flush():
        nonlocal cur
        if cur is not None and cur[1] < text_len and cur[2] <= text_len:
            out.append(tuple(cur))
        cur = None
    for p, c, (s, e) in zip(pred, conf, offsets):
        if s == 0 and e == 0:
            continue
        label = id2label.get(int(p), f"LABEL_{int(p)}")
        if label.startswith("B-"):
            flush()
            cur = [label[2:], s, e, np.float32(c)]
        elif label.startswith("I-"):
            if cur is not None and cur[0] == label[2:]:
                cur[2] = e
                cur[3] = np.float32((cur[3] + np.float32(c)) / np.float32(2.0))
        else:
            flush()
    flush()
    return out


def mmbert_embed_onnx(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor,
                      target_layer: Optional[int] = None, target_dim: Optional[int] = None) -> np.ndarray:
    """onnx-binding MmBertEmbeddingModel::encode (embedding/mmbert_embedding.rs:637-700): hidden states -> masked
    mean pool -> truncate_dimension -> l2_normalize with x / max(||x||, 1e-12) (embedding/pooling.rs:61-82)."""
    L = cfg.num_hidden_layers if not target_layer or target_layer > cfg.num_hidden_layers else target_layer
    emb = masked_mean_pool(modernbert_forward(weights, cfg, ids, mask, L), mask)
    if target_dim and target_dim < cfg.hidden_size:
        emb = emb[:, :target_dim]
    norm = emb.pow(2).sum(1, keepdim=True).sqrt().clamp_min(1e-12)
    return (emb / norm).numpy()


def mmbert_embed(weights, cfg: ModernBertConfig, ids: torch.Tensor, mask: torch.Tensor,
                 target_layer: Optional[int] = None, target_dim: Optional[int] = None) -> np.ndarray:
    """MmBertEmbeddingModel::embedding_forward_with_matryoshka (mmbert_embedding.rs:630-709) +
    l2_normalize (:781-796): encoder to `target_layer` (1-indexed count) -> final_norm -> masked mean
    -> narrow(0..dim) -> x / (||x||_2 + 1e-12)."""
    L = cfg.num_hidden_layers if target_layer is None else target_layer
    if L == 0 or L > cfg.num_hidden_layers:
        raise ValueError("target_layer must be in 1..num_layers")
    hidden = modernbert_forward(weights, cfg, ids, mask, L)
    emb = masked_mean_pool(hidden, mask)
    if target_dim is not None and target_dim < cfg.hidden_size:
        emb = emb[:, :target_dim]
    norm = emb.pow(2).sum(1, keepdim=True).sqrt() + 1e-12
    return (emb / norm).numpy()


# --------------------------------------------------------------------------------------
# BERT (candle-transformers models/bert.rs semantics)
# --------------------------------------------------------------------------------------
def bert_forward(weights: Dict[str, torch.Tensor], cfg: BertConfig, ids: torch.Tensor,
                 mask: torch.Tensor, prefix: str = "bert") -> torch.Tensor:
    """candle BertModel::forward(input_ids, token_type_ids=0, Some(mask)) used at
    traditional/bert.rs:230-234, core/similarity.rs:213-217, lora/bert_lora.rs:569."""
    p = (prefix + ".") if prefix else ""
    B, S = ids.shape
    nH, D = cfg.num_attention_heads, cfg.head_dim
    E = p + "embeddings."
    x = F.embedding(ids.long(), weights[E + "word_embeddings.weight"])
    x = x + weights[E + "token_type_embeddings.weight"][0][None, None, :]
    x = x + weights[E + "position_embeddings.weight"][:S][None, :, :]
    x = layer_norm(x, weights[E + "LayerNorm.weight"], weights[E + "LayerNorm.bias"], cfg.layer_norm_eps)
    amask = global_mask_4d(mask)  # get_extended_attention_mask: (1-mask)*f32::MIN
    for li in range(cfg.num_hidden_layers):
        Lp = f"{p}encoder.layer.{li}."
        def lin(t, name):
            return t @ weights[Lp + name + ".weight"].t() + weights[Lp + name + ".bias"]
        q = lin(x, "attention.self.query").reshape(B, S, nH, D).transpose(1, 2)
        k = lin(x, "attention.self.key").reshape(B, S, nH, D).transpose(1, 2)
        v = lin(x, "attention.self.value").reshape(B, S, nH, D).transpose(1, 2)
        att = (q @ k.transpose(-2, -1)) / math.sqrt(D)
        att = torch.softmax(att + amask, dim=-1)
        ctx = (att @ v).transpose(1, 2).reshape(B, S, nH * D)
        x = layer_norm(lin(ctx, "attention.output.dense") + x,
                       weights[Lp + "attention.output.LayerNorm.weight"],
                       weights[Lp + "attention.output.LayerNorm.bias"], cfg.layer_norm_eps)
        inter = gelu_erf(lin(x, "intermediate.dense"))           # HiddenAct::Gelu => erf
        x = layer_norm(lin(inter, "output.dense") + x,
                       weights[Lp + "output.LayerNorm.weight"],
                       weights[Lp + "output.LayerNorm.bias"], cfg.layer_norm_eps)
    return x


def bert_classify(weights, cfg: BertConfig, ids: torch.Tensor, mask: torch.Tensor,
                  pooler_transposed: bool = True):
    """TraditionalBertClassifier::classify_text (traditional/bert.rs:222-255).

    CLS -> pooler -> tanh -> classifier -> softmax -> LAST-max argmax.
    `pooler_transposed=True` follows bert.rs:107 (`Linear::new(pooler_weight.t(), bias)` => y = x @ P);
    False follows lora/bert_lora.rs:534-538 (`candle_nn::linear` => y = x @ P^T).
    """
    hidden = bert_forward(weights, cfg, ids, mask)
    cls_tok = hidden[:, 0]
    P = weights["bert.pooler.dense.weight"]
    pooled = cls_tok @ (P if pooler_transposed else P.t()) + weights["bert.pooler.dense.bias"]
    pooled = torch.tanh(pooled)
    logits = pooled @ weights["classifier.weight"].t() + weights["classifier.bias"]
    probs = torch.softmax(logits, dim=-1).numpy()
    cls = np.array([argmax_last(r) for r in probs], dtype=np.int64)
    conf = np.array([probs[i, c] for i, c in enumerate(cls)], dtype=np.float32)
    return {"logits": logits.numpy(), "probs": probs, "cls": cls, "conf": conf}


def bert_classify_tokens(weights, cfg: BertConfig, ids: torch.Tensor, mask: torch.Tensor):
    """TraditionalBertTokenClassifier (traditional/bert.rs:542-592): classifier per token, softmax,
    per-token max_by (LAST max)."""
    hidden = bert_forward(weights, cfg, ids, mask)
    logits = hidden @ weights["classifier.weight"].t() + weights["classifier.bias"]
    probs = torch.softmax(logits, dim=-1).numpy()
    pred = np.array([[argmax_last(r) for r in row] for row in probs], dtype=np.int64)
    return {"logits": logits.numpy(), "probs": probs, "pred": pred}


def bert_similarity_embedding(weights, cfg: BertConfig, ids: torch.Tensor, mask: torch.Tensor,
                              prefix: str = "") -> np.ndarray:
    """BertSimilarity::get_embedding (core/similarity.rs:189-228): UNMASKED token sum / sum(mask)
    (batch 1 => identical to masked), then normalize_l2 WITHOUT epsilon (:338-341)."""
    hidden = bert_forward(weights, cfg, ids, mask, prefix=prefix)
    pooled = hidden.sum(1) / mask.to(torch.float32).sum(1, keepdim=True)
    return (pooled / pooled.pow(2).sum(1, keepdim=True).sqrt()).numpy()


# --------------------------------------------------------------------------------------
# BIO decode (host-side, integer/fp tiny) -- traditional/modernbert.rs:1478-1567
# --------------------------------------------------------------------------------------
def bio_decode(pred: Sequence[int], conf: Sequence[float], offsets: Sequence[Tuple[int, int]],
               id2label: Dict[int, str]) -> List[Tuple[str, int, int, float]]:
    """Merge B-/I- tags into (entity_type, start, end, confidence) spans.

    Skips special tokens whose offsets are (0,0); a B-X starts a new entity; I-X extends the
    current entity when the type matches (running pairwise mean confidence (c+c')/2, NOT an
    average); anything else closes the current entity.
    """
    out: List[Tuple[str, int, int, float]] = []
    cur: Optional[List] = None
    for p, c, (s, e) in zip(pred, conf, offsets):
        if s == 0 and e == 0:
            continue
        label = id2label.get(int(p), "O")
        if label.startswith("B-"):
            if cur is not None:
                out.append(tuple(cur))
            cur = [label[2:], s, e, float(c)]
        elif label.startswith("I-") and cur is not None and cur[0] == label[2:]:
            cur[2] = e
            cur[3] = (cur[3] + float(c)) / 2.0
        else:
            if cur is not None:
                out.append(tuple(cur))
                cur = None
    if cur is not None:
        out.append(tuple(cur))
    return out


def hallucination_spans(pred: Sequence[int], conf: Sequence[float], offsets: Sequence[Tuple[int, int]],
                        answer_start: int, answer: bytes, threshold: float):
    """detect_hallucinations (candle-binding/src/ffi/classify.rs:1536-1660) after the token classifier: tokens that
    start inside the answer, class 1 with confidence >= threshold (0.5 unless 0 < threshold <= 1) extend a span
    (span confidence = max token confidence), anything else closes it; spans must slice the answer cleanly.
    Returns (has_hallucination, overall_confidence, [(text, start, end, confidence)])."""
    thr = threshold if 0.0 < threshold <= 1.0 else 0.5
    spans, cur = [], None
    n_hall = n_ans = 0
    max_conf = np.float32(0.0)

    def close():
        nonlocal cur
        if cur is not None and cur[0] >= 0 and cur[1] > cur[0] and cur[1] <= len(answer):
            spans.append((answer[cur[0]:cur[1]], cur[0], cur[1], cur[2]))
        cur = None
    for p, c, (s, e) in zip(pred, conf, offsets):
        if s < answer_start:
            continue
        n_ans += 1
        c = np.float32(c)
        if int(p) == 1 and c >= np.float32(thr):
            n_hall += 1
            max_conf = max(max_conf, c)
            if cur is None:
                cur = [s - answer_start, e - answer_start, c]
            else:
                cur[1] = e - answer_start
            cur[2] = max(cur[2], c)
        else:
            close()
    close()
    has = len(spans) > 0
    overall = max_conf if has else (np.float32(1.0) - np.float32(n_hall) / np.float32(n_ans) if n_ans else np.float32(1.0))
    return has, float(overall), spans


def nli_result(cls: int, conf: float):
    """classify_nli (ffi/classify.rs:1766-1795): label + the other two classes reported as an even split."""
    rest = (np.float32(1.0) - np.float32(conf)) / np.float32(2.0)
    probs = [rest, rest, rest]
    probs[cls] = np.float32(conf)
    return cls, [float(x) for x in probs]


def shannon_entropy(probs: np.ndarray) -> float:
    """src/semantic-router/pkg/utils/entropy/entropy.go:24 -- -sum p log2 p over p>0 (reasoning-need)."""
    p = probs[probs > 0].astype(np.float64)
    return float(-(p * np.log2(p)).sum())
