"""ModernBERT checkpoints whose attn_norm layout differs from the usual one (none on layer 0, one on every later layer).
The reference loads attn_norm with `.ok()` (candle_models/modernbert.rs:266-271), so any layer may have it or not:

* layer 0 WITH attn_norm: the LayerNorm runs on the fp32 embedding output, and Wqkv is not folded;
* a later layer WITHOUT attn_norm (identity): Wqkv multiplies fp16(x) rebuilt from the fp16-pair residual stream.

Both go through the classifier and the embedding head against the oracle, at the tolerances of test_encoder_parity_gpu.py."""
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu

LOGIT_RTOL = 1e-3      # x max(1, max|logit|)
PROB_ATOL = 1e-3
EMB_ATOL = 1e-3
CFG = dict(vocab_size=1000, num_hidden_layers=5, max_position_embeddings=1024, pad_token_id=0)


def _layer0_norm(w, cfg, rng):
    w["model.layers.0.attn_norm.weight"] = (0.5 + rng.random(cfg.hidden_size)).astype(np.float32)


def _middle_identity(w, cfg, rng):
    del w["model.layers.2.attn_norm.weight"]


@pytest.mark.parametrize("edit", [_layer0_norm, _middle_identity], ids=["layer0_attn_norm", "middle_identity_norm"])
def test_modernbert_attn_norm_layout(srlib, cuda, edit):
    cfg = eo.ModernBertConfig(**CFG)
    w = synth.make_modernbert_weights(cfg, 14, seed=41)
    rng = np.random.default_rng(41)
    # residual-stream rows with a spread of about 3 instead of 1: a LayerNorm skipped where the checkpoint has one,
    # or applied where it has none, moves the outputs far past the tolerances
    w["model.embeddings.norm.weight"] *= np.float32(3.0)
    edit(w, cfg, rng)
    seqs = synth.make_ids(rng, [1, 129, 300, 64, 517], cfg.vocab_size)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(14)})
        m = srlib.Model(d, device=0)
        out = m.classify_ids(seqs)
        emb = m.embed_ids(seqs)
        m.close()
    wt = {k: torch.from_numpy(v) for k, v in w.items()}
    for i, s in enumerate(seqs):
        ids, mask = torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long)
        ref = eo.modernbert_classify(wt, cfg, ids, mask)
        ref_emb = eo.mmbert_embed(wt, cfg, ids, mask)[0]
        dl = np.abs(ref["logits"][0] - out["logits"][i]).max()
        de = np.abs(ref_emb - emb[i]).max()
        print(f"{edit.__name__} len {len(s)}: max|dlogit| {dl:.2e} scale {np.abs(ref['logits']).max():.1f} max|demb| {de:.2e}")
        assert dl < LOGIT_RTOL * max(1.0, float(np.abs(ref["logits"]).max())), (i, len(s))
        assert np.abs(ref["probs"][0] - out["probs"][i]).max() < PROB_ATOL, (i, len(s))
        assert ref["cls"][0] == out["cls"][i], (i, len(s))
        assert de < EMB_ATOL, (i, len(s))
