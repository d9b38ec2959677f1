"""The strict bound of BASELINE's north star -- "logits and embeddings within 1e-3 fp32" -- as an ABSOLUTE bound on the logits
of the x8-scaled synthetic heads (SURVEY 8d), met by the precise path (sr_model_set_precise: every GEMM operand as an fp16
hi + lo pair on the same wgmma kernel, fp32 in between; csrc/precise.cu), at 5 layers and at the full 22-layer depth.
Also measured here: what the production (fp16-operand) path gives on the same inputs, and its error on an UN-scaled head
(classifier std 0.02, logits ~1): that is inside 1e-3 absolute without the precise path."""
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu
ABS = 1e-3


def _t(w):
    return {k: torch.from_numpy(v) for k, v in w.items()}


def _ref(wt, cfg, s):
    return eo.modernbert_classify(wt, cfg, torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long))


def _errs(m, wt, cfg, seqs):
    out = m.classify_ids(seqs)
    dl = dp = scale = 0.0
    for i, s in enumerate(seqs):
        r = _ref(wt, cfg, s)
        dl = max(dl, float(np.abs(r["logits"][0] - out["logits"][i]).max()))
        dp = max(dp, float(np.abs(r["probs"][0] - out["probs"][i]).max()))
        scale = max(scale, float(np.abs(r["logits"]).max()))
        assert int(r["cls"][0]) == int(out["cls"][i])
    return dl, dp, scale


@pytest.mark.parametrize("layers,vocab,lens", [(5, 1000, [17, 96, 129, 130, 200, 511, 512]), (22, 50368, [512, 64, 300])])
def test_precise_path_meets_the_absolute_bound(srlib, cuda, layers, vocab, lens):
    cfg = eo.ModernBertConfig(vocab_size=vocab, num_hidden_layers=layers, max_position_embeddings=1024, pad_token_id=0)
    w = synth.make_modernbert_weights(cfg, 14, seed=7 if layers == 5 else 1234)
    wt = _t(w)
    rng = np.random.default_rng(5)
    seqs = synth.make_ids(rng, lens, cfg.vocab_size)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {i: f"cat{i}" for i in range(14)})
        m = srlib.Model(d, device=0)
        dl0, dp0, scale = _errs(m, wt, cfg, seqs)                        # production path (fp16 operands)
        m.set_precise(True)
        dl1, dp1, _ = _errs(m, wt, cfg, seqs)
        # embeddings through the same path (early exit + matryoshka)
        e = m.embed_ids(seqs, target_layer=min(6, layers), target_dim=256)
        for i, s in enumerate(seqs):
            r = eo.mmbert_embed(wt, cfg, torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long),
                                min(6, layers), 256)[0]
            assert np.abs(e[i] - r).max() < 1e-5
        # the batch still equals one prompt per call, and switching back restores the production path bit for bit
        o_b = m.classify_ids(seqs)
        o_1 = m.classify_ids([seqs[1]])
        assert np.abs(o_1["logits"][0] - o_b["logits"][1]).max() < 1e-5
        m.set_precise(False)
        dl2, _, _ = _errs(m, wt, cfg, seqs)
        m.close()
    print(f"L={layers}: logit scale {scale:.2f}; production max|dlogit| {dl0:.3e} max|dprob| {dp0:.3e}; "
          f"precise max|dlogit| {dl1:.3e} max|dprob| {dp1:.3e}")
    assert dl1 < ABS and dp1 < 1e-4                                     # the north star's bound, absolute, on x8 logits
    # the production path on the SAME x8-scaled head: ~5e-4 relative on the logits, which a x8 head turns into up to
    # ~1e-3 on a probability (measured 1.04e-3 on a 64-token prompt at 22 layers); see the un-scaled head below
    assert dl0 < 1e-3 * max(1.0, scale) and dp0 < 2e-3
    assert dl2 == dl0


def test_production_path_on_an_unscaled_head(srlib, cuda):
    """The x8 classifier of the synthetic models (SURVEY 8d) multiplies every error by 8.  With the classifier at its
    natural scale (std 0.02: logits of order 1) the fp16-operand path itself is inside 1e-3 absolute at full depth."""
    cfg = eo.ModernBertConfig(vocab_size=50368, num_hidden_layers=22, max_position_embeddings=1024, pad_token_id=0)
    w = synth.make_modernbert_weights(cfg, 14, seed=1234)
    w["classifier.weight"] = (w["classifier.weight"] / np.float32(8.0)).astype(np.float32)
    wt = _t(w)
    rng = np.random.default_rng(6)
    seqs = synth.make_ids(rng, [512, 128, 333], cfg.vocab_size)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {i: f"cat{i}" for i in range(14)})
        m = srlib.Model(d, device=0)
        out = m.classify_ids(seqs)
        m.close()
    dl = max(float(np.abs(_ref(wt, cfg, s)["logits"][0] - out["logits"][i]).max()) for i, s in enumerate(seqs))
    print(f"un-scaled head, 22 layers, production path: max|dlogit| {dl:.3e}")
    assert dl < ABS
