"""End-to-end parity of the CUDA path (through the C ABI, host buffers) against the CPU oracle on the same
seeded synthetic models, and against the committed golden fixtures (tests/golden/, produced by gen_golden.py).

Tolerances (BASELINE.json north_star: "class indices bit-exact, logits and embeddings within 1e-3 fp32"):
  * class indices / top-1: bit-exact (token predictions: bit-exact wherever the oracle's top-2 logit margin
    exceeds the drift bound, and > 99 % overall);
  * embeddings (unit vectors) and sequence probabilities (what the reference ABI returns): 1e-3 absolute;
  * logits: 1e-3 RELATIVE to the logit scale, |dlogit| <= 1e-3 * max(1, max|logit|) -- the synthetic
    classifier is scaled x8 (SURVEY 8d) so logits reach ~13 and an absolute 1e-3 would be 7.7e-5 relative,
    below what fp16 operands (2^-11) can give; the encoder GEMMs run fp16 x fp16 -> fp32 as the north star
    prescribes.  Token-level probabilities (no pooling to average the drift): 3e-3 absolute.
Measured values are printed (pytest -s)."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

MB_SMALL = dict(vocab_size=1000, num_hidden_layers=5, max_position_embeddings=1024, pad_token_id=0)
BERT_SMALL = dict(vocab_size=1000, num_hidden_layers=3)
LOGIT_RTOL = 1e-3      # x max(1, max|logit|)
PROB_ATOL = 1e-3
TOKEN_PROB_ATOL = 3e-3
EMB_ATOL = 1e-3


def logit_tol(ref_logits):
    return LOGIT_RTOL * max(1.0, float(np.abs(ref_logits).max()))


def _t(w):
    return {k: torch.from_numpy(v) for k, v in w.items()}


def _one(s):
    return torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long)


@pytest.fixture(scope="module")
def mb_small(srlib, cuda):
    cfg = eo.ModernBertConfig(**MB_SMALL)
    w = synth.make_modernbert_weights(cfg, 14, seed=7)
    d = tempfile.mkdtemp(prefix="srb_mb_")
    synth.write_model_dir(d, cfg, w, {i: f"cat{i}" for i in range(14)})
    m = srlib.Model(d, device=0)
    yield cfg, w, m, d
    m.close()


def test_modernbert_golden_and_oracle(mb_small):
    cfg, w, m, _ = mb_small
    g = np.load(os.path.join(GOLD, "modernbert_small.npz"))
    lengths = g["lengths"].tolist()
    seqs = np.split(g["ids"].astype(np.int32), np.cumsum(lengths)[:-1])
    out = m.classify_ids(seqs)                      # one packed varlen batch
    dl = np.abs(out["logits"] - g["logits"]).max()
    dp = np.abs(out["probs"] - g["probs"]).max()
    print(f"modernbert small: max|dlogit|={dl:.3e} max|dprob|={dp:.3e} logit scale={np.abs(g['logits']).max():.2f}")
    assert (out["cls"] == g["cls"]).all()
    assert dl < logit_tol(g["logits"]) and dp < PROB_ATOL
    # reference operating mode: one prompt per call gives the same answer as the packed batch
    for i in (0, 3, 4):
        o1 = m.classify_ids([seqs[i]])
        assert np.abs(o1["logits"][0] - out["logits"][i]).max() < 1e-5
        assert o1["cls"][0] == out["cls"][i]
    # probabilities sum to one; confidence is the arg-max probability
    assert np.allclose(out["probs"].sum(1), 1.0, atol=1e-5)
    assert np.allclose(out["conf"], out["probs"][np.arange(len(seqs)), out["cls"]])


def test_modernbert_embedding_matryoshka(mb_small):
    cfg, w, m, _ = mb_small
    g = np.load(os.path.join(GOLD, "modernbert_small.npz"))
    lengths = g["lengths"].tolist()
    seqs = np.split(g["ids"].astype(np.int32), np.cumsum(lengths)[:-1])
    e = m.embed_ids(seqs, target_layer=3, target_dim=256)
    ef = m.embed_ids(seqs)
    print("emb l3/d256 max|d|", np.abs(e - g["emb_l3_d256"]).max(), "full", np.abs(ef - g["emb_full"]).max())
    assert np.abs(e - g["emb_l3_d256"]).max() < EMB_ATOL
    assert np.abs(ef - g["emb_full"]).max() < EMB_ATOL
    assert np.allclose(np.linalg.norm(e, axis=1), 1.0, atol=1e-5)
    assert np.allclose(np.linalg.norm(ef, axis=1), 1.0, atol=1e-5)
    # identical text => similarity ~ 1 (semantic-router_test.go:283-331), determinism (<= 1e-6, :255-278)
    e2 = m.embed_ids(seqs, target_layer=3, target_dim=256)
    assert np.abs(e - e2).max() <= 1e-6


def test_modernbert_tokens(srlib, cuda):
    cfg = eo.ModernBertConfig(**MB_SMALL)
    w = synth.make_modernbert_weights(cfg, 35, seed=7)
    g = np.load(os.path.join(GOLD, "modernbert_small.npz"))
    lengths = g["lengths"].tolist()[:3]
    seqs = np.split(g["ids"].astype(np.int32), np.cumsum(g["lengths"])[:-1])[:3]
    with tempfile.TemporaryDirectory() as d:
        c = cfg.to_json(synth.pii_id2label())
        synth.write_model_dir(d, cfg, w, synth.pii_id2label())
        m = srlib.Model(d, device=0)
        out = m.classify_tokens_ids(seqs)
        m.close()
    dl = np.abs(out["logits"] - g["tok_logits"]).max()
    print(f"token head: max|dlogit|={dl:.3e}")
    assert dl < logit_tol(g["tok_logits"])
    # predictions must match wherever the oracle's top-2 margin exceeds the drift; report exact-match rate
    gl = np.sort(g["tok_logits"], axis=1)
    margin = gl[:, -1] - gl[:, -2]
    safe = margin > 2 * logit_tol(g["tok_logits"])
    assert (out["pred"][safe] == g["tok_pred"][safe]).all()
    assert (out["pred"] == g["tok_pred"]).mean() > 0.99


def test_modernbert_multi_head_shared_encoder(srlib, cuda, mb_small):
    """BASELINE cfg 3 analogue: one encoder pass + 3 heads == three independent classifiers with identical
    encoder weights (the reference runs three separate encoders, parallel_engine.rs:85-104)."""
    cfg, w, m, _ = mb_small
    w2 = dict(w)
    w2.update({k: v for k, v in synth.make_modernbert_weights(cfg, 2, seed=21).items()
               if k.startswith(("head.", "classifier."))})
    w3 = dict(w)
    w3.update({k: v for k, v in synth.make_modernbert_weights(cfg, 35, seed=22).items()
               if k.startswith(("head.", "classifier."))})
    rng = np.random.default_rng(3)
    seqs = synth.make_ids(rng, [256, 100, 31], cfg.vocab_size)
    with tempfile.TemporaryDirectory() as d2, tempfile.TemporaryDirectory() as d3:
        synth.write_model_dir(d2, cfg, w2, {0: "benign", 1: "jailbreak"})
        synth.write_model_dir(d3, cfg, w3, synth.pii_id2label())
        h2 = m.add_head(d2, token_level=0)
        h3 = m.add_head(d3, token_level=1)
        probs, cls = m.classify_multi_ids(seqs, [0, h2, h3], [False, False, True])
    for i, s in enumerate(seqs):
        ids, mask = _one(s)
        r1 = eo.modernbert_classify(_t(w), cfg, ids, mask)
        r2 = eo.modernbert_classify(_t(w2), cfg, ids, mask)
        assert cls[0][i] == r1["cls"][0] and cls[1][i] == r2["cls"][0]
        assert np.abs(probs[0][i] - r1["probs"][0]).max() < PROB_ATOL
        assert np.abs(probs[1][i] - r2["probs"][0]).max() < PROB_ATOL
    r3 = eo.modernbert_classify_tokens(_t(w3), cfg, *_one(seqs[1]))
    sl = slice(256, 356)
    assert np.abs(probs[2][sl] - r3["probs"][0]).max() < TOKEN_PROB_ATOL


def test_modernbert_long_and_edge_lengths(mb_small):
    """Ragged / edge cases: single token, window boundary (129/130), > 512 tokens, 1000 tokens."""
    cfg, w, m, _ = mb_small
    rng = np.random.default_rng(9)
    seqs = synth.make_ids(rng, [1, 129, 130, 1000, 513], cfg.vocab_size)
    out = m.classify_ids(seqs)
    wt = _t(w)
    for i, s in enumerate(seqs):
        ref = eo.modernbert_classify(wt, cfg, *_one(s))
        assert np.abs(ref["logits"][0] - out["logits"][i]).max() < logit_tol(ref["logits"]), (i, len(s))
        assert ref["cls"][0] == out["cls"][i]


def test_bert_golden(srlib, cuda):
    cfg = eo.BertConfig(**BERT_SMALL)
    w = synth.make_bert_weights(cfg, 14, seed=11)
    g = np.load(os.path.join(GOLD, "bert_small.npz"))
    seqs = np.split(g["ids"].astype(np.int32), np.cumsum(g["lengths"])[:-1])
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(14)})
        m = srlib.Model(d, device=0)
        out = m.classify_ids(seqs, pooler_mode=0)       # traditional/bert.rs:107 (x @ P)
        out_l = m.classify_ids(seqs, pooler_mode=1)     # lora/bert_lora.rs:534 (x @ P^T)
        emb = m.embed_ids(seqs)
        m.close()
    print("bert: max|dlogit|", np.abs(out["logits"] - g["logits"]).max(), np.abs(out_l["logits"] - g["logits_lora"]).max(),
          "emb", np.abs(emb - g["emb"]).max())
    assert np.abs(out["logits"] - g["logits"]).max() < logit_tol(g["logits"])
    assert np.abs(out_l["logits"] - g["logits_lora"]).max() < logit_tol(g["logits_lora"])
    assert (out["cls"] == g["cls"]).all()
    assert np.abs(emb - g["emb"]).max() < EMB_ATOL


def test_no_cpu_fallback_errors(srlib, cuda):
    with pytest.raises(srlib.SrError):
        srlib.Model("/nonexistent/model/dir", device=0)
    with pytest.raises(srlib.SrError):
        srlib.Model("/tmp", device=99)


def test_graph_replay_survives_workspace_regrow(srlib, mb_small):
    """Small calls replay a captured CUDA graph; a later larger batch reallocates workspace buffers (more sequences,
    more tokens, more output rows).  The captured graph must be dropped, not replayed against freed pointers."""
    cfg, w, _, d = mb_small
    m = srlib.Model(d, device=0)                         # fresh workspace: nothing grown yet
    rng = np.random.default_rng(17)
    small = synth.make_ids(rng, [40, 23], cfg.vocab_size)
    a = m.classify_ids(small)                            # eager + capture
    b = m.classify_ids(small)                            # replay
    m.classify_ids(synth.make_ids(rng, [9] * 200, cfg.vocab_size))      # more sequences than the first allocation
    c = m.classify_ids(small)
    m.classify_ids(synth.make_ids(rng, [700] * 12, cfg.vocab_size))     # more tokens
    e = m.classify_ids(small)
    for o in (b, c, e):
        assert np.array_equal(a["probs"], o["probs"]) and np.array_equal(a["cls"], o["cls"])
    ref = eo.modernbert_classify(_t(w), cfg, *_one(small[0]))
    assert np.abs(ref["probs"][0] - e["probs"][0]).max() < PROB_ATOL
    m.close()


def test_modernbert_long_context_embeddings(srlib, cuda):
    """mmBERT-32k-style long inputs on the embedding path (mmbert_embedding.rs:82-101: 32 768 positions): a 4 096-token
    prompt against the oracle (global + local layer), 16 384 and 32 768 tokens through properties only (the oracle's
    dense score tensor does not fit), alone and packed next to short prompts."""
    cfg = eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=4, max_position_embeddings=32768, pad_token_id=0,
                              local_rope_theta=160000.0)
    w = synth.make_modernbert_weights(cfg, 2, seed=77)
    rng = np.random.default_rng(77)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {0: "a", 1: "b"})
        m = srlib.Model(d, device=0)
        seqs = synth.make_ids(rng, [4096, 17, 16384, 130, 32768], cfg.vocab_size)
        e = m.embed_ids(seqs, target_layer=0, target_dim=256)
        assert np.isfinite(e).all() and np.abs(np.linalg.norm(e, axis=1) - 1.0).max() < 1e-3
        for i in (0, 2, 4):                                   # a long prompt alone == the same prompt inside the packed batch
            e1 = m.embed_ids([seqs[i]], target_layer=0, target_dim=256)
            assert np.abs(e1[0] - e[i]).max() <= 1e-6, i
        for i in (0, 1):
            ids, mask = _one(seqs[i])
            ref = eo.mmbert_embed(_t(w), cfg, ids, mask, None, 256)[0]
            print("long-context embed len", len(seqs[i]), "max|d|", np.abs(ref - e[i]).max())
            assert np.abs(ref - e[i]).max() < EMB_ATOL
        m.close()


def test_minilm_heads_of_32(srlib, cuda):
    """all-MiniLM-L6/L12 shape (SURVEY appendix B: H = 384, 12 heads x 32, FFN 1536), the reference's default similarity
    / cache model: the heads are zero-padded to 64 at load time and run on the head_dim-64 kernels.  Classification and
    the similarity embedding against the oracle, small ragged batch and a batch large enough to give every GEMM worker several tiles."""
    cfg = eo.BertConfig(vocab_size=1000, hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=3)
    w = synth.make_bert_weights(cfg, 14, seed=13)
    rng = np.random.default_rng(13)
    seqs = synth.make_ids(rng, [128, 5, 77, 300], cfg.vocab_size)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(14)})
        m = srlib.Model(d, device=0)
        out = m.classify_ids(seqs, pooler_mode=0)
        emb = m.embed_ids(seqs)
        big = seqs + synth.make_ids(rng, [256] * 12, cfg.vocab_size)        # 3 582 tokens: several tiles per worker
        out_big = m.classify_ids(big, pooler_mode=0)
        m.close()
    wt = _t(w)
    for i, s in enumerate(seqs):
        ids, mask = _one(s)
        ref = eo.bert_classify(wt, cfg, ids, mask)
        dl = np.abs(ref["logits"][0] - out["logits"][i]).max()
        de = np.abs(eo.bert_similarity_embedding(wt, cfg, ids, mask, prefix="bert")[0] - emb[i]).max()
        db = np.abs(ref["logits"][0] - out_big["logits"][i]).max()
        print(f"minilm len {len(s)}: max|dlogit| {dl:.2e} (in the large batch {db:.2e}) max|demb| {de:.2e} scale {np.abs(ref['logits']).max():.1f}")
        assert dl < logit_tol(ref["logits"]) and db < logit_tol(ref["logits"])
        assert de < EMB_ATOL
        assert np.abs(ref["probs"][0] - out["probs"][i]).max() < PROB_ATOL
