"""BertSimilarity under a tokenizer.json that carries fixed-length padding (core/similarity.rs:189-222): the reference clones
the tokenizer as loaded, so "padding": {"strategy": {"Fixed": n}} -- the sentence-transformers MiniLM files ship it -- makes it
encode every text to n positions, run the encoder over the pad positions as QUERIES (they are only masked as keys) and divide
the UNMASKED token sum by the number of real tokens.  Reproduced on the device (sr_embed_ids_padded: kv_lens in the
attention, divisor lengths in the pooling) and through the text ABI (init_similarity_model / get_text_embedding /
calculate_similarity); expected values from the oracle fed with the padded ids and mask HuggingFace `tokenizers` produces."""
import ctypes as C
import os
import shutil
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth, tokenizer_fixtures as tf

pytestmark = pytest.mark.gpu


class EmbRes(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_float)), ("length", C.c_int), ("error", C.c_bool), ("model_type", C.c_int),
                ("sequence_length", C.c_int), ("processing_time_ms", C.c_float)]


def _t(w):
    return {k: torch.from_numpy(v) for k, v in w.items()}


def test_ids_level_pads_are_queries_and_are_summed(srlib, cuda):
    cfg = eo.BertConfig(vocab_size=600, num_hidden_layers=3)
    w = synth.make_bert_weights(cfg, 2, seed=401)
    w = {(k[len("bert."):] if k.startswith("bert.") else k): v for k, v in w.items()}
    rng = np.random.default_rng(3)
    real = [5, 17, 32, 100, 131]
    padded = [32, 32, 32, 128, 256]                          # tiles of the attention kernel: inside one, across two
    seqs = []
    for r, n in zip(real, padded):
        s = np.zeros(n, dtype=np.int32)
        s[:r] = synth.make_ids(rng, [r], cfg.vocab_size)[0]
        seqs.append(s)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, cfg, w, {0: "a", 1: "b"})
        m = srlib.Model(d, device=0)
        got = m.embed_ids_padded(seqs, real)
        plain = m.embed_ids([s[:r] for s, r in zip(seqs, real)])
        m.close()
    wt = _t(w)
    for i, (s, r) in enumerate(zip(seqs, real)):
        mask = torch.zeros(1, len(s), dtype=torch.long)
        mask[0, :r] = 1
        want = eo.bert_similarity_embedding(wt, cfg, torch.from_numpy(s[None].astype(np.int64)), mask)[0]
        assert np.abs(got[i] - want).max() < 1e-3, (i, np.abs(got[i] - want).max())
        assert abs(np.linalg.norm(got[i]) - 1.0) < 1e-4
        if r < len(s):                                       # the quirk is visible: it is NOT the embedding of the real tokens alone
            assert np.abs(got[i] - plain[i]).max() > 1e-3


def test_text_abi_with_a_fixed_padding_tokenizer(srlib, cuda):
    from tokenizers import Tokenizer
    inst = os.path.join(os.path.dirname(srlib.LIB_PATH), "libcandle_semantic_router_fixedpad_instance.so")
    shutil.copyfile(srlib.LIB_PATH, inst)                    # fresh global slots
    L = C.CDLL(inst)
    cfg = eo.BertConfig(vocab_size=600, num_hidden_layers=3)
    w = synth.make_bert_weights(cfg, 2, seed=402)
    w = {(k[len("bert."):] if k.startswith("bert.") else k): v for k, v in w.items()}
    d = tempfile.mkdtemp(prefix="srb_fixedpad_")
    try:
        tp = os.path.join(d, "tokenizer.json")
        tf.BUILDERS["bert"](tp)
        hf = Tokenizer.from_file(tp)
        hf.enable_padding(length=48, pad_id=hf.token_to_id("[PAD]"), pad_token="[PAD]")
        hf.save(tp)                                          # the file now carries "padding": {"strategy": {"Fixed": 48}, ...}
        synth.write_model_dir(d, cfg, w, {0: "a", 1: "b"})
        hf = Tokenizer.from_file(tp)
        hf.enable_truncation(max_length=512)
        L.init_similarity_model.argtypes, L.init_similarity_model.restype = [C.c_char_p, C.c_bool], C.c_bool
        L.get_text_embedding.argtypes, L.get_text_embedding.restype = [C.c_char_p, C.c_int], EmbRes
        L.free_embedding.argtypes = [C.POINTER(C.c_float), C.c_int]
        L.calculate_similarity.argtypes, L.calculate_similarity.restype = [C.c_char_p, C.c_char_p, C.c_int], C.c_float
        assert L.init_similarity_model(d.encode(), True)
        wt = _t(w)
        texts = ["What is the derivative of x^2?", "hello", "word " * 90, "naïve café 数学"]
        embs = []
        for text in texts:
            enc = hf.encode(text)
            ids = torch.tensor([enc.ids], dtype=torch.long)
            mask = torch.tensor([enc.attention_mask], dtype=torch.long)
            assert len(enc.ids) >= 48 and (len(enc.ids) == 48) == (int(mask.sum()) <= 48)
            want = eo.bert_similarity_embedding(wt, cfg, ids, mask)[0]
            r = L.get_text_embedding(text.encode(), 0)
            assert not r.error and r.length == cfg.hidden_size
            got = np.ctypeslib.as_array(r.data, (r.length,)).copy()
            L.free_embedding(r.data, r.length)
            assert np.abs(got - want).max() < 1e-3, (text[:20], np.abs(got - want).max())
            embs.append(want)
        s = L.calculate_similarity(texts[0].encode(), texts[1].encode(), 512)
        assert abs(s - float(np.dot(embs[0], embs[1]))) < 2e-3
    finally:
        shutil.rmtree(d, ignore_errors=True)
        try:
            os.remove(inst)
        except OSError:
            pass
