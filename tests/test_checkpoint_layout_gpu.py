"""Checkpoint layouts the loader must read the same way on every path (csrc/engine.cu: tensor_prefix, layer_projections).

* Tensor-name prefixes: one synthetic ModernBERT checkpoint under each prefix the reference loaders try ("model.",
  "_orig_mod.model.", none, "_orig_mod.") gives byte-identical logits / probabilities and hidden rows through the ordinary
  load, the precise path and the shared-LoRA pass; one BERT checkpoint with and without "bert." does the same, and a
  head-only directory still finds "bert." through its pooler.
* A checkpoint replaced in place (os.replace, as a trainer saving checkpoints does): the precise path of a model loaded
  afterwards from the same directory builds its weights from the new file, not from an earlier mapping."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu

MB_PREFIXES = ["model", "_orig_mod.model", "", "_orig_mod"]
TASKS = [(8, 16.0, 5), (16, 32.0, 3)]   # rank, alpha, classes


def _hidden(srlib, m, rows):
    """Host copy of the first `rows` rows of the model's fp32 hidden states (sr_dev_hidden)."""
    ptr = srlib.lib().sr_dev_hidden(m.handle)
    assert ptr

    class _Dev:
        __cuda_array_interface__ = {"data": (int(ptr), False), "shape": (rows, m.hidden), "typestr": "<f4", "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy()


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _modernbert_dirs(cfg, tmp, prefix):
    """The base checkpoint and two unmerged-LoRA task checkpoints over it, every encoder tensor under `prefix`."""
    base = synth.make_modernbert_weights(cfg, 4, seed=61, prefix=prefix)
    p = (prefix + ".") if prefix else ""
    H, I = cfg.hidden_size, cfg.intermediate_size
    d0 = synth.write_model_dir(os.path.join(tmp, "base"), cfg, base, {i: f"c{i}" for i in range(4)})
    dirs = []
    for task, (rank, alpha, ncls) in enumerate(TASKS):
        w = dict(base)
        head = synth.make_modernbert_weights(cfg, ncls, seed=70 + task)
        for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias"):
            w[k] = head[k]
        rng = np.random.default_rng(80 + task)
        for li in range(cfg.num_hidden_layers):
            for name, (o, i) in (("attn.Wqkv", (3 * H, H)), ("attn.Wo", (H, H)), ("mlp.Wi", (2 * I, H)), ("mlp.Wo", (H, I))):
                stem = f"{p}layers.{li}.{name}"
                w[stem + ".lora_A.weight"] = (rng.standard_normal((rank, i)) * 0.02).astype(np.float32)
                w[stem + ".lora_B.weight"] = (rng.standard_normal((o, rank)) * 0.02).astype(np.float32)
        d = synth.write_model_dir(os.path.join(tmp, f"task{task}"), cfg, w, {i: f"c{i}" for i in range(ncls)})
        json.dump({"rank": rank, "alpha": alpha}, open(os.path.join(d, "lora_config.json"), "w"))
        dirs.append(d)
    return d0, dirs


def _modernbert_results(srlib, cfg, prefix, seqs):
    T = sum(len(s) for s in seqs)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        d0, dirs = _modernbert_dirs(cfg, tmp, prefix)
        m = srlib.Model(d0, device=0)
        r = m.classify_ids(seqs)
        out["logits"], out["probs"], out["hidden"] = r["logits"], r["probs"], _hidden(srlib, m, T)
        m.set_precise(True)
        r = m.classify_ids(seqs)
        out["precise_logits"], out["precise_hidden"] = r["logits"], _hidden(srlib, m, T)
        m.close()
        m = srlib.LoraSharedModel(dirs, [0, 0], device=0)
        probs, cls, _ = m.classify_shared_ids(seqs)
        for t in range(len(dirs)):
            out[f"lora_probs{t}"], out[f"lora_cls{t}"] = probs[t], cls[t]
        out["lora_hidden"] = _hidden(srlib, m, T)   # task 0's copy of the rows
        m.close()
    return out


def test_modernbert_prefixes_give_identical_results(srlib, cuda):
    cfg = eo.ModernBertConfig(vocab_size=600, num_hidden_layers=3, max_position_embeddings=1024, pad_token_id=0)
    seqs = synth.make_ids(np.random.default_rng(9), [5, 130, 77], cfg.vocab_size)
    ref = _modernbert_results(srlib, cfg, MB_PREFIXES[0], seqs)
    for prefix in MB_PREFIXES[1:]:
        got = _modernbert_results(srlib, cfg, prefix, seqs)
        assert got.keys() == ref.keys()
        for k in ref:
            assert _same(got[k], ref[k]), (prefix, k)


def test_bert_prefixes_give_identical_results(srlib, cuda):
    cfg = eo.BertConfig(vocab_size=600, num_hidden_layers=2, max_position_embeddings=512)
    seqs = synth.make_ids(np.random.default_rng(10), [5, 130, 77], cfg.vocab_size)
    T = sum(len(s) for s in seqs)
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for prefix in ("bert", ""):
            w = synth.make_bert_weights(cfg, 4, seed=62, prefix=prefix)
            d = synth.write_model_dir(os.path.join(tmp, prefix or "none"), cfg, w, {i: f"c{i}" for i in range(4)})
            # head-only checkpoint: classifier + pooler, no embeddings to name the prefix
            hd = synth.write_model_dir(os.path.join(tmp, (prefix or "none") + "_head"), cfg,
                                       {k: v for k, v in w.items() if k.startswith("classifier.") or "pooler." in k},
                                       {i: f"c{i}" for i in range(4)})
            m = srlib.Model(d, device=0)
            r = m.classify_ids(seqs, pooler_mode=1)
            hidden = _hidden(srlib, m, T)
            r_head = m.classify_ids(seqs, head=m.add_head(hd), pooler_mode=1)
            m.close()
            assert _same(r_head["logits"], r["logits"]), prefix   # the head-only copy found the same pooler
            res.append((r["logits"], r["probs"], hidden))
    for a, b in zip(*res):
        assert _same(a, b)


def test_precise_path_reads_a_replaced_checkpoint(srlib, cuda):
    """Model A from D with the precise path on; B replaces D/model.safetensors; A is closed.  A model loaded from D on the
    same thread must run B's weights on the precise path too."""
    cfg = eo.ModernBertConfig(vocab_size=600, num_hidden_layers=3, max_position_embeddings=1024, pad_token_id=0)
    seqs = synth.make_ids(np.random.default_rng(11), [17, 200, 64], cfg.vocab_size)
    wa = synth.make_modernbert_weights(cfg, 6, seed=91)
    wb = synth.make_modernbert_weights(cfg, 6, seed=92)
    with tempfile.TemporaryDirectory() as tmp:
        d = synth.write_model_dir(os.path.join(tmp, "ckpt"), cfg, wa, {i: f"c{i}" for i in range(6)})
        db = synth.write_model_dir(os.path.join(tmp, "next"), cfg, wb, {i: f"c{i}" for i in range(6)})
        a = srlib.Model(d, device=0)
        a.set_precise(True)
        a.classify_ids(seqs)
        os.replace(os.path.join(db, "model.safetensors"), os.path.join(d, "model.safetensors"))
        a.close()
        m = srlib.Model(d, device=0)
        m.set_precise(True)
        out = m.classify_ids(seqs)
        m.close()
    wt = {k: torch.from_numpy(v) for k, v in wb.items()}
    for i, s in enumerate(seqs):
        ref = eo.modernbert_classify(wt, cfg, torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long))
        dl = float(np.abs(ref["logits"][0] - out["logits"][i]).max())
        dp = float(np.abs(ref["probs"][0] - out["probs"][i]).max())
        assert dl < 1e-3 and dp < 1e-4, (len(s), dl, dp)   # test_precise_gpu.py's bound
