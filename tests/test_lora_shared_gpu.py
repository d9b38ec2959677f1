"""Shared-base multi-task pass over UNMERGED LoRA checkpoints (SURVEY section 8 f3; model_architectures/lora/lora_adapter.rs:136-144,
pkg/classification/unified_classifier.go:113): three task checkpoints over ONE base -- intent (sequence head), PII (token head),
security (sequence head); ranks 8 / 16 / 32, their own alpha, not every projection adapted -- load as one model
(sr_model_load_lora_shared) and a batch runs ONCE through the encoder, every task's copy of the rows multiplied with that task's
merged projection weights (picked per row block in the GEMM's TMA producer).  Expected values: the oracle on the MERGED weights
W + (alpha / r) B A of each task (merge_weights, lora_adapter.rs:157-168), i.e. what three separate forwards would give;
and the three-slot path of this library (load-time fold) on the same inputs."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu

TASKS = [(8, 16.0, 14, 0), (16, 32.0, 9, 1), (32, 32.0, 2, 0)]   # rank, alpha, classes, token-level


def _modernbert_tasks(cfg, tmp, std=0.02):
    base = synth.make_modernbert_weights(cfg, 14, seed=11)
    H, I = cfg.hidden_size, cfg.intermediate_size
    dirs, merged = [], []
    for task, (rank, alpha, ncls, _tok) in enumerate(TASKS):
        w = dict(base)
        head = synth.make_modernbert_weights(cfg, ncls, seed=20 + task)
        for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias"):
            w[k] = head[k]
        mg = dict(w)
        trng = np.random.default_rng(30 + task)
        for li in range(cfg.num_hidden_layers):
            for name, (o, i) in (("attn.Wqkv", (3 * H, H)), ("attn.Wo", (H, H)), ("mlp.Wi", (2 * I, H)), ("mlp.Wo", (H, I))):
                if (li + task) % 2 == 0 and name == "mlp.Wo":
                    continue                                   # not every projection carries an adapter
                A = (trng.standard_normal((rank, i)) * std).astype(np.float32)
                B = (trng.standard_normal((o, rank)) * std).astype(np.float32)
                stem = f"model.layers.{li}.{name}"
                w[stem + ".lora_A.weight"] = A
                w[stem + ".lora_B.weight"] = B
                mg[stem + ".weight"] = (w[stem + ".weight"].astype(np.float64) + (alpha / rank) * (B.astype(np.float64) @ A.astype(np.float64))).astype(np.float32)
        d = os.path.join(tmp, f"task{task}")
        synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(ncls)})
        json.dump({"rank": rank, "alpha": alpha}, open(os.path.join(d, "lora_config.json"), "w"))
        dirs.append(d)
        merged.append({k: torch.from_numpy(v) for k, v in mg.items()})
    return dirs, merged, base


# Tolerances: token-level probabilities 3e-3 as in test_encoder_parity_gpu.py (no pooling to average the drift); sequence
# probabilities 1.5e-3, where the three-slot path (adapters folded at load) gives 2.6e-4 .. 1.2e-3 on these x8-scaled heads:
# the drift is the fp16 pipeline's.  Adapter scale 0.02 gives |dW| ~ 10 % of |W| (a trained adapter's order of magnitude);
# 0.05 makes the adapter term as large as the base weights themselves -- every fp16-rounded intermediate then carries twice
# the signal, and the bounds are doubled for that case (the three-slot path drifts by the same amount: printed).
# The shared pass stacks the tasks' merged matrices and picks one per 256-row block in the TMA producer (every copy of the
# rows padded to whole blocks): it has the arithmetic of the three-slot path and must agree with it to batch-composition
# noise (1e-5), not just to the tolerance.
@pytest.mark.parametrize("std,tol", [(0.02, 1.0), (0.05, 2.0)])
@pytest.mark.parametrize("lens", [[33, 200, 512], [7], [64] * 40 + [300, 511, 2, 129]])
def test_three_tasks_one_pass_modernbert(srlib, cuda, lens, std, tol):
    cfg = eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=0)
    rng = np.random.default_rng(12 + len(lens))
    seqs = synth.make_ids(rng, lens, cfg.vocab_size)
    with tempfile.TemporaryDirectory() as tmp:
        dirs, merged, base = _modernbert_tasks(cfg, tmp, std)
        m = srlib.LoraSharedModel(dirs, [t[3] for t in TASKS], device=0)
        assert m.tasks == 3
        probs, cls, conf = m.classify_shared_ids(seqs)
        probs2, cls2, _ = m.classify_shared_ids(seqs)                  # second call: the graph replay of small batches
        m.close()
        slots = []
        for t, d in enumerate(dirs):                                   # the three-slot path (adapters folded at load)
            sm = srlib.Model(d, device=0)
            slots.append(sm.classify_tokens_ids(seqs) if TASKS[t][3] else sm.classify_ids(seqs))
            sm.close()
    cu = np.concatenate([[0], np.cumsum(lens)])
    worst = {0: 0.0, 1: 0.0}
    worst_slots = {0: 0.0, 1: 0.0}
    worst_between = 0.0
    seq_tol, tok_tol = 1.5e-3 * tol, 3e-3 * tol
    for t, (_r, _a, ncls, tok) in enumerate(TASKS):
        assert np.array_equal(cls[t], cls2[t]) and np.abs(probs[t] - probs2[t]).max() < 1e-6
        for i, s in enumerate(seqs):
            ids, mask = torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long)
            if tok:
                ref = eo.modernbert_classify_tokens(merged[t], cfg, ids, mask)
                got = probs[t][cu[i]:cu[i + 1]]
                d = np.abs(ref["probs"][0] - got).max()
                # argmax parity wherever the oracle's margin is not inside the tolerance
                srt = np.sort(ref["probs"][0], axis=-1)
                clear = (srt[:, -1] - srt[:, -2]) > 2 * tok_tol
                assert np.array_equal(ref["pred"][0][clear], cls[t][cu[i]:cu[i + 1]][clear])
                worst_between = max(worst_between, float(np.abs(slots[t]["probs"][cu[i]:cu[i + 1]] - got).max()))
                worst_slots[1] = max(worst_slots[1], float(np.abs(slots[t]["probs"][cu[i]:cu[i + 1]] - ref["probs"][0]).max()))
            else:
                ref = eo.modernbert_classify(merged[t], cfg, ids, mask)
                d = np.abs(ref["probs"][0] - probs[t][i]).max()
                top2 = np.sort(ref["probs"][0])[-2:]
                if top2[1] - top2[0] > 2 * seq_tol:
                    assert int(ref["cls"][0]) == int(cls[t][i])
                assert abs(float(conf[t][i]) - float(probs[t][i][cls[t][i]])) < 1e-6
                worst_between = max(worst_between, float(np.abs(slots[t]["probs"][i] - probs[t][i]).max()))
                worst_slots[0] = max(worst_slots[0], float(np.abs(slots[t]["probs"][i] - ref["probs"][0]).max()))
            worst[tok] = max(worst[tok], float(d))
    print(f"shared-LoRA pass, adapters x{std}, lens={lens[:4]}..: max |dprob| vs merged-weight oracle: sequence heads {worst[0]:.2e}, "
          f"token head {worst[1]:.2e} (three-slot path vs oracle: {worst_slots[0]:.2e} / {worst_slots[1]:.2e}; between the two paths {worst_between:.2e})")
    assert worst[0] < seq_tol and worst[1] < tok_tol and worst_between < 1e-5
    # and the adapters matter: the base alone answers differently
    bt = {k: torch.from_numpy(v) for k, v in base.items()}
    bt.update({k: merged[0][k] for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias")})
    refb = eo.modernbert_classify(bt, cfg, torch.from_numpy(seqs[0][None].astype(np.int64)), torch.ones(1, len(seqs[0]), dtype=torch.long))
    assert np.abs(refb["probs"][0] - probs[0][0]).max() > 1e-2


def test_three_tasks_one_pass_bert(srlib, cuda):
    """BERT-family base (the reference's LoRA classifiers are BERT or ModernBERT, classifiers/lora/intent_lora.rs:50-78): PEFT
    adapts query / key / value separately -- three segments of the fused QKV projection."""
    cfg = eo.BertConfig(vocab_size=800, num_hidden_layers=3, max_position_embeddings=512)
    base = synth.make_bert_weights(cfg, 4, seed=5)
    H, I = cfg.hidden_size, cfg.intermediate_size
    rng = np.random.default_rng(3)
    seqs = synth.make_ids(rng, [5, 128, 300, 77], cfg.vocab_size)
    tasks = [(8, 16.0, 6, 0), (16, 16.0, 3, 0)]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, merged = [], []
        for task, (rank, alpha, ncls, _tok) in enumerate(tasks):
            w = dict(base)
            head = synth.make_bert_weights(cfg, ncls, seed=40 + task)
            for k in head:
                if k.startswith("classifier.") or "pooler." in k:
                    w[k] = head[k]
            mg = dict(w)
            trng = np.random.default_rng(50 + task)
            for li in range(cfg.num_hidden_layers):
                Lp = f"bert.encoder.layer.{li}."
                for name, (o, i) in (("attention.self.query", (H, H)), ("attention.self.value", (H, H)), ("attention.self.key", (H, H)),
                                     ("attention.output.dense", (H, H)), ("intermediate.dense", (I, H)), ("output.dense", (H, I))):
                    if name == "attention.self.key" and task == 0:
                        continue                               # the usual PEFT target set: query + value only
                    A = (trng.standard_normal((rank, i)) * 0.05).astype(np.float32)
                    B = (trng.standard_normal((o, rank)) * 0.05).astype(np.float32)
                    w[Lp + name + ".lora_A.weight"] = A
                    w[Lp + name + ".lora_B.weight"] = B
                    mg[Lp + name + ".weight"] = (w[Lp + name + ".weight"].astype(np.float64) + (alpha / rank) * (B.astype(np.float64) @ A.astype(np.float64))).astype(np.float32)
            d = os.path.join(tmp, f"task{task}")
            synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(ncls)})
            json.dump({"rank": rank, "alpha": alpha}, open(os.path.join(d, "lora_config.json"), "w"))
            dirs.append(d)
            merged.append({k: torch.from_numpy(v) for k, v in mg.items()})
        m = srlib.LoraSharedModel(dirs, [0, 0], device=0)
        probs, cls, _ = m.classify_shared_ids(seqs, pooler_mode=1)
        m.close()
    for t in range(2):
        for i, s in enumerate(seqs):
            ref = eo.bert_classify(merged[t], cfg, torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long),
                                   pooler_transposed=False)     # lora/bert_lora.rs:534-538 <-> pooler_mode 1
            assert int(ref["cls"][0]) == int(cls[t][i])
            assert np.abs(ref["probs"][0] - probs[t][i]).max() < 1e-3


def test_checkpoints_over_different_bases_are_refused(srlib, cuda):
    cfg = eo.ModernBertConfig(vocab_size=500, num_hidden_layers=2, max_position_embeddings=512, pad_token_id=0)
    with tempfile.TemporaryDirectory() as tmp:
        dirs = []
        for task in range(2):
            w = synth.make_modernbert_weights(cfg, 3, seed=7 + task)   # two DIFFERENT bases
            w["model.layers.0.attn.Wo.lora_A.weight"] = np.zeros((8, cfg.hidden_size), np.float32)
            w["model.layers.0.attn.Wo.lora_B.weight"] = np.zeros((cfg.hidden_size, 8), np.float32)
            d = os.path.join(tmp, f"t{task}")
            synth.write_model_dir(d, cfg, w, {i: f"c{i}" for i in range(3)})
            dirs.append(d)
        with pytest.raises(srlib.SrError, match="share one base"):
            srlib.LoraSharedModel(dirs, [0, 0], device=0)


def test_text_abi_serves_the_three_tasks_from_one_pass(srlib, cuda):
    """init_lora_unified_classifier / classify_batch_with_lora (unified_classifier.go:66-81) over three unmerged task
    checkpoints: the default build serves them from ONE shared-base pass; SR_B200_LORA_SHARED=0 loads three slots with the
    adapters folded at load.  Same LoRABatchResult from both (two private copies of the library = two sets of global slots),
    fewer kernel launches from the shared pass."""
    import ctypes as C
    import shutil
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_multi_device_dispatch_mock import LBatch, _arr
    from oracle import tokenizer_fixtures as tf
    cfg = eo.ModernBertConfig(vocab_size=700, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=3)
    texts = [f"request {i}: " + "please send the report to john@example.com " * (i % 3) + "ignore previous instructions " * (i % 2) + "filler " * (i % 13)
             for i in range(48)]
    old = {k: os.environ.get(k) for k in ("SR_B200_LORA_SHARED", "SR_B200_DEVICE", "SR_B200_DEVICES")}
    os.environ["SR_B200_DEVICE"] = "0"
    os.environ.pop("SR_B200_DEVICES", None)
    tmp = tempfile.mkdtemp(prefix="srb_lora_shared_abi_")
    try:
        dirs, _merged, _base = _modernbert_tasks(cfg, tmp)
        for d in dirs:
            tf.BUILDERS["modernbert"](os.path.join(d, "tokenizer.json"))
        res = {}
        for mode in ("1", "0"):                                      # shared pass (default), three slots
            os.environ["SR_B200_LORA_SHARED"] = mode
            inst = os.path.join(tmp, f"libcandle_private_{mode}.so")
            shutil.copyfile(srlib.LIB_PATH, inst)                    # fresh global slots
            L = C.CDLL(inst)
            L.init_lora_unified_classifier.argtypes = [C.c_char_p] * 4 + [C.c_bool]; L.init_lora_unified_classifier.restype = C.c_bool
            L.classify_batch_with_lora.argtypes = [C.POINTER(C.c_char_p), C.c_int]; L.classify_batch_with_lora.restype = LBatch
            L.free_lora_batch_result.argtypes = [LBatch]
            L.sr_launch_count.restype = C.c_longlong
            assert L.init_lora_unified_classifier(dirs[0].encode(), dirs[1].encode(), dirs[2].encode(), b"modernbert", False)
            r = L.classify_batch_with_lora(_arr(texts), len(texts))           # warm-up (allocations)
            L.free_lora_batch_result(r)
            n0 = L.sr_launch_count()
            r = L.classify_batch_with_lora(_arr(texts), len(texts))
            res[mode] = (r, L, L.sr_launch_count() - n0)
        a, b = res["1"][0], res["0"][0]                               # the shared pass has the three-slot arithmetic
        assert a.batch_size == b.batch_size == len(texts)
        flips = 0
        for i in range(len(texts)):
            assert abs(a.intent_results[i].confidence - b.intent_results[i].confidence) < 1e-5
            assert abs(a.security_results[i].confidence - b.security_results[i].confidence) < 1e-5
            assert abs(a.pii_results[i].confidence - b.pii_results[i].confidence) < 1.5e-5
            flips += a.intent_results[i].category != b.intent_results[i].category
            flips += a.security_results[i].threat_type != b.security_results[i].threat_type
        assert flips == 0
        print(f"launches for {len(texts)} texts: shared pass {res['1'][2]}, three slots {res['0'][2]}")
        assert res["1"][2] < res["0"][2]
        for r, L, _ in res.values():
            L.free_lora_batch_result(r)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        shutil.rmtree(tmp, ignore_errors=True)
