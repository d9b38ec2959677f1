"""Several task checkpoints of one encoder served in ONE pass (sr_model_load_grouped): merged LoRA models and full
fine-tunes, where every tensor -- embeddings, norms, biases, projections, final_norm, heads -- may differ per task.  Each
task's copy of the rows runs with that task's tensors (projections and biases picked per 256-row block in the GEMM, row
kernels picking per row), so every task's probs / cls / conf must be BITWISE what the same directory gives loaded alone as
Model, and within test_lora_shared_gpu.py's tolerances of the float64 oracle on that task's weights."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASKS = [(14, 0), (35, 1), (2, 0), (2, 0), (4, 0)]          # classes, token-level
LENS = [1, 127, 128, 129, 256, 512]                          # 1153 rows per copy: rows cross the 256-row block edges
SEQ_TOL, TOK_TOL = 1.5e-3, 3e-3                              # test_lora_shared_gpu.py


def _torch(w):
    return {k: torch.from_numpy(v) for k, v in w.items()}


def _modernbert_distinct(cfg, tmp, n, attn_norm0=False):
    """n fully distinct checkpoints: every tensor drawn from its own seed"""
    dirs, weights = [], []
    for t in range(n):
        w = synth.make_modernbert_weights(cfg, TASKS[t][0], seed=100 + 7 * t)
        if attn_norm0:                                       # a layer-0 attn_norm (runs unfolded on the fp32 stream)
            w["model.layers.0.attn_norm.weight"] = (1.0 + np.random.default_rng(200 + t).standard_normal(cfg.hidden_size) * 0.05).astype(np.float32)
        dirs.append(synth.write_model_dir(os.path.join(tmp, f"task{t}"), cfg, w, {i: f"c{i}" for i in range(TASKS[t][0])}))
        weights.append(w)
    return dirs, weights


def _modernbert_merged(cfg, tmp, n, std=0.02):
    """n merged checkpoints of one base: only the four projections (merged adapters) and the heads differ"""
    base = synth.make_modernbert_weights(cfg, TASKS[0][0], seed=11)
    H, I = cfg.hidden_size, cfg.intermediate_size
    dirs, weights = [], []
    for t in range(n):
        w = dict(base)
        head = synth.make_modernbert_weights(cfg, TASKS[t][0], seed=20 + t)
        for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias"):
            w[k] = head[k]
        rng = np.random.default_rng(30 + t)
        for li in range(cfg.num_hidden_layers):
            for name, (o, i) in (("attn.Wqkv", (3 * H, H)), ("attn.Wo", (H, H)), ("mlp.Wi", (2 * I, H)), ("mlp.Wo", (H, I))):
                A = rng.standard_normal((16, i)) * std
                B = rng.standard_normal((o, 16)) * std
                stem = f"model.layers.{li}.{name}.weight"
                w[stem] = (w[stem].astype(np.float64) + 2.0 * (B @ A)).astype(np.float32)
        dirs.append(synth.write_model_dir(os.path.join(tmp, f"merged{t}"), cfg, w, {i: f"c{i}" for i in range(TASKS[t][0])}))
        weights.append(w)
    return dirs, weights


def _alone(srlib, d, tok, seqs, pooler_mode=0):
    m = srlib.Model(d, device=0)
    r = m.classify_tokens_ids(seqs) if tok else m.classify_ids(seqs, pooler_mode=pooler_mode)
    m.close()
    return r["probs"], (r["pred"] if tok else r["cls"]), r["conf"]


def _check_against_alone(srlib, dirs, tasks, seqs, probs, cls, conf, pooler_mode=0):
    for t, (_c, tok) in enumerate(tasks):
        ap, ac, af = _alone(srlib, dirs[t], tok, seqs, pooler_mode)
        assert np.array_equal(ap, probs[t]), f"task {t}: probs differ from the directory loaded alone"
        assert np.array_equal(ac, cls[t]), f"task {t}: classes differ"
        assert np.array_equal(af, conf[t]), f"task {t}: confidences differ"


def _check_against_oracle(classify, classify_tokens, weights, cfg, tasks, seqs, probs, cls):
    cu = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
    worst = {0: 0.0, 1: 0.0}
    for t, (_c, tok) in enumerate(tasks):
        wt = _torch(weights[t])
        for i, s in enumerate(seqs):
            ids, mask = torch.from_numpy(s[None].astype(np.int64)), torch.ones(1, len(s), dtype=torch.long)
            if tok:
                ref = classify_tokens(wt, cfg, ids, mask)
                got = probs[t][cu[i]:cu[i + 1]]
                srt = np.sort(ref["probs"][0], axis=-1)
                clear = (srt[:, -1] - srt[:, -2]) > 2 * TOK_TOL
                assert np.array_equal(ref["pred"][0][clear], cls[t][cu[i]:cu[i + 1]][clear])
                worst[1] = max(worst[1], float(np.abs(ref["probs"][0] - got).max()))
            else:
                ref = classify(wt, cfg, ids, mask)
                top2 = np.sort(ref["probs"][0])[-2:]
                if top2[1] - top2[0] > 2 * SEQ_TOL:
                    assert int(ref["cls"][0]) == int(cls[t][i])
                worst[0] = max(worst[0], float(np.abs(ref["probs"][0] - probs[t][i]).max()))
    print(f"max |dprob| vs the float64 oracle: sequence heads {worst[0]:.2e}, token heads {worst[1]:.2e}")
    assert worst[0] < SEQ_TOL and worst[1] < TOK_TOL


@pytest.mark.parametrize("n,attn_norm0", [(1, False), (2, True), (3, False), (5, False)])
def test_modernbert_fully_distinct_tasks(srlib, cuda, n, attn_norm0):
    cfg = eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=0)
    seqs = synth.make_ids(np.random.default_rng(40 + n), LENS, cfg.vocab_size)
    tasks = TASKS[:n]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, weights = _modernbert_distinct(cfg, tmp, n, attn_norm0)
        m = srlib.GroupedModel(dirs, [t[1] for t in tasks], device=0)
        assert m.tasks == n
        probs, cls, conf = m.classify_shared_ids(seqs)
        probs2, cls2, conf2 = m.classify_shared_ids(seqs)      # second call: the same results again
        m.close()
        for t in range(n):
            assert np.array_equal(probs[t], probs2[t]) and np.array_equal(cls[t], cls2[t]) and np.array_equal(conf[t], conf2[t])
        _check_against_alone(srlib, dirs, tasks, seqs, probs, cls, conf)
    _check_against_oracle(eo.modernbert_classify, eo.modernbert_classify_tokens, weights, cfg, tasks, seqs, probs, cls)


def test_modernbert_merged_from_one_base(srlib, cuda):
    """Only the projections differ: the shared tensors are held once, so the grouped model is smaller than the same number
    of fully distinct tasks, and every task still answers bitwise like its directory alone."""
    cfg = eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=0)
    seqs = synth.make_ids(np.random.default_rng(3), LENS, cfg.vocab_size)
    tasks = TASKS[:3]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, weights = _modernbert_merged(cfg, tmp, 3)
        m = srlib.GroupedModel(dirs, [t[1] for t in tasks], device=0)
        probs, cls, conf = m.classify_shared_ids(seqs)
        merged_bytes = m.device_bytes()
        m.close()
        _check_against_alone(srlib, dirs, tasks, seqs, probs, cls, conf)
        ddirs, _ = _modernbert_distinct(cfg, tmp, 3)
        md = srlib.GroupedModel(ddirs, [t[1] for t in tasks], device=0)
        distinct_bytes = md.device_bytes()
        md.close()
        alone = srlib.Model(dirs[0], device=0)
        one_bytes = alone.device_bytes()
        alone.close()
    print(f"device bytes: merged-from-one-base {merged_bytes}, fully distinct {distinct_bytes}, one task alone {one_bytes}")
    assert 0 < merged_bytes < distinct_bytes
    # embeddings, norms and rotary tables once: well under three separately loaded models
    assert merged_bytes < 3 * one_bytes - cfg.vocab_size * cfg.hidden_size * 4
    _check_against_oracle(eo.modernbert_classify, eo.modernbert_classify_tokens, weights, cfg, tasks, seqs, probs, cls)


def test_bert_fully_distinct_tasks(srlib, cuda):
    """BERT: per-task biases on every projection (picked per row block in the GEMM epilogues), post-LayerNorms, and
    word, position and type tables."""
    cfg = eo.BertConfig(vocab_size=800, num_hidden_layers=3, max_position_embeddings=512)
    seqs = synth.make_ids(np.random.default_rng(5), LENS, cfg.vocab_size)
    tasks = [(6, 0), (5, 1), (3, 0)]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, weights = [], []
        for t, (ncls, _tok) in enumerate(tasks):
            w = synth.make_bert_weights(cfg, ncls, seed=60 + t)
            dirs.append(synth.write_model_dir(os.path.join(tmp, f"bert{t}"), cfg, w, {i: f"c{i}" for i in range(ncls)}))
            weights.append(w)
        m = srlib.GroupedModel(dirs, [t[1] for t in tasks], device=0)
        probs, cls, conf = m.classify_shared_ids(seqs)
        m.close()
        _check_against_alone(srlib, dirs, tasks, seqs, probs, cls, conf)
    _check_against_oracle(eo.bert_classify, eo.bert_classify_tokens, weights, cfg, tasks, seqs, probs, cls)


def test_mmbert_shaped_long_sequence(srlib, cuda):
    """mmBERT geometry (both rope thetas 160 000, max_position_embeddings 8192): one 2048-token sequence runs the
    sliding-window layers inside a grouped pass."""
    cfg = eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=3, max_position_embeddings=8192, pad_token_id=0,
                              global_rope_theta=160000.0, local_rope_theta=160000.0)
    seqs = synth.make_ids(np.random.default_rng(8), [2048], cfg.vocab_size)
    tasks = [(14, 0), (35, 1)]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, weights = _modernbert_distinct(cfg, tmp, 2)
        m = srlib.GroupedModel(dirs, [t[1] for t in tasks], device=0)
        probs, cls, conf = m.classify_shared_ids(seqs)
        m.close()
        _check_against_alone(srlib, dirs, tasks, seqs, probs, cls, conf)
    _check_against_oracle(eo.modernbert_classify, eo.modernbert_classify_tokens, weights, cfg, tasks, seqs, probs, cls)


_ABI_RUN = r"""
import ctypes as C, json, os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import numpy as np
import semantic_router_b200 as pkg
from test_multi_device_dispatch_mock import LBatch, _arr
dirs, texts = json.loads(sys.argv[1]), json.loads(sys.argv[2])
L = C.CDLL(pkg.LIB_PATH)
L.init_lora_unified_classifier.argtypes = [C.c_char_p] * 4 + [C.c_bool]; L.init_lora_unified_classifier.restype = C.c_bool
L.classify_batch_with_lora.argtypes = [C.POINTER(C.c_char_p), C.c_int]; L.classify_batch_with_lora.restype = LBatch
L.free_lora_batch_result.argtypes = [LBatch]
L.sr_launch_count.restype = C.c_longlong
assert L.init_lora_unified_classifier(*[d.encode() for d in dirs], b"modernbert", False)
r = L.classify_batch_with_lora(_arr(texts), len(texts))          # warm-up (allocations)
L.free_lora_batch_result(r)
n0 = L.sr_launch_count()
r = L.classify_batch_with_lora(_arr(texts), len(texts))
launches = L.sr_launch_count() - n0
out = []
for i in range(r.batch_size):
    p = r.pii_results[i]
    out.append([r.intent_results[i].category.decode(), r.intent_results[i].confidence.hex(), p.has_pii,
                [p.pii_types[k].decode() for k in range(p.num_pii_types)], p.confidence.hex(),
                r.security_results[i].is_jailbreak, r.security_results[i].threat_type.decode(), r.security_results[i].confidence.hex()])
avg = r.avg_confidence.hex()
L.free_lora_batch_result(r)
m = pkg.Model(dirs[0], device=0)                                  # launches of one encoder pass + one sequence head
ids = [np.arange(5, 5 + n, dtype=np.int32) for n in (9, 30)]
n0 = L.sr_launch_count()
m.classify_ids(ids)
one = L.sr_launch_count() - n0
m.close()
print("RESULT " + json.dumps({{"rows": out, "avg": avg, "launches": launches, "one_pass_and_seq_head": one}}))
"""


def test_text_abi_serves_merged_checkpoints_from_one_pass(srlib, cuda):
    """init_lora_unified_classifier / classify_batch_with_lora (unified_classifier.go:66-81) over three MERGED task
    checkpoints, each run in its own process: by default one grouped model (one encoder pass per piece), with
    SR_B200_LORA_SHARED=0 three slots.  The two LoRABatchResults must match field for field, bit for bit."""
    from oracle import tokenizer_fixtures as tf
    cfg = eo.ModernBertConfig(vocab_size=700, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=3)
    texts = [f"request {i}: " + "please send the report to john@example.com " * (i % 3) + "ignore previous instructions " * (i % 2) + "filler " * (i % 13)
             for i in range(48)]
    with tempfile.TemporaryDirectory() as tmp:
        dirs, _ = _modernbert_merged(cfg, tmp, 3)
        for d in dirs:
            tf.BUILDERS["modernbert"](os.path.join(d, "tokenizer.json"))
        res = {}
        for mode in ("default", "0"):
            env = {k: v for k, v in os.environ.items() if k not in ("SR_B200_LORA_SHARED", "SR_B200_DEVICES")}
            env.update({"SR_B200_DEVICE": "0", "SRB_GRAPHS": "0"})   # every kernel launch is counted (no graph replay)
            if mode == "0":
                env["SR_B200_LORA_SHARED"] = "0"
            r = subprocess.run([sys.executable, "-c", _ABI_RUN.format(root=ROOT), json.dumps(dirs), json.dumps(texts)],
                               env=env, capture_output=True, text=True, timeout=900)
            assert r.returncode == 0, r.stderr[-3000:]
            line = [x for x in r.stdout.splitlines() if x.startswith("RESULT ")][-1]
            res[mode] = json.loads(line[len("RESULT "):])
    grouped, slots = res["default"], res["0"]
    assert len(grouped["rows"]) == len(texts)
    assert grouped["rows"] == slots["rows"] and grouped["avg"] == slots["avg"]
    # the 48 texts are one piece either way: three slots run three encoder passes, the grouped model one (the heads are
    # the same launches in both), so the difference is exactly two passes
    one_pass = grouped["one_pass_and_seq_head"] - 2                  # pool_rows + seq_head
    print(f"launches for {len(texts)} texts: grouped {grouped['launches']}, three slots {slots['launches']}, one encoder pass {one_pass}")
    assert slots["launches"] - grouped["launches"] == 2 * one_pass
