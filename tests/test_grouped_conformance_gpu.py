"""Every task of a grouped pass (sr_model_load_grouped + sr_classify_lora_shared_ids) against the same directory loaded alone
and against float64, through the C ABI only.  include/sr_b200.h promises that each task's results are bitwise what the task
gives loaded alone as Model; this file holds the grouped pass to that on its hidden rows as well as its heads.

For every case the grouped model classifies one batch, `sr_dev_hidden` is read for tasks * T1p rows (T1p: the batch's T1
rows padded to whole 256-row blocks), and each task's directory is loaded alone and run on the same batch:
  * rows [t T1p, t T1p + T1) are bitwise the alone model's hidden rows (the pad rows after them are read by nobody);
  * the same rows are within oracle/hidden_oracle.py's per-row bound (U16) of the float64 forward on task t's weights;
  * probs, classes and confidences are bitwise the alone model's.

Cases: every ModernBERT geometry of hidden_oracle.GEOMETRIES on trained-like weights (the GeGLU N = 640 / 2176 / 5248 / 8192
end in a partial 192-column tile of the wide kernel, whose last rows belong to the next task's matrix); 1, 2 and 8 tasks
(8 x 256 rows: the call runs as a captured graph); T1 = 1, 255, 256, 257, 512 and a pack crossing the 256-row edges; a
graph replayed on a second batch with the same key; tasks sharing some embeddings and norms but not others; BERT at H 384 /
768 / 1024 with a bias per task on every projection, both pooler modes; max_position_embeddings 128 (the pad rows split into
sequences the position table covers); a BERT intermediate_size the grouped GEMMs cannot pick per task, refused at load.
Run with -s for the worst error / bound of every case."""
import ctypes as C
import os
import tempfile
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, hidden_oracle as ho, synth

pytestmark = pytest.mark.gpu

PACK = [1, 63, 64, 65, 129, 130, 257, 511, 512]      # T1 = 1732: 60 pad rows per task
TASKS = [(5, 0), (7, 1), (3, 0), (2, 0), (4, 1), (6, 0), (9, 0), (2, 1)]    # (classes, token-level)
DEV = "cuda"


def _hidden(srlib, m, rows):
    ptr = srlib.lib().sr_dev_hidden(m.handle)
    assert ptr

    class _Dev:
        __cuda_array_interface__ = {"data": (int(ptr), False), "shape": (rows, m.hidden), "typestr": "<f4", "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").clone()


def _same(a, b):
    return a.shape == b.shape and bool((a.view(torch.int32) == b.view(torch.int32)).all())


def _same_np(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _offsets(seqs):
    return np.concatenate([[0], np.cumsum([len(s) for s in seqs])])


# ---- checkpoints ----------------------------------------------------------------------------------------------------
def _head(cfg, num_classes, seed):
    """synth's ModernBERT head (head.dense, head.norm, classifier) for hidden size cfg.hidden_size"""
    w = synth.make_modernbert_weights(replace(cfg, num_hidden_layers=0, vocab_size=1), num_classes, seed=seed)
    return {k: v for k, v in w.items() if k.startswith(("head.", "classifier."))}


def _modernbert_task(cfg, t, seed0=300):
    w = ho.modernbert_weights(cfg, "trained", seed=seed0 + 17 * t)
    w.update(_head(cfg, TASKS[t][0], seed0 + 17 * t + 5))
    return w


def _write(tmp, name, cfg, w, num_classes):
    return synth.write_model_dir(os.path.join(tmp, name), cfg, w, {i: f"c{i}" for i in range(num_classes)})


class Tasks:
    """Task checkpoints written to one temporary directory: dirs[t], weights[t], tasks[t] = (classes, token-level)"""

    def __init__(self, cfg, weights, tasks, tmp, tag="task"):
        self.cfg, self.weights, self.tasks = cfg, weights, tasks
        self.dirs = [_write(tmp, f"{tag}{t}", cfg, w, tasks[t][0]) for t, w in enumerate(weights)]

    def pick(self, idx):
        """the tasks idx, in that order"""
        s = object.__new__(Tasks)
        s.cfg = self.cfg
        s.weights, s.tasks, s.dirs = ([x[i] for i in idx] for x in (self.weights, self.tasks, self.dirs))
        return s


def _modernbert_tasks(cfg, n, tmp, seed0=300):
    return Tasks(cfg, [_modernbert_task(cfg, t, seed0) for t in range(n)], TASKS[:n], tmp)


def _bert_tasks(cfg, tasks, tmp, seed0=60):
    return Tasks(cfg, [synth.make_bert_weights(cfg, c, seed=seed0 + t) for t, (c, _tok) in enumerate(tasks)], tasks, tmp,
                 "bert")


# ---- one grouped call, the alone models, float64 ----------------------------------------------------------------------
def _grouped_call(srlib, m, seqs, pooler_mode=0):
    """per task: probs, cls, conf and the task's T1 hidden rows of one classify_shared_ids call"""
    probs, cls, conf = m.classify_shared_ids(seqs, pooler_mode)
    T1 = int(_offsets(seqs)[-1])
    T1p = -(-T1 // 256) * 256
    hid = _hidden(srlib, m, m.tasks * T1p)
    return [dict(probs=probs[t], cls=cls[t], conf=conf[t], rows=hid[t * T1p:t * T1p + T1]) for t in range(m.tasks)]


def _alone(srlib, d, tok, seqs, pooler_mode=0):
    m = srlib.Model(d, device=0)
    try:
        r = m.classify_tokens_ids(seqs) if tok else m.classify_ids(seqs, pooler_mode=pooler_mode)
        rows = _hidden(srlib, m, int(_offsets(seqs)[-1]))
    finally:
        m.close()
    return dict(probs=r["probs"], cls=r["pred"] if tok else r["cls"], conf=r["conf"], rows=rows)


def _refs(cfg, w, seqs):
    """float64 hidden rows after every layer, per sequence, on the weights w"""
    w64 = ho.to64(w, DEV)
    if isinstance(cfg, eo.BertConfig):
        return [ho.bert_hidden64(w64, cfg, s) for s in seqs]
    return [ho.modernbert_hidden64(w64, cfg, s, cfg.num_hidden_layers) for s in seqs]


def _check(srlib, name, got, ts, seqs, pooler_mode=0, refs=None):
    """got: _grouped_call's results; refs: per task, _refs of that task (computed here when None)"""
    off = _offsets(seqs)
    worst = []
    for t, (_c, tok) in enumerate(ts.tasks):
        a = _alone(srlib, ts.dirs[t], tok, seqs, pooler_mode)
        assert _same(got[t]["rows"], a["rows"]), f"{name}: task {t}: hidden rows differ from the directory loaded alone"
        for k in ("probs", "cls", "conf"):
            assert _same_np(got[t][k], a[k]), f"{name}: task {t}: {k} differ from the directory loaded alone"
        r = refs[t] if refs is not None else _refs(ts.cfg, ts.weights[t], seqs)
        worst.append(max(ho.worst_over_bound(got[t]["rows"][off[i]:off[i + 1]], r[i], ts.cfg.num_hidden_layers, ho.U16)
                         for i in range(len(seqs))))
    print(f"{name}: worst error / bound per task: " + " ".join(f"{v:.3f}" for v in worst))
    assert max(worst) <= 1.0, (name, worst)


def _serve(srlib, name, ts, seqs, pooler_mode=0):
    m = srlib.GroupedModel(ts.dirs, [tok for _c, tok in ts.tasks], device=0)
    try:
        assert m.tasks == len(ts.dirs)
        got = _grouped_call(srlib, m, seqs, pooler_mode)
    finally:
        m.close()
    _check(srlib, name, got, ts, seqs, pooler_mode)


# ---- ModernBERT ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geo", list(ho.GEOMETRIES))
def test_modernbert_geometries(srlib, cuda, geo):
    """three tasks (one token-level) of trained-like weights at ho.depth(geo) layers"""
    cfg = ho.modernbert_config(geo, ho.depth(geo))
    seqs = synth.make_ids(np.random.default_rng(41), PACK, cfg.vocab_size)
    with tempfile.TemporaryDirectory() as tmp:
        _serve(srlib, f"{geo} T1 {sum(PACK)}", _modernbert_tasks(cfg, 3, tmp), seqs)


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    """eight small-384 tasks of trained-like weights"""
    cfg = ho.modernbert_config("small-384", ho.depth("small-384"))
    return _modernbert_tasks(cfg, 8, str(tmp_path_factory.mktemp("grouped_small")))


@pytest.mark.parametrize("n", [1, 2, 8])
def test_task_counts(srlib, cuda, small, n):
    """8 tasks x 256 rows = 2048: the pass is captured as a graph on the first call and replayed on the second"""
    seqs = synth.make_ids(np.random.default_rng(43 + n), [1, 60, 130, 40], small.cfg.vocab_size)
    ts = small.pick(range(n))
    m = srlib.GroupedModel(ts.dirs, [tok for _c, tok in ts.tasks], device=0)
    try:
        got = _grouped_call(srlib, m, seqs)
        again = _grouped_call(srlib, m, seqs)
    finally:
        m.close()
    for t in range(n):
        for k in ("probs", "cls", "conf"):
            assert _same_np(got[t][k], again[t][k]), (t, k)
        assert _same(got[t]["rows"], again[t]["rows"]), t
    _check(srlib, f"small-384 {n} tasks", got, ts, seqs)


@pytest.mark.parametrize("lens", [[1], [255], [256], [257], [512], [200, 100, 250, 10, 3]],
                         ids=["T1-1", "T1-255", "T1-256", "T1-257", "T1-512", "pack-563"])
def test_batch_edges(srlib, cuda, small, lens):
    """a pad of 255 rows, of 1 row, none, and a pack whose sequences cross the 256- and 512-row block edges"""
    seqs = synth.make_ids(np.random.default_rng(sum(lens)), lens, small.cfg.vocab_size)
    _serve(srlib, f"small-384 lens {lens}", small.pick(range(3)), seqs)


def test_graph_replay_on_another_batch(srlib, cuda, small):
    """[100, 150] then [150, 100] with other ids: one graph key (batch 2, T1 250, max_len 150), so the second call replays
    the graph captured on the first; each call's results are the alone models' on its own batch"""
    ts = small.pick(range(3))
    first = synth.make_ids(np.random.default_rng(50), [100, 150], small.cfg.vocab_size)
    second = synth.make_ids(np.random.default_rng(51), [150, 100], small.cfg.vocab_size)
    m = srlib.GroupedModel(ts.dirs, [tok for _c, tok in ts.tasks], device=0)
    try:
        a = _grouped_call(srlib, m, first)
        b = _grouped_call(srlib, m, second)
        a2 = _grouped_call(srlib, m, first)
    finally:
        m.close()
    _check(srlib, "graph: first batch", a, ts, first)
    _check(srlib, "graph: second batch, replayed", b, ts, second)
    for t in range(3):
        assert _same(a[t]["rows"], a2[t]["rows"]) and _same_np(a[t]["probs"], a2[t]["probs"]), t


def test_partial_sharing(srlib, cuda, tmp_path):
    """Four tasks: embeddings A, B, A, B; layer 1's mlp_norm A, A, B, B; final_norm shared by tasks 0 - 2, task 3's own;
    every other tensor per task.  The loader keeps one device copy of each shared tensor and every task still gets its
    own results."""
    cfg = ho.modernbert_config("small-384", ho.depth("small-384"))
    distinct = [_modernbert_task(cfg, t, seed0=500) for t in range(4)]
    mixed = [dict(w) for w in distinct]
    for t in (2, 3):
        for k in ("model.embeddings.tok_embeddings.weight", "model.embeddings.norm.weight"):
            mixed[t][k] = distinct[t - 2][k]
    mixed[1]["model.layers.1.mlp_norm.weight"] = distinct[0]["model.layers.1.mlp_norm.weight"]
    mixed[3]["model.layers.1.mlp_norm.weight"] = distinct[2]["model.layers.1.mlp_norm.weight"]
    for t in (1, 2):
        mixed[t]["model.final_norm.weight"] = distinct[0]["model.final_norm.weight"]
    ts = Tasks(cfg, mixed, TASKS[:4], str(tmp_path), "mixed")
    td = Tasks(cfg, distinct, TASKS[:4], str(tmp_path), "distinct")
    seqs = synth.make_ids(np.random.default_rng(52), [300, 7, 129, 64], cfg.vocab_size)
    m = srlib.GroupedModel(ts.dirs, [tok for _c, tok in ts.tasks], device=0)
    try:
        got = _grouped_call(srlib, m, seqs)
        mixed_bytes = m.device_bytes()
    finally:
        m.close()
    md = srlib.GroupedModel(td.dirs, [tok for _c, tok in td.tasks], device=0)
    distinct_bytes = md.device_bytes()
    md.close()
    print(f"device bytes: partly shared {mixed_bytes}, fully distinct {distinct_bytes}")
    # two of the four embedding tables are held once
    assert mixed_bytes <= distinct_bytes - 2 * cfg.vocab_size * cfg.hidden_size * 4
    _check(srlib, "small-384 partly shared tensors", got, ts, seqs)


# ---- BERT ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,hidden,inter", [(6, 384, 1536), (12, 768, 3072), (16, 1024, 4096)])
def test_bert_tasks(srlib, cuda, tmp_path, heads, hidden, inter):
    """three tasks with their own biases on every projection (each 256-row block adds its task's in the GEMM epilogues);
    the sequence heads under pooler_mode 0 (pooler) and 1"""
    cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=hidden, num_hidden_layers=3, num_attention_heads=heads,
                        intermediate_size=inter)
    ts = _bert_tasks(cfg, [(6, 0), (5, 1), (3, 0)], str(tmp_path))
    seqs = synth.make_ids(np.random.default_rng(53), PACK, cfg.vocab_size)
    refs = [_refs(cfg, w, seqs) for w in ts.weights]
    m = srlib.GroupedModel(ts.dirs, [tok for _c, tok in ts.tasks], device=0)
    try:
        got = {mode: _grouped_call(srlib, m, seqs, mode) for mode in (0, 1)}
    finally:
        m.close()
    for mode in (0, 1):
        _check(srlib, f"BERT H {hidden} pooler_mode {mode}", got[mode], ts, seqs, mode, refs)


# ---- the pad rows against a short position table --------------------------------------------------------------------
@pytest.mark.parametrize("lens", [[10], [100, 28], [100, 27]], ids=["10", "100-28", "100-27"])
@pytest.mark.parametrize("arch", ["modernbert", "bert"])
def test_pad_within_max_position_embeddings(srlib, cuda, tmp_path, arch, lens):
    """max_position_embeddings 128: a prompt each task serves alone is served grouped.  The 246 pad rows of a 10-token
    batch (129 of [100, 27]) run as sequences of at most 128 rows."""
    if arch == "modernbert":
        cfg = replace(ho.modernbert_config("small-384", 4), max_position_embeddings=128)
        ts = Tasks(cfg, [_modernbert_task(cfg, t, seed0=700) for t in range(2)], TASKS[:2], str(tmp_path))
    else:
        cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=384, num_hidden_layers=2, num_attention_heads=6,
                            intermediate_size=1536, max_position_embeddings=128)
        ts = _bert_tasks(cfg, TASKS[:2], str(tmp_path))
    seqs = synth.make_ids(np.random.default_rng(54), lens, cfg.vocab_size)
    _serve(srlib, f"{arch} max_position_embeddings 128, lens {lens}", ts, seqs)


# ---- a BERT intermediate_size the grouped GEMMs cannot serve ---------------------------------------------------------
def test_bert_intermediate_size_not_a_multiple_of_128(srlib, cuda, tmp_path):
    """I = 1088: Wi (N = I) ends in half a 128-column tile, so two tasks cannot pick their matrices per row block.  The
    grouped load refuses them; each directory alone, and as a group of one, still serves."""
    cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                        intermediate_size=1088)
    ts = _bert_tasks(cfg, [(3, 0), (4, 0)], str(tmp_path))
    dirs = (C.c_char_p * 2)(*[d.encode() for d in ts.dirs])
    h = C.c_void_p()
    assert srlib.lib().sr_model_load_grouped(dirs, None, 2, 0, C.byref(h)) != 0
    assert not h.value
    assert f"{ts.dirs[0]}: intermediate_size 1088 must be a multiple of 128" in srlib.lib().sr_last_error().decode()
    seqs = synth.make_ids(np.random.default_rng(55), [40, 200], cfg.vocab_size)
    for t in range(2):
        _serve(srlib, f"BERT I 1088 task {t} as a group of one", ts.pick([t]), seqs)
