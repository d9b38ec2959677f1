"""Every row of the encoder's hidden states against float64 (oracle/hidden_oracle.py), through the C ABI only: a model is loaded
from a synthetic checkpoint, `sr_forward_dev` runs 1 ... L layers on one packed batch and `sr_dev_hidden` is read back, on the
production path and on the precise path.  Each element must be within hidden_oracle.row_bound of the float64 forward of the same
fp32 checkpoint; tests/test_hidden_oracle.py holds the CPU evidence for that bound.

Geometries: every hidden size the loader accepts (384 / 768 / 1024) with I % 128 == 64, I < H, N = 5248, global layers every
1 / 2 / 3 / 4, windows 32 / 64 / 128, local rope theta above the global one, eps 1e-6; the plain, the trained-like and the
wide weight family; both attn_norm layouts that leave the LayerNorm fold; packs whose totals sit one past a multiple of 128 and of 256; a
pack of ~20 000 tokens; 22 layers; BERT at 384 (heads of 32) / 768 / 1024 and through `sr_embed_ids_padded`.
Bitwise: alone = inside the pack, a shallower run after a deeper one = the shallower run first, repeat = first, precise on then
off = production.  Run with -s for the worst error over the bound of every case."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, hidden_oracle as ho, synth

pytestmark = pytest.mark.gpu

L = 4
PACK = [1, 63, 64, 65, 129, 130, 257, 511, 512]
DEV = "cuda"


def _hidden(srlib, m, rows):
    ptr = srlib.lib().sr_dev_hidden(m.handle)
    assert ptr

    class _Dev:
        __cuda_array_interface__ = {"data": (int(ptr), False), "shape": (rows, m.hidden), "typestr": "<f4", "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").clone()


def _forward(srlib, m, seqs, depth):
    """[T, H] fp32 rows (on the device) after `depth` layers of one packed batch; exactly T rows are read"""
    ids, cu = srlib.pack(seqs)
    T, B = len(ids), len(seqs)
    lib = srlib.lib()
    assert lib.sr_reserve(m.handle, T, B, B) == 0
    d_ids, d_cu = torch.from_numpy(ids).cuda(), torch.from_numpy(cu).cuda()
    torch.cuda.synchronize()
    assert lib.sr_forward_dev(m.handle, d_ids.data_ptr(), d_cu.data_ptr(), B, T, max(len(s) for s in seqs), depth) == 0
    assert lib.sr_sync(m.handle) == 0
    return _hidden(srlib, m, T)


class _load:
    """A model from a checkpoint directory that lives as long as the model (the precise path reads it when it is enabled)"""

    def __init__(self, srlib, cfg, w):
        self.tmp = tempfile.TemporaryDirectory()
        self.m = srlib.Model(synth.write_model_dir(os.path.join(self.tmp.name, "m"), cfg, w), device=0)

    def __enter__(self):
        return self.m

    def __exit__(self, *exc):
        self.m.close()
        self.tmp.cleanup()


def _check(got, seqs, refs, depth, u, which=None):
    """worst (error / bound) over the rows of the sequences `which` (all), refs[i] = float64 rows per depth of sequence i"""
    assert bool(torch.isfinite(got).all())
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
    return max(ho.worst_over_bound(got[off[i]:off[i + 1]], refs[i], depth, u) for i in (which or range(len(seqs))))


def _same(a, b):
    return a.shape == b.shape and bool((a.view(torch.int32) == b.view(torch.int32)).all())


def _modernbert_case(srlib, name, cfg, w, seqs, depths, sample=None, bitwise=True):
    w64 = ho.to64(w, DEV)
    which = list(range(len(seqs))) if sample is None else sample
    refs = {i: ho.modernbert_hidden64(w64, cfg, seqs[i], max(depths)) for i in which}
    with _load(srlib, cfg, w) as m:
        rows = {}
        for path, u in (("production", ho.U16), ("precise", ho.precise_u(cfg))):
            m.set_precise(path == "precise")
            worst = []
            for d in depths:
                rows[path, d] = _forward(srlib, m, seqs, d)
                worst.append(_check(rows[path, d], seqs, refs, d, u, which))
            print(f"{name} {path}: worst error / bound at depths {list(depths)}: " + " ".join(f"{v:.3f}" for v in worst))
            assert max(worst) <= 1.0, (name, path, worst)
        m.set_precise(False)                                       # precise on, then off: the production rows again
        d0, dL = depths[0], depths[-1]
        assert _same(_forward(srlib, m, seqs, dL), rows["production", dL])           # ... and a repeat = the first run
        if bitwise:
            # a shallower run after the deepest one: nothing is carried in row_stats or the pivot records
            assert _same(_forward(srlib, m, seqs, d0), rows["production", d0])
            off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
            for i in (0, len(seqs) // 2, len(seqs) - 1):           # a sequence alone = the same sequence inside the pack
                for d in (d0, dL):
                    assert _same(_forward(srlib, m, [seqs[i]], d), rows["production", d][off[i]:off[i + 1]]), (name, i, d)


@pytest.mark.parametrize("family", ho.FAMILIES)
@pytest.mark.parametrize("geo", list(ho.GEOMETRIES))
def test_modernbert_geometries(srlib, cuda, geo, family):
    """ho.depth(geo) layers: past the second global layer.  The wide family is the one on which tests/test_hidden_oracle.py
    shows a wrong layer kind, window or rope table > 10x the bound at every geometry."""
    layers = ho.depth(geo)
    cfg = ho.modernbert_config(geo, layers)
    seqs = synth.make_ids(np.random.default_rng(21), PACK, cfg.vocab_size)
    _modernbert_case(srlib, f"{geo} {family}", cfg, ho.modernbert_weights(cfg, family), seqs, range(1, layers + 1))


@pytest.mark.parametrize("layout", ["layer0-attn-norm", "layer2-without"])
def test_modernbert_attn_norm_layouts(srlib, cuda, layout):
    """the unfolded routes of encoder_forward: LayerNorm of the fp32 embedding rows, and hl_to_f32 + cast"""
    cfg = ho.modernbert_config("base-768", L)
    w = ho.modernbert_weights(cfg, "trained", layer0_attn_norm=layout == "layer0-attn-norm",
                              drop_attn_norm=(2,) if layout == "layer2-without" else ())
    seqs = synth.make_ids(np.random.default_rng(23), PACK, cfg.vocab_size)
    _modernbert_case(srlib, f"base-768 trained {layout}", cfg, w, seqs, range(1, L + 1))


@pytest.mark.parametrize("total", [128 * 9 + 1, 256 * 5 + 1])
def test_modernbert_pack_one_past_a_row_block(srlib, cuda, total):
    cfg = ho.modernbert_config("base-768", L)
    lens = [300, 17, 512, 64]
    lens.append(total - sum(lens))
    seqs = synth.make_ids(np.random.default_rng(24), lens, cfg.vocab_size)
    _modernbert_case(srlib, f"base-768 trained T {total}", cfg, ho.modernbert_weights(cfg, "trained"), seqs, [1, L])


def test_modernbert_large_pack(srlib, cuda):
    """~20 000 tokens: every GEMM worker takes several tiles; the oracle runs on a seeded sample of the sequences"""
    cfg = ho.modernbert_config("large-1024", L)
    rng = np.random.default_rng(25)
    lens = [int(n) for n in rng.integers(1, 513, size=78)]
    seqs = synth.make_ids(rng, lens, cfg.vocab_size)
    sample = sorted(int(i) for i in rng.choice(len(seqs), 8, replace=False))
    _modernbert_case(srlib, f"large-1024 trained T {sum(lens)}", cfg, ho.modernbert_weights(cfg, "trained"), seqs, [1, L],
                     sample=sample, bitwise=False)


def test_modernbert_full_depth(srlib, cuda):
    cfg = ho.modernbert_config("base-768", 22)
    seqs = synth.make_ids(np.random.default_rng(26), PACK, cfg.vocab_size)
    for family in ("plain", "trained"):
        _modernbert_case(srlib, f"base-768 {family} 22 layers", cfg, ho.modernbert_weights(cfg, family), seqs, [11, 22],
                         sample=[0, 3, 5, 8])


@pytest.mark.parametrize("heads,hidden,inter", [(12, 384, 1536), (12, 768, 3072), (16, 1024, 4096)])
def test_bert_hidden_rows(srlib, cuda, heads, hidden, inter):
    layers = 3
    cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                        intermediate_size=inter)
    w = synth.make_bert_weights(cfg, 0, seed=27, with_pooler=False)
    w64 = ho.to64(w, DEV)
    seqs = synth.make_ids(np.random.default_rng(28), PACK, cfg.vocab_size)
    with _load(srlib, cfg, w) as m:
        refs = [ho.bert_hidden64(w64, cfg, s) for s in seqs]
        got = _forward(srlib, m, seqs, 0)
        worst = _check(got, seqs, refs, layers, ho.U16)
        print(f"BERT H {hidden} heads {heads}: worst error / bound after {layers} layers {worst:.3f}")
        assert worst <= 1.0
        assert _same(_forward(srlib, m, seqs, 0), got)
        assert _same(_forward(srlib, m, [seqs[5]], 0), got[sum(PACK[:5]):sum(PACK[:6])])
        if hidden == 384:     # fixed padding: every position is a query, positions >= real_len are masked as keys
            real = [1, 40, 64, 65, 100, 130, 200, 300, 512]
            refs = [ho.bert_hidden64(w64, cfg, s, r) for s, r in zip(seqs, real)]
            m.embed_ids_padded(seqs, real)
            worst = _check(_hidden(srlib, m, sum(PACK)), seqs, refs, layers, ho.U16)
            print(f"BERT H {hidden} through sr_embed_ids_padded: worst error / bound {worst:.3f}")
            assert worst <= 1.0


@pytest.mark.parametrize("fields,message", [
    (dict(hidden_size=512, num_attention_heads=8, intermediate_size=1152), "hidden_size unsupported"),
    (dict(hidden_size=768, num_attention_heads=12, intermediate_size=1136), "intermediate_size must be a multiple of 64"),
    # I % 64 == 32: the GeGLU GEMM (N = 2 I, 128-column tiles) cannot run it; the loader used to accept it and every forward failed
    (dict(hidden_size=768, num_attention_heads=12, intermediate_size=1120), "intermediate_size must be a multiple of 64"),
    (dict(hidden_size=384, num_attention_heads=6, intermediate_size=288), "intermediate_size must be a multiple of 64"),
    (dict(hidden_size=384, num_attention_heads=12, intermediate_size=1152), "head_dim 32 unsupported"),
])
def test_loader_refusals(srlib, cuda, fields, message):
    cfg = eo.ModernBertConfig(vocab_size=ho.VOCAB, num_hidden_layers=1, max_position_embeddings=1024, pad_token_id=0, **fields)
    w = synth.make_modernbert_weights(cfg, 0, seed=29, with_head=False)
    with tempfile.TemporaryDirectory() as tmp:
        d = synth.write_model_dir(os.path.join(tmp, "m"), cfg, w)
        h = C.c_void_p()
        assert srlib.lib().sr_model_load(d.encode(), 0, C.byref(h)) != 0
        assert not h.value                                           # no model returned
        assert message in srlib.lib().sr_last_error().decode()
