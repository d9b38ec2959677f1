"""Every hidden row of long sequences and of the benchmark-sized batch against float64, through the C ABI only (`sr_reserve`,
`sr_forward_dev`, `sr_dev_hidden`), on the production path at hidden_oracle.row_bound(U16) and on the precise path at
precise_u(cfg).  The float64 forward is hidden_oracle.modernbert_hidden64_long on the GPU, in calls of at most BATCH_TOKENS
tokens; tests/test_hidden_oracle.py shows it equal to the dense forward, the restated engine inside the bound at 4096
tokens, and a rope row read at a wrong position past 2048 rejected by > 10x.

  * mmBERT geometry (H 768, I 1152, global every 3, window 128, both thetas 160 000), depths 1 ... 4: 2049 and 8192 tokens
    at max_position_embeddings 8192 (all three families at 8192), 32 768 tokens at 32 768 (plain and trained-like);
  * [17, 8192, 63, 2049] packed, so row blocks straddle sequences at far positions; the 8192-token sequence alone is
    bitwise the same rows inside the pack;
  * the 256 x 512 = 131 072-row batch of the benchmark: base-768 at 22 layers (plain, trained-like; every row at depth 22,
    production path) and large-1024 (N = 5248, the widest GEMM the engine launches) at 4 layers on both paths;
  * max_position_embeddings + 1 tokens refused on both paths with the hidden buffer bitwise untouched.
Run with -s for the worst error over the bound of every case."""
import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo, hidden_oracle as ho, synth
from test_encoder_hidden_conformance_gpu import DEV, _check, _forward, _hidden, _load, _same

pytestmark = pytest.mark.gpu

L = 4
MMBERT = dict(hidden_size=768, num_attention_heads=12, intermediate_size=1152, global_attn_every_n_layers=3,
              local_attention=128, global_rope_theta=160000.0, local_rope_theta=160000.0)
# Tokens per call of the float64 forward: 8 * 16384 * (7 H + 4 I) bytes of activations, 1.3 GB at H 768 / I 1152 and 2.3 GB at
# H 1024 / I 2624, plus one chunk's scores, held under SCORES values (512 MB) by the query chunk.  Longer sequences run alone.
BATCH_TOKENS = 16384
SCORES = 2 ** 26
PATHS = {"production": lambda cfg: ho.U16, "precise": ho.precise_u}


def _mmbert(max_pos, layers=L):
    return eo.ModernBertConfig(vocab_size=ho.VOCAB, num_hidden_layers=layers, max_position_embeddings=max_pos, pad_token_id=0,
                               **MMBERT)


def _oracle(w64, cfg, seqs, depths):
    """(sequence indices, {index: Hidden64}) per call of the float64 forward: sequences of one length, BATCH_TOKENS at most
    (one sequence when it is longer)"""
    by_len = {}
    for i, s in enumerate(seqs):
        by_len.setdefault(len(s), []).append(i)
    for n, idx in by_len.items():
        step = max(1, BATCH_TOKENS // n)
        for j in range(0, len(idx), step):
            part = idx[j:j + step]
            q_chunk = max(1, min(ho.Q_CHUNK, SCORES // (len(part) * cfg.num_attention_heads * n)))
            refs = ho.modernbert_hidden64_long(w64, cfg, np.stack([seqs[i] for i in part]), depths, q_chunk=q_chunk)
            yield part, dict(zip(part, refs))


def _long_case(srlib, name, cfg, w, seqs, depths, paths=tuple(PATHS)):
    """Rows of every sequence after each depth on each path, all within the bound; returns the rows by (path, depth)"""
    with _load(srlib, cfg, w) as m:
        rows = {}
        for path in paths:
            m.set_precise(path == "precise")
            for d in depths:
                rows[path, d] = _forward(srlib, m, seqs, d)
        m.set_precise(False)
    worst = dict.fromkeys(rows, 0.0)
    for which, refs in _oracle(ho.to64(w, DEV), cfg, seqs, depths):
        for (path, d), got in rows.items():
            worst[path, d] = max(worst[path, d], _check(got, seqs, refs, d, PATHS[path](cfg), which))
        del refs
    for path in paths:
        print(f"{name} {path}: worst error / bound at depths {list(depths)}: " +
              " ".join(f"{worst[path, d]:.3f}" for d in depths))
    assert max(worst.values()) <= 1.0, (name, worst)
    return rows


@pytest.mark.parametrize("S,max_pos,family", [
    (2049, 8192, "trained"),
    (8192, 8192, "plain"), (8192, 8192, "trained"), (8192, 8192, "wide"),
    (32768, 32768, "plain"), (32768, 32768, "trained"),
])
def test_mmbert_long_sequence(srlib, cuda, S, max_pos, family):
    """One sequence up to max_position_embeddings: rope rows and windows at every far position, global layers over all keys
    (the precise path's attention sums each 32-key tile and then adds it to the running sums of the row)"""
    cfg = _mmbert(max_pos)
    seqs = synth.make_ids(np.random.default_rng(S + 31), [S], cfg.vocab_size)
    _long_case(srlib, f"mmBERT {family} S {S} (max_position_embeddings {max_pos})", cfg, ho.modernbert_weights(cfg, family),
               seqs, range(1, L + 1))


def test_mmbert_long_sequence_in_unaligned_pack(srlib, cuda):
    cfg = _mmbert(8192)
    w = ho.modernbert_weights(cfg, "trained")
    seqs = synth.make_ids(np.random.default_rng(32), [17, 8192, 63, 2049], cfg.vocab_size)
    rows = _long_case(srlib, "mmBERT trained pack [17, 8192, 63, 2049]", cfg, w, seqs, [1, L])
    with _load(srlib, cfg, w) as m:
        for d in (1, L):
            assert _same(_forward(srlib, m, [seqs[1]], d), rows["production", d][17:17 + 8192]), d


@pytest.mark.parametrize("family", ["plain", "trained"])
def test_benchmark_batch_full_depth(srlib, cuda, family):
    """modernbert-base-b256-s512: every one of the 131 072 rows after 22 layers"""
    cfg = ho.modernbert_config("base-768", 22)
    seqs = synth.make_ids(np.random.default_rng(33), [512] * 256, cfg.vocab_size)
    _long_case(srlib, f"base-768 {family} 256 x 512, 22 layers", cfg, ho.modernbert_weights(cfg, family), seqs, [22],
               paths=("production",))


def test_benchmark_batch_widest_gemm(srlib, cuda):
    """large-1024 (I 2624: the N = 5248 GeGLU GEMM) at 131 072 rows"""
    cfg = ho.modernbert_config("large-1024", L)
    seqs = synth.make_ids(np.random.default_rng(34), [512] * 256, cfg.vocab_size)
    _long_case(srlib, "large-1024 trained 256 x 512", cfg, ho.modernbert_weights(cfg, "trained"), seqs, [1, L])


def test_position_limit(srlib, cuda):
    """max_position_embeddings tokens run; one more is refused by sr_forward_dev on both paths before anything is launched,
    and the hidden buffer keeps the previous forward's rows bit for bit"""
    P = 8192
    cfg = _mmbert(P, layers=1)
    ids = synth.make_ids(np.random.default_rng(35), [P + 1], cfg.vocab_size)[0]
    lib = srlib.lib()
    with _load(srlib, cfg, ho.modernbert_weights(cfg, "plain")) as m:
        assert lib.sr_reserve(m.handle, P + 1, 1, 1) == 0
        d_ids = torch.from_numpy(ids.astype(np.int32)).cuda()
        d_cu = torch.tensor([0, P + 1], dtype=torch.int32, device="cuda")
        for path in PATHS:
            m.set_precise(path == "precise")
            got = _forward(srlib, m, [ids[:P]], 1)
            assert bool(torch.isfinite(got).all()), path
            before = _hidden(srlib, m, P + 1)
            torch.cuda.synchronize()
            assert lib.sr_forward_dev(m.handle, d_ids.data_ptr(), d_cu.data_ptr(), 1, P + 1, P + 1, 1) != 0, path
            assert lib.sr_sync(m.handle) == 0
            assert _same(_hidden(srlib, m, P + 1), before), path
        m.set_precise(False)
