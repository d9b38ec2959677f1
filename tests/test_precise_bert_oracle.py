"""CPU checks of oracle/bert_precise_oracle.py, the precise path's BERT / MiniLM forms: the fp32 attention at heads of 32
and 64 with and without key lengths and the fp32 GELU equal plain torch float64 computations; at head dim 64 without key
lengths the attention reference and restatement are bitwise oracle/precise_oracle.py's; the float32 restatements stay inside
their bounds with a margin >= 2 on every input family of precise_oracle; each wrong kernel of BERT_MUTATIONS leaves the
bound by more than 10x on some family; and the float32 BERT forward over split-pair weights (bert_precise_restated) stays
inside hidden_oracle's precise per-row bound of the float64 forward with a margin >= 2 at H 384 (heads of 32), 768 and
1024."""
import math

import numpy as np
import pytest
import torch

from oracle import bert_precise_oracle as bpo, encoder_oracle as eo, hidden_oracle as ho, precise_oracle as po, synth

LENS = [1, 31, 32, 33, 64, 65, 130]
KV = [1, 1, 31, 32, 33, 64, 129]          # 1, 31, 32, 33, len - 1 and len among them


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


def _ratio(got, ref_value, bound):
    r = (torch.as_tensor(np.asarray(got)).double() - ref_value).abs() / bound
    return float(torch.nan_to_num(r, nan=torch.inf).max())


# ---- values --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head_dim", [32, 64])
@pytest.mark.parametrize("kv", [False, True])
def test_attention_value_is_masked_softmax_attention(head_dim, kv):
    nH, cu = 2, _cu(LENS)
    kv_lens = KV if kv else None
    qkv = bpo.make_qkv("random", cu, nH, seed=1, head_dim=head_dim)
    ref = bpo.attention(qkv, cu, nH, 0, head_dim=head_dim, kv_lens=kv_lens)
    x = qkv.double().view(-1, 3, nH, head_dim)
    for b, L in enumerate(LENS):
        s = slice(cu[b], cu[b + 1])
        att = torch.einsum("ihd,jhd->hij", x[s, 0], x[s, 1]) / math.sqrt(head_dim)
        if kv:
            att[..., KV[b]:] = -torch.inf
        want = torch.einsum("hij,jhd->ihd", torch.softmax(att, -1), x[s, 2]).reshape(L, nH * head_dim)
        torch.testing.assert_close(ref.value[s], want, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("family", ["sink", "constant", "random"])
@pytest.mark.parametrize("window", [0, 33])
def test_head_dim_64_without_key_lengths_is_precise_oracle(family, window):
    """the ModernBERT form: bitwise precise_oracle's inputs, reference, bound and restatement; key lengths >= len change
    nothing"""
    cu = _cu(LENS)
    qkv = bpo.make_qkv(family, cu, 2, window, seed=2)
    assert torch.equal(qkv, po.make_qkv(family, cu, 2, window, seed=2))
    a, b = bpo.attention(qkv, cu, 2, window), po.attention(qkv, cu, 2, window)
    assert torch.equal(a.value, b.value) and torch.equal(a.bound, b.bound)
    got = bpo.restate_attention(qkv.numpy(), cu, 2, window)
    assert np.array_equal(got.view(np.int32), po.restate_attention(qkv.numpy(), cu, 2, window).view(np.int32))
    if window == 0:
        c = bpo.attention(qkv, cu, 2, 0, kv_lens=LENS)
        assert torch.equal(a.value, c.value) and torch.equal(a.bound, c.bound)
        assert np.array_equal(got.view(np.int32), bpo.restate_attention(qkv.numpy(), cu, 2, 0, kv_lens=LENS).view(np.int32))


def test_gelu_value_is_gelu_erf():
    x = torch.linspace(-10, 10, 4001)
    torch.testing.assert_close(bpo.gelu(x).value, eo.gelu_erf(x.double()), rtol=1e-12, atol=1e-13)


def test_kernel_scale_is_fp32_of_the_inverse_square_root():
    assert bpo.scale_of(64) == 0.125
    assert bpo.scale_of(32) == float(np.float32(1.0 / math.sqrt(32.0)))


# ---- restatements inside, mutations outside -----------------------------------------------------------------------
@pytest.mark.parametrize("family", po.FAMILIES)
@pytest.mark.parametrize("head_dim", [32, 64])
@pytest.mark.parametrize("kv", [False, True])
def test_attention_restatement_within_bound(family, head_dim, kv):
    cu = _cu(LENS)
    kv_lens = KV if kv else None
    qkv = bpo.make_qkv(family, cu, 2, seed=3, head_dim=head_dim, kv_lens=kv_lens)
    ref = bpo.attention(qkv, cu, 2, 0, head_dim=head_dim, kv_lens=kv_lens)
    got = bpo.restate_attention(qkv.numpy(), cu, 2, 0, head_dim=head_dim, kv_lens=kv_lens)
    assert _ratio(got, ref.value, ref.bound) <= 0.5, family


@pytest.mark.parametrize("mut,head_dim,kv", [("scale_64_at_32", 32, False), ("scale_64_at_32", 32, True),
                                             ("kv_ignored", 32, True), ("kv_ignored", 64, True),
                                             ("kv_plus_one", 32, True), ("kv_plus_one", 64, True)])
def test_attention_mutations_leave_the_bound(mut, head_dim, kv):
    cu = _cu(LENS)
    kv_lens = KV if kv else None
    worst = 0.0
    for family in po.FAMILIES:
        qkv = bpo.make_qkv(family, cu, 2, seed=3, head_dim=head_dim, kv_lens=kv_lens)
        ref = bpo.attention(qkv, cu, 2, 0, head_dim=head_dim, kv_lens=kv_lens)
        bad = bpo.restate_attention(qkv.numpy(), cu, 2, 0, head_dim=head_dim, kv_lens=kv_lens, mut=mut)
        worst = max(worst, _ratio(bad, ref.value, ref.bound))
    assert worst > 10.0, (mut, worst)


def test_gelu_restatement_and_mutation():
    g = torch.Generator().manual_seed(5)
    x = torch.cat([torch.linspace(-10, 10, 2001), 3 * torch.randn(4000, generator=g), torch.tensor([0.0, -0.0, 1e-30])])
    ref = bpo.gelu(x)
    assert _ratio(bpo.restate_gelu(x.numpy()), ref.value, ref.bound) <= 0.5
    assert _ratio(bpo.restate_gelu(x.numpy(), mut="gelu_tanh"), ref.value, ref.bound) > 10.0


# ---- the whole BERT forward ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,hidden,inter", [(12, 384, 1536), (12, 768, 3072), (16, 1024, 4096)])
def test_bert_precise_restated_within_the_precise_bound(heads, hidden, inter):
    layers = 3
    cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                        intermediate_size=inter)
    w = synth.make_bert_weights(cfg, 0, seed=27, with_pooler=False)
    w64 = ho.to64(w)
    u = ho.precise_u(cfg)
    seqs = synth.make_ids(np.random.default_rng(28), [1, 65, 130], cfg.vocab_size)
    cases = [(s, None) for s in seqs] + [(seqs[2], 100)]
    for s, real in cases:
        ref = ho.bert_hidden64(w64, cfg, s, real)
        got = bpo.bert_precise_restated(w, cfg, s, real)
        for d in range(1, layers + 1):
            worst = ho.worst_over_bound(got[d - 1], ref, d, u)
            assert worst <= 0.5, (hidden, len(s), real, d, worst)
